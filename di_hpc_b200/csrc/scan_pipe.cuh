// scan_pipe.cuh -- TMA-staged column-scan pipeline shared by every T-recurrence of the path
// (GAE fwd/bwd, episodic GAE fwd/bwd, TD-lambda, V-trace return, UPGO return), and its launcher.
//
// Layout reminder: all scan operands are (T,B) with B contiguous.  One CTA owns a tile of BT adjacent columns for ALL
// of T.  A producer lane streams (TT x BT) boxes of each input tensor through an ST-deep shared-memory ring with
// cp.async.bulk.tensor (TMA) + mbarrier expect-tx; BT consumer threads (one per column, bank-conflict-free row reads)
// walk the rows of the box in scan order and carry the recurrence state in registers across boxes.
//
//   ScanPipe<NF, NB, NOUT, BT, TT, ST, NTAB>
//     NF   fp32 input boxes                 maps.m[0..NF)
//     NB   uint8 input boxes (masks)        maps.m[NF..NF+NB); a byte box of a multiple of 32 columns and 4 rows is a
//                                           multiple of 128 bytes, so every box of a stage stays 128-byte aligned
//     NTAB fp32 constants per row (`rowtab`, e.g. GAE's d_t and 1/d_t), one 1-D bulk copy per stage, padded to 128 B
//     NOUT fp32 outputs staged in shared memory (two buffers each) and TMA-stored as (TT x BT) boxes; 0 = the body
//          stores its own results
//
//   * no thread ever issues a global load in the steady state: all input traffic is bulk async,
//     ST-1 boxes per CTA are in flight while one is being consumed
//   * consumers never __syncthreads(): full[]/empty[] mbarriers only (plus, with NOUT > 0, one named barrier over
//     the consumer threads per box before its outputs are handed to the TMA unit)
//   * rows/columns outside an input tensor are zero-filled by the TMA unit; rows/columns outside an output tensor map
//     are clipped by it, so only bodies that store their own results mask their stores
//
// The reference walks the same recurrence with one thread per column issuing dependent scalar
// loads (include/hpc/rll/cuda/rl_utils/gae_kernel.h:17-27, td_lambda_kernel.h:17-31,
// vtrace_kernel.h:161-180, upgo_kernel.h:18-35); this file is the TMA-pipelined re-design of that loop.
#pragma once
#include "common.cuh"

namespace hpcrll {

template <int N>
struct TmapPack {
    CUtensorMap m[N];
};
template <>
struct TmapPack<0> {};

template <int NF, int NB, int NOUT, int BT, int TT, int ST, int NTAB>
struct ScanPipe {
    static_assert(BT % 32 == 0, "column tile must be whole warps");
    static_assert(TT % 4 == 0, "row tile must keep byte boxes 128-byte and the row table 16-byte aligned");
    static_assert(NB == 0 || NOUT > 0, "byte inputs reach the body through the staged-output call form only");
    static constexpr int kConsumerWarps = BT / 32;
    static constexpr int kThreads = BT + 32;  // + one producer warp
    static constexpr int kBoxBytes = TT * BT * 4;
    static constexpr int kByteBoxBytes = TT * BT;
    static constexpr int kTabOff = NF * kBoxBytes + NB * kByteBoxBytes;
    static constexpr int kTabBytes = ((TT * NTAB * 4 + 127) / 128) * 128;
    static constexpr int kStageBytes = kTabOff + kTabBytes;
    static constexpr uint32_t kTxBytes = kTabOff + TT * NTAB * 4;
    static constexpr int kOutBytes = 2 * NOUT * kBoxBytes;
    static constexpr int kSmemBytes = ST * kStageBytes + kOutBytes + 2 * ST * 8;
    static constexpr int kTabN = NTAB > 0 ? NTAB : 1;
    static constexpr int kNB = NB > 0 ? NB : 1;

    // Runs the whole pipeline for the column tile starting at col0.  Consumer thread c (column col0+c) calls, for t in
    // scan order, with x[k] = fp32 input k and m[k] = byte input k at (t, col0+c), rt[k] = rowtab[t*NTAB + k]:
    //   NOUT == 0: body.step(t, x, rt)
    //   NOUT  > 0: body.step(t, x, rt, m, o), o[k] = value of output k at (t, col0+c);
    //              rt and m have one unused element when NTAB or NB is 0
    template <bool REVERSE, class Body>
    static __device__ __forceinline__ void run(const TmapPack<NF + NB>& maps, const TmapPack<NOUT>& omaps,
                                               const float* __restrict__ rowtab, int T, int col0, Body& body) {
        // dynamic shared memory starts at the CTA's shared window base (no static smem in these
        // kernels), so the declared alignment holds; keeping the pointer un-cast lets the compiler
        // emit LDS (shared-space) loads instead of generic ones.
        extern __shared__ __align__(1024) unsigned char smem[];
        float* obuf = reinterpret_cast<float*>(smem + ST * kStageBytes);
        uint64_t* full = reinterpret_cast<uint64_t*>(smem + ST * kStageBytes + kOutBytes);
        uint64_t* empty = full + ST;

        const int tid = threadIdx.x;
        const int nT = (T + TT - 1) / TT;

        if (tid == 0) {
#pragma unroll
            for (int s = 0; s < ST; ++s) {
                mbar_init(&full[s], 1);
                mbar_init(&empty[s], kConsumerWarps);
            }
            fence_mbar_init();
        }
        __syncthreads();

        if (tid >= BT) {
            // ---------------- producer warp: one elected lane feeds the ring ----------------
            if (tid == BT) {
#pragma unroll
                for (int k = 0; k < NF + NB; ++k) prefetch_tmap(&maps.m[k]);
                for (int it = 0; it < nT; ++it) {
                    const int s = it % ST;
                    if (it >= ST) mbar_wait(&empty[s], ((it / ST) & 1) ^ 1);
                    const int j = REVERSE ? nT - 1 - it : it;
                    unsigned char* st = smem + s * kStageBytes;
                    mbar_arrive_expect_tx(&full[s], kTxBytes);
#pragma unroll
                    for (int k = 0; k < NF; ++k) tma_load_2d(st + k * kBoxBytes, &maps.m[k], col0, j * TT, &full[s]);
#pragma unroll
                    for (int k = 0; k < NB; ++k)
                        tma_load_2d(st + NF * kBoxBytes + k * kByteBoxBytes, &maps.m[NF + k], col0, j * TT, &full[s]);
                    if (NTAB > 0) bulk_load_1d(st + kTabOff, rowtab + j * TT * NTAB, TT * NTAB * 4, &full[s]);
                }
            }
            return;
        }

        // -------------------- consumers: one column per thread --------------------
        const int c = tid;
        if constexpr (NOUT > 0) {
            if (tid == 0) {
#pragma unroll
                for (int k = 0; k < NOUT; ++k) prefetch_tmap(&omaps.m[k]);
            }
        }
        // one row i of the stage: a macro rather than a function, because even an inlined call changes the machine
        // code nvcc emits for the two loops below
#define HPC_SCAN_ROW(ROW)                                                                            \
    do {                                                                                             \
        const int i = ROW;                                                                           \
        float x[NF];                                                                                 \
        _Pragma("unroll") for (int k = 0; k < NF; ++k) x[k] = st[(k * TT + i) * BT + c];             \
        float rt[kTabN];                                                                             \
        _Pragma("unroll") for (int k = 0; k < NTAB; ++k) rt[k] = tab[i * NTAB + k];                  \
        if constexpr (NOUT == 0) {                                                                   \
            body.step(j * TT + i, x, rt);                                                            \
        } else {                                                                                     \
            unsigned m[kNB];                                                                         \
            _Pragma("unroll") for (int k = 0; k < NB; ++k) m[k] = sb[(k * TT + i) * BT + c];         \
            float o[NOUT];                                                                           \
            body.step(j * TT + i, x, rt, m, o);                                                      \
            _Pragma("unroll") for (int k = 0; k < NOUT; ++k) ob[(k * TT + i) * BT + c] = o[k];       \
        }                                                                                            \
    } while (0)
        for (int it = 0; it < nT; ++it) {
            const int s = it % ST;
            const int j = REVERSE ? nT - 1 - it : it;
            const float* st = reinterpret_cast<const float*>(smem + s * kStageBytes);
            const unsigned char* sb = smem + s * kStageBytes + NF * kBoxBytes;
            const float* tab = st + kTabOff / 4;
            float* ob = obuf + (it & 1) * (NOUT * TT * BT);
            mbar_wait(&full[s], (it / ST) & 1);
            const int rows = min(TT, T - j * TT);
            if (rows == TT) {
#pragma unroll
                for (int ii = 0; ii < TT; ++ii) HPC_SCAN_ROW(REVERSE ? TT - 1 - ii : ii);
            } else {
                for (int ii = 0; ii < rows; ++ii) HPC_SCAN_ROW(REVERSE ? rows - 1 - ii : ii);
            }
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(&empty[s]);  // input stage free again
            if constexpr (NOUT > 0) {
                // hand the finished output box to the TMA unit.  The buffer written NEXT (the other one) was stored
                // one box ago: thread 0 waits for that store to have read it before anybody passes the barrier.
                fence_proxy_async_smem();
                if (tid == 0) bulk_wait_group_read<0>();
                named_bar_sync(1, BT);
                if (tid == 0) {
#pragma unroll
                    for (int k = 0; k < NOUT; ++k) tma_store_2d(&omaps.m[k], col0, j * TT, ob + k * TT * BT);
                    bulk_commit_group();
                }
            }
        }
#undef HPC_SCAN_ROW
        if constexpr (NOUT > 0) {
            if (tid == 0) bulk_wait_group<0>();
        }
    }
};

// One operand of scan_column: base pointer and row pitch in elements.
template <class P>
struct ColOp {
    P p;
    int64_t ld;
};

// The generic regime of the same scans, for operands TMA cannot describe (misaligned pointers or pitches): the calling
// thread walks column `col` over rows [0, T) in scan order with streaming loads, 8 rows in flight, 64-bit indexing.
// The body is called as in ScanPipe::run, with x[k] = in[k] and m[k] = mk[k] (a NULL mask reads as 0) at (t, col),
// rt[k] = rowtab[t*NTAB + k]; with NOUT > 0, o[k] is stored to out[k] at (t, col).
template <int NF, int NB, int NOUT, int NTAB, bool REVERSE, class Body>
__device__ __forceinline__ void scan_column(const ColOp<const float*> (&in)[NF],
                                            const ColOp<const uint8_t*> (&mk)[NB > 0 ? NB : 1],
                                            const float* __restrict__ rowtab,
                                            const ColOp<float*> (&out)[NOUT > 0 ? NOUT : 1], int64_t T, int64_t col,
                                            Body& body) {
    static_assert(NTAB == 0 || NTAB == 2, "the row table is read as (d_t, 1/d_t) pairs");
    constexpr int U = 8, kNB = NB > 0 ? NB : 1, kTabN = NTAB > 0 ? NTAB : 1;
    const auto load = [&](int64_t t, float (&x)[NF], unsigned (&m)[kNB], float (&rt)[kTabN]) {
#pragma unroll
        for (int k = 0; k < NF; ++k) x[k] = ld_stream(in[k].p + t * in[k].ld + col);
#pragma unroll
        for (int k = 0; k < NB; ++k) m[k] = ld_mask(mk[k].p, t * mk[k].ld + col);
        if constexpr (NTAB == 2) {
            const float2 d = __ldg(reinterpret_cast<const float2*>(rowtab) + t);
            rt[0] = d.x;
            rt[1] = d.y;
        }
    };
    const auto step = [&](int64_t t, const float (&x)[NF], const unsigned (&m)[kNB], const float (&rt)[kTabN]) {
        if constexpr (NOUT == 0) {
            body.step(static_cast<int>(t), x, rt);
        } else {
            float o[NOUT];
            body.step(static_cast<int>(t), x, rt, m, o);
#pragma unroll
            for (int k = 0; k < NOUT; ++k) st_stream(out[k].p + t * out[k].ld + col, o[k]);
        }
    };
    const auto row = [&](int64_t n) { return REVERSE ? T - 1 - n : n; };
    int64_t n = 0;
    for (; n + U <= T; n += U) {
        float x[U][NF], rt[U][kTabN];
        unsigned m[U][kNB];
#pragma unroll
        for (int u = 0; u < U; ++u) load(row(n + u), x[u], m[u], rt[u]);
#pragma unroll
        for (int u = 0; u < U; ++u) step(row(n + u), x[u], m[u], rt[u]);
    }
    for (; n < T; ++n) {
        float x[NF], rt[kTabN];
        unsigned m[kNB];
        load(row(n), x, m, rt);
        step(row(n), x, m, rt);
    }
}

// Host: opts Kernel into Pipe's dynamic shared memory, launches it on `grid` CTAs of Pipe::kThreads and checks the
// launch.  The opt-in record is keyed by the kernel itself: several scan kernels share one function type.
template <class Pipe, auto Kernel, class... A>
int launch_scan(unsigned grid, cudaStream_t stream, A... args) {
    static SmemOptIn opt;
    if (int rc = opt.ensure(Kernel, Pipe::kSmemBytes)) return rc;
    Kernel<<<grid, Pipe::kThreads, Pipe::kSmemBytes, stream>>>(args...);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

}  // namespace hpcrll
