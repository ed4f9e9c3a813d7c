// scan_pipe.cuh -- TMA-staged column-scan pipeline shared by every T-recurrence of the path
// (GAE fwd/bwd, TD-lambda, V-trace return, UPGO return).
//
// Layout reminder: all scan operands are (T,B) fp32 with B contiguous.  One CTA owns a tile of BT
// adjacent columns for ALL of T.  A producer lane streams (TT x BT) boxes of each of the NIN input
// tensors through an ST-deep shared-memory ring with cp.async.bulk.tensor (TMA) + mbarrier
// expect-tx; BT consumer threads (one per column, bank-conflict-free row reads) walk the rows of
// the box in scan order and carry the recurrence state in registers across boxes.  Optional
// per-row constants (`rowtab`, e.g. GAE's denominators d_t and 1/d_t) ride in the same stage as a 1-D bulk copy.
//
//   * no thread ever issues a global load in the steady state: all input traffic is bulk async,
//     ST-1 boxes per CTA are in flight while one is being consumed
//   * consumers never __syncthreads(): full[]/empty[] mbarriers only
//   * rows/columns outside the tensor are zero-filled by the TMA unit; callers mask their stores
//
// The reference walks the same recurrence with one thread per column issuing dependent scalar
// loads (include/hpc/rll/cuda/rl_utils/gae_kernel.h:17-27, td_lambda_kernel.h:17-31,
// vtrace_kernel.h:161-180, upgo_kernel.h:18-35); this file is the TMA-pipelined re-design of that loop.
#pragma once
#include "common.cuh"

namespace hpcrll {

template <int NIN>
struct TmapPack {
    CUtensorMap m[NIN];
};

template <int NIN, int BT, int TT, int ST, int NTAB>
struct ScanPipe {
    static_assert(BT % 32 == 0, "column tile must be whole warps");
    static_assert(TT % 4 == 0, "row tile must keep the row table 16B aligned");
    static constexpr int kConsumerWarps = BT / 32;
    static constexpr int kThreads = BT + 32;  // + one producer warp
    static constexpr int kBoxBytes = TT * BT * 4;
    static constexpr int kTabBytes = ((TT * NTAB * 4 + 127) / 128) * 128;  // NTAB fp32 constants per row
    static constexpr int kStageBytes = NIN * kBoxBytes + kTabBytes;
    static constexpr uint32_t kTxBytes = NIN * kBoxBytes + TT * NTAB * 4;
    static constexpr int kTabN = NTAB > 0 ? NTAB : 1;
    static constexpr int kSmemBytes = ST * kStageBytes + 2 * ST * 8;

    // Runs the whole pipeline for the column tile starting at col0.
    //   body.step(t, x, rt): called by consumer thread c (column col0+c) for t in scan order,
    //   x[k] = input k at (t, col0+c), rt[k] = rowtab[t*NTAB + k] (per-row constants).
    template <bool REVERSE, class Body>
    static __device__ __forceinline__ void run(const TmapPack<NIN>& maps, const float* __restrict__ rowtab, int T,
                                               int col0, Body& body) {
        // dynamic shared memory starts at the CTA's shared window base (no static smem in these
        // kernels), so the declared alignment holds; keeping the pointer un-cast lets the compiler
        // emit LDS (shared-space) loads instead of generic ones.
        extern __shared__ __align__(1024) unsigned char smem[];
        uint64_t* full = reinterpret_cast<uint64_t*>(smem + ST * kStageBytes);
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
                for (int k = 0; k < NIN; ++k) prefetch_tmap(&maps.m[k]);
                for (int it = 0; it < nT; ++it) {
                    const int s = it % ST;
                    if (it >= ST) mbar_wait(&empty[s], ((it / ST) & 1) ^ 1);
                    const int j = REVERSE ? nT - 1 - it : it;
                    unsigned char* st = smem + s * kStageBytes;
                    mbar_arrive_expect_tx(&full[s], kTxBytes);
#pragma unroll
                    for (int k = 0; k < NIN; ++k) tma_load_2d(st + k * kBoxBytes, &maps.m[k], col0, j * TT, &full[s]);
                    if (NTAB > 0) bulk_load_1d(st + NIN * kBoxBytes, rowtab + j * TT * NTAB, TT * NTAB * 4, &full[s]);
                }
            }
            return;
        }

        // -------------------- consumers: one column per thread --------------------
        const int c = tid;
        for (int it = 0; it < nT; ++it) {
            const int s = it % ST;
            const int j = REVERSE ? nT - 1 - it : it;
            const float* st = reinterpret_cast<const float*>(smem + s * kStageBytes);
            const float* tab = st + NIN * TT * BT;
            mbar_wait(&full[s], (it / ST) & 1);
            const int rows = min(TT, T - j * TT);
            if (rows == TT) {
#pragma unroll
                for (int ii = 0; ii < TT; ++ii) {
                    const int i = REVERSE ? TT - 1 - ii : ii;
                    float x[NIN];
#pragma unroll
                    for (int k = 0; k < NIN; ++k) x[k] = st[(k * TT + i) * BT + c];
                    float rt[kTabN];
#pragma unroll
                    for (int k = 0; k < NTAB; ++k) rt[k] = tab[i * NTAB + k];
                    body.step(j * TT + i, x, rt);
                }
            } else {
                for (int ii = 0; ii < rows; ++ii) {
                    const int i = REVERSE ? rows - 1 - ii : ii;
                    float x[NIN];
#pragma unroll
                    for (int k = 0; k < NIN; ++k) x[k] = st[(k * TT + i) * BT + c];
                    float rt[kTabN];
#pragma unroll
                    for (int k = 0; k < NTAB; ++k) rt[k] = tab[i * NTAB + k];
                    body.step(j * TT + i, x, rt);
                }
            }
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(&empty[s]);
        }
    }
};

// ScanPipeOut -- the same pipeline with the OUTPUT side staged as well: consumers put their per-step results
// into a (TT x BT) shared-memory box per output tensor and one thread hands finished boxes to the TMA unit
// (cp.async.bulk.tensor store), double-buffered, so HBM sees whole (TT x BT) write bursts instead of one
// 128-byte line per warp per row.  Costs one named barrier over the consumer threads per box.
//   body.step(t, x, rt, o): as above, plus o[k] = value of output k at (t, col0+c)
//   rows/columns outside an output tensor map are clipped by the TMA unit
template <int NIN, int NOUT, int BT, int TT, int ST, int NTAB>
struct ScanPipeOut {
    using In = ScanPipe<NIN, BT, TT, ST, NTAB>;
    static constexpr int kThreads = In::kThreads;
    static constexpr int kBoxBytes = In::kBoxBytes;
    static constexpr int kStageBytes = In::kStageBytes;
    static constexpr int kOutBytes = 2 * NOUT * kBoxBytes;  // two buffers per output
    static constexpr int kSmemBytes = ST * kStageBytes + kOutBytes + 2 * ST * 8;

    template <bool REVERSE, class Body>
    static __device__ __forceinline__ void run(const TmapPack<NIN>& maps, const TmapPack<NOUT>& omaps,
                                               const float* __restrict__ rowtab, int T, int col0, Body& body) {
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
                mbar_init(&empty[s], In::kConsumerWarps);
            }
            fence_mbar_init();
        }
        __syncthreads();

        if (tid >= BT) {
            if (tid == BT) {
#pragma unroll
                for (int k = 0; k < NIN; ++k) prefetch_tmap(&maps.m[k]);
                for (int it = 0; it < nT; ++it) {
                    const int s = it % ST;
                    if (it >= ST) mbar_wait(&empty[s], ((it / ST) & 1) ^ 1);
                    const int j = REVERSE ? nT - 1 - it : it;
                    unsigned char* st = smem + s * kStageBytes;
                    mbar_arrive_expect_tx(&full[s], In::kTxBytes);
#pragma unroll
                    for (int k = 0; k < NIN; ++k) tma_load_2d(st + k * kBoxBytes, &maps.m[k], col0, j * TT, &full[s]);
                    if (NTAB > 0) bulk_load_1d(st + NIN * kBoxBytes, rowtab + j * TT * NTAB, TT * NTAB * 4, &full[s]);
                }
            }
            return;
        }

        const int c = tid;
        if (tid == 0) {
#pragma unroll
            for (int k = 0; k < NOUT; ++k) prefetch_tmap(&omaps.m[k]);
        }
        for (int it = 0; it < nT; ++it) {
            const int s = it % ST;
            const int j = REVERSE ? nT - 1 - it : it;
            const float* st = reinterpret_cast<const float*>(smem + s * kStageBytes);
            const float* tab = st + NIN * TT * BT;
            float* ob = obuf + (it & 1) * (NOUT * TT * BT);
            mbar_wait(&full[s], (it / ST) & 1);
            const int rows = min(TT, T - j * TT);
            if (rows == TT) {
#pragma unroll
                for (int ii = 0; ii < TT; ++ii) {
                    const int i = REVERSE ? TT - 1 - ii : ii;
                    float x[NIN], o[NOUT];
#pragma unroll
                    for (int k = 0; k < NIN; ++k) x[k] = st[(k * TT + i) * BT + c];
                    float rt[In::kTabN];
#pragma unroll
                    for (int k = 0; k < NTAB; ++k) rt[k] = tab[i * NTAB + k];
                    body.step(j * TT + i, x, rt, o);
#pragma unroll
                    for (int k = 0; k < NOUT; ++k) ob[(k * TT + i) * BT + c] = o[k];
                }
            } else {
                for (int ii = 0; ii < rows; ++ii) {
                    const int i = REVERSE ? rows - 1 - ii : ii;
                    float x[NIN], o[NOUT];
#pragma unroll
                    for (int k = 0; k < NIN; ++k) x[k] = st[(k * TT + i) * BT + c];
                    float rt[In::kTabN];
#pragma unroll
                    for (int k = 0; k < NTAB; ++k) rt[k] = tab[i * NTAB + k];
                    body.step(j * TT + i, x, rt, o);
#pragma unroll
                    for (int k = 0; k < NOUT; ++k) ob[(k * TT + i) * BT + c] = o[k];
                }
            }
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(&empty[s]);  // input stage free again
            // hand the finished output box to the TMA unit.  The buffer written NEXT (the other one) was
            // stored one box ago: thread 0 waits for that store to have read it before anybody passes the barrier.
            fence_proxy_async_smem();
            if (tid == 0) bulk_wait_group_read<0>();
            named_bar_sync(1, BT);
            if (tid == 0) {
#pragma unroll
                for (int k = 0; k < NOUT; ++k) tma_store_2d(&omaps.m[k], col0, j * TT, ob + k * TT * BT);
                bulk_commit_group();
            }
        }
        if (tid == 0) bulk_wait_group<0>();
    }
};

// ScanPipeMix -- ScanPipeOut with byte-wide inputs next to the fp32 ones (episode masks) and no row table.
// maps.m[0..NF) are fp32 (TT x BT) boxes, maps.m[NF..NF+NB) uint8 (TT x BT) boxes (a byte box of a multiple of 32
// columns and 4 rows is a multiple of 128 bytes, so every box of a stage stays 128-byte aligned).  Outputs are fp32
// and TMA-stored as in ScanPipeOut.
//   body.step(t, x, m, o): x[k] = fp32 input k, m[k] = byte input k at (t, col0+c); o[k] = output k
template <int NF, int NB, int NOUT, int BT, int TT, int ST>
struct ScanPipeMix {
    static_assert(BT % 32 == 0, "column tile must be whole warps");
    static_assert(TT % 4 == 0, "byte boxes must stay 128-byte aligned");
    static constexpr int kConsumerWarps = BT / 32;
    static constexpr int kThreads = BT + 32;  // + one producer warp
    static constexpr int kBoxBytes = TT * BT * 4;
    static constexpr int kByteBoxBytes = TT * BT;
    static constexpr int kStageBytes = NF * kBoxBytes + NB * kByteBoxBytes;
    static constexpr uint32_t kTxBytes = kStageBytes;
    static constexpr int kNB = NB > 0 ? NB : 1;
    static constexpr int kOutBytes = 2 * NOUT * kBoxBytes;  // two buffers per output
    static constexpr int kSmemBytes = ST * kStageBytes + kOutBytes + 2 * ST * 8;

    template <bool REVERSE, class Body>
    static __device__ __forceinline__ void run(const TmapPack<NF + NB>& maps, const TmapPack<NOUT>& omaps, int T,
                                               int col0, Body& body) {
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
                }
            }
            return;
        }

        const int c = tid;
        if (tid == 0) {
#pragma unroll
            for (int k = 0; k < NOUT; ++k) prefetch_tmap(&omaps.m[k]);
        }
        for (int it = 0; it < nT; ++it) {
            const int s = it % ST;
            const int j = REVERSE ? nT - 1 - it : it;
            const float* st = reinterpret_cast<const float*>(smem + s * kStageBytes);
            const unsigned char* sb = smem + s * kStageBytes + NF * kBoxBytes;
            float* ob = obuf + (it & 1) * (NOUT * TT * BT);
            mbar_wait(&full[s], (it / ST) & 1);
            const int rows = min(TT, T - j * TT);
            if (rows == TT) {
#pragma unroll
                for (int ii = 0; ii < TT; ++ii) {
                    const int i = REVERSE ? TT - 1 - ii : ii;
                    float x[NF], o[NOUT];
                    unsigned m[kNB];
#pragma unroll
                    for (int k = 0; k < NF; ++k) x[k] = st[(k * TT + i) * BT + c];
#pragma unroll
                    for (int k = 0; k < NB; ++k) m[k] = sb[(k * TT + i) * BT + c];
                    body.step(j * TT + i, x, m, o);
#pragma unroll
                    for (int k = 0; k < NOUT; ++k) ob[(k * TT + i) * BT + c] = o[k];
                }
            } else {
                for (int ii = 0; ii < rows; ++ii) {
                    const int i = REVERSE ? rows - 1 - ii : ii;
                    float x[NF], o[NOUT];
                    unsigned m[kNB];
#pragma unroll
                    for (int k = 0; k < NF; ++k) x[k] = st[(k * TT + i) * BT + c];
#pragma unroll
                    for (int k = 0; k < NB; ++k) m[k] = sb[(k * TT + i) * BT + c];
                    body.step(j * TT + i, x, m, o);
#pragma unroll
                    for (int k = 0; k < NOUT; ++k) ob[(k * TT + i) * BT + c] = o[k];
                }
            }
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(&empty[s]);
            fence_proxy_async_smem();
            if (tid == 0) bulk_wait_group_read<0>();
            named_bar_sync(1, BT);
            if (tid == 0) {
#pragma unroll
                for (int k = 0; k < NOUT; ++k) tma_store_2d(&omaps.m[k], col0, j * TT, ob + k * TT * BT);
                bulk_commit_group();
            }
        }
        if (tid == 0) bulk_wait_group<0>();
    }
};

}  // namespace hpcrll
