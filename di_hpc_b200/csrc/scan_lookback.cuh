// scan_lookback.cuh -- single-launch T-split of the column scans for the SMALL-BATCH regime (round 2).
//
// The column-scan kernels (scan_pipe.cuh) give every column tile ONE CTA for all of T: at the reference's own test
// shapes (T=1024, B=64: tests/test_gae.py:10-11, tests/test_tdlambda.py:10-11) that is 2 CTAs on a 132-SM H100 and
// the scan is a 1024-step dependent chain per thread.  Every recurrence of the path is first-order affine,
// x_t = a_t * x_{t+-1} + b_t, so T can be cut into S segments that run as independent CTAs:
//
//   grid = S segments x (B/32) column tiles, one warp per CTA, lane = column
//   1. the CTA takes a ticket (atomicAdd) -> its position k in SCAN ORDER; tickets are handed out in launch order, so
//      every segment a CTA will ever wait for already holds an earlier ticket, i.e. is running or done: no deadlock
//      whatever the residency (the classic decoupled-look-back ordering argument)
//   2. it loads its rows into shared memory (coalesced, all loads in flight at once), scans them from a ZERO carry
//      and PUBLISHES the segment aggregate (A = prod a_t, Bagg = result) per column
//   3. LOOK-BACK: it folds the aggregates of segments 0..k-1 (32 loads in flight at a time, each polled until its
//      tag shows this launch's epoch) into its carry-in:  c <- A_j * c + B_j
//   4. it re-scans its rows from shared memory with the true carry and writes the outputs.
//
// Aggregates are 64-bit words (epoch << 32 | float bits): one relaxed 8-byte store/load is atomic, so the value and
// its "ready" tag can never be seen torn and no fence is needed.  The epoch lives in DEVICE memory and is bumped by the
// last CTA of every launch (which also resets the ticket counter), so the scratch needs no memset between launches and
// the scheme survives CUDA-graph replay (kernel arguments are frozen at capture; the epoch is not an argument).
// Scratch is library-owned, zero-initialised once per (device, stream): launches that share it are stream-ordered.
//
// Re-association: a segment boundary replaces the sequential rounding of the carry by one fused multiply-add per
// predecessor, so results agree with the serial scan to ~1e-7 relative instead of bit for bit (tests: 2e-6).  The
// wide-batch TMA path stays bit-exact.  SURVEY.md 8(f) item 2; VERDICT r1 item 7.
#pragma once
#include "common.cuh"

namespace hpcrll {

constexpr int kLbCols = 32;      // columns per CTA = one warp
constexpr int kLbChunkRows = 32; // rows staged in shared memory at a time
constexpr int kLbMaxSeg = 64;

struct LbCtl {
    unsigned ticket, done, epoch, pad;
};

struct LbScratch {
    LbCtl* ctl = nullptr;
    unsigned long long* words = nullptr;  // [k][col][2] (A-word, B-word); constant-coefficient ops use the B-word only
    size_t cap_words = 0;
};

struct LbGeom {
    int S = 1;      // segments
    int L = 0;      // rows per segment (multiple of 8)
    int tiles = 0;  // column tiles of kLbCols
};

// host (scan_lookback.cu)
bool lookback_geometry(int op, int64_t T, int64_t B, LbGeom* g);
int lookback_scratch(const LbGeom& g, int64_t B, cudaStream_t stream, LbScratch* out);

#ifdef __CUDACC__

struct LbTile {
    int k;     // position in scan order (0 = first segment scanned)
    int tile;  // column tile
    int vid;   // ticket
    unsigned epoch;
};

__device__ __forceinline__ unsigned long long lb_ld(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void lb_st(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long lb_pack(unsigned epoch, float x) {
    return (static_cast<unsigned long long>(epoch) << 32) | static_cast<unsigned long long>(__float_as_uint(x));
}

// one warp per CTA: lane 0 takes the ticket and reads the epoch, both are broadcast by shuffle.  Grids that are
// certainly co-resident (kLbResidentCtas: 8 one-warp CTAs per SM on 132 SMs; the largest of these kernels stages 20 KB
// of shared memory, 11 CTAs per SM) use blockIdx as their ticket -- every CTA is running, so nobody can wait for one
// that has not started -- and save the atomic's round trip before the first load.
constexpr unsigned kLbResidentCtas = 1024;
__device__ __forceinline__ LbTile lb_begin(LbCtl* ctl, int tiles) {
    unsigned vid = blockIdx.x, epoch = 0;
    if (threadIdx.x == 0) {
        if (gridDim.x > kLbResidentCtas) vid = atomicAdd(&ctl->ticket, 1u);
        asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(epoch) : "l"(&ctl->epoch) : "memory");
    }
    vid = __shfl_sync(0xffffffffu, vid, 0);
    epoch = __shfl_sync(0xffffffffu, epoch, 0);
    LbTile t;
    t.vid = static_cast<int>(vid);
    t.k = t.vid / tiles;
    t.tile = t.vid - t.k * tiles;
    t.epoch = epoch;
    return t;
}

// the last CTA of the launch re-arms the scratch: ticket = done = 0, epoch + 1
__device__ __forceinline__ void lb_end(LbCtl* ctl, int total, unsigned epoch) {
    __syncwarp();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned d = atomicAdd(&ctl->done, 1u);
        if (d == static_cast<unsigned>(total) - 1u) {
            ctl->ticket = 0u;
            ctl->done = 0u;
            __threadfence();
            unsigned e = epoch + 1u;
            if (e == 0u) e = 1u;  // 0 is the "never written" tag of fresh scratch
            asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(&ctl->epoch), "r"(e) : "memory");
        }
    }
}

template <bool CONSTA>
__device__ __forceinline__ void lb_publish(unsigned long long* words, int k, int col, int Bpad, unsigned epoch, float A,
                                           float Bagg) {
    unsigned long long* w = words + (static_cast<size_t>(k) * Bpad + col) * 2;
    if (!CONSTA) lb_st(w, lb_pack(epoch, A));
    lb_st(w + 1, lb_pack(epoch, Bagg));
}

// carry into segment k = F_{k-1}( ... F_0(0)),  F_j(c) = A_j*c + B_j.  CONSTA: every A_j that matters equals AL
// (= a^L: only full-length segments ever feed a successor, see the kernels).
template <bool CONSTA>
__device__ __forceinline__ float lb_fold(const unsigned long long* words, int k, int col, int Bpad, unsigned epoch,
                                         float AL) {
    float c = 0.f;
    constexpr int U = 32;  // loads in flight per round: one L2 round trip folds up to 32 predecessors
    for (int j0 = 0; j0 < k; j0 += U) {
        unsigned long long wa[U], wb[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (j0 + u < k) {
                const unsigned long long* w = words + (static_cast<size_t>(j0 + u) * Bpad + col) * 2;
                if (!CONSTA) wa[u] = lb_ld(w);
                wb[u] = lb_ld(w + 1);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (j0 + u < k) {
                const unsigned long long* w = words + (static_cast<size_t>(j0 + u) * Bpad + col) * 2;
                while (static_cast<unsigned>(wb[u] >> 32) != epoch) wb[u] = lb_ld(w + 1);
                float A = AL;
                if (!CONSTA) {
                    while (static_cast<unsigned>(wa[u] >> 32) != epoch) wa[u] = lb_ld(w);
                    A = __uint_as_float(static_cast<unsigned>(wa[u]));
                }
                c = fmaf(A, c, __uint_as_float(static_cast<unsigned>(wb[u])));
            }
        }
    }
    return c;
}

// stage rows [r0, r0+rows) of one (rows x B) operand into shared memory: dst[i*32 + lane] (time order), zeros beyond B
__device__ __forceinline__ void lb_stage(float* dst, const float* __restrict__ src, int64_t ld, int r0, int rows, int col,
                                         bool valid) {
    const float* p = src + static_cast<int64_t>(r0) * ld + col;
    int i = 0;
    for (; i + 8 <= rows; i += 8) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = valid ? __ldg(p + static_cast<int64_t>(i + u) * ld) : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) dst[(i + u) * kLbCols + threadIdx.x] = v[u];
    }
    for (; i < rows; ++i) dst[i * kLbCols + threadIdx.x] = valid ? __ldg(p + static_cast<int64_t>(i) * ld) : 0.f;
}

// Drives one segment: both passes over the chunks of rows [t0, t1), in scan order.
//   Fac::make(pass, t_edge, carry) -> Body with its boundary state loaded at t_edge (t1 when REVERSE, else t0) and
//                                     the carry; pass 0 gets carry 0 and must not store, pass 1 the folded carry
//   Fac::step(body, t, x)          -> one step; x[k] = operand k at (t, col); Fac loads any per-row constants itself
//   Fac::state(body), Fac::coef(body) -> carried scalar / coefficient of the LAST step (coef ignored when CONSTA)
//   Fac::finish(body, t0, t1)      -> after pass 1: per-segment epilogue (e.g. loss partials, GAE's row T)
template <int NIN, bool REVERSE, bool CONSTA, class Fac>
__device__ __forceinline__ void lb_segment(const Fac& fac, const float* const (&in)[NIN], const int64_t (&ld)[NIN], int t0,
                                           int t1, int col, bool valid, const LbTile& lt, unsigned long long* words,
                                           int Bpad, float AL, float* smem) {
    const int len = t1 - t0;
    const bool single = len <= kLbChunkRows;
    float carry = 0.f;
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {
        auto body = fac.make(pass, REVERSE ? t1 : t0, carry);
        float Aprod = 1.f;
#pragma unroll 1
        for (int done = 0; done < len; done += kLbChunkRows) {
            const int rows = min(kLbChunkRows, len - done);
            const int c0 = REVERSE ? t1 - done - rows : t0 + done;
            if (!(single && pass == 1)) {
                __syncwarp();
#pragma unroll
                for (int k = 0; k < NIN; ++k) lb_stage(smem + k * kLbChunkRows * kLbCols, in[k], ld[k], c0, rows, col, valid);
                __syncwarp();
            }
            int ii = 0;
            for (; ii + 8 <= rows; ii += 8) {  // 8 rows per trip: the shared-memory reads of a trip are issued together
                float x[8][NIN];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int i = REVERSE ? rows - 1 - (ii + u) : ii + u;
#pragma unroll
                    for (int k = 0; k < NIN; ++k) x[u][k] = smem[(k * kLbChunkRows + i) * kLbCols + threadIdx.x];
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int i = REVERSE ? rows - 1 - (ii + u) : ii + u;
                    fac.step(body, c0 + i, x[u]);
                    if (!CONSTA && pass == 0) Aprod *= Fac::coef(body);
                }
            }
            for (; ii < rows; ++ii) {
                const int i = REVERSE ? rows - 1 - ii : ii;
                float x[NIN];
#pragma unroll
                for (int k = 0; k < NIN; ++k) x[k] = smem[(k * kLbChunkRows + i) * kLbCols + threadIdx.x];
                fac.step(body, c0 + i, x);
                if (!CONSTA && pass == 0) Aprod *= Fac::coef(body);
            }
        }
        if (pass == 0) {
            lb_publish<CONSTA>(words, lt.k, col, Bpad, lt.epoch, Aprod, Fac::state(body));
            carry = lb_fold<CONSTA>(words, lt.k, col, Bpad, lt.epoch, AL);
        } else {
            fac.finish(body, t0, t1);
        }
    }
}

#endif  // __CUDACC__

}  // namespace hpcrll
