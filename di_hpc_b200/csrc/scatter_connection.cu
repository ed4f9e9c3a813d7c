// scatter_connection.cu -- ScatterConnection (AlphaStar-style entity scatter) forward and backward for sm_90a.
//
// Semantics: hpc_rll/origin/scatter_connection.py (torch on the CPU), exposed by hpc_rll/torch_utils/network/
// scatter_connection.py:  x (B,M,N) fp32, location (B,M,2) int64 (y, x)  ->  out (B,N,H,W)
//   out[b,:,y,x] = 0 where no entity lands;
//   cover: the row of the entity with the LARGEST m among those that land on the cell;
//   add:   the sequential fp32 sum over those entities in increasing m, starting from +0.0.
// Backward (both modes): grad_x[b,m,:] = grad_out[b,:,y_m,x_m]  (torch's derivative of scatter / scatter_add w.r.t. src).
// Deliberate deviation (DESIGN.md section 7): an entity with y outside [0,H) or x outside [0,W) is dropped -- it writes
// nothing and its gradient is zero (origin flattens b*HW + y*W + x unchecked and writes into a neighbouring sample/row).
//
// Both passes are deterministic and use no atomics of any kind:
//   forward  one CTA owns (sample b, channel chunk, cell tile).  It compacts the entities of b that land in the tile
//            (block-wide prefix scan, m order kept), ranks them by (cell, m) in shared memory, stages their x rows in
//            that order and then walks the cells with contiguous (float4 where aligned) stores: every output element is
//            written exactly once -- no memset followed by a scatter.  Each thread finds a cell's entity run once and
//            reuses it across the channel chunk.  M > 1024 is handled in passes of 1024 entities (later passes
//            read-modify-write only the cells they touch, in m order, so the result is the same).
//   backward a gather.  Dense regime (many entities per cell-plane byte): the CTA stages grad_out[b, n0:n0+NC, :]
//            through shared memory with coalesced loads; sparse regime: each entity reads its own 32-byte sectors.
//            The regime follows from the shape (8*M >= H*W and the plane slab fits), never from a user option.
#include <algorithm>

#include "common.cuh"

namespace hpcrll {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunk = 1024;                   // entities per forward pass
constexpr int kPerThread = kChunk / kThreads;  // consecutive entities per thread in the compaction
constexpr int kIdxBits = 10;                   // composite key = local cell << 10 | compacted index
constexpr int kMaxTile = 4096;                 // cells per forward CTA
constexpr int kStageBytes = 96 * 1024;         // forward: staged x rows
constexpr int kSlabBytes = 64 * 1024;          // backward dense regime: staged grad_out planes
constexpr int kRowsInFlight = 8;               // global loads a thread issues before it stores them to shared memory

struct FwdArgs {
    const float* x;
    const int64_t* loc;
    float* out;
    int64_t M, N, H, W, HW;
    int nc_max;  // channels per CTA
    int stride;  // row pitch of the staged x rows (odd: conflict-free column reads)
    int tile;    // cells per CTA
    int mc;      // entity capacity of the shared-memory arrays (min(M, kChunk) rounded up to 4)
    int64_t ntiles, nchunks;
};

__device__ __forceinline__ int64_t cell_of(const int64_t* loc, int64_t e, int64_t H, int64_t W) {
    const int64_t y = loc[2 * e], x = loc[2 * e + 1];
    return (y >= 0 && y < H && x >= 0 && x < W) ? y * W + x : -1;
}

// value of a cell whose sorted entities are [r0, r1), given its value so far (0 in the first pass)
template <bool ADD>
__device__ __forceinline__ float run_value(float acc, int r0, int r1, const float* xn, int stride) {
    if (ADD) {
        for (int r = r0; r < r1; ++r) acc += xn[r * stride];
        return acc;
    }
    return r1 > r0 ? xn[(r1 - 1) * stride] : acc;
}

template <bool VEC, bool ADD>
__global__ void __launch_bounds__(kThreads) scatter_conn_fwd_kernel(const FwdArgs a) {
    constexpr int V = VEC ? 4 : 1;
    extern __shared__ __align__(16) unsigned char smem[];
    uint32_t* comp = reinterpret_cast<uint32_t*>(smem);  // mc + 4 (sentinel padding to a multiple of 4)
    int* ment = reinterpret_cast<int*>(comp + a.mc + 4);  // compacted index -> entity within the pass
    int* scell = ment + a.mc;                             // sorted position -> local cell
    int* srow = scell + a.mc;                             // sorted position -> entity within the pass
    int* wsum = srow + a.mc;                              // per-warp counts of the compaction scan
    float* xs = reinterpret_cast<float*>(wsum + 16);      // staged x rows, sorted order, pitch a.stride

    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    int64_t blk = blockIdx.x;
    const int64_t tile = blk % a.ntiles;
    blk /= a.ntiles;
    const int64_t chunk = blk % a.nchunks;
    const int64_t b = blk / a.nchunks;
    const int64_t c0 = tile * a.tile;
    const int tile_len = static_cast<int>(min(static_cast<int64_t>(a.tile), a.HW - c0));
    const int64_t n0 = chunk * a.nc_max;
    const int nc = static_cast<int>(min(static_cast<int64_t>(a.nc_max), a.N - n0));
    // work split of the write phase: G groups of V cells; with fewer groups than threads, P threads share a group's
    // channels so that the whole CTA stores
    const int G = tile_len / V;
    const int P = G >= kThreads ? 1 : kThreads / G;
    const int part = P > 1 ? t / G : 0;
    const int g0 = P > 1 ? t % G : t;
    const int gstep = P > 1 ? G : kThreads;

    const int64_t* __restrict__ loc = a.loc + b * a.M * 2;
    const float* __restrict__ xb = a.x + b * a.M * a.N + n0;
    float* __restrict__ ob = a.out + (b * a.N + n0) * a.HW + c0;

    for (int64_t m0 = 0;;) {
        const int cnt = static_cast<int>(min(static_cast<int64_t>(kChunk), a.M - m0));  // 0 when M == 0
        // 1. entities t*4 .. t*4+3 of this pass that land in the tile (local cell, or -1)
        int lc[kPerThread];
        int mine = 0;
#pragma unroll
        for (int i = 0; i < kPerThread; ++i) {
            const int e = t * kPerThread + i;
            lc[i] = -1;
            if (e < cnt) {
                const int64_t c = cell_of(loc, m0 + e, a.H, a.W);
                if (c >= c0 && c - c0 < tile_len) lc[i] = static_cast<int>(c - c0);  // dropped entities: c == -1
            }
            mine += lc[i] >= 0;
        }
        // 2. stable compaction: block-wide exclusive scan of the per-thread counts
        int incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();  // also: every thread has finished reading the previous pass's arrays
        int off = 0, K = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
            const int s = wsum[w];
            off += w < warp ? s : 0;
            K += s;
        }
        int pos = off + incl - mine;
#pragma unroll
        for (int i = 0; i < kPerThread; ++i) {
            if (lc[i] >= 0) {
                comp[pos] = (static_cast<uint32_t>(lc[i]) << kIdxBits) | static_cast<uint32_t>(pos);
                ment[pos] = t * kPerThread + i;
                ++pos;
            }
        }
        const int K4 = (K + 3) & ~3;
        if (t < K4 - K) comp[K + t] = 0xffffffffu;  // larger than every key: never counted
        __syncthreads();
        // 3. rank by (cell, m): the keys are distinct, so the rank is the number of smaller keys
        const uint4* comp4 = reinterpret_cast<const uint4*>(comp);
        for (int e = t; e < K; e += kThreads) {
            const uint32_t key = comp[e];
            int r = 0;
            for (int j = 0; j < K4 / 4; ++j) {
                const uint4 q = comp4[j];
                r += (q.x < key) + (q.y < key) + (q.z < key) + (q.w < key);
            }
            scell[r] = static_cast<int>(key >> kIdxBits);
            srow[r] = ment[e];
        }
        __syncthreads();
        // 4. stage the x rows of the tile's entities in sorted order: lane = channel (nc <= 32), kRowsInFlight rows
        //    per warp with all their loads issued before the first shared-memory store
        for (int r0 = warp * kRowsInFlight; r0 < K; r0 += kWarps * kRowsInFlight) {
            float v[kRowsInFlight];
#pragma unroll
            for (int i = 0; i < kRowsInFlight; ++i) {
                const int r = r0 + i;
                v[i] = r < K && lane < nc ? __ldg(xb + (m0 + srow[r]) * a.N + lane) : 0.f;
            }
#pragma unroll
            for (int i = 0; i < kRowsInFlight; ++i)
                if (r0 + i < K && lane < nc) xs[(r0 + i) * a.stride + lane] = v[i];
        }
        __syncthreads();
        // 5. write the tile: a cell's value is the last row of its run (cover), the in-order sum (add), or 0
        const bool first = m0 == 0;
        if (part < P) {
            for (int g = g0; g < G; g += gstep) {
                const int lcell = g * V;
                int lo = 0, hi = K;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (scell[mid] < lcell) lo = mid + 1;
                    else hi = mid;
                }
                int bnd[V + 1];  // cell lcell + j holds sorted entities [bnd[j], bnd[j+1])
                bnd[0] = lo;
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    int p = bnd[j];
                    while (p < K && scell[p] == lcell + j) ++p;
                    bnd[j + 1] = p;
                }
                if (!first && bnd[V] == lo) continue;  // a later pass leaves cells it does not touch alone
                for (int n = part; n < nc; n += P) {
                    float* dst = ob + static_cast<int64_t>(n) * a.HW + lcell;
                    float v[V];
                    if (first) {
#pragma unroll
                        for (int j = 0; j < V; ++j) v[j] = 0.f;
                    } else if constexpr (VEC) {
                        const float4 o = *reinterpret_cast<const float4*>(dst);
                        v[0] = o.x;
                        v[1] = o.y;
                        v[2] = o.z;
                        v[3] = o.w;
                    } else {
                        v[0] = dst[0];
                    }
                    const float* xn = xs + n;
                    v[0] = run_value<ADD>(v[0], bnd[0], bnd[1], xn, a.stride);
                    if constexpr (VEC) {
                        v[1] = run_value<ADD>(v[1], bnd[1], bnd[2], xn, a.stride);
                        v[2] = run_value<ADD>(v[2], bnd[2], bnd[3], xn, a.stride);
                        v[3] = run_value<ADD>(v[3], bnd[3], bnd[4], xn, a.stride);
                    }
                    if constexpr (VEC) {
                        *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                    } else {
                        dst[0] = v[0];
                    }
                }
            }
        }
        m0 += kChunk;
        if (m0 >= a.M) break;
    }
}

struct BwdArgs {
    const float* grad_out;
    const int64_t* loc;
    float* grad_x;
    int64_t B, M, N, H, W, HW;
    int nc_max;  // dense: channels per CTA
    int stride;  // dense: row pitch of the staged planes (odd)
    int lanes;   // lanes per entity row (power of two <= 32)
    int lshift;  // log2(lanes)
    int64_t nchunks;
};

// sparse regime: a group of `lanes` lanes per entity row (b, m); each read is its own 32-byte sector of grad_out
__global__ void __launch_bounds__(kThreads) scatter_conn_bwd_gather_kernel(const BwdArgs a) {
    const int lane = threadIdx.x & 31, sub = lane & (a.lanes - 1);
    const int rows_per_warp = 32 >> a.lshift;
    const int64_t rows = a.B * a.M;
    const int64_t gw = (static_cast<int64_t>(blockIdx.x) * kWarps + (threadIdx.x >> 5)) * rows_per_warp +
                       (lane >> a.lshift);
    const int64_t step = static_cast<int64_t>(gridDim.x) * kWarps * rows_per_warp;
    for (int64_t row = gw; row < rows; row += step) {
        const int64_t b = row / a.M;
        const int64_t cell = cell_of(a.loc, row, a.H, a.W);
        const float* __restrict__ src = a.grad_out + b * a.N * a.HW + cell;
        float* __restrict__ dst = a.grad_x + row * a.N;
        if (cell >= 0) {
            for (int64_t n = sub; n < a.N; n += a.lanes) dst[n] = __ldg(src + n * a.HW);
        } else {
            for (int64_t n = sub; n < a.N; n += a.lanes) dst[n] = 0.f;
        }
    }
}

// dense regime: one CTA per (b, channel chunk) stages the contiguous planes grad_out[b, n0:n0+nc, :] and then gathers
// every entity's row out of shared memory
__global__ void __launch_bounds__(kThreads) scatter_conn_bwd_dense_kernel(const BwdArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    float* slab = reinterpret_cast<float*>(smem);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, sub = lane & (a.lanes - 1);
    const int64_t chunk = blockIdx.x % a.nchunks, b = blockIdx.x / a.nchunks;
    const int64_t n0 = chunk * a.nc_max;
    const int nc = static_cast<int>(min(static_cast<int64_t>(a.nc_max), a.N - n0));
    const int hw = static_cast<int>(a.HW);  // the dense regime needs nc * HW floats in shared memory
    const float* __restrict__ src = a.grad_out + (b * a.N + n0) * a.HW;
    for (int i0 = t; i0 < nc * hw; i0 += kThreads * kRowsInFlight) {
        float v[kRowsInFlight];
#pragma unroll
        for (int k = 0; k < kRowsInFlight; ++k) {
            const int i = i0 + k * kThreads;
            v[k] = i < nc * hw ? __ldg(src + i) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < kRowsInFlight; ++k) {
            const int i = i0 + k * kThreads, j = i / hw;
            if (i < nc * hw) slab[j * a.stride + (i - j * hw)] = v[k];
        }
    }
    __syncthreads();
    const int rows_per_warp = 32 >> a.lshift;
    const int64_t* __restrict__ loc = a.loc + b * a.M * 2;
    float* __restrict__ gx = a.grad_x + b * a.M * a.N + n0;
    for (int64_t m = static_cast<int64_t>(warp) * rows_per_warp + (lane >> a.lshift); m < a.M;
         m += kWarps * rows_per_warp) {
        const int64_t cell = cell_of(loc, m, a.H, a.W);
        float* dst = gx + m * a.N;
        for (int j = sub; j < nc; j += a.lanes) dst[j] = cell >= 0 ? slab[j * a.stride + cell] : 0.f;
    }
}

SmemOptIn g_fwd_opt[4];
SmemOptIn g_bwd_opt;

int lanes_for(int64_t n) {
    int l = 1;
    while (l < 32 && l < n) l <<= 1;
    return l;
}
int log2i(int v) {
    int s = 0;
    while ((1 << s) < v) ++s;
    return s;
}

bool mul_ok(int64_t a, int64_t b, int64_t* out) { return !__builtin_mul_overflow(a, b, out); }

int check_sizes(int64_t B, int64_t M, int64_t N, int64_t H, int64_t W, int64_t* HW) {
    HPC_REQUIRE(B >= 0 && M >= 0 && N >= 0 && H >= 0 && W >= 0,
                "scatter_connection: negative size (B=%lld M=%lld N=%lld H=%lld W=%lld)", (long long)B, (long long)M,
                (long long)N, (long long)H, (long long)W);
    int64_t bm, bm2, bmn, bn, bnhw;
    HPC_REQUIRE(mul_ok(H, W, HW) && mul_ok(B, M, &bm) && mul_ok(bm, 2, &bm2) && mul_ok(bm, N, &bmn) &&
                    mul_ok(B, N, &bn) && mul_ok(bn, *HW, &bnhw),
                "scatter_connection: sizes overflow 64-bit indexing");
    return HPC_RLL_OK;
}

}  // namespace

int scatter_connection_forward(const float* x, const int64_t* location, float* out, int64_t B, int64_t M, int64_t N,
                               int64_t H, int64_t W, int mode, cudaStream_t stream) {
    int64_t HW = 0;
    if (int rc = check_sizes(B, M, N, H, W, &HW)) return rc;
    HPC_REQUIRE(mode == HPC_RLL_SCATTER_COVER || mode == HPC_RLL_SCATTER_ADD, "scatter_connection: unknown mode %d",
                mode);
    HPC_REQUIRE((x || B * M * N == 0) && (location || B * M == 0) && (out || B * N * HW == 0),
                "scatter_connection_forward: null pointer");
    if (B * N * HW == 0) return HPC_RLL_OK;
    FwdArgs a;
    a.x = x;
    a.loc = location;
    a.out = out;
    a.M = M;
    a.N = N;
    a.H = H;
    a.W = W;
    a.HW = HW;
    a.mc = static_cast<int>((std::min<int64_t>(std::max<int64_t>(M, 1), kChunk) + 3) & ~int64_t(3));
    int nc = static_cast<int>(std::min<int64_t>(N, 32));  // <= 32: one lane per channel when staging x rows
    while (nc > 1 && static_cast<int64_t>(a.mc) * (nc | 1) * 4 > kStageBytes) nc >>= 1;
    a.nc_max = nc;
    a.stride = nc | 1;
    a.nchunks = (N + nc - 1) / nc;
    const bool vec = HW % 4 == 0 && aligned16(out);
    int tile = static_cast<int>(std::min<int64_t>(HW, kMaxTile));
    if (vec) tile = (tile + 3) & ~3;
    const int64_t want = 4LL * sm_count();
    while (B * a.nchunks * ((HW + tile - 1) / tile) < want && tile >= 512) tile = vec ? ((tile / 2 + 3) & ~3) : tile / 2;
    a.tile = tile;
    a.ntiles = (HW + tile - 1) / tile;
    const int64_t blocks = B * a.nchunks * a.ntiles;
    HPC_REQUIRE(blocks <= INT32_MAX, "scatter_connection_forward: problem too large for one launch");
    const int smem = (a.mc + 4) * 4 + 3 * a.mc * 4 + 16 * 4 + a.mc * a.stride * 4;
    const bool add = mode == HPC_RLL_SCATTER_ADD;
    auto launch = [&](auto kernel, SmemOptIn& opt) -> int {
        if (int rc = opt.ensure(kernel, smem)) return rc;
        kernel<<<static_cast<unsigned>(blocks), kThreads, smem, stream>>>(a);
        return HPC_RLL_OK;
    };
    int rc;
    if (vec) rc = add ? launch(scatter_conn_fwd_kernel<true, true>, g_fwd_opt[0])
                      : launch(scatter_conn_fwd_kernel<true, false>, g_fwd_opt[1]);
    else rc = add ? launch(scatter_conn_fwd_kernel<false, true>, g_fwd_opt[2])
                  : launch(scatter_conn_fwd_kernel<false, false>, g_fwd_opt[3]);
    if (rc) return rc;
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

int scatter_connection_backward(const float* grad_out, const int64_t* location, float* grad_x, int64_t B, int64_t M,
                                int64_t N, int64_t H, int64_t W, cudaStream_t stream) {
    int64_t HW = 0;
    if (int rc = check_sizes(B, M, N, H, W, &HW)) return rc;
    HPC_REQUIRE((grad_out || B * N * HW == 0) && (location || B * M == 0) && (grad_x || B * M * N == 0),
                "scatter_connection_backward: null pointer");
    if (B * M * N == 0) return HPC_RLL_OK;
    BwdArgs a;
    a.grad_out = grad_out;
    a.loc = location;
    a.grad_x = grad_x;
    a.B = B;
    a.M = M;
    a.N = N;
    a.H = H;
    a.W = W;
    a.HW = HW;
    // dense when a 32-byte sector per (entity, channel) would read more than the planes themselves, and
    // enough channels of the planes fit in shared memory
    int nc = static_cast<int>(std::min<int64_t>(N, 32));
    while (nc > 1 && static_cast<int64_t>(nc) * (HW | 1) * 4 > kSlabBytes) nc >>= 1;
    const bool dense = M >= (HW + 7) / 8 && static_cast<int64_t>(nc) * (HW | 1) * 4 <= kSlabBytes &&
                       nc >= std::min<int64_t>(N, 4);
    if (dense) {
        a.nc_max = nc;
        a.stride = static_cast<int>(HW | 1);
        a.nchunks = (N + nc - 1) / nc;
        a.lanes = lanes_for(nc);
        a.lshift = log2i(a.lanes);
        const int64_t blocks = B * a.nchunks;
        HPC_REQUIRE(blocks <= INT32_MAX, "scatter_connection_backward: problem too large for one launch");
        const int smem = nc * a.stride * 4;
        if (int rc = g_bwd_opt.ensure(scatter_conn_bwd_dense_kernel, smem)) return rc;
        scatter_conn_bwd_dense_kernel<<<static_cast<unsigned>(blocks), kThreads, smem, stream>>>(a);
    } else {
        a.nc_max = 0;
        a.stride = 0;
        a.nchunks = 1;
        a.lanes = lanes_for(N);
        a.lshift = log2i(a.lanes);
        const int64_t rows_per_cta = static_cast<int64_t>(kWarps) * (32 >> a.lshift);
        const int64_t blocks = std::min<int64_t>((B * M + rows_per_cta - 1) / rows_per_cta, 64LL * sm_count());
        scatter_conn_bwd_gather_kernel<<<static_cast<unsigned>(blocks), kThreads, 0, stream>>>(a);
    }
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_scatter_connection_forward(const float* x, const int64_t* location, float* out, int64_t B, int64_t M,
                                       int64_t N, int64_t H, int64_t W, int mode, void* stream) {
    HPC_NVTX("scatter_connection_forward");
    return hpcrll::scatter_connection_forward(x, location, out, B, M, N, H, W, mode, hpcrll::as_stream(stream));
}

int hpc_rll_scatter_connection_backward(const float* grad_out, const int64_t* location, float* grad_x, int64_t B,
                                        int64_t M, int64_t N, int64_t H, int64_t W, void* stream) {
    HPC_NVTX("scatter_connection_backward");
    return hpcrll::scatter_connection_backward(grad_out, location, grad_x, B, M, N, H, W, hpcrll::as_stream(stream));
}

}  // extern "C"
