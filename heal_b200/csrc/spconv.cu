// Sparse 3-D convolution for the SECOND middle encoder (VoxelBackBone8x) and HeightCompression.
// Reference call sites: opencood/models/sub_modules/sparse_backbone_3d.py:48-91 (layer list), :114-130
// (SparseConvTensor + forward), opencood/models/sub_modules/height_compression.py:21-23 (.dense() + fold D into C).
// The reference delegates to spconv (third party, not vendored, not pinned, absent here); semantics restated in
// oracle/sparse_conv.py: cross-correlation evaluated only at active output sites —
//   SubMConv3d   : output sites = input sites;
//   SparseConv3d : output sites = every site reached by at least one active input under the kernel,
//                  out = floor((in + 2*pad - k) / stride) + 1 per axis.
// Design: "output-stationary" rulebook. For each output row we store the input row feeding each of the K
// kernel offsets (-1 if inactive), built with a GPU hash table; the convolution is then ONE gather-GEMM kernel per
// layer with BatchNorm1d folded and ReLU fused, no atomics and no intermediate buffers, deterministic per row.
// Output-site order of a strided conv = order of first generation by (input row, kernel offset), made
// deterministic with atomicMin + a prefix sum (same trick as the voxelizer).
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr uint32_t SP_EMPTY = 0xFFFFFFFFu;
// Every kernel below loops over the LIVE rows (device count) with a grid-stride loop and is launched with a machine-sized grid:
// row capacities are worst-case bounds (2x per strided level), the live counts are a fraction of them, and a capacity-sized
// grid spent most of its blocks on an early exit (HeightCompression: 64 M threads for 3 M elements).
constexpr int SP_MAX_BLOCKS = HEAL_NUM_SMS * 16;
inline unsigned sp_grid(long long work, int threads) {
    long long b = (work + threads - 1) / threads;
    return (unsigned)(b < 1 ? 1 : (b > SP_MAX_BLOCKS ? SP_MAX_BLOCKS : b));
}
constexpr int SP_SCAN = 1024;

struct SpGeom {
    int Z, Y, X;          // spatial shape of the tensor the keys index
    uint32_t tmask; int tshift;
};

__device__ __forceinline__ uint32_t sp_key(int b, int z, int y, int x, const SpGeom& g) {
    return (((uint32_t)b * g.Z + z) * g.Y + y) * g.X + x;
}
__device__ __forceinline__ uint32_t sp_hash(uint32_t key, const SpGeom& g) { return (key * 2654435761u) >> g.tshift; }

__device__ __forceinline__ int sp_lookup(const uint32_t* __restrict__ keys, const int* __restrict__ vals, uint32_t key, const SpGeom& g) {
    uint32_t s = sp_hash(key, g);
    while (true) {
        uint32_t k = keys[s];
        if (k == key) return vals[s];
        if (k == SP_EMPTY) return -1;
        s = (s + 1) & g.tmask;
    }
}

__global__ void k_sp_build(const int4* __restrict__ coords, const int* __restrict__ m_dev, int M, SpGeom g,
                           uint32_t* __restrict__ keys, int* __restrict__ vals) {
    int Md = m_dev ? min(M, m_dev[0]) : M;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Md; i += gridDim.x * blockDim.x) {
        int4 c = coords[i];
        uint32_t key = sp_key(c.x, c.y, c.z, c.w, g);
        uint32_t s = sp_hash(key, g);
        while (true) {
            uint32_t prev = atomicCAS(&keys[s], SP_EMPTY, key);
            if (prev == SP_EMPTY || prev == key) break;
            s = (s + 1) & g.tmask;
        }
        vals[s] = i;
    }
}

struct KShape { int kz, ky, kx, sz, sy, sx, pz, py, px; };

// SubM: nbr[i][k] = row of the input site at coords[i] + (k - center)
__global__ void k_sp_subm_nbr(const int4* __restrict__ coords, const int* __restrict__ m_dev, int M, SpGeom g, KShape ks,
                              const uint32_t* __restrict__ keys, const int* __restrict__ vals, int* __restrict__ nbr) {
    const int K = ks.kz * ks.ky * ks.kx;
    int Md = m_dev ? min(M, m_dev[0]) : M;
    const long long total = (long long)Md * K, stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        int i = (int)(t / K), k = (int)(t % K);
        int dz = k / (ks.ky * ks.kx), dy = (k / ks.kx) % ks.ky, dx = k % ks.kx;
        int4 c = coords[i];
        int z = c.y + dz - ks.kz / 2, y = c.z + dy - ks.ky / 2, x = c.w + dx - ks.kx / 2;
        int r = -1;
        if (z >= 0 && z < g.Z && y >= 0 && y < g.Y && x >= 0 && x < g.X) r = sp_lookup(keys, vals, sp_key(c.x, z, y, x, g), g);
        nbr[t] = r;
    }
}

// strided conv, pass 1: each (input i, offset k) proposes an output site; the smallest proposer id wins the site
__global__ void k_sp_propose(const int4* __restrict__ coords, const int* __restrict__ m_dev, int M, SpGeom go, KShape ks,
                             uint32_t* __restrict__ okeys, int* __restrict__ ofirst, int* __restrict__ cand_slot, int* __restrict__ overflow) {
    const int K = ks.kz * ks.ky * ks.kx;
    int Md = m_dev ? min(M, m_dev[0]) : M;
    const long long total = (long long)Md * K, stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    int i = (int)(t / K), k = (int)(t % K);
    int dz = k / (ks.ky * ks.kx), dy = (k / ks.kx) % ks.ky, dx = k % ks.kx;
    int4 c = coords[i];
    int nz = c.y + ks.pz - dz, ny = c.z + ks.py - dy, nx = c.w + ks.px - dx;
    int slot = -1;
    if (nz >= 0 && ny >= 0 && nx >= 0 && nz % ks.sz == 0 && ny % ks.sy == 0 && nx % ks.sx == 0) {
        int oz = nz / ks.sz, oy = ny / ks.sy, ox = nx / ks.sx;
        if (oz < go.Z && oy < go.Y && ox < go.X) {
            uint32_t key = sp_key(c.x, oz, oy, ox, go);
            uint32_t s = sp_hash(key, go);
            // The table holds 2 x out_capacity slots.  With more distinct output sites than slots (an undersized capacity) an
            // unbounded probe would spin forever: give up after one sweep, drop the candidate and raise the overflow flag.
            bool found = false;
            for (uint32_t probe = 0; probe <= go.tmask; ++probe) {
                uint32_t prev = atomicCAS(&okeys[s], SP_EMPTY, key);
                if (prev == SP_EMPTY || prev == key) { found = true; break; }
                s = (s + 1) & go.tmask;
            }
            if (found) {
                atomicMin(&ofirst[s], (int)t);
                slot = (int)s;
            } else {
                atomicExch(overflow, 1);
            }
        }
    }
    cand_slot[t] = slot;
    }
}

// pass 2: per input row, number of output sites it generates first (<= K)
__global__ void k_sp_count_first(const int* __restrict__ m_dev, int M, int K, const int* __restrict__ ofirst,
                                 const int* __restrict__ cand_slot, int* __restrict__ cnt) {
    int Md = m_dev ? min(M, m_dev[0]) : M;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < M; i += gridDim.x * blockDim.x) {      // the scan reads all M entries
        int n = 0;
        if (i < Md)
            for (int k = 0; k < K; ++k) { int s = cand_slot[(size_t)i * K + k]; n += (s >= 0 && ofirst[s] == i * K + k) ? 1 : 0; }
        cnt[i] = n;
    }
}

__global__ void k_sp_scan_local(const int* __restrict__ in, int n, int* __restrict__ local_excl, int* __restrict__ block_sums) {
    __shared__ int warp_tot[32];
    int i = blockIdx.x * SP_SCAN + threadIdx.x;
    int v = (i < n) ? in[i] : 0;
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    if (w == 0) {
        int t = warp_tot[lane], ti = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += u; }
        warp_tot[lane] = ti - t;
        if (lane == 31) block_sums[blockIdx.x] = ti;
    }
    __syncthreads();
    if (i < n) local_excl[i] = inc - v + warp_tot[w];
}
__global__ void k_sp_scan_blocks(int* __restrict__ block_sums, int nblocks, int* __restrict__ total_out) {
    __shared__ int warp_tot[32];
    int t = threadIdx.x;
    int v = (t < nblocks) ? block_sums[t] : 0;
    int lane = t & 31, w = t >> 5, inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    if (w == 0) {
        int x = warp_tot[lane], xi = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, xi, o); if (lane >= o) xi += u; }
        warp_tot[lane] = xi - x;
    }
    __syncthreads();
    int excl = inc - v + warp_tot[w];
    if (t < nblocks) block_sums[t] = excl;
    if (t == nblocks - 1) total_out[0] = excl + v;
}

// pass 3: assign output rows in (input row, offset) order, write coords and the site -> row map
__global__ void k_sp_assign(const int4* __restrict__ coords, const int* __restrict__ m_dev, int M, SpGeom go, KShape ks,
                            const uint32_t* __restrict__ okeys, const int* __restrict__ ofirst, const int* __restrict__ cand_slot,
                            const int* __restrict__ local_excl, const int* __restrict__ block_off, int cap,
                            int* __restrict__ ovals, int4* __restrict__ out_coords) {
    const int K = ks.kz * ks.ky * ks.kx;
    int Md = m_dev ? min(M, m_dev[0]) : M;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Md; i += gridDim.x * blockDim.x) {
    int rank = local_excl[i] + block_off[i / SP_SCAN];
    for (int k = 0; k < K; ++k) {
        int s = cand_slot[(size_t)i * K + k];
        if (s >= 0 && ofirst[s] == i * K + k) {
            if (rank < cap) {
                ovals[s] = rank;
                uint32_t key = okeys[s];
                int x = (int)(key % (uint32_t)go.X); key /= (uint32_t)go.X;
                int y = (int)(key % (uint32_t)go.Y); key /= (uint32_t)go.Y;
                int z = (int)(key % (uint32_t)go.Z); int b = (int)(key / (uint32_t)go.Z);
                out_coords[rank] = make_int4(b, z, y, x);
            } else ovals[s] = -1;
            ++rank;
        }
    }
    }
}

// a full hash table dropped candidates: report more rows than the capacity so that callers see the overflow
__global__ void k_sp_flag_overflow(const int* __restrict__ overflow, int cap, int* __restrict__ out_rows) {
    if (threadIdx.x == 0 && blockIdx.x == 0 && overflow[0] && out_rows[0] <= cap) out_rows[0] = cap + 1;
}

// pass 4: nbr[out_row][k] = i
__global__ void k_sp_link(const int* __restrict__ m_dev, int M, int K, const int* __restrict__ cand_slot,
                          const int* __restrict__ ovals, int* __restrict__ nbr) {
    int Md = m_dev ? min(M, m_dev[0]) : M;
    const long long total = (long long)Md * K, stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        int s = cand_slot[t];
        if (s < 0) continue;
        int r = ovals[s];
        if (r >= 0) nbr[(size_t)r * K + (t % K)] = (int)(t / K);
    }
}

// ---- gather-GEMM: out[r][:] = act(bias + sum_k in[nbr[r][k]][:] . W[k]) ------------------------------
template <int CIN, int COUT>
__global__ void __launch_bounds__(128)
k_sp_gather_gemm(const float* __restrict__ in, const int* __restrict__ nbr, const int* __restrict__ m_dev, int M, int K,
                 const float* __restrict__ W, const float* __restrict__ bias, int relu, float* __restrict__ out) {
    constexpr int ROWS = 32;
    constexpr int CPT = COUT / 4;                     // output channels per thread (4 threads per row)
    __shared__ float sA[ROWS][CIN + 1];
    __shared__ __align__(16) float sW[CIN][COUT];
    __shared__ int sN[ROWS];
    const int Md = m_dev ? min(M, m_dev[0]) : M;
    const int r0 = blockIdx.x * ROWS;
    if (r0 >= Md) return;
    const int row = threadIdx.x >> 2, cg = threadIdx.x & 3;
    float acc[CPT];
#pragma unroll
    for (int j = 0; j < CPT; ++j) acc[j] = 0.f;
    for (int k = 0; k < K; ++k) {
        __syncthreads();
        if (threadIdx.x < ROWS) {
            int r = r0 + threadIdx.x;
            sN[threadIdx.x] = (r < Md) ? nbr[(size_t)r * K + k] : -1;
        }
        __syncthreads();
        int any = 0;
#pragma unroll 8
        for (int j = 0; j < ROWS; ++j) any |= (sN[j] >= 0);
        if (!any) continue;                             // block-uniform
        for (int t = threadIdx.x; t < ROWS * CIN; t += blockDim.x) {
            int rr = t / CIN, ci = t % CIN;
            int src = sN[rr];
            sA[rr][ci] = (src >= 0) ? __ldg(in + (size_t)src * CIN + ci) : 0.f;
        }
        for (int t = threadIdx.x; t < CIN * COUT / 4; t += blockDim.x)
            reinterpret_cast<float4*>(&sW[0][0])[t] = __ldg(reinterpret_cast<const float4*>(W + (size_t)k * CIN * COUT) + t);
        __syncthreads();
        if (sN[row] >= 0) {
#pragma unroll 4
            for (int ci = 0; ci < CIN; ++ci) {
                float a = sA[row][ci];
#pragma unroll
                for (int j = 0; j < CPT; ++j) acc[j] = fmaf(a, sW[ci][cg * CPT + j], acc[j]);
            }
        }
    }
    int r = r0 + row;
    if (r < Md) {
#pragma unroll
        for (int j = 0; j < CPT; ++j) {
            float v = acc[j] + (bias ? bias[cg * CPT + j] : 0.f);
            out[(size_t)r * COUT + cg * CPT + j] = relu ? fmaxf(v, 0.f) : v;
        }
    }
}

// HeightCompression: dense (B, C*D, H, W) channels-last; channel index = c*D + z
__global__ void k_sp_to_bev(const float* __restrict__ feats, const int4* __restrict__ coords, const int* __restrict__ m_dev, int M,
                            int C, int D, int H, int W, float* __restrict__ out) {
    int Md = m_dev ? min(M, m_dev[0]) : M;
    const long long total = (long long)Md * C, stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        int i = (int)(t / C), c = (int)(t % C);
        int4 cd = coords[i];
        if (cd.y < 0 || cd.y >= D || cd.z < 0 || cd.z >= H || cd.w < 0 || cd.w >= W) continue;
        out[(((size_t)cd.x * H + cd.z) * W + cd.w) * (size_t)(C * D) + (size_t)c * D + cd.y] = feats[t];
    }
}

int table_log2(int n) { int lg = 10; while ((1 << lg) < 2 * n) ++lg; return lg; }
SpGeom make_geom(const int* shape, int lg) {
    SpGeom g; g.Z = shape[0]; g.Y = shape[1]; g.X = shape[2]; g.tmask = (1u << lg) - 1; g.tshift = 32 - lg; return g;
}

template <int CIN, int COUT>
int launch_gg(const float* in, const int* nbr, const int* m_dev, int M, int K, const float* W, const float* b, int relu, float* out, cudaStream_t st) {
    k_sp_gather_gemm<CIN, COUT><<<(M + 31) / 32, 128, 0, st>>>(in, nbr, m_dev, M, K, W, b, relu, out);
    return heal_check_launch();
}

}  // namespace

extern "C" size_t heal_spconv_table_size(int capacity) { return (size_t)1 << table_log2(capacity > 0 ? capacity : 1); }

extern "C" int heal_spconv_build_table(const int* coords, const int* num_rows_dev, int capacity, const int* spatial_shape3_host, int batch,
                                       uint32_t* table_keys, int* table_vals, void* stream_) {
    if (!coords || !table_keys || !table_vals || capacity < 1) return HEAL_ERR_ARG;
    unsigned long long cells = (unsigned long long)spatial_shape3_host[0] * spatial_shape3_host[1] * spatial_shape3_host[2] * (unsigned long long)batch;
    if (cells >= 0xFFFFFFFFull) return HEAL_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    int lg = table_log2(capacity);
    SpGeom g = make_geom(spatial_shape3_host, lg);
    size_t ts = (size_t)1 << lg;
    cudaMemsetAsync(table_keys, 0xFF, ts * 4, st);
    k_sp_build<<<sp_grid(capacity, 256), 256, 0, st>>>((const int4*)coords, num_rows_dev, capacity, g, table_keys, table_vals);
    return heal_check_launch(1);
}

extern "C" int heal_spconv_subm_neighbors(const int* coords, const int* num_rows_dev, int capacity, const int* spatial_shape3_host,
                                          const int* ksize3_host, const uint32_t* table_keys, const int* table_vals, int table_capacity,
                                          int* nbr_out, void* stream_) {
    if (!coords || !table_keys || !table_vals || !nbr_out || capacity < 1) return HEAL_ERR_ARG;
    KShape ks; ks.kz = ksize3_host[0]; ks.ky = ksize3_host[1]; ks.kx = ksize3_host[2];
    ks.sz = ks.sy = ks.sx = 1; ks.pz = ks.py = ks.px = 0;
    int K = ks.kz * ks.ky * ks.kx;
    SpGeom g = make_geom(spatial_shape3_host, table_log2(table_capacity));
    long long total = (long long)capacity * K;
    k_sp_subm_nbr<<<sp_grid(total, 256), 256, 0, (cudaStream_t)stream_>>>((const int4*)coords, num_rows_dev, capacity, g, ks,
                                                                                     table_keys, table_vals, nbr_out);
    return heal_check_launch();
}

extern "C" size_t heal_spconv_strided_workspace(int in_capacity, int out_capacity, int kvol) {
    size_t M = (size_t)(in_capacity > 0 ? in_capacity : 1);
    size_t ts = (size_t)1 << table_log2(out_capacity > 0 ? out_capacity : 1);
    return heal_align_up(M * kvol * 4, 256) + heal_align_up(M * 4, 256) * 2 + heal_align_up((M / SP_SCAN + 4) * 4, 256) +
           heal_align_up(ts * 4, 256) + 256 + 4096;
}

extern "C" int heal_spconv_strided_rulebook(const int* in_coords, const int* in_rows_dev, int in_capacity,
                                            const int* out_spatial_shape3_host, int batch,
                                            const int* ksize3_host, const int* stride3_host, const int* pad3_host,
                                            int out_capacity, int* out_coords, int* out_rows_dev,
                                            uint32_t* out_table_keys, int* out_table_vals, int* nbr_out,
                                            void* workspace, size_t workspace_bytes, void* stream_) {
    if (!in_coords || !out_coords || !out_rows_dev || !out_table_keys || !out_table_vals || !nbr_out) return HEAL_ERR_ARG;
    if (in_capacity < 1 || out_capacity < 1 || in_capacity > SP_SCAN * SP_SCAN) return HEAL_ERR_ARG;
    KShape ks;
    ks.kz = ksize3_host[0]; ks.ky = ksize3_host[1]; ks.kx = ksize3_host[2];
    ks.sz = stride3_host[0]; ks.sy = stride3_host[1]; ks.sx = stride3_host[2];
    ks.pz = pad3_host[0]; ks.py = pad3_host[1]; ks.px = pad3_host[2];
    const int K = ks.kz * ks.ky * ks.kx;
    if (workspace_bytes < heal_spconv_strided_workspace(in_capacity, out_capacity, K)) return HEAL_ERR_WORKSPACE;
    unsigned long long cells = (unsigned long long)out_spatial_shape3_host[0] * out_spatial_shape3_host[1] * out_spatial_shape3_host[2] * (unsigned long long)batch;
    if (cells >= 0xFFFFFFFFull) return HEAL_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    int lg = table_log2(out_capacity);
    SpGeom go = make_geom(out_spatial_shape3_host, lg);
    size_t ts = (size_t)1 << lg;
    HealArena ar(workspace, workspace_bytes);
    int* cand_slot = ar.take<int>((size_t)in_capacity * K);
    int* cnt = ar.take<int>(in_capacity);
    int* local_excl = ar.take<int>(in_capacity);
    int nb = (in_capacity + SP_SCAN - 1) / SP_SCAN;
    int* block_off = ar.take<int>(nb + 2);
    int* ofirst = ar.take<int>(ts);                        // per site: smallest proposer id (input row * K + offset)
    int* overflow = ar.take<int>(1);
    if (!ar.ok()) return HEAL_ERR_WORKSPACE;
    cudaMemsetAsync(overflow, 0, 4, st);
    cudaMemsetAsync(out_table_keys, 0xFF, ts * 4, st);
    cudaMemsetAsync(ofirst, 0x7F, ts * 4, st);
    cudaMemsetAsync(nbr_out, 0xFF, (size_t)out_capacity * K * 4, st);
    long long total = (long long)in_capacity * K;
    unsigned gt = sp_grid(total, 256), gm = sp_grid(in_capacity, 256);
    k_sp_propose<<<gt, 256, 0, st>>>((const int4*)in_coords, in_rows_dev, in_capacity, go, ks, out_table_keys, ofirst, cand_slot, overflow);
    k_sp_count_first<<<gm, 256, 0, st>>>(in_rows_dev, in_capacity, K, ofirst, cand_slot, cnt);
    k_sp_scan_local<<<nb, SP_SCAN, 0, st>>>(cnt, in_capacity, local_excl, block_off);
    k_sp_scan_blocks<<<1, SP_SCAN, 0, st>>>(block_off, nb, out_rows_dev);
    k_sp_assign<<<gm, 256, 0, st>>>((const int4*)in_coords, in_rows_dev, in_capacity, go, ks, out_table_keys, ofirst, cand_slot,
                                    local_excl, block_off, out_capacity, out_table_vals, (int4*)out_coords);
    k_sp_link<<<gt, 256, 0, st>>>(in_rows_dev, in_capacity, K, cand_slot, out_table_vals, nbr_out);
    k_sp_flag_overflow<<<1, 32, 0, st>>>(overflow, out_capacity, out_rows_dev);
    return heal_check_launch(7);
}

extern "C" int heal_spconv_gather_gemm(const float* in_feats, const int* nbr, const int* out_rows_dev, int out_capacity, int kvol,
                                       const float* weight, const float* bias, int c_in, int c_out, int relu,
                                       float* out_feats, void* stream_) {
    if (!in_feats || !nbr || !weight || !out_feats || out_capacity < 1) return HEAL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
#define GG(ci, co) if (c_in == ci && c_out == co) return launch_gg<ci, co>(in_feats, nbr, out_rows_dev, out_capacity, kvol, weight, bias, relu, out_feats, st)
    GG(4, 16); GG(16, 16); GG(16, 32); GG(32, 32); GG(32, 64); GG(64, 64); GG(64, 128);
#undef GG
    return HEAL_ERR_UNSUPPORTED;
}

extern "C" int heal_sparse_to_bev(const float* feats, const int* coords, const int* rows_dev, int capacity, int C, int D, int H, int W,
                                  float* bev_out, void* stream_) {
    if (!feats || !coords || !bev_out || capacity < 1) return HEAL_ERR_ARG;
    long long total = (long long)capacity * C;
    k_sp_to_bev<<<sp_grid(total, 256), 256, 0, (cudaStream_t)stream_>>>(feats, (const int4*)coords, rows_dev, capacity, C, D, H, W, bev_out);
    return heal_check_launch();
}
