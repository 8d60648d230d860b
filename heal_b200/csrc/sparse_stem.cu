// Sparse stem: the first residual block's two stride-2 convolutions evaluated directly from the pillar list, so the dense
// (B, ny, nx, 64) BEV canvas of PointPillarScatter is never materialised (335 MB zero-fill + two full reads at 5 x 512^2).
// Reference ops fused: PointPillarScatter.forward (point_pillar_scatter.py:19-77) -> BasicBlock.conv1 (3x3, stride 2, pad 1) +
// bn1 + ReLU and BasicBlock.downsample (1x1, stride 2) + bn (resblock.py:48-64, 178-187).  Only ~4.6 % of the pillars' cells
// are occupied; an output pixel gathers the <= 9 occupied input cells under its window through an id map (pillar row or -1),
// every other pixel is just ReLU(folded bias).  fp32 FMA math, any output storage format.
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

struct StemP {
    const float* feats;     // (M, 64) pillar features
    const int* idmap;       // (B, ny, nx) pillar row or -1
    const float* w1;        // [9][64][64] (tap, cin, cout), BN folded
    const float* b1;        // [64]
    const float* w2;        // [64][64] (cin, cout) 1x1 stride-2 downsample, BN folded
    const float* b2;        // [64]
    ActV out1, out2;        // (B, Ho, Wo, 64)
    int B, ny, nx, Ho, Wo;
};

__device__ __forceinline__ void store2(const ActV& a, size_t pix, int c, float x, float y) {
    size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (a.fmt == 0) { *reinterpret_cast<float2*>(reinterpret_cast<float*>(a.p) + idx) = make_float2(x, y); return; }
    __nv_bfloat16* b = reinterpret_cast<__nv_bfloat16*>(a.p) + idx;
    __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    *reinterpret_cast<__nv_bfloat162*>(b) = h;
    if (a.fmt == 2) {
        float2 hf = __bfloat1622float2(h);
        *reinterpret_cast<__nv_bfloat162*>(b + a.plane) = __floats2bfloat162_rn(x - hf.x, y - hf.y);
    }
}

__global__ void __launch_bounds__(256)
k_sparse_stem(StemP p) {
    const int lane = threadIdx.x & 31;
    const long long npix = (long long)p.B * p.Ho * p.Wo;
    const float2 bias1 = *reinterpret_cast<const float2*>(p.b1 + 2 * lane);
    const float2 bias2 = *reinterpret_cast<const float2*>(p.b2 + 2 * lane);
    for (long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pix < npix;
         pix += (long long)gridDim.x * (blockDim.x >> 5)) {
        const int ox = (int)(pix % p.Wo); long long t = pix / p.Wo;
        const int oy = (int)(t % p.Ho); const int b = (int)(t / p.Ho);
        int id = -1;
        if (lane < 9) {
            int iy = 2 * oy - 1 + lane / 3, ix = 2 * ox - 1 + lane % 3;
            if (iy >= 0 && iy < p.ny && ix >= 0 && ix < p.nx) id = __ldg(p.idmap + ((size_t)b * p.ny + iy) * p.nx + ix);
        }
        unsigned hits = __ballot_sync(0xffffffffu, id >= 0);
        float2 a1 = bias1, a2 = bias2;
        while (hits) {
            const int tap = __ffs(hits) - 1;
            hits &= hits - 1;
            const int pid = __shfl_sync(0xffffffffu, id, tap);
            const float2 f = *reinterpret_cast<const float2*>(p.feats + (size_t)pid * 64 + 2 * lane);
            const float* w = p.w1 + (size_t)tap * 64 * 64 + 2 * lane;
#pragma unroll 8
            for (int k = 0; k < 64; ++k) {
                const float fk = __shfl_sync(0xffffffffu, (k & 1) ? f.y : f.x, k >> 1);
                const float2 wv = __ldg(reinterpret_cast<const float2*>(w + (size_t)k * 64));
                a1.x = fmaf(fk, wv.x, a1.x); a1.y = fmaf(fk, wv.y, a1.y);
            }
            if (tap == 4) {                         // centre cell (2oy, 2ox) is the 1x1 stride-2 downsample's input
                const float* w2 = p.w2 + 2 * lane;
#pragma unroll 8
                for (int k = 0; k < 64; ++k) {
                    const float fk = __shfl_sync(0xffffffffu, (k & 1) ? f.y : f.x, k >> 1);
                    const float2 wv = __ldg(reinterpret_cast<const float2*>(w2 + (size_t)k * 64));
                    a2.x = fmaf(fk, wv.x, a2.x); a2.y = fmaf(fk, wv.y, a2.y);
                }
            }
        }
        store2(p.out1, (size_t)pix, 2 * lane, fmaxf(a1.x, 0.f), fmaxf(a1.y, 0.f));
        store2(p.out2, (size_t)pix, 2 * lane, a2.x, a2.y);
    }
}

// ---- tensor-core variant (split-bf16, fp32-equivalent) ------------------------------------------------------------------------
// The SIMT kernel above streams a 16 KB tap matrix from L1 for every occupied (pixel, tap) pair and is bound by that
// (110 M warp instructions at 5 x 512^2).  Here a warp owns 16 consecutive output pixels of a row (one m16 row block of
// mma.sync.m16n8k16) and keeps both 16x64 fp32 outputs in registers; for each of the 9 taps that has at least one hit among the 16
// pixels it gathers the hit pillars' features as the A fragments (zero rows elsewhere), splits them into bf16 hi/lo and issues
// a_lo*b_hi + a_hi*b_lo + a_hi*b_hi against the tap's 64x64 weights, which all ten matrices (9 taps + the 1x1 downsample) keep
// resident in shared memory as bf16 hi/lo, [cout][cin] with a 72-element pitch (conflict-free 32-bit B-fragment loads).
// Deterministic: taps are accumulated in order 0..8, exactly like the SIMT kernel.  Persistent grid: one CTA per SM.
constexpr int ST_PITCH = 72;                                   // bf16 elements per weight row in smem
constexpr int ST_MAT = 64 * ST_PITCH;                          // elements per matrix plane
constexpr int ST_SMEM = 10 * 2 * ST_MAT * 2;                   // 10 matrices x (hi, lo) x 2 B = 184320 B

__device__ __forceinline__ void mma_bf16_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split2(float x, float y, uint32_t& hi, uint32_t& lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    float2 hf = __bfloat1622float2(h);
    __nv_bfloat162 l = __floats2bfloat162_rn(x - hf.x, y - hf.y);
    hi = *reinterpret_cast<uint32_t*>(&h); lo = *reinterpret_cast<uint32_t*>(&l);
}

__global__ void __launch_bounds__(256, 1)
k_sparse_stem_tc(StemP p) {
    extern __shared__ __align__(16) uint8_t st_smem[];
    __nv_bfloat16* W = reinterpret_cast<__nv_bfloat16*>(st_smem);      // [mat 0..9][plane][cout 64][ST_PITCH]
    // weights: fp32 (tap, cin, cout) -> bf16 hi/lo, transposed to [cout][cin]
    for (int i = threadIdx.x; i < 10 * 64 * 64; i += blockDim.x) {
        const int m = i / 4096, r = i % 4096, ci = r / 64, co = r % 64;
        const float w = (m < 9) ? __ldg(p.w1 + (size_t)m * 4096 + r) : __ldg(p.w2 + r);
        const __nv_bfloat16 h = __float2bfloat16_rn(w);
        W[(m * 2 + 0) * ST_MAT + co * ST_PITCH + ci] = h;
        W[(m * 2 + 1) * ST_MAT + co * ST_PITCH + ci] = __float2bfloat16_rn(w - __bfloat162float(h));
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int groups_per_row = p.Wo / 16;
    const long long ngroups = (long long)p.B * p.Ho * groups_per_row;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    float bias1[8][2], bias2[8][2];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        bias1[j][0] = __ldg(p.b1 + 8 * j + 2 * t); bias1[j][1] = __ldg(p.b1 + 8 * j + 2 * t + 1);
        bias2[j][0] = __ldg(p.b2 + 8 * j + 2 * t); bias2[j][1] = __ldg(p.b2 + 8 * j + 2 * t + 1);
    }
    for (long long grp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); grp < ngroups; grp += nwarps) {
        const int gx = (int)(grp % groups_per_row); long long t2 = grp / groups_per_row;
        const int oy = (int)(t2 % p.Ho); const int b = (int)(t2 / p.Ho);
        const int ox0 = gx * 16;
        // lanes 0..15: the 9 pillar ids under pixel (oy, ox0 + lane)
        int ids[9];
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            ids[tap] = -1;
            if (lane < 16) {
                const int iy = 2 * oy - 1 + tap / 3, ix = 2 * (ox0 + lane) - 1 + tap % 3;
                if (iy >= 0 && iy < p.ny && ix >= 0 && ix < p.nx) ids[tap] = __ldg(p.idmap + ((size_t)b * p.ny + iy) * p.nx + ix);
            }
        }
        float d1[8][4], d2[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) { d1[j][e] = 0.f; d2[j][e] = 0.f; }
        }
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
            int my = -1;
#pragma unroll
            for (int q = 0; q < 9; ++q) if (q == tap) my = ids[q];
            if (__ballot_sync(0xffffffffu, my >= 0) == 0u) continue;
            const int pid0 = __shfl_sync(0xffffffffu, my, g), pid1 = __shfl_sync(0xffffffffu, my, g + 8);
            // A fragments for the 4 K steps: rows g / g+8 = pixels g / g+8 of the group, zero rows where the tap misses
            uint32_t ah[4][4], al[4][4];
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                float2 x0 = make_float2(0.f, 0.f), x1 = x0, x2 = x0, x3 = x0;
                if (pid0 >= 0) {
                    const float* f = p.feats + (size_t)pid0 * 64 + s * 16 + 2 * t;
                    x0 = __ldg(reinterpret_cast<const float2*>(f)); x2 = __ldg(reinterpret_cast<const float2*>(f + 8));
                }
                if (pid1 >= 0) {
                    const float* f = p.feats + (size_t)pid1 * 64 + s * 16 + 2 * t;
                    x1 = __ldg(reinterpret_cast<const float2*>(f)); x3 = __ldg(reinterpret_cast<const float2*>(f + 8));
                }
                split2(x0.x, x0.y, ah[s][0], al[s][0]); split2(x1.x, x1.y, ah[s][1], al[s][1]);
                split2(x2.x, x2.y, ah[s][2], al[s][2]); split2(x3.x, x3.y, ah[s][3], al[s][3]);
            }
            const int nmat = (tap == 4) ? 2 : 1;                // the centre tap also feeds the 1x1 stride-2 downsample
            for (int mm = 0; mm < nmat; ++mm) {
                const __nv_bfloat16* Wh = W + ((mm == 0 ? tap : 9) * 2 + 0) * ST_MAT;
                const __nv_bfloat16* Wl = Wh + ST_MAT;
#pragma unroll
                for (int s = 0; s < 4; ++s) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int o = (8 * j + g) * ST_PITCH + s * 16 + 2 * t;
                        const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(Wh + o), bh1 = *reinterpret_cast<const uint32_t*>(Wh + o + 8);
                        const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(Wl + o), bl1 = *reinterpret_cast<const uint32_t*>(Wl + o + 8);
                        float* d = (mm == 0) ? d1[j] : d2[j];
                        mma_bf16_16816(d, al[s], bh0, bh1);
                        mma_bf16_16816(d, ah[s], bl0, bl1);
                        mma_bf16_16816(d, ah[s], bh0, bh1);
                    }
                }
            }
        }
        // epilogue: row g -> pixel ox0+g (c0,c1), row g+8 -> pixel ox0+g+8 (c2,c3); channels 8j+2t, 8j+2t+1
        const size_t pix0 = ((size_t)b * p.Ho + oy) * p.Wo + ox0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = 8 * j + 2 * t;
            store2(p.out1, pix0 + g, c, fmaxf(d1[j][0] + bias1[j][0], 0.f), fmaxf(d1[j][1] + bias1[j][1], 0.f));
            store2(p.out1, pix0 + g + 8, c, fmaxf(d1[j][2] + bias1[j][0], 0.f), fmaxf(d1[j][3] + bias1[j][1], 0.f));
            store2(p.out2, pix0 + g, c, d2[j][0] + bias2[j][0], d2[j][1] + bias2[j][1]);
            store2(p.out2, pix0 + g + 8, c, d2[j][2] + bias2[j][0], d2[j][3] + bias2[j][1]);
        }
    }
}

__global__ void k_fill_idmap(const int4* __restrict__ coords, const int* __restrict__ m_dev, int M, int ny, int nx, int* __restrict__ idmap) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int Md = m_dev ? min(M, m_dev[0]) : M;
    if (i >= Md) return;
    int4 c = coords[i];   // [b, z, y, x]
    idmap[((size_t)c.x * ny + c.z) * nx + (c.y + c.w)] = i;
}

}  // namespace

extern "C" int heal_pillar_idmap(const int* voxel_coords, const int* num_voxels_dev, int num_voxels, int batch, int ny, int nx,
                                 int* idmap_out, void* stream_) {
    if (!voxel_coords || !idmap_out || batch < 1) return HEAL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaMemsetAsync(idmap_out, 0xFF, (size_t)batch * ny * nx * sizeof(int), st);
    if (num_voxels > 0)
        k_fill_idmap<<<(num_voxels + 255) / 256, 256, 0, st>>>((const int4*)voxel_coords, num_voxels_dev, num_voxels, ny, nx, idmap_out);
    return heal_check_launch();
}

extern "C" int heal_sparse_stem(const float* pillar_features, const int* idmap, int batch, int ny, int nx,
                                const float* w_conv3x3, const float* b_conv3x3, const float* w_down1x1, const float* b_down1x1,
                                int channels, const heal_act_t* out_conv, const heal_act_t* out_down, void* stream_) {
    if (!pillar_features || !idmap || !w_conv3x3 || !b_conv3x3 || !w_down1x1 || !b_down1x1 || !out_conv || !out_down) return HEAL_ERR_ARG;
    if (channels != 64 || (ny & 1) || (nx & 1)) return HEAL_ERR_UNSUPPORTED;
    if ((out_conv->cstride & 1) || (out_conv->coffset & 1) || (out_down->cstride & 1) || (out_down->coffset & 1)) return HEAL_ERR_UNSUPPORTED;
    StemP p;
    p.feats = pillar_features; p.idmap = idmap; p.w1 = w_conv3x3; p.b1 = b_conv3x3; p.w2 = w_down1x1; p.b2 = b_down1x1;
    p.out1.p = out_conv->data; p.out1.fmt = out_conv->fmt; p.out1.cs = out_conv->cstride; p.out1.co = out_conv->coffset; p.out1.plane = out_conv->plane_stride;
    p.out2.p = out_down->data; p.out2.fmt = out_down->fmt; p.out2.cs = out_down->cstride; p.out2.co = out_down->coffset; p.out2.plane = out_down->plane_stride;
    p.B = batch; p.ny = ny; p.nx = nx; p.Ho = ny / 2; p.Wo = nx / 2;
    long long npix = (long long)batch * p.Ho * p.Wo;
    long long blocks = (npix + 7) / 8;
    long long cap = (long long)HEAL_NUM_SMS * 32;
    k_sparse_stem<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream_>>>(p);
    return heal_check_launch();
}

extern "C" int heal_sparse_stem_tc(const float* pillar_features, const int* idmap, int batch, int ny, int nx,
                                   const float* w_conv3x3, const float* b_conv3x3, const float* w_down1x1, const float* b_down1x1,
                                   int channels, const heal_act_t* out_conv, const heal_act_t* out_down, void* stream_) {
    if (!pillar_features || !idmap || !w_conv3x3 || !b_conv3x3 || !w_down1x1 || !b_down1x1 || !out_conv || !out_down) return HEAL_ERR_ARG;
    if (channels != 64 || (ny & 1) || (nx & 31)) return HEAL_ERR_UNSUPPORTED;            // output rows in groups of 16 pixels
    if ((out_conv->cstride & 1) || (out_conv->coffset & 1) || (out_down->cstride & 1) || (out_down->coffset & 1)) return HEAL_ERR_UNSUPPORTED;
    StemP p;
    p.feats = pillar_features; p.idmap = idmap; p.w1 = w_conv3x3; p.b1 = b_conv3x3; p.w2 = w_down1x1; p.b2 = b_down1x1;
    p.out1.p = out_conv->data; p.out1.fmt = out_conv->fmt; p.out1.cs = out_conv->cstride; p.out1.co = out_conv->coffset; p.out1.plane = out_conv->plane_stride;
    p.out2.p = out_down->data; p.out2.fmt = out_down->fmt; p.out2.cs = out_down->cstride; p.out2.co = out_down->coffset; p.out2.plane = out_down->plane_stride;
    p.B = batch; p.ny = ny; p.nx = nx; p.Ho = ny / 2; p.Wo = nx / 2;
    static size_t attr_set[HEAL_MAX_DEVICES] = {};
    if (!heal_ensure_dyn_smem(k_sparse_stem_tc, ST_SMEM, attr_set)) return HEAL_ERR_LAUNCH;
    long long ngroups = (long long)batch * p.Ho * (p.Wo / 16);
    long long blocks = (ngroups + 7) / 8;
    k_sparse_stem_tc<<<(unsigned)(blocks < HEAL_NUM_SMS ? blocks : HEAL_NUM_SMS), 256, ST_SMEM, (cudaStream_t)stream_>>>(p);
    return heal_check_launch();
}
