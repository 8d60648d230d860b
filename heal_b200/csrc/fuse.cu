// Multi-agent BEV feature fusion kernels (channels-last):
//   heal_pyramid_fuse_level : warp(feat) + warp(score) -> mask -> softmax over agents -> weighted sum
//       reference: opencood/models/fuse_modules/pyramid_fuse.py:17-63 (weighted_fuse) and :143-164
//       (score = sigmoid(occ) + 1e-4, camera crop mask in eval mode)
//   heal_att_fuse           : warp -> per-pixel scaled dot-product attention over agents, ego row only
//       reference: opencood/models/fuse_modules/fusion_in_one.py:126-151 (AttFusion), :41-45
//   heal_max_fuse           : warp -> max over agents (MaxFusion, fusion_in_one.py:87-124)
// All three fold warp_affine_simple (torch_transformation_utils.py:323-332 = F.affine_grid with an fp64
// theta, cast to fp32, then F.grid_sample bilinear / zeros padding) into the fusion so the warped
// per-agent maps never exist in HBM.
//   heal_warp_affine, heal_v2v_aggregate, heal_gru_gate : the non-conv steps of V2VNetFusion (fusion_in_one.py:203-318),
//       whose message and GRU convolutions run on the conv engine between them.
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int MAX_AGENTS = 8;

struct Tap {
    int off[4];    // source pixel index (within the agent's map) or -1 when out of bounds
    float w[4];    // bilinear weights (nw, ne, sw, se)
};

// affine_grid (fp64, then cast to fp32) + grid_sample unnormalisation; pytorch semantics.
__device__ __forceinline__ Tap make_tap(const double* __restrict__ th, int oh, int ow, int H, int W, int align) {
    double xb, yb;
    if (align) {
        xb = (W > 1) ? (-1.0 + 2.0 * ow / (double)(W - 1)) : 0.0;
        yb = (H > 1) ? (-1.0 + 2.0 * oh / (double)(H - 1)) : 0.0;
    } else {
        xb = (2.0 * ow + 1.0) / (double)W - 1.0;
        yb = (2.0 * oh + 1.0) / (double)H - 1.0;
    }
    float gx = (float)(th[0] * xb + th[1] * yb + th[2]);
    float gy = (float)(th[3] * xb + th[4] * yb + th[5]);
    float ix, iy;
    if (align) { ix = ((gx + 1.f) / 2.f) * (float)(W - 1); iy = ((gy + 1.f) / 2.f) * (float)(H - 1); }
    else { ix = ((gx + 1.f) * (float)W - 1.f) / 2.f; iy = ((gy + 1.f) * (float)H - 1.f) / 2.f; }
    float fx = floorf(ix), fy = floorf(iy);
    // clamp before the int cast so that huge/NaN coordinates become plainly out of bounds
    int x0 = (fx >= -2.f && fx <= (float)(W + 1)) ? (int)fx : -2;
    int y0 = (fy >= -2.f && fy <= (float)(H + 1)) ? (int)fy : -2;
    int x1 = x0 + 1, y1 = y0 + 1;
    float wx1 = ix - fx, wx0 = (fx + 1.f) - ix, wy1 = iy - fy, wy0 = (fy + 1.f) - iy;
    Tap t;
    bool xi0 = (x0 >= 0 && x0 < W), xi1 = (x1 >= 0 && x1 < W), yi0 = (y0 >= 0 && y0 < H), yi1 = (y1 >= 0 && y1 < H);
    t.off[0] = (xi0 && yi0) ? y0 * W + x0 : -1;  t.w[0] = wx0 * wy0;   // nw
    t.off[1] = (xi1 && yi0) ? y0 * W + x1 : -1;  t.w[1] = wx1 * wy0;   // ne
    t.off[2] = (xi0 && yi1) ? y1 * W + x0 : -1;  t.w[2] = wx0 * wy1;   // sw
    t.off[3] = (xi1 && yi1) ? y1 * W + x1 : -1;  t.w[3] = wx1 * wy1;   // se
    return t;
}

struct FuseP {
    ActV feat;             // (n, H, W, C) channels-last view (fp32 / bf16 / split-bf16)
    const float* occ;      // (n, H, W) occupancy logits
    const double* theta;   // (n, 2, 3) fp64: affine[b, 0, j]
    const int* crop;       // (n, 4) [h0, h1, w0, w1] window where the score is kept, or nullptr
    ActV out;              // (rows, W, C): the output slab, pixel 0 = (row0, 0)
    int n, H, W, C, align;
    int row0, rows;        // output rows [row0, row0 + rows) (row-sharded fusion tail); whole map: 0, H
    long long foff[MAX_AGENTS];   // element offset of agent j's map from feat.p (dense stack: j*H*W*cstride; gathered buffer: any)
    long long ooff[MAX_AGENTS];   // element offset of agent j's occupancy map from occ
};

__device__ __forceinline__ ActV agent_view(const ActV& f, long long off) {
    ActV v = f;
    v.p = (f.fmt == 0) ? (void*)(reinterpret_cast<float*>(f.p) + off) : (void*)(reinterpret_cast<__nv_bfloat16*>(f.p) + off);
    return v;
}

// FUSE_PIX pixels per 256-thread block, chosen by the host so that FUSE_PIX * C / 4 == 256 (one 4-channel chunk per thread)
// and small maps still fill the machine (64x64x256 -> 1024 blocks).
template <int FUSE_PIX>
__global__ void __launch_bounds__(256)
k_pyramid_fuse(FuseP p) {
    __shared__ Tap sTap[FUSE_PIX][MAX_AGENTS];
    __shared__ float sScore[FUSE_PIX][MAX_AGENTS];
    const int HW = p.rows * p.W;                   // pixels of the output slab; `pix` below is slab-local
    const int pix0 = blockIdx.x * FUSE_PIX;
    // phase 1: tap geometry + warped score per (pixel, agent)
    for (int it = threadIdx.x; it < FUSE_PIX * p.n; it += blockDim.x) {
        int j = it % p.n, lp = it / p.n;
        int pix = pix0 + lp;
        if (pix >= HW) continue;
        Tap t = make_tap(p.theta + 6 * j, p.row0 + pix / p.W, pix % p.W, p.H, p.W, p.align);
        const float* occ = p.occ + p.ooff[j];
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (t.off[k] >= 0) {
                float sc = 1.f / (1.f + expf(-occ[t.off[k]])) + 1e-4f;
                if (p.crop) {
                    int y = t.off[k] / p.W, x = t.off[k] % p.W;
                    const int* c = p.crop + 4 * j;
                    if (!(y >= c[0] && y < c[1] && x >= c[2] && x < c[3])) sc = 0.f;
                }
                s += sc * t.w[k];
            }
        }
        sTap[lp][j] = t;
        sScore[lp][j] = s;
    }
    __syncthreads();
    // phase 2: masked softmax over agents (score == 0 -> -inf; all -inf -> NaN -> 0), folded into tap weights
    if (threadIdx.x < FUSE_PIX && pix0 + threadIdx.x < HW) {
        int lp = threadIdx.x;
        float mx = -INFINITY;
        for (int j = 0; j < p.n; ++j) { float s = sScore[lp][j]; if (s != 0.f) mx = fmaxf(mx, s); }
        float den = 0.f;
        float e[MAX_AGENTS];
        for (int j = 0; j < p.n; ++j) {
            float s = sScore[lp][j];
            e[j] = (s != 0.f) ? expf(s - mx) : 0.f;
            den += e[j];
        }
        for (int j = 0; j < p.n; ++j) {
            float wgt = (den > 0.f) ? e[j] / den : 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) sTap[lp][j].w[k] *= wgt;
        }
    }
    __syncthreads();
    // phase 3: thread = (pixel, 4-channel chunk)
    const int chunks = p.C / 4;
    for (int it = threadIdx.x; it < FUSE_PIX * chunks; it += blockDim.x) {
        int ch = it % chunks, lp = it / chunks;
        int pix = pix0 + lp;
        if (pix >= HW) continue;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < p.n; ++j) {
            // warped feature (bilinear), then weighted; the four tap loads are issued together, then the FMAs in tap order
            float4 v[4];
            float w[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                int off = sTap[lp][j].off[k];
                w[k] = sTap[lp][j].w[k];
                v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (off >= 0) v[k] = act_load4(agent_view(p.feat, p.foff[j]), (size_t)off, ch * 4);
                else w[k] = 0.f;
            }
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                a.x = fmaf(v[k].x, w[k], a.x); a.y = fmaf(v[k].y, w[k], a.y);
                a.z = fmaf(v[k].z, w[k], a.z); a.w = fmaf(v[k].w, w[k], a.w);
            }
            acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
        }
        act_store4(p.out, (size_t)pix, ch * 4, acc);
    }
}

// Split-bf16 features (the tc32 engine format), 8 channels per thread: 16 B loads per plane and tap, offsets precomputed as
// element indices -- the generic kernel above is instruction-bound (41.5 M warp instructions for the 256x256x64 level), this one
// issues ~1.6x fewer per channel.  Same arithmetic order (hi + lo, FMA over the 4 taps, sum over agents) => identical results.
template <int FUSE_PIX>
__global__ void __launch_bounds__(256)
k_pyramid_fuse_split8(FuseP p) {
    __shared__ Tap sTap[FUSE_PIX][MAX_AGENTS];
    __shared__ float sScore[FUSE_PIX][MAX_AGENTS];
    const int HW = p.rows * p.W;
    const int pix0 = blockIdx.x * FUSE_PIX;
    for (int it = threadIdx.x; it < FUSE_PIX * p.n; it += blockDim.x) {
        int j = it % p.n, lp = it / p.n;
        int pix = pix0 + lp;
        if (pix >= HW) continue;
        Tap t = make_tap(p.theta + 6 * j, p.row0 + pix / p.W, pix % p.W, p.H, p.W, p.align);
        const float* occ = p.occ + p.ooff[j];
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (t.off[k] >= 0) {
                float sc = 1.f / (1.f + expf(-occ[t.off[k]])) + 1e-4f;
                if (p.crop) {
                    int y = t.off[k] / p.W, x = t.off[k] % p.W;
                    const int* c = p.crop + 4 * j;
                    if (!(y >= c[0] && y < c[1] && x >= c[2] && x < c[3])) sc = 0.f;
                }
                s += sc * t.w[k];
                t.off[k] = t.off[k] * p.feat.cs + p.feat.co;      // element index of the tap's first channel inside agent j's map
            }
        }
        sTap[lp][j] = t;
        sScore[lp][j] = s;
    }
    __syncthreads();
    if (threadIdx.x < FUSE_PIX && pix0 + threadIdx.x < HW) {
        int lp = threadIdx.x;
        float mx = -INFINITY;
        for (int j = 0; j < p.n; ++j) { float s = sScore[lp][j]; if (s != 0.f) mx = fmaxf(mx, s); }
        float den = 0.f;
        float e[MAX_AGENTS];
        for (int j = 0; j < p.n; ++j) {
            float s = sScore[lp][j];
            e[j] = (s != 0.f) ? expf(s - mx) : 0.f;
            den += e[j];
        }
        for (int j = 0; j < p.n; ++j) {
            float wgt = (den > 0.f) ? e[j] / den : 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) sTap[lp][j].w[k] *= wgt;
        }
    }
    __syncthreads();
    const int chunks = p.C / 8;
    const __nv_bfloat16* hi = reinterpret_cast<const __nv_bfloat16*>(p.feat.p);
    const __nv_bfloat16* lo = hi + p.feat.plane;
    for (int it = threadIdx.x; it < FUSE_PIX * chunks; it += blockDim.x) {
        int ch = it % chunks, lp = it / chunks;
        int pix = pix0 + lp;
        if (pix >= HW) continue;
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
        for (int j = 0; j < p.n; ++j) {
            const __nv_bfloat16* hj = hi + p.foff[j];
            const __nv_bfloat16* lj = lo + p.foff[j];
            uint4 vh[4], vl[4];
            float w[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int off = sTap[lp][j].off[k];
                w[k] = sTap[lp][j].w[k];
                vh[k] = make_uint4(0u, 0u, 0u, 0u); vl[k] = make_uint4(0u, 0u, 0u, 0u);
                if (off >= 0) {
                    vh[k] = __ldg(reinterpret_cast<const uint4*>(hj + off + ch * 8));
                    vl[k] = __ldg(reinterpret_cast<const uint4*>(lj + off + ch * 8));
                } else {
                    w[k] = 0.f;
                }
            }
            float a[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) a[e] = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t* h32 = reinterpret_cast<const uint32_t*>(&vh[k]);
                const uint32_t* l32 = reinterpret_cast<const uint32_t*>(&vl[k]);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float x0 = __uint_as_float(h32[q] << 16) + __uint_as_float(l32[q] << 16);
                    float x1 = __uint_as_float(h32[q] & 0xffff0000u) + __uint_as_float(l32[q] & 0xffff0000u);
                    a[2 * q] = fmaf(x0, w[k], a[2 * q]);
                    a[2 * q + 1] = fmaf(x1, w[k], a[2 * q + 1]);
                }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] += a[e];
        }
        act_store4(p.out, (size_t)pix, ch * 8, make_float4(acc[0], acc[1], acc[2], acc[3]));
        act_store4(p.out, (size_t)pix, ch * 8 + 4, make_float4(acc[4], acc[5], acc[6], acc[7]));
    }
}

struct AttP {
    ActV feat; const double* theta; ActV out;
    int n, H, W, C, align;
    float inv_sqrt_dim;
};

// one warp per output pixel; lane covers channels {4*lane + 128*q}.  Every agent's warped feature vector is sampled ONCE and
// kept in registers for both the ego-row scores and the weighted sum (the first version sampled twice = 2x the HBM reads).
template <int Q>
__global__ void __launch_bounds__(256)
k_att_fuse(AttP p) {
    const int HW = p.H * p.W;
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int pix = blockIdx.x * (blockDim.x >> 5) + warp;
    if (pix >= HW) return;
    float4 xs[MAX_AGENTS][Q];
    float sc[MAX_AGENTS];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < MAX_AGENTS; ++j) {
        if (j < p.n) {
            const Tap t = make_tap(p.theta + 6 * j, pix / p.W, pix % p.W, p.H, p.W, p.align);
#pragma unroll
            for (int q = 0; q < Q; ++q) xs[j][q] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int off = t.off[k];
                if (off >= 0) {
                    const float w = t.w[k];
#pragma unroll
                    for (int q = 0; q < Q; ++q) {
                        const float4 v = act_load4(p.feat, (size_t)j * HW + off, 4 * lane + 128 * q);
                        xs[j][q].x = fmaf(v.x, w, xs[j][q].x); xs[j][q].y = fmaf(v.y, w, xs[j][q].y);
                        xs[j][q].z = fmaf(v.z, w, xs[j][q].z); xs[j][q].w = fmaf(v.w, w, xs[j][q].w);
                    }
                }
            }
            float d = 0.f;
#pragma unroll
            for (int q = 0; q < Q; ++q) d += xs[0][q].x * xs[j][q].x + xs[0][q].y * xs[j][q].y + xs[0][q].z * xs[j][q].z + xs[0][q].w * xs[j][q].w;
            d = warp_sum(d) * p.inv_sqrt_dim;
            sc[j] = d;
            mx = fmaxf(mx, d);
        }
    }
    float den = 0.f;
#pragma unroll
    for (int j = 0; j < MAX_AGENTS; ++j) if (j < p.n) { sc[j] = expf(sc[j] - mx); den += sc[j]; }
    float4 acc[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < MAX_AGENTS; ++j) {
        if (j < p.n) {
            const float a = sc[j] / den;
#pragma unroll
            for (int q = 0; q < Q; ++q) {
                acc[q].x = fmaf(a, xs[j][q].x, acc[q].x); acc[q].y = fmaf(a, xs[j][q].y, acc[q].y);
                acc[q].z = fmaf(a, xs[j][q].z, acc[q].z); acc[q].w = fmaf(a, xs[j][q].w, acc[q].w);
            }
        }
    }
#pragma unroll
    for (int q = 0; q < Q; ++q) act_store4(p.out, (size_t)pix, 4 * lane + 128 * q, acc[q]);
}

// Split-bf16 features, 8 channels per lane (16-byte loads per plane and tap), C <= 256: half the load instructions of the
// generic kernel and 128-thread blocks (4 pixels) for more resident blocks per SM -- the generic version, with 8-byte loads and
// larger blocks, was latency-bound under a profiler on the B200 build.
template <int NA>
__global__ void __launch_bounds__(128)
k_att_fuse_split8(AttP p) {
    const int HW = p.H * p.W;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pix = blockIdx.x * 4 + warp;
    if (pix >= HW) return;
    const int c0 = 8 * lane;
    const bool active = c0 < p.C;
    const __nv_bfloat16* hi = reinterpret_cast<const __nv_bfloat16*>(p.feat.p) + p.feat.co + c0;
    const __nv_bfloat16* lo = hi + p.feat.plane;
    float xs[NA][8];
    float sc[NA];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < NA; ++j) {
        if (j < p.n) {
            const Tap t = make_tap(p.theta + 6 * j, pix / p.W, pix % p.W, p.H, p.W, p.align);
            uint4 vh[4], vl[4];
            float w[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                vh[k] = make_uint4(0u, 0u, 0u, 0u); vl[k] = make_uint4(0u, 0u, 0u, 0u);
                w[k] = t.w[k];
                if (t.off[k] >= 0 && active) {
                    const size_t e = ((size_t)j * HW + t.off[k]) * (size_t)p.feat.cs;
                    vh[k] = __ldg(reinterpret_cast<const uint4*>(hi + e));
                    vl[k] = __ldg(reinterpret_cast<const uint4*>(lo + e));
                } else w[k] = 0.f;
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) xs[j][e] = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t* h32 = reinterpret_cast<const uint32_t*>(&vh[k]);
                const uint32_t* l32 = reinterpret_cast<const uint32_t*>(&vl[k]);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float x0 = __uint_as_float(h32[q] << 16) + __uint_as_float(l32[q] << 16);
                    const float x1 = __uint_as_float(h32[q] & 0xffff0000u) + __uint_as_float(l32[q] & 0xffff0000u);
                    xs[j][2 * q] = fmaf(x0, w[k], xs[j][2 * q]);
                    xs[j][2 * q + 1] = fmaf(x1, w[k], xs[j][2 * q + 1]);
                }
            }
            float d = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) d += xs[0][e] * xs[j][e];
            d = warp_sum(d) * p.inv_sqrt_dim;
            sc[j] = d;
            mx = fmaxf(mx, d);
        }
    }
    float den = 0.f;
#pragma unroll
    for (int j = 0; j < NA; ++j) if (j < p.n) { sc[j] = expf(sc[j] - mx); den += sc[j]; }
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
    for (int j = 0; j < NA; ++j) {
        if (j < p.n) {
            const float a = sc[j] / den;
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = fmaf(a, xs[j][e], acc[e]);
        }
    }
    if (active) {
        act_store4(p.out, (size_t)pix, c0, make_float4(acc[0], acc[1], acc[2], acc[3]));
        act_store4(p.out, (size_t)pix, c0 + 4, make_float4(acc[4], acc[5], acc[6], acc[7]));
    }
}

// 8 channels of a pixel with 16 B stores per plane (fp32: two float4); the rounding of act_store4.
__device__ __forceinline__ void act_store8(const ActV& a, size_t pix, int c, const float (&v)[8]) {
    const size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (a.fmt == 0) {
        float4* f = reinterpret_cast<float4*>(reinterpret_cast<float*>(a.p) + idx);
        f[0] = make_float4(v[0], v[1], v[2], v[3]);
        f[1] = make_float4(v[4], v[5], v[6], v[7]);
        return;
    }
    __nv_bfloat16* b = reinterpret_cast<__nv_bfloat16*>(a.p) + idx;
    uint4 h, l;
    __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&h);
    __nv_bfloat162* l2 = reinterpret_cast<__nv_bfloat162*>(&l);
#pragma unroll
    for (int q = 0; q < 4; ++q) h2[q] = __floats2bfloat162_rn(v[2 * q], v[2 * q + 1]);
    *reinterpret_cast<uint4*>(b) = h;
    if (a.fmt == 2) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 hf = __bfloat1622float2(h2[q]);
            l2[q] = __floats2bfloat162_rn(v[2 * q] - hf.x, v[2 * q + 1] - hf.y);
        }
        *reinterpret_cast<uint4*>(b + a.plane) = l;
    }
}

// C = 64 (the first level of the multi-scale models): 8 lanes per output pixel, 8 channels per lane, 4 pixels per warp and 16
// per 128-thread block, so all 32 lanes load even though a pixel has only 64 channels.  FMT is the input format (0 f32,
// 1 bf16, 2 split-bf16): each tap is 32 B per lane in fp32 (two float4), 16 B per plane otherwise.  Every agent's warped 8-channel
// slice is sampled once (FMA over the taps in nw, ne, sw, se order, as in k_att_fuse_split8) and kept in registers for both the
// ego-row scores and the weighted sum; the score is reduced over the pixel's 8 lanes with 3 xor shuffles.
template <int NA, int FMT>
__global__ void __launch_bounds__(128)
k_att_fuse_g8(AttP p) {
    const int HW = p.H * p.W;
    if (blockIdx.x * 16 + (threadIdx.x >> 5) * 4 >= HW) return;      // whole warp past the map (the shuffles need all 32 lanes)
    const int pix_raw = blockIdx.x * 16 + (threadIdx.x >> 3);
    const bool valid = pix_raw < HW;
    const int pix = valid ? pix_raw : HW - 1;                        // a partial warp's tail lanes recompute the last pixel
    const int c0 = 8 * (threadIdx.x & 7);
    constexpr int R = FMT == 1 ? 1 : 2;                              // uint4 per tap: fp32 8 floats, split hi + lo, bf16 hi
    const size_t lo_off = FMT == 2 ? p.feat.plane : 0;
    float xs[NA][8];
    float sc[NA];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < NA; ++j) {
        if (j < p.n) {
            const Tap t = make_tap(p.theta + 6 * j, pix / p.W, pix % p.W, p.H, p.W, p.align);
            uint4 v[4][R];
            float w[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
#pragma unroll
                for (int r = 0; r < R; ++r) v[k][r] = make_uint4(0u, 0u, 0u, 0u);
                w[k] = t.w[k];
                if (t.off[k] >= 0) {
                    const size_t e = ((size_t)j * HW + t.off[k]) * (size_t)p.feat.cs + (size_t)(p.feat.co + c0);
                    if (FMT == 0) {
                        const uint4* f = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(p.feat.p) + e);
                        v[k][0] = __ldg(f);
                        v[k][R - 1] = __ldg(f + 1);
                    } else {
                        const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(p.feat.p) + e;
                        v[k][0] = __ldg(reinterpret_cast<const uint4*>(h));
                        if (FMT == 2) v[k][R - 1] = __ldg(reinterpret_cast<const uint4*>(h + lo_off));
                    }
                } else {
                    w[k] = 0.f;
                }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) xs[j][e] = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float x[8];
                const uint32_t* a32 = reinterpret_cast<const uint32_t*>(&v[k][0]);
                const uint32_t* b32 = reinterpret_cast<const uint32_t*>(&v[k][R - 1]);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (FMT == 0) {
                        x[q] = __uint_as_float(a32[q]);
                        x[4 + q] = __uint_as_float(b32[q]);
                    } else if (FMT == 1) {
                        x[2 * q] = __uint_as_float(a32[q] << 16);
                        x[2 * q + 1] = __uint_as_float(a32[q] & 0xffff0000u);
                    } else {
                        x[2 * q] = __uint_as_float(a32[q] << 16) + __uint_as_float(b32[q] << 16);
                        x[2 * q + 1] = __uint_as_float(a32[q] & 0xffff0000u) + __uint_as_float(b32[q] & 0xffff0000u);
                    }
                }
#pragma unroll
                for (int e = 0; e < 8; ++e) xs[j][e] = fmaf(x[e], w[k], xs[j][e]);
            }
            float d = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) d += xs[0][e] * xs[j][e];
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
            d *= p.inv_sqrt_dim;
            sc[j] = d;
            mx = fmaxf(mx, d);
        }
    }
    float den = 0.f;
#pragma unroll
    for (int j = 0; j < NA; ++j) if (j < p.n) { sc[j] = expf(sc[j] - mx); den += sc[j]; }
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
    for (int j = 0; j < NA; ++j) {
        if (j < p.n) {
            const float a = sc[j] / den;
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = fmaf(a, xs[j][e], acc[e]);
        }
    }
    if (valid) act_store8(p.out, (size_t)pix, c0, acc);
}

// ---- MaxFusion / V2VNetFusion (fusion_in_one.py:87-124, :203-318) ---------------------------------------------------------
// One thread per (image, pixel, 4-channel chunk); blockIdx.y is the image inside the launch.  Every thread recomputes its taps
// with make_tap (a few fp64 FMAs), so the arithmetic per tap is the one the attention / pyramid kernels use.

// bilinear sample of 4 channels of one image, zeros padding: FMA over the in-bounds taps in (nw, ne, sw, se) order
__device__ __forceinline__ float4 tap_sample4(const ActV& a, long long img_pix0, const Tap& t, int c) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (t.off[k] >= 0) {
            const float4 v = act_load4(a, (size_t)(img_pix0 + t.off[k]), c);
            const float w = t.w[k];
            s.x = fmaf(v.x, w, s.x); s.y = fmaf(v.y, w, s.y); s.z = fmaf(v.z, w, s.z); s.w = fmaf(v.w, w, s.w);
        }
    }
    return s;
}

struct MaxP { ActV feat; const double* theta; ActV out; int n, H, W, C, align; };

// out = max over agents of warp(feat_j, theta_j).  A pixel warped in from outside agent j's map samples 0, and that 0 takes part
// in the max (torch.max over the warped stack).
__global__ void __launch_bounds__(256) k_max_fuse(MaxP p) {
    const int chunks = p.C >> 2, HW = p.H * p.W;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)HW * chunks) return;
    const int pix = (int)(g / chunks), c = (int)(g % chunks) * 4;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < p.n; ++j) {
        const Tap t = make_tap(p.theta + 6 * j, pix / p.W, pix % p.W, p.H, p.W, p.align);
        const float4 v = tap_sample4(p.feat, (long long)j * HW, t, c);
        if (j == 0) m = v;
        else { m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w); }
    }
    act_store4(p.out, (size_t)pix, c, m);
}

constexpr int WARP_BATCH = 256;    // output images per heal_warp_affine launch (source indices travel in the parameter block)

struct WarpP { ActV src; const double* theta; ActV out; int H, W, C, k0; int src_img[WARP_BATCH]; };

// out image k0 + y = grid_sample(src image src_img[y], theta[k0 + y])
__global__ void __launch_bounds__(256) k_warp_affine(WarpP p) {
    const int chunks = p.C >> 2, HW = p.H * p.W;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)HW * chunks) return;
    const int pix = (int)(g / chunks), c = (int)(g % chunks) * 4;
    const int k = p.k0 + blockIdx.y;
    const Tap t = make_tap(p.theta + 6 * (long long)k, pix / p.W, pix % p.W, p.H, p.W, 0);
    act_store4(p.out, (size_t)k * HW + pix, c, tap_sample4(p.src, (long long)p.src_img[blockIdx.y] * HW, t, c));
}

constexpr int AGG_BATCH = 64;      // updated nodes per heal_v2v_aggregate launch

struct AggP {
    ActV q, pn, x, out; const double* theta;
    int H, W, C, agg_max, gru, u0;
    int4 node[AGG_BATCH];          // (x image, P image, first pair row, number of neighbours n) of updated node u0 + y
};

// One V2VNet node update.  msg_ij = mask_ij * (Q_ij + P_i) with Q_ij = W[:, :C] (*) warp(x_j, theta_ij) and P_i = W[:, C:] (*) x_i
// + b: the message conv of cat[warp(x_j), x_i] split along K, so P_i is computed once per node.  mask_ij = warp(ones, theta_ij) is
// the sum of the in-bounds tap weights (fractional on border pixels).  agg_i = mean over all n neighbours (self included, /n) or
// their max; with the GRU the output is the GRU conv input [x_i | agg_i], without it the next node feature x_i + agg_i.
__global__ void __launch_bounds__(256) k_v2v_aggregate(AggP p) {
    const int chunks = p.C >> 2, HW = p.H * p.W;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)HW * chunks) return;
    const int pix = (int)(g / chunks), c = (int)(g % chunks) * 4;
    const int4 nd = p.node[blockIdx.y];
    const int u = p.u0 + blockIdx.y;
    const float4 pi = act_load4(p.pn, (size_t)nd.y * HW + pix, c);
    float4 acc = p.agg_max ? make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < nd.w; ++j) {
        const long long row = (long long)nd.z + j;
        const Tap t = make_tap(p.theta + 6 * row, pix / p.W, pix % p.W, p.H, p.W, 0);
        float m = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) m += (t.off[k] >= 0) ? t.w[k] : 0.f;
        const float4 q = act_load4(p.q, (size_t)(row * HW + pix), c);
        const float4 v = make_float4(m * (q.x + pi.x), m * (q.y + pi.y), m * (q.z + pi.z), m * (q.w + pi.w));
        if (p.agg_max) { acc.x = fmaxf(acc.x, v.x); acc.y = fmaxf(acc.y, v.y); acc.z = fmaxf(acc.z, v.z); acc.w = fmaxf(acc.w, v.w); }
        else { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
    }
    if (!p.agg_max) {
        const float inv = (float)nd.w;
        acc.x /= inv; acc.y /= inv; acc.z /= inv; acc.w /= inv;
    }
    const float4 xi = act_load4(p.x, (size_t)nd.x * HW + pix, c);
    const size_t opix = (size_t)u * HW + pix;
    if (p.gru) {
        act_store4(p.out, opix, c, xi);
        act_store4(p.out, opix, p.C + c, acc);
    } else {
        act_store4(p.out, opix, c, make_float4(xi.x + acc.x, xi.y + acc.y, xi.z + acc.z, xi.w + acc.w));
    }
}

// ConvGRU cell with a zero hidden state: h' = sigmoid(z) * tanh(c), z = channels [0, C) and c = channels [C, 2C) of the GRU conv
// output (update-gate rows of conv_gates stacked over conv_can; the reset gate multiplies h = 0 and drops out).
__global__ void __launch_bounds__(256) k_gru_gate(ActV zc, ActV out, long long npix, int C) {
    const int chunks = C >> 2;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= npix * chunks) return;
    const size_t pix = (size_t)(g / chunks);
    const int c = (int)(g % chunks) * 4;
    const float4 z = act_load4(zc, pix, c), cc = act_load4(zc, pix, C + c);
    const float4 h = make_float4((1.f / (1.f + expf(-z.x))) * tanhf(cc.x), (1.f / (1.f + expf(-z.y))) * tanhf(cc.y),
                                 (1.f / (1.f + expf(-z.z))) * tanhf(cc.z), (1.f / (1.f + expf(-z.w))) * tanhf(cc.w));
    act_store4(out, pix, c, h);
}

// ---- Where2commFusion attention core (fusion_in_one.py:431-484, where2comm_attn.py:64-103) ---------------------------------
// nn.MultiheadAttention with one query (the warped ego) over the scene's n warped agents, per pixel and head.  The k | v in-
// projection is a per-pixel linear map, so it commutes with the bilinear warp (zero-padded taps contribute nothing): the
// kernel samples the projection of the UNWARPED maps and adds the bias afterwards.
constexpr int MHA_C = 256;         // embed dim (every baseline yaml has in_head 256)
constexpr int MHA_HEADS = 8;       // EncodeLayer's n_head; dim_head 32 = 8 lanes of 4 channels
constexpr int MHA_PIX = 256 / (MHA_C / 4);      // pixels per 256-thread block
constexpr int MHA_SCENES = 64;     // scenes per heal_ego_mha launch (their agent ranges travel in the parameter block)

struct MhaP {
    ActV q, kv, out; const float* kv_bias; const double* theta;
    int H, W, b0;
    float scale;
    int2 scene[MHA_SCENES];        // (first kv / theta image, agents n) of scene b0 + blockIdx.y
};

// thread = (pixel, 4 channels); the 8 lanes of a head reduce q.k by shuffles, and a warp never spans two pixels.  The taps of
// the block's (pixel, agent) pairs are computed once into shared memory; each agent's sampled k and v stay in registers.
__global__ void __launch_bounds__(256) k_ego_mha(MhaP p) {
    __shared__ Tap sTap[MHA_PIX][MAX_AGENTS];
    const int HW = p.H * p.W;
    const int b = p.b0 + blockIdx.y, first = p.scene[blockIdx.y].x, n = p.scene[blockIdx.y].y;
    const int pix0 = blockIdx.x * MHA_PIX;
    for (int it = threadIdx.x; it < MHA_PIX * n; it += blockDim.x) {
        const int lp = it / n, j = it % n, pix = pix0 + lp;
        if (pix < HW) sTap[lp][j] = make_tap(p.theta + 6 * (long long)(first + j), pix / p.W, pix % p.W, p.H, p.W, 0);
    }
    __syncthreads();
    const int lp = threadIdx.x / (MHA_C / 4), pix = pix0 + lp;
    if (pix >= HW) return;                                           // whole warps: 32 threads share one pixel
    const int c = (threadIdx.x % (MHA_C / 4)) * 4;
    float4 qv = act_load4(p.q, (size_t)b * HW + pix, c);
    qv.x *= p.scale; qv.y *= p.scale; qv.z *= p.scale; qv.w *= p.scale;
    const float4 bk = __ldg(reinterpret_cast<const float4*>(p.kv_bias + c));
    const float4 bv = __ldg(reinterpret_cast<const float4*>(p.kv_bias + MHA_C + c));
    float4 v[MAX_AGENTS];
    float s[MAX_AGENTS];
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < MAX_AGENTS; ++j) {
        if (j < n) {
            const Tap t = sTap[lp][j];
            const long long img0 = (long long)(first + j) * HW;
            float4 k = tap_sample4(p.kv, img0, t, c);
            v[j] = tap_sample4(p.kv, img0, t, MHA_C + c);
            k.x += bk.x; k.y += bk.y; k.z += bk.z; k.w += bk.w;
            v[j].x += bv.x; v[j].y += bv.y; v[j].z += bv.z; v[j].w += bv.w;
            float d = qv.x * k.x + qv.y * k.y + qv.z * k.z + qv.w * k.w;
            d += __shfl_xor_sync(0xffffffffu, d, 1);
            d += __shfl_xor_sync(0xffffffffu, d, 2);
            d += __shfl_xor_sync(0xffffffffu, d, 4);
            s[j] = d;
            m = fmaxf(m, d);
        }
    }
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < MAX_AGENTS; ++j) if (j < n) { s[j] = expf(s[j] - m); sum += s[j]; }
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < MAX_AGENTS; ++j) {
        if (j < n) {
            const float a = s[j] / sum;
            acc.x = fmaf(a, v[j].x, acc.x); acc.y = fmaf(a, v[j].y, acc.y);
            acc.z = fmaf(a, v[j].z, acc.z); acc.w = fmaf(a, v[j].w, acc.w);
        }
    }
    act_store4(p.out, (size_t)b * HW + pix, c, acc);
}

}  // namespace

static inline ActV to_view(const heal_act_t* a) {
    ActV v;
    v.p = a->data; v.fmt = a->fmt; v.cs = a->cstride; v.co = a->coffset; v.plane = a->plane_stride;
    return v;
}

// Views read / written 4 channels at a time (act_load4 / act_store4): every 4-channel group must start 16 B-aligned in fp32
// and 8 B-aligned in each bf16 plane, so the base pointer as well as the channel stride, offset and plane stride.
static inline bool aligned4(const heal_act_t* a) {
    const uintptr_t need = a->fmt == 0 ? 15 : 7;
    return ((uintptr_t)a->data & need) == 0 && (a->cstride & 3) == 0 && (a->coffset & 3) == 0 &&
           (a->fmt == 0 || (a->plane_stride & 3) == 0);
}
// The 8-channel split kernels load 16 B per plane: a 16 B-aligned base and channel groups of 8.
static inline bool aligned8_split(const heal_act_t* a) {
    return a->fmt == 2 && ((uintptr_t)a->data & 15) == 0 && (a->cstride & 7) == 0 && (a->coffset & 7) == 0 &&
           (a->plane_stride & 7) == 0;
}
// k_att_fuse_g8 loads and stores 16 B per plane and 8-channel group: a 16 B-aligned base, channel groups of 8 in bf16 / split
// (fp32 reads two float4, so groups of 4 do, which is aligned4).
static inline bool aligned16(const heal_act_t* a) {
    if (a->fmt == 0) return aligned4(a);
    return (a->fmt == 1 || a->fmt == 2) && ((uintptr_t)a->data & 15) == 0 && (a->cstride & 7) == 0 && (a->coffset & 7) == 0 &&
           (a->fmt == 1 || (a->plane_stride & 7) == 0);
}

template <int FMT>
static void launch_att_g8(const AttP& p, int grid, cudaStream_t st) {
    if (p.n <= 5) k_att_fuse_g8<5, FMT><<<grid, 128, 0, st>>>(p);         // register file sized for the scene
    else k_att_fuse_g8<MAX_AGENTS, FMT><<<grid, 128, 0, st>>>(p);
}

extern "C" int heal_pyramid_fuse_level(const heal_act_t* feat, const float* occ, const double* theta,
                                       const int* crop_windows, int n_agents, int H, int W, int C, int align_corners,
                                       const long long* agent_feat_offsets_host, const long long* agent_occ_offsets_host,
                                       int row0, int rows, const heal_act_t* out, void* stream_) {
    if (!feat || !feat->data || !occ || !theta || !out || !out->data) return HEAL_ERR_ARG;
    if (n_agents < 1 || n_agents > MAX_AGENTS) return HEAL_ERR_UNSUPPORTED;
    if (rows <= 0) { row0 = 0; rows = H; }
    if (row0 < 0 || row0 + rows > H) return HEAL_ERR_ARG;
    if ((C & 3) || !aligned4(feat) || !aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    FuseP p;
    p.feat = to_view(feat); p.occ = occ; p.theta = theta; p.crop = crop_windows; p.out = to_view(out);
    p.n = n_agents; p.H = H; p.W = W; p.C = C; p.align = align_corners;
    p.row0 = row0; p.rows = rows;
    bool off8 = true;
    for (int j = 0; j < MAX_AGENTS; ++j) {
        p.foff[j] = (j < n_agents) ? (agent_feat_offsets_host ? agent_feat_offsets_host[j] : (long long)j * H * W * feat->cstride) : 0;
        p.ooff[j] = (j < n_agents) ? (agent_occ_offsets_host ? agent_occ_offsets_host[j] : (long long)j * H * W) : 0;
        if (p.foff[j] & 7) off8 = false;
        if (p.foff[j] & 3) return HEAL_ERR_UNSUPPORTED;
    }
    cudaStream_t st = (cudaStream_t)stream_;
    const int HW = rows * W;
    // split-bf16 input, 16 B-aligned channel groups (base pointer included), per-agent element indices that fit 31 bits:
    // the 8-channel kernel; any other view takes the generic one
    if (aligned8_split(feat) && (C & 7) == 0 && off8 && (long long)H * W * feat->cstride < (1LL << 31)) {
        if (C >= 256)      k_pyramid_fuse_split8<8><<<(HW + 7) / 8, 256, 0, st>>>(p);
        else if (C >= 128) k_pyramid_fuse_split8<16><<<(HW + 15) / 16, 256, 0, st>>>(p);
        else               k_pyramid_fuse_split8<32><<<(HW + 31) / 32, 256, 0, st>>>(p);
        return heal_check_launch();
    }
    if (C >= 256)      k_pyramid_fuse<4><<<(HW + 3) / 4, 256, 0, st>>>(p);
    else if (C >= 128) k_pyramid_fuse<8><<<(HW + 7) / 8, 256, 0, st>>>(p);
    else if (C >= 64)  k_pyramid_fuse<16><<<(HW + 15) / 16, 256, 0, st>>>(p);
    else               k_pyramid_fuse<32><<<(HW + 31) / 32, 256, 0, st>>>(p);
    return heal_check_launch();
}

extern "C" int heal_att_fuse(const heal_act_t* feat, const double* theta, int n_agents, int H, int W, int C,
                             const heal_act_t* out, void* stream_) {
    if (!feat || !feat->data || !theta || !out || !out->data) return HEAL_ERR_ARG;
    if (n_agents < 1 || n_agents > MAX_AGENTS) return HEAL_ERR_UNSUPPORTED;
    if (C == 64) {
        if (!aligned16(feat) || !aligned16(out)) return HEAL_ERR_UNSUPPORTED;
    } else if ((C % 128) || C > 512 || !aligned4(feat) || !aligned4(out)) {
        return HEAL_ERR_UNSUPPORTED;
    }
    AttP p;
    p.feat = to_view(feat); p.theta = theta; p.out = to_view(out); p.n = n_agents; p.H = H; p.W = W; p.C = C; p.align = 0;
    p.inv_sqrt_dim = 1.0f / sqrtf((float)C);
    cudaStream_t st = (cudaStream_t)stream_;
    if (C == 64) {
        const int grid = (H * W + 15) / 16;
        if (feat->fmt == 0) launch_att_g8<0>(p, grid, st);
        else if (feat->fmt == 1) launch_att_g8<1>(p, grid, st);
        else launch_att_g8<2>(p, grid, st);
        return heal_check_launch();
    }
    if (aligned8_split(feat) && C <= 256) {
        if (n_agents <= 5) k_att_fuse_split8<5><<<(H * W + 3) / 4, 128, 0, st>>>(p);       // register file sized for the scene
        else k_att_fuse_split8<MAX_AGENTS><<<(H * W + 3) / 4, 128, 0, st>>>(p);
        return heal_check_launch();
    }
    int grid = (H * W + 7) / 8;
    switch (C / 128) {
        case 1: k_att_fuse<1><<<grid, 256, 0, st>>>(p); break;
        case 2: k_att_fuse<2><<<grid, 256, 0, st>>>(p); break;
        case 3: k_att_fuse<3><<<grid, 256, 0, st>>>(p); break;
        default: k_att_fuse<4><<<grid, 256, 0, st>>>(p); break;
    }
    return heal_check_launch();
}

static inline long long grid_x(int H, int W, int C) { return ((long long)H * W * (C / 4) + 255) / 256; }

extern "C" int heal_max_fuse(const heal_act_t* feat, const double* theta, int n_agents, int H, int W, int C,
                             const heal_act_t* out, void* stream_) {
    if (!feat || !feat->data || !theta || !out || !out->data || H < 1 || W < 1) return HEAL_ERR_ARG;
    if (n_agents < 1 || (C & 3) || !aligned4(feat) || !aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    MaxP p;
    p.feat = to_view(feat); p.theta = theta; p.out = to_view(out); p.n = n_agents; p.H = H; p.W = W; p.C = C; p.align = 0;
    k_max_fuse<<<(unsigned)grid_x(H, W, C), 256, 0, (cudaStream_t)stream_>>>(p);
    return heal_check_launch();
}

extern "C" int heal_warp_affine(const heal_act_t* src, const int* src_index_host, const double* theta, int n_out,
                                int H, int W, int C, const heal_act_t* out, void* stream_) {
    if (!src || !src->data || !src_index_host || !theta || !out || !out->data || n_out < 0 || H < 1 || W < 1) return HEAL_ERR_ARG;
    if ((C & 3) || !aligned4(src) || !aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    WarpP p;
    p.src = to_view(src); p.theta = theta; p.out = to_view(out); p.H = H; p.W = W; p.C = C;
    int launches = 0;
    for (int k0 = 0; k0 < n_out; k0 += WARP_BATCH) {
        const int nb = n_out - k0 < WARP_BATCH ? n_out - k0 : WARP_BATCH;
        p.k0 = k0;
        for (int y = 0; y < nb; ++y) {
            if (src_index_host[k0 + y] < 0) return HEAL_ERR_ARG;
            p.src_img[y] = src_index_host[k0 + y];
        }
        k_warp_affine<<<dim3((unsigned)grid_x(H, W, C), nb), 256, 0, (cudaStream_t)stream_>>>(p);
        ++launches;
    }
    return heal_check_launch(launches);
}

extern "C" int heal_v2v_aggregate(const heal_act_t* q, const heal_act_t* p_node, const heal_act_t* x, const double* theta,
                                  const int* nodes_host, int n_nodes, int H, int W, int C, int agg_max, int gru,
                                  const heal_act_t* out, void* stream_) {
    if (!q || !q->data || !p_node || !p_node->data || !x || !x->data || !theta || !nodes_host || !out || !out->data) return HEAL_ERR_ARG;
    if (n_nodes < 0 || H < 1 || W < 1) return HEAL_ERR_ARG;
    if ((C & 3) || !aligned4(q) || !aligned4(p_node) || !aligned4(x) || !aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    AggP p;
    p.q = to_view(q); p.pn = to_view(p_node); p.x = to_view(x); p.out = to_view(out); p.theta = theta;
    p.H = H; p.W = W; p.C = C; p.agg_max = agg_max ? 1 : 0; p.gru = gru ? 1 : 0;
    int launches = 0;
    for (int u0 = 0; u0 < n_nodes; u0 += AGG_BATCH) {
        const int nb = n_nodes - u0 < AGG_BATCH ? n_nodes - u0 : AGG_BATCH;
        p.u0 = u0;
        for (int y = 0; y < nb; ++y) {
            const int* nd = nodes_host + 4 * (u0 + y);
            if (nd[0] < 0 || nd[1] < 0 || nd[2] < 0 || nd[3] < 1) return HEAL_ERR_ARG;
            p.node[y] = make_int4(nd[0], nd[1], nd[2], nd[3]);
        }
        k_v2v_aggregate<<<dim3((unsigned)grid_x(H, W, C), nb), 256, 0, (cudaStream_t)stream_>>>(p);
        ++launches;
    }
    return heal_check_launch(launches);
}

extern "C" int heal_ego_mha(const heal_act_t* q, const heal_act_t* kv, const float* kv_bias, const double* theta,
                            const int* n_agents_host, int B, int H, int W, int C, int heads, const heal_act_t* out,
                            void* stream_) {
    if (!q || !q->data || !kv || !kv->data || !kv_bias || !theta || !n_agents_host || !out || !out->data) return HEAL_ERR_ARG;
    if (B < 0 || H < 1 || W < 1 || q->fmt < 0 || q->fmt > 2 || kv->fmt < 0 || kv->fmt > 2 || out->fmt < 0 || out->fmt > 2)
        return HEAL_ERR_ARG;
    if (C != MHA_C || heads != MHA_HEADS) return HEAL_ERR_UNSUPPORTED;
    if (!aligned4(q) || !aligned4(kv) || !aligned4(out) || ((uintptr_t)kv_bias & 15)) return HEAL_ERR_UNSUPPORTED;
    if ((long long)H * W >= (1LL << 31)) return HEAL_ERR_UNSUPPORTED;      // pixel indices are ints
    for (int b = 0; b < B; ++b)          // every count before the first launch, so a bad one leaves the output untouched
        if (n_agents_host[b] < 1 || n_agents_host[b] > MAX_AGENTS) return HEAL_ERR_ARG;
    MhaP p;
    p.q = to_view(q); p.kv = to_view(kv); p.out = to_view(out); p.kv_bias = kv_bias; p.theta = theta;
    p.H = H; p.W = W;
    p.scale = (float)sqrt(1.0 / (double)(C / heads));      // PyTorch's q * sqrt(1 / dim_head), in fp32
    const unsigned grid = (unsigned)(((long long)H * W + MHA_PIX - 1) / MHA_PIX);
    int first = 0, launches = 0;
    for (int b0 = 0; b0 < B; b0 += MHA_SCENES) {
        const int nb = B - b0 < MHA_SCENES ? B - b0 : MHA_SCENES;
        p.b0 = b0;
        for (int z = 0; z < nb; ++z) {
            p.scene[z] = make_int2(first, n_agents_host[b0 + z]);
            first += n_agents_host[b0 + z];
        }
        k_ego_mha<<<dim3(grid, (unsigned)nb), 256, 0, (cudaStream_t)stream_>>>(p);
        ++launches;
    }
    return heal_check_launch(launches);
}

extern "C" int heal_gru_gate(const heal_act_t* zc, long long npix, int C, const heal_act_t* out, void* stream_) {
    if (!zc || !zc->data || !out || !out->data || npix < 0) return HEAL_ERR_ARG;
    if ((C & 3) || !aligned4(zc) || !aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    if (npix == 0) return HEAL_OK;
    const long long blocks = (npix * (C / 4) + 255) / 256;
    k_gru_gate<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream_>>>(to_view(zc), to_view(out), npix, C);
    return heal_check_launch();
}
