// Multi-agent BEV feature fusion kernels (channels-last):
//   heal_pyramid_fuse_level : warp(feat) + warp(score) -> mask -> softmax over agents -> weighted sum
//       reference: opencood/models/fuse_modules/pyramid_fuse.py:17-63 (weighted_fuse) and :143-164
//       (score = sigmoid(occ) + 1e-4, camera crop mask in eval mode)
//   heal_att_fuse           : warp -> per-pixel scaled dot-product attention over agents, ego row only
//       reference: opencood/models/fuse_modules/fusion_in_one.py:126-151 (AttFusion), :41-45
// Both fold warp_affine_simple (torch_transformation_utils.py:323-332 = F.affine_grid with an fp64
// theta, cast to fp32, then F.grid_sample bilinear / zeros padding) into the fusion so the warped
// per-agent maps never exist in HBM.
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

}  // namespace

static inline ActV to_view(const heal_act_t* a) {
    ActV v;
    v.p = a->data; v.fmt = a->fmt; v.cs = a->cstride; v.co = a->coffset; v.plane = a->plane_stride;
    return v;
}

extern "C" int heal_pyramid_fuse_level(const heal_act_t* feat, const float* occ, const double* theta,
                                       const int* crop_windows, int n_agents, int H, int W, int C, int align_corners,
                                       const long long* agent_feat_offsets_host, const long long* agent_occ_offsets_host,
                                       int row0, int rows, const heal_act_t* out, void* stream_) {
    if (!feat || !feat->data || !occ || !theta || !out || !out->data) return HEAL_ERR_ARG;
    if (n_agents < 1 || n_agents > MAX_AGENTS) return HEAL_ERR_UNSUPPORTED;
    if (rows <= 0) { row0 = 0; rows = H; }
    if (row0 < 0 || row0 + rows > H) return HEAL_ERR_ARG;
    if ((C & 3) || (feat->cstride & 3) || (feat->coffset & 3) || (out->cstride & 3) || (out->coffset & 3)) return HEAL_ERR_UNSUPPORTED;
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
    // split-bf16 input, 16 B-aligned channel groups, per-agent element indices that fit 31 bits: the 8-channel kernel
    if (feat->fmt == 2 && (C & 7) == 0 && (feat->cstride & 7) == 0 && (feat->coffset & 7) == 0 && (feat->plane_stride & 7) == 0 && off8 &&
        (long long)H * W * feat->cstride < (1LL << 31)) {
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
    if ((C % 128) || C > 512 || (feat->cstride & 3) || (feat->coffset & 3) || (out->cstride & 3) || (out->coffset & 3)) return HEAL_ERR_UNSUPPORTED;
    AttP p;
    p.feat = to_view(feat); p.theta = theta; p.out = to_view(out); p.n = n_agents; p.H = H; p.W = W; p.C = C; p.align = 0;
    p.inv_sqrt_dim = 1.0f / sqrtf((float)C);
    cudaStream_t st = (cudaStream_t)stream_;
    if (feat->fmt == 2 && C <= 256 && (C & 7) == 0 && (feat->cstride & 7) == 0 && (feat->coffset & 7) == 0 && (feat->plane_stride & 7) == 0) {
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
