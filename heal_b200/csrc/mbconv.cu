// EfficientNet-B0 camera trunk of Lift-Splat-Shoot (`camera_encoder: EfficientNet`; opencood/models/sub_modules/lss_submodule.py:39-138
// runs efficientnet_pytorch's stem and 16 MBConv blocks, then two `Up` stages).  All trunk tensors are dense channels-last fp32.
//   k_stem_conv_swish      3x3 / stride 2 conv 3 -> 32 straight from the NCHW image, pad (0, 1), folded BN, swish
//   k_dwconv_bn_swish      depthwise 3x3 | 5x5, stride 1 | 2, per-side pads, folded BN, swish; per-block channel sums of the output
//   k_dwconv_sum_finish    ordered sum of those partials -> (image, channel) sums for the squeeze-and-excitation mean
//   k_se_gate              mean -> reduce (C -> Csq) -> swish -> expand (Csq -> C) -> sigmoid, one block per image
//   k_pwconv               1x1 conv as a register-tiled fp32 GEMM over pixels: optional per-(image, Cin) gate on the input (the SE
//                          multiply, so the gated tensor is never stored), folded BN, optional swish, optional residual
//   k_upsample2x_concat    `Up`'s front half: [x2 | bilinear x2 (align_corners) of x1 | zeros] in the conv engine's activation format
// The layers are narrow (16 .. 1152 channels) and HBM / launch bound; the dense 3x3 convolutions of `Up`, which carry the FLOPs,
// run on the wgmma engine (csrc/conv2d_tc.cu).  No float atomics: the channel sums are the same bits on every run.
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

__device__ __forceinline__ float swish(float v) { return v / (1.f + expf(-v)); }

// ---- stem -------------------------------------------------------------------------------------------------------------------
// thread = (output pixel, 4 of the 32 output channels); weights [27][32] (row = (ci * 3 + ky) * 3 + kx) staged in shared memory
__global__ void __launch_bounds__(256)
k_stem_conv_swish(const float* __restrict__ img, int N, int Cimg, int H, int W, const float* __restrict__ w,
                  const float* __restrict__ bias, float* __restrict__ out, int Ho, int Wo) {
    __shared__ float4 ws[27 * 8];
    for (int i = threadIdx.x; i < 27 * 8; i += blockDim.x) ws[i] = ldg_f4(w + 4 * i);
    __syncthreads();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)N * Ho * Wo * 8) return;
    const int cq = (int)(t & 7);
    long long pix = t >> 3;
    const int ox = (int)(pix % Wo); pix /= Wo;
    const int oy = (int)(pix % Ho); const int n = (int)(pix / Ho);
    float4 acc = ldg_f4(bias + 4 * cq);
    const float* base = img + (size_t)n * Cimg * H * W;
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int y = 2 * oy + ky;                       // pad top 0, bottom 1
            if (y >= H) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int x = 2 * ox + kx;                   // pad left 0, right 1
                if (x >= W) continue;
                const float v = __ldg(base + ((size_t)ci * H + y) * W + x);
                const float4 wv = ws[((ci * 3 + ky) * 3 + kx) * 8 + cq];
                acc.x = fmaf(v, wv.x, acc.x); acc.y = fmaf(v, wv.y, acc.y);
                acc.z = fmaf(v, wv.z, acc.z); acc.w = fmaf(v, wv.w, acc.w);
            }
        }
    }
    acc.x = swish(acc.x); acc.y = swish(acc.y); acc.z = swish(acc.z); acc.w = swish(acc.w);
    stg_f4(out + (size_t)t * 4, acc);
}

// ---- depthwise conv + BN + swish + channel sums -------------------------------------------------------------------------------
struct DwP {
    const float* in; const float* w; const float* bias; float* out; float* partial;
    int N, H, W, C, k, stride, pad_t, pad_l, Ho, Wo;
    int lx, ly, slabs, chunks;         // thread tile: lx channel quads x ly pixel lanes; `slabs` channel slabs; `chunks` pixel chunks
};
constexpr int DW_ITERS = 8;            // output pixels per pixel lane
constexpr int DW_THREADS = 256;

// grid (chunks, slabs, N).  Thread (cx, py): channel quad slab * lx + cx, pixels chunk * ly * DW_ITERS + it * ly + py.  Each block
// writes the sum of its outputs per channel to partial[(n * chunks + chunk) * C + c], added in a fixed order.
__global__ void __launch_bounds__(DW_THREADS)
k_dwconv_bn_swish(DwP p) {
    __shared__ float4 red[DW_THREADS];
    const int cx = threadIdx.x % p.lx, py = threadIdx.x / p.lx;
    const int q = blockIdx.y * p.lx + cx;                    // channel quad
    const int n = blockIdx.z;
    const bool live = py < p.ly && q * 4 < p.C;
    float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live) {
        const int c = q * 4;
        const float4 b = ldg_f4(p.bias + c);
        const int HW = p.Ho * p.Wo;
        const float* img = p.in + (size_t)n * p.H * p.W * p.C;
        for (int it = 0; it < DW_ITERS; ++it) {
            const int pix = (blockIdx.x * DW_ITERS + it) * p.ly + py;
            if (pix >= HW) break;
            const int oy = pix / p.Wo, ox = pix - oy * p.Wo;
            float4 acc = b;
            for (int ky = 0; ky < p.k; ++ky) {
                const int y = oy * p.stride - p.pad_t + ky;
                if (y < 0 || y >= p.H) continue;
                for (int kx = 0; kx < p.k; ++kx) {
                    const int x = ox * p.stride - p.pad_l + kx;
                    if (x < 0 || x >= p.W) continue;
                    const float4 v = ldg_f4(img + ((size_t)y * p.W + x) * p.C + c);
                    const float4 wv = ldg_f4(p.w + (size_t)(ky * p.k + kx) * p.C + c);
                    acc.x = fmaf(v.x, wv.x, acc.x); acc.y = fmaf(v.y, wv.y, acc.y);
                    acc.z = fmaf(v.z, wv.z, acc.z); acc.w = fmaf(v.w, wv.w, acc.w);
                }
            }
            acc.x = swish(acc.x); acc.y = swish(acc.y); acc.z = swish(acc.z); acc.w = swish(acc.w);
            stg_f4(p.out + ((size_t)n * HW + pix) * p.C + c, acc);
            sum.x += acc.x; sum.y += acc.y; sum.z += acc.z; sum.w += acc.w;
        }
    }
    red[threadIdx.x] = sum;
    __syncthreads();
    if (py == 0 && q * 4 < p.C) {
        for (int j = 1; j < p.ly; ++j) {
            const float4 o = red[j * p.lx + cx];
            sum.x += o.x; sum.y += o.y; sum.z += o.z; sum.w += o.w;
        }
        stg_f4(p.partial + ((size_t)n * p.chunks + blockIdx.x) * p.C + q * 4, sum);
    }
}

__global__ void __launch_bounds__(256)
k_dwconv_sum_finish(const float* __restrict__ partial, int N, int C, int chunks, float* __restrict__ sums) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N * C) return;
    const int n = t / C, c = t - n * C;
    float s = 0.f;
    for (int j = 0; j < chunks; ++j) s += __ldg(partial + ((size_t)n * chunks + j) * C + c);
    sums[t] = s;
}

static void dw_tile(int C, int HoWo, int* lx, int* ly, int* slabs, int* chunks) {
    const int quads = C / 4;
    *slabs = (quads + 31) / 32;
    *lx = (quads + *slabs - 1) / *slabs;
    *ly = DW_THREADS / *lx;
    *chunks = (HoWo + *ly * DW_ITERS - 1) / (*ly * DW_ITERS);
}

// ---- squeeze-and-excitation gate -----------------------------------------------------------------------------------------------
constexpr int SE_MAX_C = 1152, SE_MAX_SQ = 64;

// one block per image: warp j computes squeezed channel j (coalesced rows of w_reduce), then thread c computes gate[c]
__global__ void __launch_bounds__(256)
k_se_gate(const float* __restrict__ sums, float inv_hw, int C, int Csq, const float* __restrict__ w_reduce,
          const float* __restrict__ b_reduce, const float* __restrict__ w_expand_t, const float* __restrict__ b_expand,
          float* __restrict__ gate) {
    __shared__ float mean[SE_MAX_C];
    __shared__ float sq[SE_MAX_SQ];
    const int n = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int c = threadIdx.x; c < C; c += blockDim.x) mean[c] = sums[(size_t)n * C + c] * inv_hw;
    __syncthreads();
    for (int j = warp; j < Csq; j += 8) {
        float s = 0.f;
        for (int c = lane; c < C; c += 32) s = fmaf(mean[c], __ldg(w_reduce + (size_t)j * C + c), s);
        s = warp_sum(s);
        if (lane == 0) sq[j] = swish(s + __ldg(b_reduce + j));
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = __ldg(b_expand + c);
        for (int j = 0; j < Csq; ++j) s = fmaf(sq[j], __ldg(w_expand_t + (size_t)j * C + c), s);
        gate[(size_t)n * C + c] = 1.f / (1.f + expf(-s));
    }
}

// ---- pointwise conv ------------------------------------------------------------------------------------------------------------
struct PwP {
    const float* in; const float* w; const float* bias; const float* gate; const float* res; float* out;
    long long M;                       // pixels (images * HW)
    int HW, Cin, Cout, swish;
};
constexpr int PW_BM = 64, PW_BN = 64, PW_BK = 16;

// block tile 64 pixels x 64 output channels, K step 16, thread tile 4 x 4.  w is [Cin][Cout].  Cin, Cout multiples of 4.
__global__ void __launch_bounds__(256)
k_pwconv(PwP p) {
    __shared__ __align__(16) float As[PW_BK][PW_BM + 4];
    __shared__ __align__(16) float Bs[PW_BK][PW_BN];
    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    const long long m0 = (long long)blockIdx.x * PW_BM;
    const int n0 = blockIdx.y * PW_BN;
    const int am = t >> 2, ak = (t & 3) * 4;                 // A loader: pixel row, k quad
    const int bk = t >> 4, bn = (t & 15) * 4;                // B loader: k row, cout quad
    const long long apix = m0 + am;
    const float* grow = (p.gate && apix < p.M) ? p.gate + (size_t)(apix / p.HW) * p.Cin : nullptr;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < p.Cin; k0 += PW_BK) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        if (apix < p.M && k0 + ak < p.Cin) {
            a = ldg_f4(p.in + (size_t)apix * p.Cin + k0 + ak);
            if (grow) {
                const float4 g = ldg_f4(grow + k0 + ak);
                a.x *= g.x; a.y *= g.y; a.z *= g.z; a.w *= g.w;
            }
        }
        As[ak + 0][am] = a.x; As[ak + 1][am] = a.y; As[ak + 2][am] = a.z; As[ak + 3][am] = a.w;
        float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k0 + bk < p.Cin && n0 + bn < p.Cout) b = ldg_f4(p.w + (size_t)(k0 + bk) * p.Cout + n0 + bn);
        *reinterpret_cast<float4*>(&Bs[bk][bn]) = b;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PW_BK; ++k) {
            const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
            const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
            const float ar[4] = {av.x, av.y, av.z, av.w};
            const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
        }
        __syncthreads();
    }
    const int co = n0 + tx * 4;
    if (co >= p.Cout) return;
    const float4 b = ldg_f4(p.bias + co);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long pix = m0 + ty * 4 + i;
        if (pix >= p.M) break;
        float4 v = make_float4(acc[i][0] + b.x, acc[i][1] + b.y, acc[i][2] + b.z, acc[i][3] + b.w);
        if (p.swish) { v.x = swish(v.x); v.y = swish(v.y); v.z = swish(v.z); v.w = swish(v.w); }
        if (p.res) {
            const float4 r = ldg_f4(p.res + (size_t)pix * p.Cout + co);
            v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
        }
        stg_f4(p.out + (size_t)pix * p.Cout + co, v);
    }
}

// ---- Up: bilinear x2 (align_corners=True) of x1, concatenated behind x2, zero tail ------------------------------------------------
struct UpP {
    ActV x1, x2, out;
    int N, H1, W1, C1, C2, Cout;
    float sy, sx;                      // (in - 1) / (out - 1), as torch's area_pixel_compute_scale with align_corners
};

// grid (pixel-quads of one image, N); thread = (output pixel, 4 output channels)
__global__ void __launch_bounds__(256)
k_upsample2x_concat(UpP p) {
    const int cq = p.Cout / 4, Ho = 2 * p.H1, Wo = 2 * p.W1, n = blockIdx.y;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= Ho * Wo * cq) return;
    const int ipix = t / cq, c = (t - ipix * cq) * 4;
    const int oy = ipix / Wo, ox = ipix - oy * Wo;
    const size_t opix = (size_t)n * Ho * Wo + ipix;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < p.C2) {
        v = act_load4(p.x2, opix, c);
    } else if (c < p.C2 + p.C1) {
        const float fy = p.sy * (float)oy, fx = p.sx * (float)ox;
        const int y0 = (int)fy, x0 = (int)fx;
        const int y1 = y0 + (y0 < p.H1 - 1), x1 = x0 + (x0 < p.W1 - 1);
        const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
        const size_t img = (size_t)n * p.H1 * p.W1;
        const int c1 = c - p.C2;
        const float4 a = act_load4(p.x1, img + (size_t)y0 * p.W1 + x0, c1), b = act_load4(p.x1, img + (size_t)y0 * p.W1 + x1, c1);
        const float4 d = act_load4(p.x1, img + (size_t)y1 * p.W1 + x0, c1), e = act_load4(p.x1, img + (size_t)y1 * p.W1 + x1, c1);
        v.x = hy * (hx * a.x + lx * b.x) + ly * (hx * d.x + lx * e.x);
        v.y = hy * (hx * a.y + lx * b.y) + ly * (hx * d.y + lx * e.y);
        v.z = hy * (hx * a.z + lx * b.z) + ly * (hx * d.z + lx * e.z);
        v.w = hy * (hx * a.w + lx * b.w) + ly * (hx * d.w + lx * e.w);
    }
    act_store4(p.out, opix, c, v);
}

static inline ActV view_of(const heal_act_t* a) {
    ActV v;
    v.p = a->data; v.fmt = a->fmt; v.cs = a->cstride; v.co = a->coffset; v.plane = a->plane_stride;
    return v;
}

static inline bool quad_aligned(const heal_act_t* a) { return !((a->cstride | a->coffset) & 3) && !((uintptr_t)a->data & 15); }

}  // namespace

extern "C" int heal_stem_conv_swish(const float* image, int N, int image_channels, int H, int W, const float* weight,
                                    const float* bias, float* out, void* stream_) {
    if (!image || !weight || !bias || !out || N < 1 || H < 2 || W < 2) return HEAL_ERR_ARG;
    if (image_channels < 3) return HEAL_ERR_UNSUPPORTED;
    const int Ho = (H - 2) / 2 + 1, Wo = (W - 2) / 2 + 1;
    const long long total = (long long)N * Ho * Wo * 8;
    k_stem_conv_swish<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(image, N, image_channels, H, W, weight,
                                                                                         bias, out, Ho, Wo);
    return heal_check_launch();
}

extern "C" size_t heal_dwconv_bn_swish_workspace(int N, int C, int Ho, int Wo) {
    if (N < 1 || C < 4 || (C & 3) || Ho < 1 || Wo < 1) return 0;
    int lx, ly, slabs, chunks;
    dw_tile(C, Ho * Wo, &lx, &ly, &slabs, &chunks);
    return (size_t)N * chunks * C * sizeof(float);
}

extern "C" int heal_dwconv_bn_swish(const float* in, int N, int H, int W, int C, const float* weight, const float* bias, int ksize,
                                    int stride, int pad_top, int pad_left, int Ho, int Wo, float* out, float* sums,
                                    void* workspace, size_t workspace_bytes, void* stream_) {
    if (!in || !weight || !bias || !out || !sums || N < 1 || H < 1 || W < 1 || Ho < 1 || Wo < 1 || pad_top < 0 || pad_left < 0)
        return HEAL_ERR_ARG;
    if ((ksize != 3 && ksize != 5) || (stride != 1 && stride != 2) || C < 4 || (C & 3)) return HEAL_ERR_UNSUPPORTED;
    DwP p;
    p.in = in; p.w = weight; p.bias = bias; p.out = out; p.partial = (float*)workspace;
    p.N = N; p.H = H; p.W = W; p.C = C; p.k = ksize; p.stride = stride; p.pad_t = pad_top; p.pad_l = pad_left; p.Ho = Ho; p.Wo = Wo;
    dw_tile(C, Ho * Wo, &p.lx, &p.ly, &p.slabs, &p.chunks);
    if (!workspace || workspace_bytes < (size_t)N * p.chunks * C * sizeof(float)) return HEAL_ERR_WORKSPACE;
    k_dwconv_bn_swish<<<dim3(p.chunks, p.slabs, N), DW_THREADS, 0, (cudaStream_t)stream_>>>(p);
    k_dwconv_sum_finish<<<(N * C + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(p.partial, N, C, p.chunks, sums);
    return heal_check_launch(2);
}

extern "C" int heal_se_gate(const float* sums, int N, int C, int Csq, int HW, const float* w_reduce, const float* b_reduce,
                            const float* w_expand_t, const float* b_expand, float* gate, void* stream_) {
    if (!sums || !w_reduce || !b_reduce || !w_expand_t || !b_expand || !gate || N < 1 || HW < 1) return HEAL_ERR_ARG;
    if (C < 1 || C > SE_MAX_C || Csq < 1 || Csq > SE_MAX_SQ) return HEAL_ERR_UNSUPPORTED;
    k_se_gate<<<N, 256, 0, (cudaStream_t)stream_>>>(sums, 1.f / (float)HW, C, Csq, w_reduce, b_reduce, w_expand_t, b_expand, gate);
    return heal_check_launch();
}

extern "C" int heal_pwconv(const float* in, int N, int HW, int Cin, int Cout, const float* weight, const float* bias,
                           const float* gate, int swish_epilogue, const float* residual, float* out, void* stream_) {
    if (!in || !weight || !bias || !out || N < 1 || HW < 1) return HEAL_ERR_ARG;
    if (Cin < 4 || (Cin & 3) || Cout < 4 || (Cout & 3)) return HEAL_ERR_UNSUPPORTED;
    PwP p;
    p.in = in; p.w = weight; p.bias = bias; p.gate = gate; p.res = residual; p.out = out;
    p.M = (long long)N * HW; p.HW = HW; p.Cin = Cin; p.Cout = Cout; p.swish = swish_epilogue;
    dim3 grid((unsigned)((p.M + PW_BM - 1) / PW_BM), (Cout + PW_BN - 1) / PW_BN);
    k_pwconv<<<grid, 256, 0, (cudaStream_t)stream_>>>(p);
    return heal_check_launch();
}

extern "C" int heal_upsample2x_concat(const heal_act_t* x1, const heal_act_t* x2, int N, int H1, int W1, int C1, int C2,
                                      const heal_act_t* out, int Cout, void* stream_) {
    if (!x1 || !x1->data || !x2 || !x2->data || !out || !out->data || N < 1 || H1 < 1 || W1 < 1) return HEAL_ERR_ARG;
    if (C1 < 4 || (C1 & 3) || C2 < 4 || (C2 & 3) || (Cout & 3) || Cout < C1 + C2) return HEAL_ERR_UNSUPPORTED;
    if (!quad_aligned(x1) || !quad_aligned(x2) || !quad_aligned(out)) return HEAL_ERR_UNSUPPORTED;
    UpP p;
    p.x1 = view_of(x1); p.x2 = view_of(x2); p.out = view_of(out);
    p.N = N; p.H1 = H1; p.W1 = W1; p.C1 = C1; p.C2 = C2; p.Cout = Cout;
    p.sy = (float)(H1 - 1) / (float)(2 * H1 - 1);
    p.sx = (float)(W1 - 1) / (float)(2 * W1 - 1);
    const long long per_image = 4LL * H1 * W1 * (Cout / 4);
    if (per_image > 0x7fffffff - 256 || N > 65535) return HEAL_ERR_UNSUPPORTED;
    k_upsample2x_concat<<<dim3((unsigned)((per_image + 255) / 256), N), 256, 0, (cudaStream_t)stream_>>>(p);
    return heal_check_launch();
}
