// ConvNeXt aligner front half: depthwise k x k convolution + bias + LayerNorm over the channels of every pixel, one kernel.
// Reference: opencood/models/sub_modules/feature_alignnet_modules.py:299-345 (ConvNeXtBlock: dwconv -> permute -> LayerNorm(eps 1e-6,
// channels_last, :12-25) -> Linear -> GELU -> Linear -> gamma -> + input).  The two Linear layers are 1x1 convolutions and run on
// the wgmma conv engine (csrc/conv2d_tc.cu, GELU / residual in its epilogue); this kernel produces their input.
// HBM-bound: reads the map once (the 7x7 neighbourhood of a pixel is shared through L1/L2 by the warps of a block, which cover
// 8 x 4 neighbouring pixels), writes it once.  One warp per pixel, lane = channel pair (C = 64) -> every tap is one coalesced
// 256 B (fp32) row read; mean / variance by warp shuffles, exactly LayerNorm's biased variance.
// heal_mean_layernorm reuses that LayerNorm after a mean over n_avg consecutive images: CoBEVT's pre-norms (n_avg = 1) and its
// mlp_head Reduce-mean over the agent slots + LayerNorm (n_avg = L; fusion_in_one.py:401-407).
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

// LayerNorm over the C channels (C = 64 .. 256, multiple of 64) of one pixel held by one warp: acc[2q], acc[2q + 1] are channels
// q * 64 + 2 * lane and + 1.  Mean and biased variance by warp shuffles (LayerNorm's definition), then the affine transform.
// The one LayerNorm of the library: the ConvNeXt front half and CoBEVT's pre-norms / head both end in it.
__device__ __forceinline__ void warp_layernorm_store(const float (&acc)[8], int C, int lane, const float* lnw, const float* lnb,
                                                     float eps, const ActV& out, size_t opix) {
    const int chunks = C / 64;
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) if (q < chunks) s += acc[2 * q] + acc[2 * q + 1];
    const float mean = warp_sum(s) / (float)C;
    float v = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) if (q < chunks) { const float d0 = acc[2 * q] - mean, d1 = acc[2 * q + 1] - mean; v += d0 * d0 + d1 * d1; }
    const float rstd = rsqrtf(warp_sum(v) / (float)C + eps);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        if (q < chunks) {
            const int c = q * 64 + 2 * lane;
            act_store1(out, opix, c, (acc[2 * q] - mean) * rstd * __ldg(lnw + c) + __ldg(lnb + c));
            act_store1(out, opix, c + 1, (acc[2 * q + 1] - mean) * rstd * __ldg(lnw + c + 1) + __ldg(lnb + c + 1));
        }
    }
}

struct DwLnP {
    ActV in, out;
    const float* w;      // [k*k][C] depthwise weights (tap-major, channel contiguous)
    const float* b;      // [C] conv bias
    const float* lnw;    // [C] LayerNorm weight
    const float* lnb;    // [C] LayerNorm bias
    int N, H, W, C, k;
    float eps;
};

// block = 32 warps = 8 (x) x 4 (y) pixels; lanes cover C in chunks of 64 (2 channels per lane per chunk)
__global__ void __launch_bounds__(1024)
k_dwconv_ln(DwLnP p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int x = blockIdx.x * 8 + (warp & 7), y = blockIdx.y * 4 + (warp >> 3), n = blockIdx.z;
    if (x >= p.W || y >= p.H) return;
    const int r = p.k / 2;
    const size_t img = (size_t)n * p.H * p.W;
    float acc[8];                                  // up to C = 256: 4 chunks x 2 channels
    const int chunks = p.C / 64;
#pragma unroll
    for (int q = 0; q < 4; ++q) { acc[2 * q] = 0.f; acc[2 * q + 1] = 0.f; }
    for (int q = 0; q < chunks; ++q) {
        const int c = q * 64 + 2 * lane;
        float a0 = p.b ? __ldg(p.b + c) : 0.f, a1 = p.b ? __ldg(p.b + c + 1) : 0.f;
        for (int dy = -r; dy <= r; ++dy) {
            const int yy = y + dy;
            if (yy < 0 || yy >= p.H) continue;
            for (int dx = -r; dx <= r; ++dx) {
                const int xx = x + dx;
                if (xx < 0 || xx >= p.W) continue;
                const float2 wv = __ldg(reinterpret_cast<const float2*>(p.w + (size_t)((dy + r) * p.k + (dx + r)) * p.C + c));
                const size_t pix = img + (size_t)yy * p.W + xx;
                const float v0 = act_load1(p.in, pix, c), v1 = act_load1(p.in, pix, c + 1);
                a0 = fmaf(v0, wv.x, a0);
                a1 = fmaf(v1, wv.y, a1);
            }
        }
        acc[2 * q] = a0; acc[2 * q + 1] = a1;
    }
    warp_layernorm_store(acc, p.C, lane, p.lnw, p.lnb, p.eps, p.out, img + (size_t)y * p.W + x);
}

struct MeanLnP {
    ActV in, out;
    const float* lnw;
    const float* lnb;
    long long npix;      // output pixels (n_out * H * W)
    int HW, C, n_avg;
    float eps;
};

// block = 8 warps = 8 output pixels.  Output image o, pixel x = LayerNorm(mean over k < n_avg of input image o * n_avg + k, pixel x)
// (n_avg = 1: a plain channels-last LayerNorm)
__global__ void __launch_bounds__(256)
k_mean_layernorm(MeanLnP p) {
    const int lane = threadIdx.x & 31;
    const long long g = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (g >= p.npix) return;
    const long long o = g / p.HW;
    const int pix = (int)(g - o * p.HW);
    const int chunks = p.C / 64;
    float acc[8];
#pragma unroll
    for (int q = 0; q < 4; ++q) { acc[2 * q] = 0.f; acc[2 * q + 1] = 0.f; }
    for (int k = 0; k < p.n_avg; ++k) {
        const size_t ip = (size_t)(o * p.n_avg + k) * p.HW + pix;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (q < chunks) {
                const int c = q * 64 + 2 * lane;
                acc[2 * q] += act_load1(p.in, ip, c);
                acc[2 * q + 1] += act_load1(p.in, ip, c + 1);
            }
        }
    }
    if (p.n_avg > 1) {
        const float n = (float)p.n_avg;
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] /= n;
    }
    warp_layernorm_store(acc, p.C, lane, p.lnw, p.lnb, p.eps, p.out, (size_t)g);
}

// 3x3 / stride-2 / pad-1 max pooling (torchvision ResNet stem), channels-last, thread = (pixel, 4 channels)
__global__ void __launch_bounds__(256)
k_maxpool3s2(ActV in, ActV out, int N, int H, int W, int C, int Ho, int Wo, int d2s) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int cq = C / 4;
    if (t >= (long long)N * Ho * Wo * cq) return;
    const int c = (int)(t % cq) * 4;
    long long pix = t / cq;
    const int ox = (int)(pix % Wo); pix /= Wo;
    const int oy = (int)(pix % Ho); const int n = (int)(pix / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int dy = 0; dy < 3; ++dy) {
        const int y = 2 * oy - 1 + dy;
        if (y < 0 || y >= H) continue;
        for (int dx = 0; dx < 3; ++dx) {
            const int x = 2 * ox - 1 + dx;
            if (x < 0 || x >= W) continue;
            // d2s: the (H, W, C) input is stored depth-to-space folded as (H/2, W/2, 4C), channel block = (y & 1) * 2 + (x & 1)
            // (the phase-major output of the space-to-depth ResNet stem convolution)
            const float4 v = d2s ? act_load4(in, ((size_t)n * (H >> 1) + (y >> 1)) * (W >> 1) + (x >> 1), (((y & 1) << 1) | (x & 1)) * C + c)
                                 : act_load4(in, ((size_t)n * H + y) * W + x, c);
            m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
        }
    }
    act_store4(out, ((size_t)n * Ho + oy) * Wo + ox, c, m);
}

static inline ActV view_of(const heal_act_t* a) {
    ActV v;
    v.p = a->data; v.fmt = a->fmt; v.cs = a->cstride; v.co = a->coffset; v.plane = a->plane_stride;
    return v;
}

// act_load4 / act_store4 move 4 channels at once: every 4-channel group starts 16 B-aligned in fp32 and 8 B-aligned in each bf16
// plane, so the base pointer as well as the channel stride, offset and (split) plane stride.
static inline bool aligned4(const heal_act_t* a) {
    const uintptr_t need = a->fmt == 0 ? 15 : 7;
    return ((uintptr_t)a->data & need) == 0 && (a->cstride & 3) == 0 && (a->coffset & 3) == 0 &&
           (a->fmt != 2 || (a->plane_stride & 3) == 0);
}

}  // namespace

extern "C" int heal_dwconv_layernorm(const heal_act_t* in, int N, int H, int W, int C, const float* dw_weight, const float* dw_bias,
                                     int ksize, const float* ln_weight, const float* ln_bias, float eps, const heal_act_t* out,
                                     void* stream_) {
    if (!in || !in->data || !out || !out->data || !dw_weight || !ln_weight || !ln_bias) return HEAL_ERR_ARG;
    if ((C % 64) || C > 256 || ksize < 1 || !(ksize & 1) || ksize > 11) return HEAL_ERR_UNSUPPORTED;
    if ((uintptr_t)dw_weight & 7) return HEAL_ERR_UNSUPPORTED;     // read as float2
    DwLnP p;
    p.in = view_of(in); p.out = view_of(out); p.w = dw_weight; p.b = dw_bias; p.lnw = ln_weight; p.lnb = ln_bias;
    p.N = N; p.H = H; p.W = W; p.C = C; p.k = ksize; p.eps = eps;
    dim3 grid((W + 7) / 8, (H + 3) / 4, N);
    k_dwconv_ln<<<grid, 1024, 0, (cudaStream_t)stream_>>>(p);
    return heal_check_launch();
}

extern "C" int heal_maxpool3x3s2(const heal_act_t* in, int N, int H, int W, int C, int depth_to_space_in, const heal_act_t* out, void* stream_) {
    if (!in || !in->data || !out || !out->data) return HEAL_ERR_ARG;
    if (depth_to_space_in && ((H | W) & 1)) return HEAL_ERR_UNSUPPORTED;
    if ((C & 3) || !aligned4(in) || !aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const long long total = (long long)N * Ho * Wo * (C / 4);
    k_maxpool3s2<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(view_of(in), view_of(out), N, H, W, C, Ho, Wo, depth_to_space_in);
    return heal_check_launch();
}

extern "C" int heal_mean_layernorm(const heal_act_t* in, int n_out, int n_avg, int H, int W, int C, const float* ln_weight,
                                   const float* ln_bias, float eps, const heal_act_t* out, void* stream_) {
    if (!in || !out || !ln_weight || !ln_bias || n_out < 0 || n_avg < 1 || H < 1 || W < 1) return HEAL_ERR_ARG;
    if ((C % 64) || C < 64 || C > 256) return HEAL_ERR_UNSUPPORTED;
    if (n_out == 0) return HEAL_OK;                 // an empty map may have no storage (a null data pointer)
    if (!in->data || !out->data) return HEAL_ERR_ARG;
    MeanLnP p;
    p.in = view_of(in); p.out = view_of(out); p.lnw = ln_weight; p.lnb = ln_bias;
    p.npix = (long long)n_out * H * W; p.HW = H * W; p.C = C; p.n_avg = n_avg; p.eps = eps;
    k_mean_layernorm<<<(unsigned)((p.npix + 7) / 8), 256, 0, (cudaStream_t)stream_>>>(p);
    return heal_check_launch();
}
