// fp32 channels-last (NHWC) 2-D convolution on the CUDA cores: the exact-fp32 companion of the
// wgmma implicit-GEMM engine (conv2d_tc.cu). It serves (a) shapes the tensor-core engine does not
// take (grouped 3x3 with 4-16 channels per group, Cin/Cout not multiples of 16, the 20-channel heads)
// and (b) as the on-device fp32 cross-check for the tensor-core path in tests.
// Reference ops replaced: nn.Conv2d / nn.ConvTranspose2d(k == stride) + eval BatchNorm2d (folded on the
// host in fp64) + ReLU + residual add, as used by
//   opencood/models/sub_modules/resblock.py:48-64,102-122 (BasicBlock / Bottleneck),
//   opencood/models/sub_modules/base_bev_backbone.py:40-86, base_bev_backbone_resnet.py:54-85,
//   opencood/models/sub_modules/downsample_conv.py:16-27, heter_pyramid_collab.py:102-107 (heads).
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

struct ConvP {
    ActV in, res, out;                       // activation views (fp32 / bf16 / split-bf16); res.p == nullptr when unused
    const float* w; const float* bias;
    int N, H, W, Cin;
    int Ho, Wo, Cout;                        // conv output grid (Ho,Wo)
    int kh, kw, stride, pad;
    int w_cs;                                // weight row stride (>= Cout, multiple of 4)
    int relu;
    int up, up_i, up_j;                      // output pixel (oh,ow) is stored at (oh*up+up_i, ow*up+up_j) of an (Ho*up, Wo*up) map
    int groups;
    int out_vec4;                            // the output view takes act_store4 (aligned4 on the host)
};

constexpr int BM = 128, BN = 64, BK = 16;

__global__ void __launch_bounds__(256)
k_conv2d_dense(ConvP p) {
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    const int tid = threadIdx.x;
    const int tm = tid / 16, tn = tid % 16;
    const long long Mtot = (long long)p.N * p.Ho * p.Wo;
    const long long m0 = (long long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;

    // loader pixels: 2 per thread
    int lp_n[2], lp_h[2], lp_w[2]; bool lp_ok[2];
    const int kq = tid % 4;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        long long m = m0 + tid / 4 + 64 * j;
        lp_ok[j] = m < Mtot;
        long long mm = lp_ok[j] ? m : 0;
        lp_w[j] = (int)(mm % p.Wo); mm /= p.Wo;
        lp_h[j] = (int)(mm % p.Ho); lp_n[j] = (int)(mm / p.Ho);
    }
    const int bk = tid / 16, bc4 = tid % 16;

    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int r = 0; r < p.kh; ++r) {
        for (int s = 0; s < p.kw; ++s) {
            for (int c0 = 0; c0 < p.Cin; c0 += BK) {
                // ---- A tile (im2col on the fly, zero fill for padding / tails) ----
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    int ih = lp_h[j] * p.stride - p.pad + r, iw = lp_w[j] * p.stride - p.pad + s;
                    int ci = c0 + kq * 4;
                    if (lp_ok[j] && ih >= 0 && ih < p.H && iw >= 0 && iw < p.W && ci < p.Cin) {
                        v = act_load4(p.in, (size_t)((size_t)lp_n[j] * p.H + ih) * p.W + iw, ci);
                    }
                    int m = tid / 4 + 64 * j;
                    As[kq * 4 + 0][m] = v.x; As[kq * 4 + 1][m] = v.y; As[kq * 4 + 2][m] = v.z; As[kq * 4 + 3][m] = v.w;
                }
                // ---- B tile ----
                {
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    int ci = c0 + bk, co = n0 + bc4 * 4;
                    if (ci < p.Cin && co < p.w_cs)
                        v = ldg_f4(p.w + ((size_t)((r * p.kw + s) * p.Cin + ci)) * p.w_cs + co);
                    *reinterpret_cast<float4*>(&Bs[bk][bc4 * 4]) = v;
                }
                __syncthreads();
#pragma unroll
                for (int k = 0; k < BK; ++k) {
                    float4 a0 = *reinterpret_cast<const float4*>(&As[k][tm * 8]);
                    float4 a1 = *reinterpret_cast<const float4*>(&As[k][tm * 8 + 4]);
                    float4 b = *reinterpret_cast<const float4*>(&Bs[k][tn * 4]);
                    float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                    float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                    for (int i = 0; i < 8; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
                }
                __syncthreads();
            }
        }
    }
    // ---- epilogue: bias (+ residual) (+ ReLU), channels-last store ----
    const int co = n0 + tn * 4;
    if (co >= p.Cout) return;
    float bv[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.bias) {
#pragma unroll
        for (int j = 0; j < 4; ++j) if (co + j < p.Cout) bv[j] = p.bias[co + j];
    }
    const int Hs = p.Ho * p.up, Ws = p.Wo * p.up;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        long long m = m0 + tm * 8 + i;
        if (m >= Mtot) break;
        long long mm = m;
        int ow = (int)(mm % p.Wo); mm /= p.Wo;
        int oh = (int)(mm % p.Ho); int n = (int)(mm / p.Ho);
        size_t pix = ((size_t)n * Hs + (size_t)(oh * p.up + p.up_i)) * Ws + (size_t)(ow * p.up + p.up_j);
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = acc[i][j] + bv[j];
        if (p.res.p) {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (co + j < p.Cout) v[j] += act_load1(p.res, pix, co + j);
        }
        if (p.relu) {
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = heal_act_fn(v[j], p.relu);
        }
        if (co + 3 < p.Cout && p.out_vec4) {
            act_store4(p.out, pix, co, make_float4(v[0], v[1], v[2], v[3]));
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (co + j < p.Cout) act_store1(p.out, pix, co + j, v[j]);
        }
    }
}

// Grouped 3x3 convolution, CG channels per group in and out (ResNeXt bottleneck conv2, groups = 32:
// resblock.py:94 with width_per_group=4 -> CG = 4 / 8 / 16). lane = group, so a warp reads a pixel's
// whole channel vector as one contiguous segment; each thread register-tiles PX output pixels along W
// so every shared-memory weight read feeds PX FMAs. blockIdx.y selects a chunk of COC output channels
// per group so that all 9 taps of the chunk's weights stay resident in shared memory while the block
// grid-strides over pixel tiles. Global weight layout: [tap][ci][co][G].
template <int CG, int COC, int PX>
__global__ void __launch_bounds__(256)
k_conv2d_grouped(ConvP p) {
    extern __shared__ float sWg[];  // [9][CG][COC][G]
    const int G = p.groups;
    const int co0 = blockIdx.y * COC;
    for (int i = threadIdx.x; i < 9 * CG * COC * G; i += blockDim.x) {
        int g_ = i % G; int t = i / G; int coc = t % COC; t /= COC; int ci = t % CG; int tap = t / CG;
        sWg[i] = p.w[(((size_t)tap * CG + ci) * CG + co0 + coc) * G + g_];
    }
    __syncthreads();
    const int g = threadIdx.x % 32 + 32 * blockIdx.z;   // group handled by this lane
    if (g >= G) return;
    const int wrp = threadIdx.x / 32, nwarps = blockDim.x / 32;
    const int wtiles = (p.Wo + PX - 1) / PX;
    const long long ntiles = (long long)p.N * p.Ho * wtiles;
    float bv[COC];
#pragma unroll
    for (int j = 0; j < COC; ++j) bv[j] = p.bias ? p.bias[g * CG + co0 + j] : 0.f;
    for (long long tile = (long long)blockIdx.x * nwarps + wrp; tile < ntiles; tile += (long long)gridDim.x * nwarps) {
        int wt = (int)(tile % wtiles); long long t2 = tile / wtiles;
        int oh = (int)(t2 % p.Ho); int n = (int)(t2 / p.Ho);
        int ow0 = wt * PX;
        float acc[PX][COC];
#pragma unroll
        for (int i = 0; i < PX; ++i)
#pragma unroll
            for (int j = 0; j < COC; ++j) acc[i][j] = 0.f;
        for (int r = 0; r < 3; ++r) {
            int ih = oh * p.stride - p.pad + r;
            if (ih < 0 || ih >= p.H) continue;
            for (int s = 0; s < 3; ++s) {
                float x[PX][CG];
#pragma unroll
                for (int i = 0; i < PX; ++i) {
                    int iw = (ow0 + i) * p.stride - p.pad + s;
                    bool ok = (iw >= 0 && iw < p.W && ow0 + i < p.Wo);
                    const size_t ipix = (size_t)((size_t)n * p.H + ih) * p.W + (ok ? iw : 0);
#pragma unroll
                    for (int q = 0; q < CG / 4; ++q) {
                        float4 v = ok ? act_load4(p.in, ipix, g * CG + q * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                        x[i][q * 4 + 0] = v.x; x[i][q * 4 + 1] = v.y; x[i][q * 4 + 2] = v.z; x[i][q * 4 + 3] = v.w;
                    }
                }
                const float* wt_ = sWg + (size_t)(r * 3 + s) * CG * COC * G;
#pragma unroll
                for (int ci = 0; ci < CG; ++ci)
#pragma unroll
                    for (int co = 0; co < COC; ++co) {
                        float wv = wt_[(ci * COC + co) * G + g];
#pragma unroll
                        for (int i = 0; i < PX; ++i) acc[i][co] = fmaf(x[i][ci], wv, acc[i][co]);
                    }
            }
        }
#pragma unroll
        for (int i = 0; i < PX; ++i) {
            int ow = ow0 + i;
            if (ow >= p.Wo) break;
            size_t pix = ((size_t)n * p.Ho + oh) * p.Wo + ow;
#pragma unroll
            for (int q = 0; q < COC / 4; ++q) {
                float v[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float t = acc[i][q * 4 + j] + bv[q * 4 + j];
                    v[j] = heal_act_fn(t, p.relu);
                }
                act_store4(p.out, pix, g * CG + co0 + q * 4, make_float4(v[0], v[1], v[2], v[3]));
            }
        }
    }
}

template <int CG, int COC, int PX>
int launch_grouped(const ConvP& p, cudaStream_t st) {
    size_t smem = (size_t)9 * CG * COC * p.groups * sizeof(float);
    if (smem > 48 * 1024) {
        if (cudaFuncSetAttribute(k_conv2d_grouped<CG, COC, PX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
            return HEAL_ERR_LAUNCH;
    }
    int wtiles = (p.Wo + PX - 1) / PX;
    long long ntiles = (long long)p.N * p.Ho * wtiles;
    long long want = (ntiles + 7) / 8;
    int per_sm = smem > 100 * 1024 ? 1 : (smem > 48 * 1024 ? 2 : 4);
    long long cap = (long long)HEAL_NUM_SMS * per_sm;
    dim3 grid((unsigned)(want < cap ? want : cap), (unsigned)(CG / COC), (unsigned)((p.groups + 31) / 32));
    k_conv2d_grouped<CG, COC, PX><<<grid, 256, smem, st>>>(p);
    return heal_check_launch();
}

}  // namespace

static inline ActV to_view(const heal_act_t* a) {
    ActV v;
    if (!a) { v.p = nullptr; v.fmt = 0; v.cs = 0; v.co = 0; v.plane = 0; return v; }
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

extern "C" int heal_conv2d_simt(const heal_act_t* in, int N, int H, int W, int Cin,
                                const float* weight, int w_cstride, const float* bias,
                                int kh, int kw, int stride, int pad, int groups,
                                const heal_act_t* residual, const heal_act_t* out, int Ho, int Wo, int Cout,
                                int upsample, int up_i, int up_j, int relu, void* stream_) {
    if (!in || !in->data || !weight || !out || !out->data) return HEAL_ERR_ARG;
    if (N < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || Ho < 1 || Wo < 1 || stride < 1 || upsample < 1) return HEAL_ERR_ARG;
    if (in->fmt < 0 || in->fmt > 2 || out->fmt < 0 || out->fmt > 2) return HEAL_ERR_ARG;
    if (!aligned4(in) || (Cin & 3)) return HEAL_ERR_UNSUPPORTED;
    ConvP p;
    p.in = to_view(in); p.res = to_view(residual); p.out = to_view(out);
    p.w = weight; p.bias = bias;
    p.N = N; p.H = H; p.W = W; p.Cin = Cin;
    p.Ho = Ho; p.Wo = Wo; p.Cout = Cout;
    p.kh = kh; p.kw = kw; p.stride = stride; p.pad = pad; p.w_cs = w_cstride; p.relu = relu;
    p.up = upsample; p.up_i = up_i; p.up_j = up_j; p.groups = groups; p.out_vec4 = aligned4(out);
    cudaStream_t st = (cudaStream_t)stream_;
    if (groups == 1) {
        if (w_cstride & 3) return HEAL_ERR_UNSUPPORTED;
        long long Mtot = (long long)N * Ho * Wo;
        dim3 grid((unsigned)((Mtot + BM - 1) / BM), (unsigned)((Cout + BN - 1) / BN));
        k_conv2d_dense<<<grid, 256, 0, st>>>(p);
        return heal_check_launch();
    }
    // grouped: 3x3, Cin == Cout, CG = Cin/groups in {4,8,16}, no residual/upsample
    if (kh != 3 || kw != 3 || Cin != Cout || residual || upsample != 1 || (groups % 32) != 0) return HEAL_ERR_UNSUPPORTED;
    if (!aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    int cg = Cin / groups;
    if (cg * groups != Cin) return HEAL_ERR_ARG;
    if (cg == 4) return launch_grouped<4, 4, 4>(p, st);
    if (cg == 8) return launch_grouped<8, 8, 4>(p, st);
    if (cg == 16) return launch_grouped<16, 4, 4>(p, st);
    return HEAL_ERR_UNSUPPORTED;
}
