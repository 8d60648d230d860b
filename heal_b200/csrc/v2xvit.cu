// V2X-ViT fusion (fusion_in_one.py:320-372, sub_modules/v2xvit_basic.py): the non-Linear steps of one encoder layer.  Every
// Linear runs on the conv engine as a 1x1 convolution; these kernels read its NHWC outputs in place.
//   heal_window_attention : softmax(q k^T + bias) v of one BaseWindowAttention branch (mswin.py:20-92) on the tensor cores
//   heal_cav_attention    : the per-pixel HGTCavAttention core (hmsa.py) with agent types 0, i.e. plain multi-head attention
//                           over the agents of a scene (relation_att / relation_msg and the scale folded into q / v)
//   heal_split_attn       : SplitAttn (split_attn.py) + the PreNorm residual: pool, gate MLP and weighted combine
//   heal_sttf_resample    : the STTF warp (v2xvit_basic.py:12-33), bilinear with align_corners=True and an fp32 2x3 matrix
// No kernel allocates, syncs or uses float atomics, so a captured graph replays bit-identically.
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

static inline ActV to_view(const heal_act_t* a) {
    ActV v;
    v.p = a->data; v.fmt = a->fmt; v.cs = a->cstride; v.co = a->coffset; v.plane = a->plane_stride;
    return v;
}

static inline bool aligned_to(const heal_act_t* a, int n) {
    return (a->cstride % n) == 0 && (a->coffset % n) == 0 && (a->fmt == 0 || (a->plane_stride % n) == 0);
}

static inline bool fmt_ok(const heal_act_t* a) { return a->fmt >= 0 && a->fmt <= 2; }

// the base pointer allows vector accesses of `elems` consecutive elements (channel offsets and strides are checked by aligned_to)
static inline bool data_aligned(const heal_act_t* a, int elems) {
    return ((uintptr_t)a->data % ((a->fmt == 0 ? 4u : 2u) * (unsigned)elems)) == 0;
}

// ---- window attention ------------------------------------------------------------------------------------------------
// CTA = (window, head, image); warp = 16 query tokens.  Token t = (w1, w2) of window (x, y) is pixel (x*w + w1, y*w + w2).
// K (token-major) and V (transposed, channel-major) of the window are staged in shared memory as bf16 hi (and lo) planes; Q
// fragments are read straight from the map.  S = Q K^T and O = P V are mma.sync m16n8k16 bf16 products with fp32
// accumulation; SPLIT adds the hi*lo and lo*hi cross products (the lo*lo term is below fp32 resolution), which makes both
// products fp32-equivalent.  The softmax is online over chunks of KC keys.

__device__ __forceinline__ uint32_t bf2_bits(__nv_bfloat162 h) { return *reinterpret_cast<uint32_t*>(&h); }

// channels (c, c+1) of pixel `pix` as packed bf16 pairs: hi = bf16(v), lo = bf16(v - hi) (0 unless SPLIT)
template <bool SPLIT>
__device__ __forceinline__ void load_pair(const ActV& a, size_t pix, int c, uint32_t& hi, uint32_t& lo) {
    const size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    lo = 0u;
    if (a.fmt == 0) {
        const float2 v = __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(a.p) + idx));
        const __nv_bfloat162 h = __floats2bfloat162_rn(v.x, v.y);
        hi = bf2_bits(h);
        if (SPLIT) {
            const float2 hf = __bfloat1622float2(h);
            lo = bf2_bits(__floats2bfloat162_rn(v.x - hf.x, v.y - hf.y));
        }
    } else {
        const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(a.p) + idx;
        hi = __ldg(reinterpret_cast<const uint32_t*>(b));
        if (SPLIT && a.fmt == 2) lo = __ldg(reinterpret_cast<const uint32_t*>(b + a.plane));
    }
}

__device__ __forceinline__ void store_pair(const ActV& a, size_t pix, int c, float x, float y) {
    const size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (a.fmt == 0) { *reinterpret_cast<float2*>(reinterpret_cast<float*>(a.p) + idx) = make_float2(x, y); return; }
    __nv_bfloat16* b = reinterpret_cast<__nv_bfloat16*>(a.p) + idx;
    const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    *reinterpret_cast<__nv_bfloat162*>(b) = h;
    if (a.fmt == 2) {
        const float2 hf = __bfloat1622float2(h);
        *reinterpret_cast<__nv_bfloat162*>(b + a.plane) = __floats2bfloat162_rn(x - hf.x, y - hf.y);
    }
}

__device__ __forceinline__ void mma_bf16(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

struct WinP {
    ActV qkv, out;          // qkv: q | k | v of the branch from the view's coffset (heads*dh channels each); out: merged heads
    const float* bias;      // (n, n) fp32, query-major: bias[i*n + j]
    int H, W, inner;        // inner = heads * dim_head
};

template <int WS, int DH>
struct WinCfg {
    static constexpr int N = WS * WS;           // tokens per window; one warp per 16 query tokens
    static constexpr int KC = N < 32 ? N : 32;  // keys per online-softmax step
    static constexpr int KP = DH + 8;           // K row pitch (bf16): conflict-free fragment loads
    static constexpr int VP = N + 8;            // V^T row pitch (bf16)
    static constexpr int PLANE = N * KP + DH * VP;
};

template <int WS, int DH, bool SPLIT>
__global__ void __launch_bounds__(WS * WS * 2, 1) k_window_attention(WinP p) {
    using Cfg = WinCfg<WS, DH>;
    constexpr int N = Cfg::N, KC = Cfg::KC, KP = Cfg::KP, VP = Cfg::VP;
    extern __shared__ __align__(16) __nv_bfloat16 wsm[];
    __nv_bfloat16* Ks[2] = {wsm, wsm + Cfg::PLANE};
    __nv_bfloat16* Vt[2] = {wsm + N * KP, wsm + Cfg::PLANE + N * KP};

    const int nwy = p.W / WS;
    const int wx = blockIdx.x / nwy, wy = blockIdx.x - wx * nwy;
    const int h = blockIdx.y, img = blockIdx.z;
    const size_t pix0 = ((size_t)img * p.H + (size_t)wx * WS) * p.W + (size_t)wy * WS;
    auto token_pix = [&](int t) { return pix0 + (size_t)(t / WS) * p.W + (t % WS); };

    for (int e = threadIdx.x; e < N * (DH / 2); e += blockDim.x) {
        const int t = e / (DH / 2), d = 2 * (e - t * (DH / 2));
        const size_t pix = token_pix(t);
        uint32_t kh, kl, vh, vl;
        load_pair<SPLIT>(p.qkv, pix, p.inner + h * DH + d, kh, kl);
        load_pair<SPLIT>(p.qkv, pix, 2 * p.inner + h * DH + d, vh, vl);
        *reinterpret_cast<uint32_t*>(Ks[0] + t * KP + d) = kh;
        const __nv_bfloat162 v2h = *reinterpret_cast<__nv_bfloat162*>(&vh);
        Vt[0][d * VP + t] = v2h.x; Vt[0][(d + 1) * VP + t] = v2h.y;
        if (SPLIT) {
            *reinterpret_cast<uint32_t*>(Ks[1] + t * KP + d) = kl;
            const __nv_bfloat162 v2l = *reinterpret_cast<__nv_bfloat162*>(&vl);
            Vt[1][d * VP + t] = v2l.x; Vt[1][(d + 1) * VP + t] = v2l.y;
        }
    }
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t4 = lane & 3;
    const int r0 = warp * 16 + g, r1 = r0 + 8;
    const size_t pq0 = token_pix(r0), pq1 = token_pix(r1);

    uint32_t qa[DH / 16][4], ql[DH / 16][4];
#pragma unroll
    for (int kk = 0; kk < DH / 16; ++kk) {
        const int c = h * DH + kk * 16 + 2 * t4;
        load_pair<SPLIT>(p.qkv, pq0, c, qa[kk][0], ql[kk][0]);
        load_pair<SPLIT>(p.qkv, pq1, c, qa[kk][1], ql[kk][1]);
        load_pair<SPLIT>(p.qkv, pq0, c + 8, qa[kk][2], ql[kk][2]);
        load_pair<SPLIT>(p.qkv, pq1, c + 8, qa[kk][3], ql[kk][3]);
    }

    float o[DH / 8][4];
#pragma unroll
    for (int dt = 0; dt < DH / 8; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    const float* b0p = p.bias + (size_t)r0 * N + 2 * t4;
    const float* b1p = p.bias + (size_t)r1 * N + 2 * t4;

    for (int j0 = 0; j0 < N; j0 += KC) {
        float s[KC / 8][4];
#pragma unroll
        for (int nt = 0; nt < KC / 8; ++nt) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
            const int krow = (j0 + nt * 8 + g) * KP + 2 * t4;
#pragma unroll
            for (int kk = 0; kk < DH / 16; ++kk) {
                const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(Ks[0] + krow + kk * 16);
                const uint32_t bh1 = *reinterpret_cast<const uint32_t*>(Ks[0] + krow + kk * 16 + 8);
                if (SPLIT) {
                    const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(Ks[1] + krow + kk * 16);
                    const uint32_t bl1 = *reinterpret_cast<const uint32_t*>(Ks[1] + krow + kk * 16 + 8);
                    mma_bf16(s[nt], ql[kk], bh0, bh1);
                    mma_bf16(s[nt], qa[kk], bl0, bl1);
                }
                mma_bf16(s[nt], qa[kk], bh0, bh1);
            }
            const float2 c0 = __ldg(reinterpret_cast<const float2*>(b0p + j0 + nt * 8));
            const float2 c1 = __ldg(reinterpret_cast<const float2*>(b1p + j0 + nt * 8));
            s[nt][0] += c0.x; s[nt][1] += c0.y; s[nt][2] += c1.x; s[nt][3] += c1.y;
        }
        float mc0 = m0, mc1 = m1;
#pragma unroll
        for (int nt = 0; nt < KC / 8; ++nt) {
            mc0 = fmaxf(mc0, fmaxf(s[nt][0], s[nt][1]));
            mc1 = fmaxf(mc1, fmaxf(s[nt][2], s[nt][3]));
        }
        mc0 = fmaxf(mc0, __shfl_xor_sync(0xffffffffu, mc0, 1)); mc0 = fmaxf(mc0, __shfl_xor_sync(0xffffffffu, mc0, 2));
        mc1 = fmaxf(mc1, __shfl_xor_sync(0xffffffffu, mc1, 1)); mc1 = fmaxf(mc1, __shfl_xor_sync(0xffffffffu, mc1, 2));
        const float corr0 = expf(m0 - mc0), corr1 = expf(m1 - mc1);     // 0 on the first chunk (m = -inf, o and l are 0)
        m0 = mc0; m1 = mc1;
        l0 *= corr0; l1 *= corr1;
#pragma unroll
        for (int dt = 0; dt < DH / 8; ++dt) { o[dt][0] *= corr0; o[dt][1] *= corr0; o[dt][2] *= corr1; o[dt][3] *= corr1; }
#pragma unroll
        for (int nt = 0; nt < KC / 8; ++nt) {
            s[nt][0] = expf(s[nt][0] - m0); s[nt][1] = expf(s[nt][1] - m0);
            s[nt][2] = expf(s[nt][2] - m1); s[nt][3] = expf(s[nt][3] - m1);
            l0 += s[nt][0] + s[nt][1]; l1 += s[nt][2] + s[nt][3];
        }
#pragma unroll
        for (int kb = 0; kb < KC / 16; ++kb) {
            // the S accumulator of key tiles 2kb, 2kb+1 is the A fragment of P for keys j0 + 16kb .. +15
            uint32_t pa[4], pl[4];
            const float* e0 = s[2 * kb];
            const float* e1 = s[2 * kb + 1];
            const float pv[8] = {e0[0], e0[1], e0[2], e0[3], e1[0], e1[1], e1[2], e1[3]};
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const __nv_bfloat162 hh = __floats2bfloat162_rn(pv[2 * r], pv[2 * r + 1]);
                pa[r] = bf2_bits(hh);
                if (SPLIT) {
                    const float2 hf = __bfloat1622float2(hh);
                    pl[r] = bf2_bits(__floats2bfloat162_rn(pv[2 * r] - hf.x, pv[2 * r + 1] - hf.y));
                }
            }
            const int vcol = j0 + kb * 16 + 2 * t4;
#pragma unroll
            for (int dt = 0; dt < DH / 8; ++dt) {
                const int vrow = (dt * 8 + g) * VP + vcol;
                const uint32_t vh0 = *reinterpret_cast<const uint32_t*>(Vt[0] + vrow);
                const uint32_t vh1 = *reinterpret_cast<const uint32_t*>(Vt[0] + vrow + 8);
                if (SPLIT) {
                    const uint32_t vl0 = *reinterpret_cast<const uint32_t*>(Vt[1] + vrow);
                    const uint32_t vl1 = *reinterpret_cast<const uint32_t*>(Vt[1] + vrow + 8);
                    mma_bf16(o[dt], pl, vh0, vh1);
                    mma_bf16(o[dt], pa, vl0, vl1);
                }
                mma_bf16(o[dt], pa, vh0, vh1);
            }
        }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
    for (int dt = 0; dt < DH / 8; ++dt) {
        const int c = h * DH + dt * 8 + 2 * t4;
        store_pair(p.out, pq0, c, o[dt][0] * i0, o[dt][1] * i0);
        store_pair(p.out, pq1, c, o[dt][2] * i1, o[dt][3] * i1);
    }
}

template <int WS, int DH, bool SPLIT>
int launch_window(const WinP& p, int windows, int heads, int n_img, cudaStream_t st) {
    static size_t smem_set[HEAL_MAX_DEVICES] = {};
    const size_t smem = (SPLIT ? 2 : 1) * (size_t)WinCfg<WS, DH>::PLANE * sizeof(__nv_bfloat16);
    if (!heal_ensure_dyn_smem(k_window_attention<WS, DH, SPLIT>, smem, smem_set)) return HEAL_ERR_LAUNCH;
    k_window_attention<WS, DH, SPLIT><<<dim3((unsigned)windows, (unsigned)heads, (unsigned)n_img), WS * WS * 2, smem, st>>>(p);
    return heal_check_launch(1);
}

template <int WS, bool SPLIT>
int launch_window_dh(const WinP& p, int dh, int windows, int heads, int n_img, cudaStream_t st) {
    if (dh == 16) return launch_window<WS, 16, SPLIT>(p, windows, heads, n_img, st);
    if (dh == 32) return launch_window<WS, 32, SPLIT>(p, windows, heads, n_img, st);
    return launch_window<WS, 64, SPLIT>(p, windows, heads, n_img, st);
}

template <bool SPLIT>
int launch_window_ws(const WinP& p, int ws, int dh, int windows, int heads, int n_img, cudaStream_t st) {
    if (ws == 4) return launch_window_dh<4, SPLIT>(p, dh, windows, heads, n_img, st);
    if (ws == 8) return launch_window_dh<8, SPLIT>(p, dh, windows, heads, n_img, st);
    return launch_window_dh<16, SPLIT>(p, dh, windows, heads, n_img, st);
}

// ---- cav attention ---------------------------------------------------------------------------------------------------
constexpr int CAV_DH = 32;
constexpr int CAV_MAX_L = 8;
constexpr int CAV_SCENES = 64;

struct CavP {
    ActV qkv, out;
    int HW, C, ego_only, b0, B;
    int2 scene[CAV_SCENES];   // (first non-ego image, real agents n) of scene b0 + z; its ego is image b0 + z
};

// thread = (pixel, 4 channels); the 8 threads of a head sit in consecutive lanes and reduce q.k by shuffles.  k and v of the
// scene's n agents stay in registers and serve all n queries (or the ego's only).
__global__ void __launch_bounds__(256) k_cav_attention(CavP p) {
    const int chunks = p.C >> 2;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = g < (long long)p.HW * chunks;
    const int pix = valid ? (int)(g / chunks) : 0, c = valid ? (int)(g % chunks) * 4 : 0;
    const int z = blockIdx.y, b = p.b0 + z;
    const int n = p.scene[z].y, other0 = p.scene[z].x;
    auto image_of = [&](int j) { return j == 0 ? b : other0 + j - 1; };
    float4 k[CAV_MAX_L], v[CAV_MAX_L];
#pragma unroll
    for (int j = 0; j < CAV_MAX_L; ++j) {
        if (j < n) {
            const size_t px = (size_t)image_of(j) * p.HW + pix;
            k[j] = act_load4(p.qkv, px, p.C + c);
            v[j] = act_load4(p.qkv, px, 2 * p.C + c);
        }
    }
    const int nq = p.ego_only ? 1 : n;
    for (int i = 0; i < nq; ++i) {
        const size_t pxi = (size_t)image_of(i) * p.HW + pix;
        const float4 q = act_load4(p.qkv, pxi, c);
        float s[CAV_MAX_L];
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < CAV_MAX_L; ++j) {
            if (j < n) {
                float d = q.x * k[j].x + q.y * k[j].y + q.z * k[j].z + q.w * k[j].w;
                d += __shfl_xor_sync(0xffffffffu, d, 1);
                d += __shfl_xor_sync(0xffffffffu, d, 2);
                d += __shfl_xor_sync(0xffffffffu, d, 4);
                s[j] = d;
                m = fmaxf(m, d);
            }
        }
        float sum = 0.f;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < CAV_MAX_L; ++j) {
            if (j < n) {
                const float e = expf(s[j] - m);
                sum += e;
                acc.x = fmaf(e, v[j].x, acc.x); acc.y = fmaf(e, v[j].y, acc.y);
                acc.z = fmaf(e, v[j].z, acc.z); acc.w = fmaf(e, v[j].w, acc.w);
            }
        }
        const float inv = 1.f / sum;
        const size_t pxo = p.ego_only ? (size_t)b * p.HW + pix : pxi;
        if (valid) act_store4(p.out, pxo, c, make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv));
    }
}

// ---- SplitAttn -------------------------------------------------------------------------------------------------------
constexpr int SPLIT_SLABS = 32;     // pixel slabs of the pooled sum; their partials are added in a fixed order
constexpr int SPLIT_C = 256;        // SplitAttn(256) is hard-coded in PyramidWindowAttention

struct PoolP { ActV o; int HW, C; float* partial; };

// partial[img][slab][c] = sum over the slab's pixels of (o_0 + o_1 + o_2)[c]; o holds the three branch outputs side by side
__global__ void __launch_bounds__(256) k_split_pool(PoolP p) {
    __shared__ float4 red[256];
    const int chunks = p.C >> 2, lanes = 256 / chunks;
    const int c4 = threadIdx.x % chunks, pl = threadIdx.x / chunks;
    const int slab = blockIdx.x, img = blockIdx.y;
    const long long a = (long long)p.HW * slab / SPLIT_SLABS, e = (long long)p.HW * (slab + 1) / SPLIT_SLABS;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long px = a + pl; px < e; px += lanes) {
        const size_t pix = (size_t)img * p.HW + px;
        const float4 s = act_load4(p.o, pix, 4 * c4), m = act_load4(p.o, pix, p.C + 4 * c4), b = act_load4(p.o, pix, 2 * p.C + 4 * c4);
        acc.x += s.x + m.x + b.x; acc.y += s.y + m.y + b.y; acc.z += s.z + m.z + b.z; acc.w += s.w + m.w + b.w;
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    if (pl == 0) {
        for (int k = 1; k < lanes; ++k) {
            const float4 r = red[k * chunks + c4];
            acc.x += r.x; acc.y += r.y; acc.z += r.z; acc.w += r.w;
        }
        stg_f4(p.partial + ((size_t)img * SPLIT_SLABS + slab) * p.C + 4 * c4, acc);
    }
}

__device__ __forceinline__ float block_sum256(float v, float* sh) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += sh[w];
    return t;
}

// one CTA per image, thread = channel: mean -> fc1 -> LayerNorm -> ReLU -> fc2 -> softmax over the 3 branches per channel
__global__ void __launch_bounds__(SPLIT_C) k_split_gate(const float* __restrict__ partial, float inv_hw,
                                                        const float* __restrict__ fc1_t, const float* __restrict__ ln_w,
                                                        const float* __restrict__ ln_b, float eps,
                                                        const float* __restrict__ fc2_t, float* __restrict__ gate) {
    constexpr int C = SPLIT_C;
    __shared__ float xs[C], red[8];
    const int c = threadIdx.x, img = blockIdx.x;
    float s = 0.f;
    for (int k = 0; k < SPLIT_SLABS; ++k) s += partial[((size_t)img * SPLIT_SLABS + k) * C + c];
    xs[c] = s * inv_hw;
    __syncthreads();
    float y = 0.f;
    for (int k = 0; k < C; ++k) y = fmaf(__ldg(fc1_t + (size_t)k * C + c), xs[k], y);
    const float mu = block_sum256(y, red) * (1.f / C);
    const float d = y - mu;
    const float var = block_sum256(d * d, red) * (1.f / C);
    const float r = fmaxf(d * rsqrtf(var + eps) * ln_w[c] + ln_b[c], 0.f);
    __syncthreads();
    xs[c] = r;
    __syncthreads();
    float z0 = 0.f, z1 = 0.f, z2 = 0.f;
    for (int k = 0; k < C; ++k) {
        const float xk = xs[k];
        const float* w = fc2_t + (size_t)k * 3 * C + c;
        z0 = fmaf(__ldg(w), xk, z0); z1 = fmaf(__ldg(w + C), xk, z1); z2 = fmaf(__ldg(w + 2 * C), xk, z2);
    }
    const float m = fmaxf(z0, fmaxf(z1, z2));
    const float e0 = expf(z0 - m), e1 = expf(z1 - m), e2 = expf(z2 - m);
    const float inv = 1.f / (e0 + e1 + e2);
    gate[(size_t)img * 3 * C + c] = e0 * inv;
    gate[(size_t)img * 3 * C + C + c] = e1 * inv;
    gate[(size_t)img * 3 * C + 2 * C + c] = e2 * inv;
}

struct CombP { ActV o, x, out; const float* gate; int HW, C; };

// out = o_0 * g_0 + o_1 * g_1 + o_2 * g_2 + x  (split_attn.py:66-68, then the PreNorm residual of v2xvit_basic.py:143)
__global__ void __launch_bounds__(256) k_split_combine(CombP p) {
    const int chunks = p.C >> 2;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)p.HW * chunks) return;
    const int img = blockIdx.y;
    const size_t pix = (size_t)img * p.HW + g / chunks;
    const int c = (int)(g % chunks) * 4;
    const float* gt = p.gate + (size_t)img * 3 * p.C + c;
    const float4 g0 = ldg_f4(gt), g1 = ldg_f4(gt + p.C), g2 = ldg_f4(gt + 2 * p.C);
    const float4 s = act_load4(p.o, pix, c), m = act_load4(p.o, pix, p.C + c), b = act_load4(p.o, pix, 2 * p.C + c);
    const float4 x = act_load4(p.x, pix, c);
    float4 r;
    r.x = s.x * g0.x + m.x * g1.x + b.x * g2.x + x.x;
    r.y = s.y * g0.y + m.y * g1.y + b.y * g2.y + x.y;
    r.z = s.z * g0.z + m.z * g1.z + b.z * g2.z + x.z;
    r.w = s.w * g0.w + m.w * g1.w + b.w * g2.w + x.w;
    act_store4(p.out, pix, c, r);
}

// ---- STTF resample ---------------------------------------------------------------------------------------------------
struct SttfP { ActV src, out; const float* theta; int H, W, C; };

// torch.linspace(-1, 1, n) in fp32 (the base grid of F.affine_grid with align_corners=True); F.affine_grid uses 0 for an axis of
// one pixel, not linspace's -1
__device__ __forceinline__ float linspace_pm1(int i, int n) {
    if (n == 1) return 0.f;
    const float step = 2.f / (float)(n - 1);
    return i < n / 2 ? -1.f + step * (float)i : 1.f - step * (float)(n - 1 - i);
}

// out image k = F.grid_sample(src image k, F.affine_grid(theta[k], align_corners=True), bilinear, zeros, align_corners=True)
__global__ void __launch_bounds__(256) k_sttf_resample(SttfP p) {
    const int chunks = p.C >> 2, HW = p.H * p.W;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)HW * chunks) return;
    const int pix = (int)(g / chunks), c = (int)(g % chunks) * 4;
    const int k = blockIdx.y, oh = pix / p.W, ow = pix - oh * p.W;
    const float* th = p.theta + 6 * (size_t)k;
    const float xb = linspace_pm1(ow, p.W), yb = linspace_pm1(oh, p.H);
    // the rounding order of PyTorch's fp32 affine_grid (base grid @ theta^T) and grid_sample unnormalisation on the CPU, so that
    // the near-identity STTF matrix moves the samples as the reference does
    const float gx = __fadd_rn(__fmaf_rn(yb, th[1], __fmul_rn(xb, th[0])), th[2]);
    const float gy = __fadd_rn(__fmaf_rn(yb, th[4], __fmul_rn(xb, th[3])), th[5]);
    const float ix = __fmul_rn(__fadd_rn(gx, 1.f), (float)(p.W - 1) * 0.5f);
    const float iy = __fmul_rn(__fadd_rn(gy, 1.f), (float)(p.H - 1) * 0.5f);
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (fx >= -2.f && fx <= (float)(p.W + 1)) ? (int)fx : -2;
    const int y0 = (fy >= -2.f && fy <= (float)(p.H + 1)) ? (int)fy : -2;
    const float wx1 = ix - fx, wx0 = (fx + 1.f) - ix, wy1 = iy - fy, wy0 = (fy + 1.f) - iy;
    const size_t base = (size_t)k * HW;
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    const int xs[4] = {x0, x0 + 1, x0, x0 + 1}, ys[4] = {y0, y0, y0 + 1, y0 + 1};
    const float ws[4] = {wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        if (xs[t] >= 0 && xs[t] < p.W && ys[t] >= 0 && ys[t] < p.H) {
            const float4 v = act_load4(p.src, base + (size_t)ys[t] * p.W + xs[t], c);
            r.x = __fadd_rn(r.x, __fmul_rn(v.x, ws[t])); r.y = __fadd_rn(r.y, __fmul_rn(v.y, ws[t]));
            r.z = __fadd_rn(r.z, __fmul_rn(v.z, ws[t])); r.w = __fadd_rn(r.w, __fmul_rn(v.w, ws[t]));
        }
    }
    act_store4(p.out, base + pix, c, r);
}

static inline unsigned grid_x(long long HW, int C) { return (unsigned)((HW * (C >> 2) + 255) / 256); }

}  // namespace

extern "C" int heal_window_attention(const heal_act_t* qkv, int n_img, int H, int W, int heads, int dim_head, int window_size,
                                     const float* bias, const heal_act_t* out, void* stream_) {
    if (!qkv || !qkv->data || !bias || !out || !out->data || n_img < 0 || H < 1 || W < 1 || heads < 1) return HEAL_ERR_ARG;
    if (!fmt_ok(qkv) || !fmt_ok(out)) return HEAL_ERR_ARG;
    if (window_size != 4 && window_size != 8 && window_size != 16) return HEAL_ERR_UNSUPPORTED;
    if (dim_head != 16 && dim_head != 32 && dim_head != 64) return HEAL_ERR_UNSUPPORTED;
    if ((H % window_size) || (W % window_size)) return HEAL_ERR_ARG;
    if (!aligned_to(qkv, 2) || !aligned_to(out, 2) || !data_aligned(qkv, 2) || !data_aligned(out, 2)) return HEAL_ERR_UNSUPPORTED;
    if ((uintptr_t)bias & 7) return HEAL_ERR_UNSUPPORTED;          // the bias is read as float2
    const long long windows = (long long)(H / window_size) * (W / window_size);
    if (windows > 0x7fffffffLL || heads > 65535 || n_img > 65535) return HEAL_ERR_UNSUPPORTED;
    if (n_img == 0) return HEAL_OK;
    WinP p;
    p.qkv = to_view(qkv); p.out = to_view(out); p.bias = bias;
    p.H = H; p.W = W; p.inner = heads * dim_head;
    cudaStream_t st = (cudaStream_t)stream_;
    // bf16 storage runs the single bf16 product; fp32 and split-bf16 storage run the split products (fp32-equivalent)
    if (qkv->fmt == 1) return launch_window_ws<false>(p, window_size, dim_head, (int)windows, heads, n_img, st);
    return launch_window_ws<true>(p, window_size, dim_head, (int)windows, heads, n_img, st);
}

extern "C" int heal_cav_attention(const heal_act_t* qkv, const int* n_agents_host, int B, int H, int W, int C, int ego_only,
                                  const heal_act_t* out, void* stream_) {
    if (!qkv || !qkv->data || !n_agents_host || !out || !out->data || B < 0 || H < 1 || W < 1 || C < 1) return HEAL_ERR_ARG;
    if (!fmt_ok(qkv) || !fmt_ok(out)) return HEAL_ERR_ARG;
    if ((C % CAV_DH) || !aligned_to(qkv, 4) || !aligned_to(out, 4) || !data_aligned(qkv, 4) || !data_aligned(out, 4))
        return HEAL_ERR_UNSUPPORTED;
    for (int b = 0; b < B; ++b)          // every count before the first launch, so a bad one leaves the output untouched
        if (n_agents_host[b] < 1 || n_agents_host[b] > CAV_MAX_L) return HEAL_ERR_ARG;
    CavP p;
    p.qkv = to_view(qkv); p.out = to_view(out); p.HW = H * W; p.C = C; p.ego_only = ego_only ? 1 : 0; p.B = B;
    int other = B, launches = 0;
    for (int b0 = 0; b0 < B; b0 += CAV_SCENES) {
        const int nb = B - b0 < CAV_SCENES ? B - b0 : CAV_SCENES;
        p.b0 = b0;
        for (int z = 0; z < nb; ++z) {
            const int n = n_agents_host[b0 + z];
            p.scene[z] = make_int2(other, n);
            other += n - 1;
        }
        k_cav_attention<<<dim3(grid_x(p.HW, C), (unsigned)nb), 256, 0, (cudaStream_t)stream_>>>(p);
        ++launches;
    }
    return heal_check_launch(launches);
}

extern "C" size_t heal_split_attn_workspace(int n_img, int C) {
    return (size_t)(n_img < 0 ? 0 : n_img) * (size_t)(SPLIT_SLABS + 3) * (size_t)(C < 0 ? 0 : C) * sizeof(float);
}

extern "C" int heal_split_attn(const heal_act_t* o, const heal_act_t* x, int n_img, int H, int W, int C, const float* fc1_t,
                               const float* ln_w, const float* ln_b, float eps, const float* fc2_t, void* workspace,
                               size_t ws_bytes, const heal_act_t* out, void* stream_) {
    if (!o || !o->data || !x || !x->data || !out || !out->data || !fc1_t || !ln_w || !ln_b || !fc2_t || !workspace) return HEAL_ERR_ARG;
    if (n_img < 0 || H < 1 || W < 1 || !fmt_ok(o) || !fmt_ok(x) || !fmt_ok(out)) return HEAL_ERR_ARG;
    if (C != SPLIT_C || !aligned_to(o, 4) || !aligned_to(x, 4) || !aligned_to(out, 4)) return HEAL_ERR_UNSUPPORTED;
    if (n_img > 65535) return HEAL_ERR_UNSUPPORTED;      // gridDim.y of the pool and combine launches
    if (!data_aligned(o, 4) || !data_aligned(x, 4) || !data_aligned(out, 4) || ((uintptr_t)workspace & 15)) return HEAL_ERR_UNSUPPORTED;
    if (ws_bytes < heal_split_attn_workspace(n_img, C)) return HEAL_ERR_WORKSPACE;
    if (n_img == 0) return HEAL_OK;
    cudaStream_t st = (cudaStream_t)stream_;
    float* partial = reinterpret_cast<float*>(workspace);
    float* gate = partial + (size_t)n_img * SPLIT_SLABS * C;
    const int HW = H * W;
    PoolP pp; pp.o = to_view(o); pp.HW = HW; pp.C = C; pp.partial = partial;
    k_split_pool<<<dim3(SPLIT_SLABS, (unsigned)n_img), 256, 0, st>>>(pp);
    k_split_gate<<<(unsigned)n_img, SPLIT_C, 0, st>>>(partial, 1.f / (float)HW, fc1_t, ln_w, ln_b, eps, fc2_t, gate);
    CombP cp; cp.o = to_view(o); cp.x = to_view(x); cp.out = to_view(out); cp.gate = gate; cp.HW = HW; cp.C = C;
    k_split_combine<<<dim3(grid_x(HW, C), (unsigned)n_img), 256, 0, st>>>(cp);
    return heal_check_launch(3);
}

extern "C" int heal_sttf_resample(const heal_act_t* src, const float* theta, int n_img, int H, int W, int C,
                                  const heal_act_t* out, void* stream_) {
    if (!src || !src->data || !theta || !out || !out->data || n_img < 0 || H < 1 || W < 1 || C < 1) return HEAL_ERR_ARG;
    if (!fmt_ok(src) || !fmt_ok(out)) return HEAL_ERR_ARG;
    if ((C & 3) || !aligned_to(src, 4) || !aligned_to(out, 4) || n_img > 65535) return HEAL_ERR_UNSUPPORTED;
    if (!data_aligned(src, 4) || !data_aligned(out, 4)) return HEAL_ERR_UNSUPPORTED;
    if (n_img == 0) return HEAL_OK;
    SttfP p; p.src = to_view(src); p.out = to_view(out); p.theta = theta; p.H = H; p.W = W; p.C = C;
    k_sttf_resample<<<dim3(grid_x((long long)H * W, C), (unsigned)n_img), 256, 0, (cudaStream_t)stream_>>>(p);
    return heal_check_launch(1);
}
