// CoBEVT window / grid attention: the softmax(q k^T + bias) v core of swap_fusion_modules.py:13-128 (Attention.forward) with the
// agent mask CoBEVT builds in fusion_in_one.py:409-429.  to_qkv and to_out are 1x1 convolutions on the conv engine; this kernel
// reads the to_qkv output map (B*L, H, W, 3C) in place and writes the merged heads (B*L, H, W, C), so no rearranged copy of the
// map ever exists.
//   window mode: window (x, y) holds pixels (x*w + w1, y*w + w2);  grid mode: pixels (w1*H/w + x, w2*W/w + y)
//   tokens of a window are ordered (l, w1, w2): agent-major, so the keys of the n_b real agents are the first n_b*w*w tokens and
//   the masked keys (padded agents, -inf in the reference) are simply not visited.  Padded agents are still queries.
// fp32 on the CUDA cores in every storage format (split-bf16 input keeps tc32 fp32-equivalent).
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int DH = 32;             // dim_head
constexpr int MAX_TOK = 128;       // tokens per window (L * w * w)
constexpr int SCENES = 64;         // scenes per launch: their real-agent counts travel in the parameter block
constexpr int KCH = 8;             // keys per online-softmax step

struct SwapP {
    ActV qkv, out;
    const float* bias;             // [head][key][query] fp32: coalesced over the queries of a CTA
    int H, W, C, L, w, grid, b0;
    int nb[SCENES];                // real agents of scene b0 + z
};

// token t = (l, w1, w2) of window (wx, wy) of scene b -> pixel index in the (B*L, H, W) map
__device__ __forceinline__ size_t token_pixel(const SwapP& p, int b, int wx, int wy, int t) {
    const int ww = p.w * p.w;
    const int l = t / ww, r = t - l * ww, w1 = r / p.w, w2 = r - w1 * p.w;
    const int row = p.grid ? w1 * (p.H / p.w) + wx : wx * p.w + w1;
    const int col = p.grid ? w2 * (p.W / p.w) + wy : wy * p.w + w2;
    return ((size_t)(b * p.L + l) * p.H + row) * p.W + col;
}

// CTA = (window, head, scene); thread = query token.  K and V rows of the valid keys are staged in shared memory; every thread
// keeps its q row and its output row in registers and runs an online softmax over the keys, KCH keys per rescale.
__global__ void __launch_bounds__(MAX_TOK) k_swap_attention(SwapP p) {
    __shared__ float4 ks[MAX_TOK][DH / 4], vs[MAX_TOK][DH / 4];
    const int nwy = p.W / p.w;
    const int wx = blockIdx.x / nwy, wy = blockIdx.x - wx * nwy;
    const int h = blockIdx.y, b = p.b0 + blockIdx.z;
    const int n = p.L * p.w * p.w;
    const int nk = p.nb[blockIdx.z] * p.w * p.w;
    for (int e = threadIdx.x; e < nk * (DH / 4); e += blockDim.x) {
        const int t = e / (DH / 4), c4 = e - t * (DH / 4);
        const size_t pix = token_pixel(p, b, wx, wy, t);
        ks[t][c4] = act_load4(p.qkv, pix, p.C + h * DH + 4 * c4);
        vs[t][c4] = act_load4(p.qkv, pix, 2 * p.C + h * DH + 4 * c4);
    }
    __syncthreads();
    const int i = threadIdx.x;
    if (i >= n) return;
    const size_t pix = token_pixel(p, b, wx, wy, i);
    float q[DH], acc[DH];
#pragma unroll
    for (int c4 = 0; c4 < DH / 4; ++c4) {
        const float4 v = act_load4(p.qkv, pix, h * DH + 4 * c4);
        q[4 * c4] = v.x; q[4 * c4 + 1] = v.y; q[4 * c4 + 2] = v.z; q[4 * c4 + 3] = v.w;
    }
#pragma unroll
    for (int d = 0; d < DH; ++d) acc[d] = 0.f;
    const float* bias = p.bias + (size_t)h * n * n + i;
    float m = -INFINITY, sum = 0.f;
    for (int j0 = 0; j0 < nk; j0 += KCH) {
        float s[KCH];
        float mc = m;
#pragma unroll
        for (int u = 0; u < KCH; ++u) {
            const int j = j0 + u;
            s[u] = -INFINITY;
            if (j < nk) {
                float dot = 0.f;
#pragma unroll
                for (int c4 = 0; c4 < DH / 4; ++c4) {
                    const float4 k = ks[j][c4];
                    dot = fmaf(q[4 * c4], k.x, dot); dot = fmaf(q[4 * c4 + 1], k.y, dot);
                    dot = fmaf(q[4 * c4 + 2], k.z, dot); dot = fmaf(q[4 * c4 + 3], k.w, dot);
                }
                s[u] = dot + __ldg(bias + (size_t)j * n);
                mc = fmaxf(mc, s[u]);
            }
        }
        const float corr = expf(m - mc);          // 0 on the first step (m = -inf, acc and sum are 0)
        sum *= corr;
#pragma unroll
        for (int d = 0; d < DH; ++d) acc[d] *= corr;
#pragma unroll
        for (int u = 0; u < KCH; ++u) {
            const int j = j0 + u;
            if (j < nk) {
                const float e = expf(s[u] - mc);
                sum += e;
#pragma unroll
                for (int c4 = 0; c4 < DH / 4; ++c4) {
                    const float4 v = vs[j][c4];
                    acc[4 * c4] = fmaf(e, v.x, acc[4 * c4]); acc[4 * c4 + 1] = fmaf(e, v.y, acc[4 * c4 + 1]);
                    acc[4 * c4 + 2] = fmaf(e, v.z, acc[4 * c4 + 2]); acc[4 * c4 + 3] = fmaf(e, v.w, acc[4 * c4 + 3]);
                }
            }
        }
        m = mc;
    }
    const float inv = 1.f / sum;
#pragma unroll
    for (int c4 = 0; c4 < DH / 4; ++c4)
        act_store4(p.out, pix, h * DH + 4 * c4,
                   make_float4(acc[4 * c4] * inv, acc[4 * c4 + 1] * inv, acc[4 * c4 + 2] * inv, acc[4 * c4 + 3] * inv));
}

static inline ActV to_view(const heal_act_t* a) {
    ActV v;
    v.p = a->data; v.fmt = a->fmt; v.cs = a->cstride; v.co = a->coffset; v.plane = a->plane_stride;
    return v;
}

static inline bool aligned4(const heal_act_t* a) {
    return (a->cstride & 3) == 0 && (a->coffset & 3) == 0 && (a->fmt == 0 || (a->plane_stride & 3) == 0);
}

// the base pointer allows the 4-channel vector accesses of act_load4 / act_store4 (16 bytes fp32, 8 bytes bf16)
static inline bool data_aligned4(const heal_act_t* a) {
    return ((uintptr_t)a->data % (a->fmt == 0 ? 16u : 8u)) == 0;
}

}  // namespace

extern "C" int heal_swap_attention(const heal_act_t* qkv, const int* n_agents_host, int B, int L, int H, int W, int C,
                                   int window_size, int grid_mode, const float* bias, const heal_act_t* out, void* stream_) {
    if (!qkv || !qkv->data || !n_agents_host || !bias || !out || !out->data) return HEAL_ERR_ARG;
    if (B < 0 || L < 1 || H < 1 || W < 1 || C < 1 || window_size < 1 || (H % window_size) || (W % window_size)) return HEAL_ERR_ARG;
    if ((C % DH) || L * window_size * window_size > MAX_TOK || !aligned4(qkv) || !aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    if (!data_aligned4(qkv) || !data_aligned4(out)) return HEAL_ERR_UNSUPPORTED;
    const long long windows = (long long)(H / window_size) * (W / window_size);
    if (C / DH > 65535 || windows > 0x7fffffffLL) return HEAL_ERR_UNSUPPORTED;
    for (int b = 0; b < B; ++b)          // every count before the first launch, so a bad one leaves the output untouched
        if (n_agents_host[b] < 1 || n_agents_host[b] > L) return HEAL_ERR_ARG;
    SwapP p;
    p.qkv = to_view(qkv); p.out = to_view(out); p.bias = bias;
    p.H = H; p.W = W; p.C = C; p.L = L; p.w = window_size; p.grid = grid_mode ? 1 : 0;
    const int n = L * window_size * window_size;
    const int threads = (n + 31) / 32 * 32;
    int launches = 0;
    for (int b0 = 0; b0 < B; b0 += SCENES) {
        const int nb = B - b0 < SCENES ? B - b0 : SCENES;
        p.b0 = b0;
        for (int z = 0; z < nb; ++z) p.nb[z] = n_agents_host[b0 + z];
        k_swap_attention<<<dim3((unsigned)windows, (unsigned)(C / DH), (unsigned)nb), threads, 0, (cudaStream_t)stream_>>>(p);
        ++launches;
    }
    return heal_check_launch(launches);
}
