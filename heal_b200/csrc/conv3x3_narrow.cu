// 3x3 / stride 1 / pad 1 convolution of a NARROW input (1 <= Cin <= 63 channels) on the Hopper tensor cores: the first decoder
// conv of NaiveCompressor (opencood/models/sub_modules/naive_compress.py), whose input is the compressed map.  heal_conv2d_tc
// takes Cin in 64-channel blocks per tap; here the GEMM's K is the whole 3x3 neighbourhood, k = tap * cinp + ci, with cinp = Cin
// rounded up to even, padded to a multiple of 16.
//
// One CTA = two consumer warpgroups = one 8 x 16 tile of output pixels (128 GEMM rows) x one 64-wide block of output channels,
// persistent over the tiles of its channel block:
//   - the folded weights of the channel block stay in shared memory for all tiles: K blocks of 64, each [hi 64 rows | lo 64 rows]
//     x 128 B, 128B-swizzled K-major (the wgmma B operand);
//   - per tile the 10 x 18 input halo is loaded once (any storage format, any channel stride; channel pairs as one load where
//     the strides allow) into bf16 hi / lo planes, pixel pitch cw words (cw = 4 mod 8: the gathers below are free of bank
//     conflicts);
//   - the A operand comes from registers: for each K step every thread gathers its fragment's bf16 pairs (k, k+1 share a tap
//     because cinp is even) from the halo through a per-CTA table of word offsets, one K step ahead of the tensor core;
//   - per K step a_hi*b_lo (+ a_lo*b_hi with split activations) + a_hi*b_hi, fp32 accumulators: the products of heal_conv2d_tc;
//   - epilogue straight from the fragments: + folded-BN bias, optional ReLU, stored in the output's format (f32, bf16, split).
#include "common.cuh"
#include "tc_prims.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int NW_THREADS = 256;
constexpr int NW_TH = 8, NW_TW = 16;                          // output tile: 128 pixels
constexpr int NW_HW = NW_TW + 2;                              // halo row length
constexpr int NW_HP = (NW_TH + 2) * NW_HW;                    // halo pixels
constexpr int NW_NB = 64;                                     // output channels per CTA
constexpr int NW_KBLK = 2 * NW_NB * 128;                      // one 64-wide K block of the [hi | lo] weights: 16 KiB
constexpr int NW_HB = 8;                                      // halo words per thread per batch of loads

struct NwP {
    ActV in, out;
    const __nv_bfloat16* w;      // [Cout/64][kb][hi 64 rows | lo 64 rows][64] bf16
    const float* bias;           // [Cout]
    int N, H, W, Cin, cinp, cw, ks, kb, Cout, relu;
    int in_pairs;                // channel pairs (c, c + 1) of the input are one aligned 4-byte (bf16, split) / 8-byte (f32) load
    int tiles_x, tiles_y, ntiles, nblk, per_nb;
};

// D(64 x 64, fp32) (+)= A(64 x 16, bf16 registers) * B(16 x 64, smem, K-major).  Register a[j] of thread t of the warpgroup holds
// the bf16 pair (k, k+1) of row 16*(t/32) + (t%32)/4 + 8*(j%2), k = 2*(t%4) + 8*(j/2).
__device__ __forceinline__ void wgmma_ra_n64(float* d, const uint32_t* a, uint64_t b, uint32_t accum) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %37, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accum));
}

__device__ __forceinline__ void store_pair(const ActV& a, size_t pix, int c, float v0, float v1) {
    const size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (a.fmt == 0) {
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(a.p) + idx) = make_float2(v0, v1);
        return;
    }
    __nv_bfloat16* b = reinterpret_cast<__nv_bfloat16*>(a.p) + idx;
    const uint32_t h = pack_bf16(v0, v1);
    *reinterpret_cast<uint32_t*>(b) = h;
    if (a.fmt == 2) *reinterpret_cast<uint32_t*>(b + a.plane) = pack_bf16(v0 - bf16_lo_f(h), v1 - bf16_hi_f(h));
}

// the halo words of input channels (c, c + 1) of pixel `pix`: hi = bf16 pair, lo = the bf16 pair of what the rounding left
// (channel c + 1 reads as zero when `two` is false)
__device__ __forceinline__ void load_pair(const ActV& a, int pairs, size_t pix, int c, bool two, uint32_t& hi, uint32_t& lo) {
    const size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (pairs && a.fmt != 0) {
        const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(a.p) + idx;
        hi = __ldg(reinterpret_cast<const uint32_t*>(b));
        lo = a.fmt == 2 ? __ldg(reinterpret_cast<const uint32_t*>(b + a.plane)) : 0u;
        if (!two) { hi &= 0xffffu; lo &= 0xffffu; }
        return;
    }
    float v0, v1;
    if (pairs) {
        const float2 v = __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(a.p) + idx));
        v0 = v.x; v1 = two ? v.y : 0.f;
    } else {
        v0 = act_load1(a, pix, c);
        v1 = two ? act_load1(a, pix, c + 1) : 0.f;
    }
    hi = pack_bf16(v0, v1);
    lo = pack_bf16(bf16_rest(v0), bf16_rest(v1));
}

template <int PLANES>
__global__ void __launch_bounds__(NW_THREADS, 1)
k_conv3x3_narrow_tc(const NwP p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uintptr_t raw_addr = reinterpret_cast<uintptr_t>(smem_raw);
    asm volatile("" : "+l"(raw_addr));
    uint8_t* smem = reinterpret_cast<uint8_t*>(raw_addr);
    if (smem_u32(smem) & 1023u) __trap();
    const uint32_t sw = smem_u32(smem);
    uint32_t* halo = reinterpret_cast<uint32_t*>(smem + (size_t)p.kb * NW_KBLK);   // [PLANES][NW_HP][cw] bf16 pairs
    int* kofs = reinterpret_cast<int*>(halo + (size_t)PLANES * NW_HP * p.cw);     // [ks * 8]: halo word of the pair (2j, 2j+1)
    const int tid = threadIdx.x;
    const int nb = blockIdx.x % p.nblk;

    {   // the channel block's weights, 16-byte chunks into the swizzled K-major layout
        const uint4* src = reinterpret_cast<const uint4*>(p.w + (size_t)nb * p.kb * (NW_KBLK / 2));
        const int chunks = p.kb * (NW_KBLK / 16);
        for (int i = tid; i < chunks; i += NW_THREADS) {
            const int blk = i >> 10, r = (i >> 3) & 127, c = i & 7;
            const uint4 v = __ldg(src + i);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};"
                         ::"r"(sw + blk * NW_KBLK + r * 128 + ((c ^ (r & 7)) << 4)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
        }
        const int taps_k = 9 * p.cinp;
        for (int j = tid; j < p.ks * 8; j += NW_THREADS) {
            const int k = 2 * j;
            int off = p.cinp / 2;                    // K padding: a zero word of halo pixel 0 (cw > cinp / 2)
            if (k < taps_k) {
                const int tap = k / p.cinp, ci = k - tap * p.cinp;
                off = ((tap / 3) * NW_HW + tap % 3) * p.cw + ci / 2;
            }
            kofs[j] = off;
        }
        fence_async_smem();
    }

    const int wg = tid >> 7, wl = (tid >> 5) & 3, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = 64 * wg + 16 * wl + g;            // this thread's tile rows r0 and r0 + 8: same tile row, columns g and g + 8
    const int ty = r0 >> 4, tx = r0 & 15;
    const uint32_t* h0 = halo + (ty * NW_HW + tx) * p.cw;
    const uint32_t* h1 = h0 + 8 * p.cw;
    const int lo = NW_HP * p.cw;

    auto gather = [&](int s, uint32_t* a) {
        const int o0 = kofs[8 * s + t], o1 = kofs[8 * s + t + 4];
        a[0] = h0[o0]; a[1] = h1[o0]; a[2] = h0[o1]; a[3] = h1[o1];
        if constexpr (PLANES == 2) { a[4] = h0[lo + o0]; a[5] = h1[lo + o0]; a[6] = h0[lo + o1]; a[7] = h1[lo + o1]; }
    };
    float d[32];
    auto mma = [&](int s, const uint32_t* a) {
        const uint32_t bb = sw + (s >> 2) * NW_KBLK + (s & 3) * 32;
        const uint64_t b_hi = gmma_desc_sw128(bb), b_lo = gmma_desc_sw128(bb + NW_KBLK / 2);
        wgmma_ra_n64(d, a, b_lo, s == 0 ? 0u : 1u);                  // a_hi * b_lo
        if constexpr (PLANES == 2) wgmma_ra_n64(d, a + 4, b_hi, 1u);  // a_lo * b_hi
        wgmma_ra_n64(d, a, b_hi, 1u);                                 // a_hi * b_hi
    };

    const int per_img = p.tiles_x * p.tiles_y;
    for (int tile = blockIdx.x / p.nblk; tile < p.ntiles; tile += p.per_nb) {
        const int n = tile / per_img, rem = tile - n * per_img;
        const int y0 = (rem / p.tiles_x) * NW_TH, x0 = (rem % p.tiles_x) * NW_TW;
        __syncthreads();                              // the previous tile's gathers are done (and, first time, the weights are in)
        // the halo, NW_HB words per thread in flight: the tile's only global-memory round trips before its MMAs
        for (int i0 = tid; i0 < NW_HP * p.cw; i0 += NW_HB * NW_THREADS) {
            uint32_t hv[NW_HB], lv[NW_HB];
#pragma unroll
            for (int u = 0; u < NW_HB; ++u) {
                const int i = i0 + u * NW_THREADS;
                const int hp = i / p.cw, c = 2 * (i - hp * p.cw);
                const int yy = y0 - 1 + hp / NW_HW, xx = x0 - 1 + hp % NW_HW;
                hv[u] = 0u; lv[u] = 0u;
                if (i < NW_HP * p.cw && yy >= 0 && yy < p.H && xx >= 0 && xx < p.W && c < p.Cin)
                    load_pair(p.in, p.in_pairs, ((size_t)n * p.H + yy) * p.W + xx, c, c + 1 < p.Cin, hv[u], lv[u]);
            }
#pragma unroll
            for (int u = 0; u < NW_HB; ++u) {
                const int i = i0 + u * NW_THREADS;
                if (i < NW_HP * p.cw) {
                    halo[i] = hv[u];
                    if constexpr (PLANES == 2) halo[lo + i] = lv[u];
                }
            }
        }
        __syncthreads();

        // one K step of gathers ahead of the tensor core: aa / ab alternate, a buffer is refilled once its MMAs have retired
        uint32_t aa[4 * PLANES], ab[4 * PLANES];
        gather(0, aa);
        for (int s = 0; s < p.ks; s += 2) {
            wgmma_fence();
            mma(s, aa);
            wgmma_commit();
            wgmma_wait<1>();
            if (s + 1 < p.ks) {
                gather(s + 1, ab);
                wgmma_fence();
                mma(s + 1, ab);
                wgmma_commit();
                wgmma_wait<1>();
            }
            if (s + 2 < p.ks) gather(s + 2, aa);
        }
        wgmma_wait<0>();

        const int y = y0 + ty;
        if (y < p.H) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int x = x0 + tx + 8 * h;
                if (x >= p.W) continue;
                const size_t pix = ((size_t)n * p.H + y) * p.W + x;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int col = nb * NW_NB + 8 * j + 2 * t;
                    if (col >= p.Cout) continue;
                    const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                    float v0 = d[4 * j + 2 * h] + bv.x, v1 = d[4 * j + 2 * h + 1] + bv.y;
                    if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                    store_pair(p.out, pix, col, v0, v1);
                }
            }
        }
    }
}

template <int PLANES>
int launch_narrow(const NwP& p, cudaStream_t st) {
    const size_t smem = (size_t)p.kb * NW_KBLK + (size_t)PLANES * NW_HP * p.cw * 4 + (size_t)p.ks * 8 * 4 + 1024;
    if (smem > 227 * 1024) return HEAL_ERR_UNSUPPORTED;
    static size_t attr_set[HEAL_MAX_DEVICES] = {};
    if (!heal_ensure_dyn_smem(k_conv3x3_narrow_tc<PLANES>, smem, attr_set)) return HEAL_ERR_LAUNCH;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_conv3x3_narrow_tc<PLANES>, NW_THREADS, smem) != cudaSuccess ||
        per_sm < 1)
        return HEAL_ERR_LAUNCH;
    NwP q = p;
    const int cap = HEAL_NUM_SMS * per_sm / q.nblk;
    q.per_nb = q.ntiles < cap ? q.ntiles : (cap > 0 ? cap : 1);
    k_conv3x3_narrow_tc<PLANES><<<q.per_nb * q.nblk, NW_THREADS, smem, st>>>(q);
    return heal_check_launch();
}

}  // namespace

extern "C" int heal_conv3x3_narrow_tc(const heal_act_t* in, int N, int H, int W, int Cin, const void* w_packed, const float* bias,
                                      int Cout, int planes, int relu, const heal_act_t* out, void* stream) {
    if (!in || !in->data || !out || !out->data || !w_packed || !bias) return HEAL_ERR_ARG;
    if (N < 1 || H < 1 || W < 1 || Cin < 1 || Cin > 63 || Cout < 16 || Cout > 256 || (Cout % 16)) return HEAL_ERR_ARG;
    if ((planes != 1 && planes != 2) || (relu != 0 && relu != 1)) return HEAL_ERR_ARG;
    if (in->fmt < 0 || in->fmt > 2 || out->fmt < 0 || out->fmt > 2) return HEAL_ERR_ARG;
    if (in->coffset < 0 || in->cstride < in->coffset + Cin || out->coffset < 0 || out->cstride < out->coffset + Cout) return HEAL_ERR_ARG;
    // fragment stores write channel pairs: even strides and offsets, 8-byte (fp32) / 4-byte (bf16) aligned data
    if ((out->cstride & 1) || (out->coffset & 1) || (out->fmt == 2 && (out->plane_stride & 1))) return HEAL_ERR_UNSUPPORTED;
    if (((uintptr_t)out->data & (out->fmt == 0 ? 7u : 3u)) || ((uintptr_t)w_packed & 15u) || ((uintptr_t)bias & 7u))
        return HEAL_ERR_UNSUPPORTED;
    const long long tiles_x = (W + NW_TW - 1) / NW_TW, tiles_y = (H + NW_TH - 1) / NW_TH, ntiles = (long long)N * tiles_x * tiles_y;
    if (ntiles > (1LL << 30)) return HEAL_ERR_UNSUPPORTED;
    NwP p;
    p.in = ActV{in->data, in->fmt, in->cstride, in->coffset, in->plane_stride};
    p.out = ActV{out->data, out->fmt, out->cstride, out->coffset, out->plane_stride};
    p.w = (const __nv_bfloat16*)w_packed; p.bias = bias;
    p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.relu = relu;
    p.in_pairs = !((in->cstride | in->coffset) & 1) && (in->fmt != 2 || !(in->plane_stride & 1)) &&
                 !((uintptr_t)in->data & (in->fmt == 0 ? 7u : 3u));
    p.cinp = (Cin + 1) & ~1;
    p.cw = ((p.cinp / 2 + 1 + 3) / 8) * 8 + 4;      // smallest word pitch >= cinp / 2 + 1 with pitch = 4 (mod 8)
    const int k = (9 * p.cinp + 15) / 16 * 16;
    p.ks = k / 16; p.kb = (k + 63) / 64;
    p.tiles_x = (int)tiles_x; p.tiles_y = (int)tiles_y; p.ntiles = (int)ntiles;
    p.nblk = (Cout + NW_NB - 1) / NW_NB; p.per_nb = 1;
    cudaStream_t st = (cudaStream_t)stream;
    return planes == 2 ? launch_narrow<2>(p, st) : launch_narrow<1>(p, st);
}
