// Sparse 3-D convolution gather-GEMM on the Hopper tensor cores (wgmma, fp32 accumulators in registers) for the
// SECOND middle encoder (VoxelBackBone8x; reference layer list: opencood/models/sub_modules/sparse_backbone_3d.py:48-91,
// post_act_block :11-30 = conv + BatchNorm1d(eps 1e-3) + ReLU; spconv semantics restated in oracle/sparse_conv.py).
//
// Output-stationary rulebook (csrc/spconv.cu): nbr[out_row][k] = input row under kernel offset k, or -1.
// GEMM view per 128-row output tile: D[128 x Cout] = sum over K-blocks  A_kb[128 x 64] . W_kb[64 x Cout]
//   A_kb row r = the gathered input rows of out-row r for the 64/Cin kernel offsets of K-block kb, side by side
//                (Cin = 64: one offset per K-block; 32: two; 16: four), zero where the rulebook says -1;
//   W_kb       = the matching offsets' (Cin x Cout) weight blocks stacked along K (zero rows for padding offsets).
// Features travel between layers as "split rows": (rows, 2*C) bf16 = [hi C | lo C], x ~= hi + lo (16 mantissa bits),
// and a product is a_hi*b_hi + a_hi*b_lo + a_lo*b_hi with fp32 accumulation: fp32-equivalent (same scheme as conv2d_tc.cu).
//
// Roles (384 threads, persistent over tiles):
//   warps 0..3  gather producers: the tile's rulebook rows go to shared memory once; per ACTIVE K-block (a K-block none of
//               the tile's 128 rows hits is skipped altogether) every thread issues sixteen 16-byte cp.async copies (8 lanes
//               per gathered row: full 128 B lines; src-size 0 zero-fills a miss) into the 128B-swizzled K-major A tile, and
//               one lane TMA-loads the K-block's weights.  Copies stay in flight across K-blocks and tiles (cp.async groups,
//               two behind), then fence.proxy.async + mbarrier arrive hand the stage to the tensor core.
//   warps 4..11 two consumer warpgroups, rows [0, 64) and [64, 128) of the tile: 4 K-steps x { a_hi x [b_hi | b_lo] (N' = 2 Cout),
//               a_lo x b_hi } per stage (Cout = 128: three N = 128 products), then the epilogue: main + aux -> fp32 scratch in
//               shared memory (one row per thread) -> + BN shift -> ReLU -> split rows (or fp32 rows) to global.
#include <cuda.h>
#include "common.cuh"
#include "tc_prims.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int SPT_THREADS = 384;
constexpr int SPT_M = 128;
constexpr int SPT_ATILE = SPT_M * 128;          // one plane of A: 128 rows x 128 B

struct SptP {
    const __nv_bfloat16* in;     // split rows: hi channels at in + row*in_pitch, lo channels at + in_lo (interleaved rows: pitch 2*CIN, lo CIN;
                                 // a planar split `Act`: pitch = pixel stride, lo = plane stride)
    long long in_pitch, in_lo, out_pitch, out_lo;
    const int* nbr;              // (capacity, K)
    const int* m_dev;            // live output rows on the device (or nullptr)
    int M;                       // capacity
    int K, KB;                   // kernel offsets, K-blocks = ceil(K / (64 / CIN))
    const float* bias;           // (COUT) folded BatchNorm shift
    int relu;
    __nv_bfloat16* out_split;    // (capacity, 2*COUT) or nullptr
    float* out_f32;              // (capacity, COUT) or nullptr
};

__device__ __forceinline__ void prod_bar() { asm volatile("bar.sync 3, 128;" ::: "memory"); }

template <int CIN, int COUT, int STAGES>
__global__ void __launch_bounds__(SPT_THREADS, 1)
k_spconv_tc(const __grid_constant__ CUtensorMap tmB, const SptP p) {
    constexpr int TPK = 64 / CIN;                   // kernel offsets per 64-wide K-block
    constexpr int CPT = CIN / 8;                    // 16-byte chunks per gathered row and plane
    constexpr int B_BYTES = 2 * COUT * 128;         // [plane][COUT rows][128 B]
    constexpr int STAGE_BYTES = 2 * SPT_ATILE + B_BYTES;
    constexpr bool NCAT = (COUT <= 64);             // a_hi x [b_hi | b_lo] as one N = 2 COUT product
    constexpr int NACC = NCAT ? 2 * COUT : COUT;    // accumulator columns (main | aux)
    constexpr int SW = COUT < 64 ? COUT : 64;       // accumulator columns per pass through the scratch
    constexpr int LA = (STAGES >= 4) ? 2 : 1;       // cp.async groups a producer keeps in flight behind the one it issues
    constexpr int KPAD = 28;                        // rulebook row pitch in shared memory (K <= 27)

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uintptr_t raw_addr = reinterpret_cast<uintptr_t>(smem_raw);
    asm volatile("" : "+l"(raw_addr));
    uint8_t* smem = reinterpret_cast<uint8_t*>(raw_addr);
    if (smem_u32(smem) & 1023u) __trap();
    const uint32_t scr = smem_u32(smem + (size_t)STAGES * STAGE_BYTES);   // fp32 scratch [128 rows][SW]
    int* snbr = reinterpret_cast<int*>(smem + (size_t)STAGES * STAGE_BYTES + SPT_M * SW * 4);
    int* sflags = snbr + SPT_M * KPAD;                                  // [STAGES] bit0 = first K-block of its tile, bit1 = last
    unsigned* smask = reinterpret_cast<unsigned*>(sflags + STAGES);     // [2] active-K-block mask of the tile being set up
    uint64_t* bars = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(smask + 2) + 7) & ~(uintptr_t)7);
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + STAGES);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, 128 + 1); mbar_init(bar_empty + 8 * s, 8); }   // 8 consumer warps
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int Md = p.m_dev ? min(p.M, p.m_dev[0]) : p.M;
    const int ntiles = (Md + SPT_M - 1) / SPT_M;

    if (warp < 4) {
        // ================================ gather producers ================================
        const int tid = threadIdx.x;                 // 0..127
        int stage = 0; uint32_t phase = 0;
        int pend[LA + 1]; int npend = 0;
#pragma unroll
        for (int i = 0; i <= LA; ++i) pend[i] = 0;
        // The tile's rulebook rows (128 x K ints, contiguous) are prefetched into REGISTERS one tile ahead: the loads fly under the
        // current tile's gathers, so a tile starts without an exposed global-memory round trip (the first version re-read them at
        // every tile start and stalled on that round trip)
        int nxt[27];
        auto fetch = [&](int tile_) {
            const long long base = (long long)tile_ * SPT_M * p.K;
            const int lim = min(SPT_M, Md - tile_ * SPT_M) * p.K;
#pragma unroll
            for (int q = 0; q < 27; ++q) {
                const int i = tid + 128 * q;
                nxt[q] = (q < p.K && i < lim) ? __ldg(p.nbr + base + i) : -1;
            }
        };
        if ((int)blockIdx.x < ntiles) fetch(blockIdx.x);
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            prod_bar();                               // every producer has issued the previous tile's copies (they read snbr)
            if (tid == 0) smask[0] = 0u;
#pragma unroll
            for (int q = 0; q < 27; ++q) {
                if (q < p.K) {
                    const int i = tid + 128 * q;
                    const int r = i / p.K, k = i - r * p.K;
                    snbr[r * KPAD + k] = nxt[q];
                }
            }
            if (tile + (int)gridDim.x < ntiles) fetch(tile + gridDim.x);
            prod_bar();
            {   // active K-blocks of this tile = OR over its rows
                unsigned m = 0;
                for (int k = 0; k < p.K; ++k) if (snbr[tid * KPAD + k] >= 0) m |= 1u << (k / TPK);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);
                if (lane == 0 && m) atomicOr(smask, m);
            }
            prod_bar();
            unsigned mask = smask[0];
            if (mask == 0u) mask = 1u;                // a tile always produces one stage (never happens: the centre / generating offset hits)
            const int kb_first = __ffs(mask) - 1, kb_last = 31 - __clz(mask);
            for (int kb = kb_first; kb <= kb_last; ++kb) {
                if (!((mask >> kb) & 1u)) continue;
                mbar_wait(bar_empty + 8 * stage, phase ^ 1);
                const uint32_t sa = smem_base + stage * STAGE_BYTES;
                if (warp == 0) {
                    if (elect_one()) {
                        sflags[stage] = (kb == kb_first ? 1 : 0) | (kb == kb_last ? 2 : 0);
                        mbar_expect_tx(bar_full + 8 * stage, (uint32_t)B_BYTES);
                        tma_load_3d(sa + 2 * SPT_ATILE, &tmB, bar_full + 8 * stage, 0, kb * COUT, 0);
                    }
                    __syncwarp();
                }
                // 8 lanes per gathered row: lane & 7 = 16-byte chunk of the 128-byte K-block row, lane >> 3 = row within a group of 4
                const int c = lane & 7;
                const int tl = c / CPT, sc = c - tl * CPT;          // offset within the K-block, chunk within that offset's row
                const int tap = kb * TPK + tl;
#pragma unroll
                for (int it = 0; it < 8; ++it) {
                    const int r = warp * 32 + it * 4 + (lane >> 3);
                    const int src = (tap < p.K) ? snbr[r * KPAD + tap] : -1;
                    const __nv_bfloat16* g = p.in + (src >= 0 ? (long long)src * p.in_pitch + sc * 8 : 0);
                    const uint32_t nb = src >= 0 ? 16u : 0u;
                    const uint32_t d = sa + r * 128 + ((c ^ (r & 7)) << 4);
                    cp_async16(d, g, nb);                            // hi plane
                    cp_async16(d + SPT_ATILE, g + (src >= 0 ? p.in_lo : 0), nb);   // lo plane
                }
                cp_async_commit();
                pend[npend++] = stage;
                if (npend > LA) {
                    cp_async_wait<LA>();
                    fence_async_smem();
                    mbar_arrive(bar_full + 8 * pend[0]);
#pragma unroll
                    for (int i = 0; i < LA; ++i) pend[i] = pend[i + 1];
                    --npend;
                }
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
        cp_async_wait<0>();
        fence_async_smem();
        for (int i = 0; i < npend; ++i) mbar_arrive(bar_full + 8 * pend[i]);
    } else {
        // ================================ consumers: wgmma + epilogue ================================
        const int wg = (warp >> 2) - 1;                // MMAs: tile rows [64 wg, 64 wg + 64)
        const int quarter = warp & 3;
        const int chalf = (warp - 4) >> 2;             // epilogue: which half of each scratch chunk this warp drains
        const int row = quarter * 32 + lane;
        constexpr int CH = (COUT >= 32) ? 32 : 16;
        float d[NACC / 2];
#pragma unroll
        for (int i = 0; i < NACC / 2; ++i) d[i] = 0.f;
        int stage = 0; uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            int prev = -1;
            while (true) {
                mbar_wait(bar_full + 8 * stage, phase);
                const int fl = sflags[stage];
                const uint32_t sa = smem_base + stage * STAGE_BYTES + (uint32_t)(wg * 64 * 128);
                const uint32_t sb = smem_base + stage * STAGE_BYTES + 2 * SPT_ATILE;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint64_t a_hi = gmma_desc_sw128(sa + k * 32), a_lo = gmma_desc_sw128(sa + SPT_ATILE + k * 32);
                    const uint64_t b = gmma_desc_sw128(sb + k * 32);
                    const uint32_t first = ((fl & 1) && k == 0) ? 0u : 1u;
                    if constexpr (NCAT) {
                        wgmma_bf16<2 * COUT>(d, a_hi, b, first);                  // [a_hi*b_hi | a_hi*b_lo]
                        wgmma_bf16<COUT>(d, a_lo, b, 1u);                         // += a_lo*b_hi
                    } else {
                        wgmma_bf16<COUT>(d, a_hi, gmma_desc_sw128(sb + COUT * 128 + k * 32), first);   // a_hi*b_lo
                        wgmma_bf16<COUT>(d, a_lo, b, 1u);
                        wgmma_bf16<COUT>(d, a_hi, b, 1u);
                    }
                }
                wgmma_commit();
                // The producers hand a stage over LA stages late (cp.async groups in flight), so keeping one stage of MMAs in
                // flight here as well needs STAGES > LA + 1: otherwise both sides wait for each other.
                if constexpr (STAGES > LA + 1) {
                    wgmma_wait<1>();                   // the previous stage's MMAs have retired: free it
                    if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
                    prev = stage;
                } else {
                    wgmma_wait<0>();
                    if (lane == 0) mbar_arrive(bar_empty + 8 * stage);
                }
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
                if (fl & 2) break;
            }
            wgmma_wait<0>();
            if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
            if constexpr (NCAT) {
#pragma unroll
                for (int i = 0; i < COUT / 2; ++i) d[i] += d[i + COUT / 2];
            }
            const int grow = tile * SPT_M + row;
#pragma unroll 1
            for (int cs = 0; cs < COUT; cs += SW) {
                epi_bar(1);
                frag_to_scratch<COUT / 2, SW>(d, scr, 64 * wg, cs);
                epi_bar(1);
                if (chalf >= SW / CH || grow >= Md) continue;
                const int c0 = cs + chalf * CH;
                uint32_t x[CH];
                scratch_row<SW, CH>(scr, row, chalf * CH, x);
#pragma unroll
                for (int g8 = 0; g8 < CH / 8; ++g8) {
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        v[j] = __uint_as_float(x[g8 * 8 + j]) + (p.bias ? __ldg(p.bias + c0 + g8 * 8 + j) : 0.f);
                        if (p.relu) v[j] = fmaxf(v[j], 0.f);
                    }
                    if (p.out_split) {
                        uint32_t hw[4], lw[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float h0 = __bfloat162float(__float2bfloat16_rn(v[2 * j])), h1 = __bfloat162float(__float2bfloat16_rn(v[2 * j + 1]));
                            hw[j] = pack_bf16(v[2 * j], v[2 * j + 1]);
                            lw[j] = pack_bf16(v[2 * j] - h0, v[2 * j + 1] - h1);
                        }
                        __nv_bfloat16* o = p.out_split + (long long)grow * p.out_pitch + c0 + g8 * 8;
                        *reinterpret_cast<uint4*>(o) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                        *reinterpret_cast<uint4*>(o + p.out_lo) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
                    }
                    if (p.out_f32) {
                        float* o = p.out_f32 + (size_t)grow * COUT + c0 + g8 * 8;
                        stg_f4(o, make_float4(v[0], v[1], v[2], v[3]));
                        stg_f4(o + 4, make_float4(v[4], v[5], v[6], v[7]));
                    }
                }
            }
        }
    }
}

template <int CIN, int COUT>
int launch_spt(const SptP& p, const void* w_packed, cudaStream_t st) {
    constexpr int STAGES = (COUT >= 128) ? 2 : (COUT >= 64 ? 3 : 4);
    constexpr int B_BYTES = 2 * COUT * 128;
    constexpr size_t SMEM = (size_t)STAGES * (2 * SPT_ATILE + B_BYTES) + (size_t)SPT_M * (COUT < 64 ? COUT : 64) * 4 + SPT_M * 28 * 4 + 512;
    static_assert(SMEM <= 227 * 1024, "shared memory budget");
    PFN_tmEncodeTiled enc = get_encode();
    if (!enc) return HEAL_ERR_DRIVER;
    CUtensorMap tmB;
    {
        cuuint64_t d[3] = {64, (cuuint64_t)p.KB * COUT, 2};
        cuuint64_t s[2] = {128, (cuuint64_t)p.KB * COUT * 128};
        cuuint32_t b[3] = {64u, (cuuint32_t)COUT, 2u};
        cuuint32_t es[3] = {1, 1, 1};
        if (enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)w_packed, d, s, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return HEAL_ERR_DRIVER;
    }
    static size_t attr_set[HEAL_MAX_DEVICES] = {};
    if (!heal_ensure_dyn_smem(k_spconv_tc<CIN, COUT, STAGES>, SMEM, attr_set)) return HEAL_ERR_LAUNCH;
    int tiles = (p.M + SPT_M - 1) / SPT_M;
    int grid = tiles < HEAL_NUM_SMS ? tiles : HEAL_NUM_SMS;
    k_spconv_tc<CIN, COUT, STAGES><<<grid, SPT_THREADS, SMEM, st>>>(tmB, p);
    return heal_check_launch();
}

// fp32 rows -> split rows [hi C | lo C]
__global__ void k_rows_to_split(const float* __restrict__ in, const int* __restrict__ m_dev, int M, int C, __nv_bfloat16* __restrict__ out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int Md = m_dev ? min(M, m_dev[0]) : M;
    if (t >= (long long)Md * C) return;
    const int r = (int)(t / C), c = (int)(t % C);
    const float v = in[t];
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    out[(size_t)r * 2 * C + c] = h;
    out[(size_t)r * 2 * C + C + c] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// PointPillars stem as a sparse 2-D convolution: rulebook of a k x k / stride-2 conv from the pillar list (cell -> pillar row id
// map) to the DENSE output grid.  nbr[(b*Ho + oy)*Wo + ox][r*k + s] = idmap[b][2oy + r - pad][2ox + s - pad] or -1.
__global__ void k_stem_rulebook(const int* __restrict__ idmap, int B, int ny, int nx, int Ho, int Wo, int k, int pad, int* __restrict__ nbr) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int K = k * k;
    if (t >= (long long)B * Ho * Wo * K) return;
    const int tap = (int)(t % K);
    long long pix = t / K;
    const int ox = (int)(pix % Wo); pix /= Wo;
    const int oy = (int)(pix % Ho); const int b = (int)(pix / Ho);
    const int y = 2 * oy + tap / k - pad, x = 2 * ox + tap % k - pad;
    nbr[t] = (y >= 0 && y < ny && x >= 0 && x < nx) ? __ldg(idmap + ((size_t)b * ny + y) * nx + x) : -1;
}

}  // namespace

extern "C" int heal_stem_rulebook(const int* idmap, int batch, int ny, int nx, int ksize, int pad, int* nbr_out, void* stream_) {
    if (!idmap || !nbr_out || batch < 1 || (ny & 1) || (nx & 1) || ksize < 1) return HEAL_ERR_ARG;
    const int Ho = ny / 2, Wo = nx / 2;
    const long long total = (long long)batch * Ho * Wo * ksize * ksize;
    k_stem_rulebook<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(idmap, batch, ny, nx, Ho, Wo, ksize, pad, nbr_out);
    return heal_check_launch();
}

extern "C" int heal_spconv_gather_gemm_tc(const void* in_split_rows, const int* nbr, const int* out_rows_dev, int out_capacity, int kvol,
                                          const void* w_packed, const float* bias, int c_in, int c_out, int relu,
                                          void* out_split_rows, float* out_f32,
                                          long long in_pitch, long long in_lo, long long out_pitch, long long out_lo, void* stream_) {
    if (!in_split_rows || !nbr || !w_packed || (!out_split_rows && !out_f32) || out_capacity < 1) return HEAL_ERR_ARG;
    if (kvol < 1 || kvol > 27) return HEAL_ERR_UNSUPPORTED;
    if (c_in != 16 && c_in != 32 && c_in != 64) return HEAL_ERR_UNSUPPORTED;
    SptP p;
    p.in = (const __nv_bfloat16*)in_split_rows; p.nbr = nbr; p.m_dev = out_rows_dev; p.M = out_capacity;
    p.K = kvol; p.KB = (kvol + (64 / c_in) - 1) / (64 / c_in);
    p.bias = bias; p.relu = relu; p.out_split = (__nv_bfloat16*)out_split_rows; p.out_f32 = out_f32;
    p.in_pitch = in_pitch > 0 ? in_pitch : 2 * c_in; p.in_lo = in_lo > 0 ? in_lo : c_in;
    p.out_pitch = out_pitch > 0 ? out_pitch : 2 * c_out; p.out_lo = out_lo > 0 ? out_lo : c_out;
    if ((p.in_pitch | p.in_lo | p.out_pitch | p.out_lo) & 7) return HEAL_ERR_UNSUPPORTED;      // 16-byte rows
    cudaStream_t st = (cudaStream_t)stream_;
#define SPT(ci, co) if (c_in == ci && c_out == co) return launch_spt<ci, co>(p, w_packed, st)
    SPT(16, 16); SPT(16, 32); SPT(32, 32); SPT(32, 64); SPT(64, 64); SPT(64, 128);
#undef SPT
    return HEAL_ERR_UNSUPPORTED;
}

extern "C" int heal_rows_to_split(const float* rows_f32, const int* rows_dev, int capacity, int channels, void* out_split_rows, void* stream_) {
    if (!rows_f32 || !out_split_rows || capacity < 1 || channels < 1) return HEAL_ERR_ARG;
    long long total = (long long)capacity * channels;
    k_rows_to_split<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(rows_f32, rows_dev, capacity, channels,
                                                                                       (__nv_bfloat16*)out_split_rows);
    return heal_check_launch();
}
