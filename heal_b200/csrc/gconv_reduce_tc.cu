// The grouped 3x3 and the 1x1 reduce of PyramidFusion's stride-1 level-1 and level-2 ResNeXt bottlenecks (resblock.py:
// Bottleneck, width = 2 C, 32 groups, no downsample) as ONE persistent wgmma kernel:
//   y = ReLU(W3 * ReLU(Wg (*) mid + b2) + b3 + x)          mid = ReLU(W1 * x + b1), written by the expand launch before it
// The grouped conv's output (as wide as mid) never leaves shared memory: the two-launch path writes it to HBM and reads it back.
//
// A work item is a 16 x 8 output-pixel tile of one image and one 128-channel block nt of the output (level 2's 256 outputs are
// two items per tile, each recomputing the tile's grouped conv: the reduce accumulators of 256 outputs do not fit next to the
// grouped ones in one warpgroup).  For each 64-channel chunk c of the width, in ascending order:
//   1. grouped 3x3: the chunk's 18 x 10 halo of mid is one 5-D TMA box (zero-filled outside the image, which is the conv's
//      padding); the 16-channel sub-block MMAs and fold of k_gconv3x3_ring on the packed diagonal weights, one sub-block at a
//      time (k_bottleneck_tc's stage 2); bias + ReLU + hi/lo split into the swizzled g chunk [plane][128 pixels][128 B].
//   2. reduce: the g chunk x the chunk's 64 K rows of W3 into accumulators that stay in registers across the chunks.
// After the last chunk: bias3, the residual (TMA-loaded into the two output staging halves), ReLU, split, TMA tensor stores.
//
// Bit-identical to conv2d_tc(Wg) -> conv2d_tc(W3, residual=x): the grouped conv keeps the MMA form, tap order, fold and rounding
// of k_gconv3x3_ring / k_conv2d_tc<64, GROUPED> (the two agree bit for bit); the reduce is k_conv2d_tc<128>'s three MMAs per K16
// step into one accumulator (a_hi*b_lo, a_lo*b_hi, a_hi*b_hi), K ascending, and its epilogue order (bias, residual hi, lo, ReLU).
//
// Roles (384 threads): warp 0 = TMA producer (loads and the output stores), warpgroups 1 and 2 = the M = 64 MMAs of one half
// of the tile each (output rows [8 wg, 8 wg + 8)).  A warpgroup's reduce reads only the g rows it wrote itself, so the two
// consumer warpgroups synchronise only through the producer's barriers.
//
// Shared memory (split activations; bf16 halves the halo, g and staging planes):
//   ring of S stages  [mid halo chunk 2 x 180 x 128 B = 45 KiB | grouped weights of the chunk 9 x 4 x 2 x 512 B = 36 KiB]
//   W3 slot           [plane][128 rows][128 B] = 32 KiB            output staging half 1 after the last chunk
//   g chunk           [plane][128 pixels][128 B] = 32 KiB          output staging half 0 after the last chunk
//   split: 2 x 81 + 32 + 32 = 226 KiB of 227 (S = 2); bf16: S = 3 (3 x 59 + 32 + 16 = 225 KiB).  Three split stages
//   would need the W3 slot or the g chunk halved (32-channel chunks, 64B swizzle); not done.
// The producer runs ahead of the MMAs by the ring: the halo and weights of chunk i + 1 (the next tile's first chunk during an
// epilogue) are in flight while chunk i is computed, and W3 of chunk i is requested when the reduce of chunk i - 1 retires.
#include <cuda.h>
#include "common.cuh"
#include "tc_prims.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int GR_THREADS = 384;
constexpr int GR_TH = 16, GR_TW = 8;                     // output tile: 16 rows x 8 pixels = the MMA's 128 rows
constexpr int GR_HW = GR_TW + 2;                         // halo tile: 18 rows x 10 pixels
constexpr int GR_HALO = (GR_TH + 2) * GR_HW;             // 180 pixels
constexpr int GR_HPLANE = GR_HALO * 128;                 // one plane of a halo chunk: 180 pixels x 64 channels bf16
constexpr int GR_TPLANE = 128 * 128;                     // one plane of a 128-pixel x 64-channel tile
constexpr int GR_WG_ROW = 3 * 4 * 2 * 512;               // one kernel row of grouped weights: [3 taps][4 sub-blocks][plane][16][32 B]
constexpr int GR_WG_CHUNK = 3 * GR_WG_ROW;               // 36 KiB
constexpr int GR_N = 128;                                // output channels per work item
constexpr int GR_W3_SLOT = 2 * GR_N * 128;               // [plane][128 rows][64 K] = 32 KiB
constexpr int GR_MAX_STAGES = 4;
constexpr int GR_SMEM_LIMIT = 227 * 1024;
constexpr uint32_t GR_MID_SBO = GR_HW * 128;             // one halo row

__host__ __device__ inline int gr_halo_bytes(int planes) { return (planes * GR_HPLANE + 1023) & ~1023; }
__host__ __device__ inline int gr_stage_bytes(int planes) { return gr_halo_bytes(planes) + GR_WG_CHUNK; }
__host__ inline int gr_fixed_bytes(int planes) { return GR_W3_SLOT + planes * GR_TPLANE + 256; }
__host__ inline int gr_stages(int planes) {
    const int s = (GR_SMEM_LIMIT - gr_fixed_bytes(planes)) / gr_stage_bytes(planes);
    return s > GR_MAX_STAGES ? GR_MAX_STAGES : s;
}

struct GrP {
    int N, H, W;
    int tiles_w, tiles_h, n_tiles, items;   // items = N * tiles_h * tiles_w * n_tiles
    int chunks;                             // width / 64
    int planes;                             // activation planes: 2 = split-bf16, 1 = bf16 (the weights always carry both)
    int stages;
    int pdl;
    const float *b2, *b3;
};

// 128B-swizzled K-major descriptor with an explicit stride byte offset (distance between 8-row groups)
__device__ __forceinline__ uint64_t desc_sw128_sbo(uint32_t saddr, uint32_t sbo) {
    return (gmma_desc_sw128(saddr) & ~(0x3FFFull << 32)) | ((uint64_t)(sbo >> 4) << 32);
}
// named barrier of one consumer warpgroup (ids 1 and 2)
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

__global__ void __launch_bounds__(GR_THREADS, 1)
k_gconv_reduce_tc(const __grid_constant__ CUtensorMap tmM, const __grid_constant__ CUtensorMap tmWg,
                  const __grid_constant__ CUtensorMap tmW3, const __grid_constant__ CUtensorMap tmR,
                  const __grid_constant__ CUtensorMap tmO, const GrP p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uintptr_t raw_addr = reinterpret_cast<uintptr_t>(smem_raw);
    asm volatile("" : "+l"(raw_addr));                    // keep shared-memory addresses run-time values (see conv2d_tc.cu)
    uint8_t* smem = reinterpret_cast<uint8_t*>(raw_addr);
    if (smem_u32(smem) & 1023u) __trap();
    const int S = p.stages;
    const int halo_bytes = gr_halo_bytes(p.planes), stage_bytes = gr_stage_bytes(p.planes);
    const uint32_t ring = smem_u32(smem);
    const uint32_t sw3 = ring + (uint32_t)(S * stage_bytes);          // W3 slot, then output staging half 1
    const uint32_t sg = sw3 + GR_W3_SLOT;                               // g chunk, then output staging half 0
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)S * stage_bytes + GR_W3_SLOT + p.planes * GR_TPLANE);
    // bars: ring full[4], ring empty[4], w3 full, w3 empty, residual full, staging ready, staging free
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + GR_MAX_STAGES);
    const uint32_t bar_w3full = smem_u32(bars + 2 * GR_MAX_STAGES), bar_w3empty = bar_w3full + 8;
    const uint32_t bar_res = bar_w3full + 16, bar_stgready = bar_w3full + 24, bar_stgfree = bar_w3full + 32;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < GR_MAX_STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }  // 8 consumer warps
        mbar_init(bar_w3full, 1); mbar_init(bar_w3empty, 8);
        mbar_init(bar_res, 1); mbar_init(bar_stgready, 8); mbar_init(bar_stgfree, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (p.pdl) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }
    const bool split = (p.planes == 2);
    const int CH = p.chunks;

    if (warp < 4) {
        regs_dec<40>();
        if (warp != 0) return;
        // ============================== producer (warp 0; one elected lane issues) ==============================
        // Item j = (work item of this CTA, chunk).  Order: the ring load of item j, then the W3 load of item j - 1 (and, after
        // the last chunk of a tile, its residual, the wait for the consumers' epilogue and the output stores), so the next
        // tile's first halo is in flight while the epilogue runs.
        auto coords = [&](int item, int& nt, int& img, int& h0, int& w0) {
            nt = item % p.n_tiles;
            int t = item / p.n_tiles;
            const int tw_i = t % p.tiles_w; t /= p.tiles_w;
            const int th_i = t % p.tiles_h; img = t / p.tiles_h;
            h0 = th_i * GR_TH; w0 = tw_i * GR_TW;
        };
        auto load_ring = [&](int j, int item, int c) {
            const int st = j % S;
            mbar_wait(bar_empty + 8 * st, (uint32_t)(((j / S) & 1) ^ 1));
            if (elect_one()) {
                int nt, img, h0, w0;
                coords(item, nt, img, h0, w0);
                const uint32_t sa = ring + (uint32_t)(st * stage_bytes), sb = sa + (uint32_t)halo_bytes;
                mbar_expect_tx(bar_full + 8 * st, (uint32_t)(p.planes * GR_HPLANE + GR_WG_CHUNK));
                tma_load_5d(sa, &tmM, bar_full + 8 * st, c * 64, w0 - 1, h0 - 1, img, 0);
                for (int r = 0; r < 3; ++r) tma_load_5d(sb + r * GR_WG_ROW, &tmWg, bar_full + 8 * st, 0, 0, 0, c * 4, r * 3);
            }
            __syncwarp();
        };
        int it = 0;                                       // tiles finished (epilogues stored)
        auto load_w3 = [&](int j, int item, int c) {
            // the slot is free: the reduce of item j - 1 has retired (within a tile), or the previous tile's stores have read it
            if (c > 0) mbar_wait(bar_w3empty, (uint32_t)((j - 1) & 1));
            int nt, img, h0, w0;
            coords(item, nt, img, h0, w0);
            if (elect_one()) {
                mbar_expect_tx(bar_w3full, (uint32_t)GR_W3_SLOT);
                tma_load_3d(sw3, &tmW3, bar_w3full, c * 64, nt * GR_N, 0);
            }
            __syncwarp();
            if (c < CH - 1) return;
            // tail of the work item: both warpgroups' last reduce has retired -> W3 slot and g chunk take the residual
            mbar_wait(bar_w3empty, (uint32_t)(j & 1));
            if (elect_one()) {
                mbar_expect_tx(bar_res, (uint32_t)(2 * p.planes * GR_TPLANE));
                tma_load_5d(sg, &tmR, bar_res, nt * GR_N, w0, h0, img, 0);
                tma_load_5d(sw3, &tmR, bar_res, nt * GR_N + 64, w0, h0, img, 0);
            }
            __syncwarp();
            mbar_wait(bar_stgready, (uint32_t)(it & 1));   // the consumers have written the output tile in place
            if (lane == 0) {                              // out-of-image pixels are clipped by the TMA unit
                tma_store_5d(&tmO, sg, nt * GR_N, w0, h0, img, 0);
                tma_store_5d(&tmO, sw3, nt * GR_N + 64, w0, h0, img, 0);
                bulk_commit();
                bulk_wait_read<0>();
                mbar_arrive(bar_stgfree);
            }
            __syncwarp();
            ++it;
        };
        int j = 0, prev_item = -1, prev_c = 0;
        for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
            for (int c = 0; c < CH; ++c, ++j) {
                load_ring(j, item, c);
                if (prev_item >= 0) load_w3(j - 1, prev_item, prev_c);
                prev_item = item; prev_c = c;
            }
        }
        if (prev_item >= 0) load_w3(j - 1, prev_item, prev_c);
        if (lane == 0) bulk_wait_all();                   // the bulk groups belong to the lane that committed them
        __syncwarp();
        return;
    }
    // ============================== consumers (warpgroups 1 and 2) ==============================
    regs_inc<232>();
    const int wg = (warp >> 2) - 1;
    // accumulator fragment (tc_prims.cuh): rows fq and fq + 8 of the warpgroup's 64, columns 8 j + fcol, +1
    const int ft = threadIdx.x & 127;
    const int fq = 16 * (ft >> 5) + ((ft & 31) >> 2), fcol = 2 * (ft & 3);
    const int frow = 64 * wg + fq;                              // tile pixel (row frow / 8, column frow % 8)
    const int fswz = frow & 7;
    const uint32_t g_row0 = sg + (uint32_t)(frow * 128 + 2 * fcol);       // pixel frow + 8 is 1024 B further
    // The reduce accumulators are zeroed by the first MMA of the chain (scale-d = 0).
    float d[64], dg[16], eg[8], gv[32];
#pragma unroll
    for (int i = 0; i < 16; ++i) dg[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) eg[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    int j = 0, it = 0;
    for (int item = blockIdx.x; item < p.items; item += gridDim.x, ++it) {
        const int nt = item % p.n_tiles;
        for (int c = 0; c < CH; ++c, ++j) {
            const int st = j % S;
            const uint32_t smid = ring + (uint32_t)(st * stage_bytes), swg = smid + (uint32_t)halo_bytes;
            mbar_wait(bar_full + 8 * st, (uint32_t)((j / S) & 1));
            // ---- 1. grouped 3x3: one 16-channel sub-block k at a time, its 9 taps in the ring kernel's order
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                wgmma_fence();
#pragma unroll
                for (int r = 0; r < 3; ++r) {
#pragma unroll
                    for (int s = 0; s < 3; ++s) {
                        const uint32_t ah = smid + (uint32_t)(((8 * wg + r) * GR_HW + s) * 128 + k * 32);
                        const uint64_t bd = gmma_desc_sw32(swg + (uint32_t)(r * GR_WG_ROW + s * 4096 + k * 1024));
                        const uint32_t f0 = (r == 0 && s == 0) ? 0u : 1u;
                        wgmma_bf16<32>(dg, desc_sw128_sbo(ah, GR_MID_SBO), bd, f0);                          // [a_hi*b_hi | a_hi*b_lo]
                        if (split) wgmma_bf16<16>(eg, desc_sw128_sbo(ah + GR_HPLANE, GR_MID_SBO), bd, f0);   // a_lo*b_hi
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
#pragma unroll
                for (int q = 0; q < 8; ++q) gv[8 * k + q] = dg[q] + (split ? dg[8 + q] + eg[q] : dg[8 + q]);   // the ring kernel's fold
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8 * st);
            // the g chunk is free: this warpgroup's reduce of the previous chunk has retired, and at a tile's first chunk the
            // previous tile's output stores have read the region
            if (c == 0 && it > 0) mbar_wait(bar_stgfree, (uint32_t)((it - 1) & 1));
            wg_bar(wg);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b2 + c * 64 + 8 * jj + fcol));
                float v[4] = {gv[4 * jj] + bb.x, gv[4 * jj + 1] + bb.y, gv[4 * jj + 2] + bb.x, gv[4 * jj + 3] + bb.y};
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = fmaxf(v[i], 0.f);
                const uint32_t a0 = g_row0 + (uint32_t)((jj ^ fswz) << 4);
                sts_b32(a0, pack_bf16(v[0], v[1])); sts_b32(a0 + 1024, pack_bf16(v[2], v[3]));
                if (split) {
                    sts_b32(a0 + GR_TPLANE, pack_bf16(bf16_rest(v[0]), bf16_rest(v[1])));
                    sts_b32(a0 + GR_TPLANE + 1024, pack_bf16(bf16_rest(v[2]), bf16_rest(v[3])));
                }
            }
            fence_async_smem();
            wg_bar(wg);
            // ---- 2. reduce: this chunk's 64 K rows of W3, accumulated across the chunks
            mbar_wait(bar_w3full, (uint32_t)(j & 1));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t ah = sg + (uint32_t)(wg * 64 * 128 + k * 32);
                const uint64_t a_hi = gmma_desc_sw128(ah);
                const uint64_t b_hi = gmma_desc_sw128(sw3 + k * 32), b_lo = gmma_desc_sw128(sw3 + GR_N * 128 + k * 32);
                const uint32_t first = (c == 0 && k == 0) ? 0u : 1u;
                wgmma_bf16<128>(d, a_hi, b_lo, first);
                if (split) wgmma_bf16<128>(d, gmma_desc_sw128(ah + GR_TPLANE), b_hi, 1u);
                wgmma_bf16<128>(d, a_hi, b_hi, 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_w3empty);
        }
        // ---- epilogue: bias3, residual (TMA-loaded into the staging halves), ReLU, split, in place
        mbar_wait(bar_res, (uint32_t)(it & 1));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t row0 = (h == 0 ? sg : sw3) + (uint32_t)(frow * 128 + 2 * fcol);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int jd = 8 * h + jj;
                const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b3 + nt * GR_N + 8 * jd + fcol));
                const uint32_t a0 = row0 + (uint32_t)((jj ^ fswz) << 4);
                float v[4] = {d[4 * jd] + bb.x, d[4 * jd + 1] + bb.y, d[4 * jd + 2] + bb.x, d[4 * jd + 3] + bb.y};
                const uint32_t rs[4] = {lds_b32(a0), lds_b32(a0 + 1024), split ? lds_b32(a0 + GR_TPLANE) : 0u,
                                        split ? lds_b32(a0 + GR_TPLANE + 1024) : 0u};
#pragma unroll
                for (int q = 0; q < 2; ++q) { v[2 * q] += bf16_lo_f(rs[q]); v[2 * q + 1] += bf16_hi_f(rs[q]); }
                if (split) {
#pragma unroll
                    for (int q = 0; q < 2; ++q) { v[2 * q] += bf16_lo_f(rs[2 + q]); v[2 * q + 1] += bf16_hi_f(rs[2 + q]); }
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = fmaxf(v[i], 0.f);
                sts_b32(a0, pack_bf16(v[0], v[1])); sts_b32(a0 + 1024, pack_bf16(v[2], v[3]));
                if (split) {
                    sts_b32(a0 + GR_TPLANE, pack_bf16(bf16_rest(v[0]), bf16_rest(v[1])));
                    sts_b32(a0 + GR_TPLANE + 1024, pack_bf16(bf16_rest(v[2]), bf16_rest(v[3])));
                }
            }
        }
        fence_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_stgready);
    }
}

}  // namespace

extern "C" int heal_gconv_reduce_tc(const void* mid, size_t mid_plane_stride, int N, int H, int W, int width, int mid_cstride,
                                    const void* w2_diag, const float* b2, const void* w3, const float* b3, int Cout,
                                    const void* res, size_t res_plane_stride, int res_cstride, int planes, int w_planes,
                                    void* out, size_t out_plane_stride, int out_cstride, int out_coffset, void* stream_) {
    if (!mid || !w2_diag || !b2 || !w3 || !b3 || !res || !out || N < 1 || H < 1 || W < 1) return HEAL_ERR_ARG;
    if (planes != 1 && planes != 2) return HEAL_ERR_ARG;
    if (w_planes != 2 || width < 64 || (width % 64) || Cout < GR_N || (Cout % GR_N)) return HEAL_ERR_UNSUPPORTED;
    if ((mid_cstride & 7) || mid_cstride < width || (res_cstride & 7) || res_cstride < Cout || (out_cstride & 7) ||
        (out_coffset & 7) || out_coffset + Cout > out_cstride) return HEAL_ERR_UNSUPPORTED;
    PFN_tmEncodeTiled enc = get_encode();
    if (!enc) return HEAL_ERR_DRIVER;
    const cuuint32_t P = (cuuint32_t)planes;
    cuuint32_t es[5] = {1, 1, 1, 1, 1};
    CUtensorMap tmM, tmWg, tmW3, tmR, tmO;
    CUresult r;
    // activation maps {C, W, H, N, plane}: the mid halo chunk (18 x 10 pixels), the residual and output halves (16 x 8 pixels)
    auto act_map = [&](CUtensorMap* tm, const void* base, size_t plane_stride, int C, int cstride, cuuint32_t bw, cuuint32_t bh) {
        cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N, (cuuint64_t)planes};
        cuuint64_t st[4] = {(cuuint64_t)cstride * 2, (cuuint64_t)W * cstride * 2, (cuuint64_t)H * W * cstride * 2,
                            (cuuint64_t)plane_stride * 2};
        if (planes == 1) st[3] = st[2] * N;
        cuuint32_t box[5] = {64u, bw, bh, 1u, P};
        return enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), dims, st, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    };
    if ((r = act_map(&tmM, mid, mid_plane_stride, width, mid_cstride, GR_HW, GR_TH + 2)) != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
    if ((r = act_map(&tmR, res, res_plane_stride, Cout, res_cstride, GR_TW, GR_TH)) != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
    if ((r = act_map(&tmO, (const __nv_bfloat16*)out + out_coffset, out_plane_stride, Cout, out_cstride, GR_TW, GR_TH)) != CUDA_SUCCESS)
        return HEAL_ERR_DRIVER;
    {
        // W3: [plane][Cout rows][width] -> per (64-channel K block, 128-row output block), smem [plane][128 rows][128 B]
        cuuint64_t d3[3] = {(cuuint64_t)width, (cuuint64_t)Cout, 2};
        cuuint64_t s3[2] = {(cuuint64_t)width * 2, (cuuint64_t)Cout * width * 2};
        cuuint32_t bx3[3] = {64u, (cuuint32_t)GR_N, 2u};
        r = enc(&tmW3, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(w3), d3, s3, bx3, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
        // grouped 3x3 diagonal sub-blocks: [plane][9 taps * width rows][16] -> per kernel row, smem [3 taps][4 sub-blocks][plane][16][32 B]
        // (the map of the ring kernel)
        cuuint64_t dg[5] = {16, 16, 2, (cuuint64_t)width / 16, 9};
        cuuint64_t sg[4] = {32, (cuuint64_t)9 * width * 32, 512, (cuuint64_t)width * 32};
        cuuint32_t bxg[5] = {16u, 16u, 2u, 4u, 3u};
        r = enc(&tmWg, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(w2_diag), dg, sg, bxg, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
    }
    GrP p;
    p.N = N; p.H = H; p.W = W;
    p.tiles_w = (W + GR_TW - 1) / GR_TW; p.tiles_h = (H + GR_TH - 1) / GR_TH;
    p.n_tiles = Cout / GR_N;
    p.items = N * p.tiles_h * p.tiles_w * p.n_tiles;
    p.chunks = width / 64;
    p.planes = planes; p.pdl = 1;
    p.stages = gr_stages(planes);
    p.b2 = b2; p.b3 = b3;
    if (p.stages < 2) return HEAL_ERR_UNSUPPORTED;
    const size_t smem = (size_t)p.stages * gr_stage_bytes(planes) + gr_fixed_bytes(planes);
    static size_t attr_set[HEAL_MAX_DEVICES] = {};
    if (!heal_ensure_dyn_smem(k_gconv_reduce_tc, GR_SMEM_LIMIT, attr_set)) return HEAL_ERR_LAUNCH;
    const int grid = p.items < HEAL_NUM_SMS ? p.items : HEAL_NUM_SMS;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(GR_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream_;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, k_gconv_reduce_tc, tmM, tmWg, tmW3, tmR, tmO, p);
    heal_launch_counter_add(1);
    return e == cudaSuccess ? HEAL_OK : HEAL_ERR_LAUNCH;
}
