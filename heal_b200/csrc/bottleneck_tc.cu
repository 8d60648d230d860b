// The stride-1 ResNeXt bottleneck of PyramidFusion's level 0 (resblock.py: Bottleneck with inplanes = planes = 64, width 128,
// 32 groups, no downsample) as ONE persistent wgmma kernel:
//   y = ReLU(W3 * ReLU(Wg (*) ReLU(W1 * x + b1) + b2) + b3 + x)
// The expanded (2x wide) maps never leave shared memory: the three-launch path writes and reads them back through HBM twice.
//
// A CTA tile is 16 x 8 output pixels of one image.  Its 18 x 10 halo of x is ONE 5-D TMA box (zero-filled outside the image);
// all weights of the block (136 KiB with both weight planes) are loaded once per persistent CTA.  For each 64-channel chunk of
// the width:
//   1. expand: the 1x1 conv over the 180 halo pixels (M = 3 x 64 rows, the last 12 discarded), bias + ReLU + hi/lo split into
//      the swizzled mid chunk [plane][180 pixels][128 B].  Mid pixels outside the image are written as 0: the grouped conv
//      zero-pads the MID map, and ReLU(b1) is not 0.
//   2. grouped 3x3: the 16-channel sub-block MMAs of k_gconv3x3_ring on the packed diagonal weights.  The 64 A rows of one
//      warpgroup are 8 output rows of 8 pixels: for tap (r, s) they start at halo pixel (8 wg + r) * 10 + s and every 8-row
//      group is one halo row (10 pixels = 1280 B) further, which is the descriptor's stride byte offset (the 128B swizzle is
//      a function of the absolute shared-memory address, so any 128 B-aligned row start is addressable).  Bias + ReLU + split
//      into the g chunk [plane][128 pixels][128 B], which takes the mid chunk's place once both warpgroups have read it.
//   3. reduce: g chunk x the chunk's K rows of W3 into accumulators that stay in registers across the chunks.
// After the last chunk: bias3, the residual (the interior of the resident x tile), ReLU, split, TMA tensor store through a
// staging tile in the same region.
//
// Every stage keeps the MMA form, K order and fold of the kernel the three-launch path runs for that shape, so the result is
// bit-identical to it: the expand is k_conv2d_tc<128>'s three-MMA form (a_hi*b_lo, a_lo*b_hi, a_hi*b_hi) issued at N = 64,
// the grouped conv k_gconv3x3_ring's, the reduce k_conv2d_tc<64>'s N-concatenated a_hi x [b_hi | b_lo] + a_lo x b_hi with
// its final fold.  The mid and g chunks are rounded to split-bf16 (or bf16) exactly as those kernels store them.
// Two warpgroups (256 threads), each the M = 64 MMAs of one half of the tile; thread 0 issues the TMA loads and stores.  No
// producer warpgroup: the reduce accumulators (96 registers) stay live while the grouped conv runs, which the 168 registers
// per thread of a 384-thread block cannot hold without spills.
#include <cuda.h>
#include "common.cuh"
#include "tc_prims.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int BT_THREADS = 256;                       // two warpgroups
constexpr int BT_TH = 16, BT_TW = 8;                        // output tile: 16 rows x 8 pixels = the MMA's 128 rows
constexpr int BT_HW = BT_TW + 2;                            // halo tile: 18 rows x 10 pixels
constexpr int BT_HALO = (BT_TH + 2) * BT_HW;                // 180 pixels
constexpr int BT_HPLANE = BT_HALO * 128;                    // one plane of a halo tile: 180 pixels x 64 channels bf16
constexpr int BT_TPLANE = 128 * 128;                        // one plane of a 128-pixel tile
constexpr int BT_C = 64, BT_WIDTH = 128, BT_CHUNKS = BT_WIDTH / 64;
// weights, both planes (hi, lo) resident for the CTA's lifetime
constexpr int BT_W1_BYTES = 2 * BT_WIDTH * 128;             // [plane][128 rows][64 K]
constexpr int BT_W3_CHUNK = 2 * BT_C * 128;                 // [plane][64 rows][64 K] per 64-channel K block
constexpr int BT_WG_ROW = 3 * 4 * 2 * 512;                  // one kernel row: [3 taps][4 sub-blocks][plane][16 rows][32 B]
constexpr int BT_WG_CHUNK = 3 * BT_WG_ROW;
constexpr int BT_W_BYTES = BT_W1_BYTES + BT_CHUNKS * BT_W3_CHUNK + BT_CHUNKS * BT_WG_CHUNK;
constexpr uint32_t BT_MID_SBO = BT_HW * 128;                // one halo row

__host__ __device__ inline int bt_halo_bytes(int planes) { return (planes * BT_HPLANE + 1023) & ~1023; }
__host__ inline size_t bt_smem_bytes(int planes) { return (size_t)BT_W_BYTES + 2 * (size_t)bt_halo_bytes(planes) + 64; }

struct BtP {
    int N, H, W;
    int tiles_w, tiles_h, tiles;
    int planes;                   // activation planes: 2 = split-bf16, 1 = bf16 (the weights always carry both planes)
    int pdl;
    const float *b1, *b2, *b3;
};

// 128B-swizzled K-major descriptor with an explicit stride byte offset (distance between 8-row groups)
__device__ __forceinline__ uint64_t desc_sw128_sbo(uint32_t saddr, uint32_t sbo) {
    return (gmma_desc_sw128(saddr) & ~(0x3FFFull << 32)) | ((uint64_t)(sbo >> 4) << 32);
}
// 16-byte chunk j of the 128 B row at saddr (128 B aligned), 128B-swizzled by the absolute address
__device__ __forceinline__ uint32_t sw_slot(uint32_t saddr, int j) { return saddr + (uint32_t)((j ^ ((saddr >> 7) & 7)) << 4); }

__global__ void __launch_bounds__(BT_THREADS, 1)
k_bottleneck_tc(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
                const __grid_constant__ CUtensorMap tmWg, const __grid_constant__ CUtensorMap tmW3,
                const __grid_constant__ CUtensorMap tmO, const BtP p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uintptr_t raw_addr = reinterpret_cast<uintptr_t>(smem_raw);
    asm volatile("" : "+l"(raw_addr));                    // keep shared-memory addresses run-time values (see conv2d_tc.cu)
    uint8_t* smem = reinterpret_cast<uint8_t*>(raw_addr);
    if (smem_u32(smem) & 1023u) __trap();
    const int halo_bytes = bt_halo_bytes(p.planes);
    const uint32_t sw1 = smem_u32(smem);
    const uint32_t sw3 = sw1 + BT_W1_BYTES;                       // [chunk][plane][64 rows][128 B]
    const uint32_t swg = sw3 + BT_CHUNKS * BT_W3_CHUNK;           // [chunk][3 kernel rows][...]
    const uint32_t sx = swg + BT_CHUNKS * BT_WG_CHUNK;            // x halo tile [plane][180][128 B]
    const uint32_t smid = sx + (uint32_t)halo_bytes;              // mid chunk [plane][180][128 B], then g chunk / output staging [plane][128][128 B]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + BT_W_BYTES + 2 * halo_bytes);
    const uint32_t bar_w = smem_u32(bars), bar_xfull = smem_u32(bars + 1);

    const int warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        mbar_init(bar_w, 1); mbar_init(bar_xfull, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (p.pdl) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }
    const bool split = (p.planes == 2);

    // thread 0 issues the TMA loads: the weights once, each x halo tile when the previous one has been consumed
    auto load_x = [&](int tile) {
        const int tw_i = tile % p.tiles_w, t2 = tile / p.tiles_w;
        const int th_i = t2 % p.tiles_h, img = t2 / p.tiles_h;
        mbar_expect_tx(bar_xfull, (uint32_t)(p.planes * BT_HPLANE));
        tma_load_5d(sx, &tmX, bar_xfull, 0, tw_i * BT_TW - 1, th_i * BT_TH - 1, img, 0);
    };
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar_w, (uint32_t)BT_W_BYTES);
        tma_load_3d(sw1, &tmW1, bar_w, 0, 0, 0);
        for (int c = 0; c < BT_CHUNKS; ++c) {
            tma_load_3d(sw3 + c * BT_W3_CHUNK, &tmW3, bar_w, c * 64, 0, 0);
            for (int r = 0; r < 3; ++r) tma_load_5d(swg + c * BT_WG_CHUNK + r * BT_WG_ROW, &tmWg, bar_w, 0, 0, 0, c * 4, r * 3);
        }
        if ((int)blockIdx.x < p.tiles) load_x(blockIdx.x);
    }
    const int wg = warp >> 2;
    // accumulator fragment (tc_prims.cuh): rows fq and fq + 8 of the warpgroup's 64, columns 8 j + fcol, +1
    const int ft = threadIdx.x & 127;
    const int fq = 16 * (ft >> 5) + ((ft & 31) >> 2), fcol = 2 * (ft & 3);
    const int frow = 64 * wg + fq;                                // tile pixel (row frow / 8, column frow % 8)
    const bool is_store = (threadIdx.x == 0);
    // The expand and reduce accumulators are zeroed right before the MMA chain that overwrites them (its first MMA has
    // scale-d = 0), so the compiler sees the old values as dead and the two share registers with the grouped ones.
    float xd[32], rd[64], re[32], dg[16], eg[8];
#pragma unroll
    for (int i = 0; i < 16; ++i) dg[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) eg[i] = 0.f;
    mbar_wait(bar_w, 0);
    int it = 0;
    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x, ++it) {
        const int tw_i = tile % p.tiles_w, t2 = tile / p.tiles_w;
        const int th_i = t2 % p.tiles_h, img = t2 / p.tiles_h;
        const int h0 = th_i * BT_TH, w0 = tw_i * BT_TW;
        mbar_wait(bar_xfull, (uint32_t)(it & 1));
#pragma unroll
        for (int i = 0; i < 32; ++i) re[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 64; ++i) rd[i] = 0.f;
        for (int c = 0; c < BT_CHUNKS; ++c) {
            // ---- 1. expand: M blocks mb of the 180-row halo tile, alternating between the warpgroups from chunk to chunk
            bool first = true;
            for (int mb = (wg + c) & 1; mb < 3; mb += 2) {
#pragma unroll
                for (int i = 0; i < 32; ++i) xd[i] = 0.f;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint32_t ah = sx + (uint32_t)(mb * 64 * 128 + k * 32);
                    const uint64_t a_hi = gmma_desc_sw128(ah);
                    const uint64_t b_hi = gmma_desc_sw128(sw1 + c * 64 * 128 + k * 32);
                    const uint64_t b_lo = gmma_desc_sw128(sw1 + BT_WIDTH * 128 + c * 64 * 128 + k * 32);
                    wgmma_bf16<64>(xd, a_hi, b_lo, k == 0 ? 0u : 1u);
                    if (split) wgmma_bf16<64>(xd, gmma_desc_sw128(ah + BT_HPLANE), b_hi, 1u);
                    wgmma_bf16<64>(xd, a_hi, b_hi, 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                if (first) {
                    // the region is free: both warpgroups' reduce MMAs of the previous chunk have retired, and the previous
                    // tile's output store has been read out
                    if (is_store) bulk_wait_read<0>();
                    epi_bar(1);
                    first = false;
                }
                bool live[2], inimg[2]; uint32_t qa[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int q = mb * 64 + fq + 8 * h;
                    const int gh = h0 - 1 + q / BT_HW, gw = w0 - 1 + q % BT_HW;
                    live[h] = q < BT_HALO;                                     // rows 180..191 of the last block are padding
                    inimg[h] = gh >= 0 && gh < p.H && gw >= 0 && gw < p.W;
                    qa[h] = smid + (uint32_t)(q * 128);
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b1 + c * 64 + 8 * j + fcol));
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (!live[h]) continue;
                        float v0 = fmaxf(xd[4 * j + 2 * h] + bb.x, 0.f), v1 = fmaxf(xd[4 * j + 2 * h + 1] + bb.y, 0.f);
                        if (!inimg[h]) { v0 = 0.f; v1 = 0.f; }
                        sts_b32(sw_slot(qa[h], j) + 2 * fcol, pack_bf16(v0, v1));
                        if (split) sts_b32(sw_slot(qa[h] + BT_HPLANE, j) + 2 * fcol, pack_bf16(bf16_rest(v0), bf16_rest(v1)));
                    }
                }
            }
            fence_async_smem();
            epi_bar(2);
            // ---- 2. grouped 3x3 on the mid chunk: output rows [8 wg, 8 wg + 8) of the tile.  One 16-channel sub-block k at a time
            // (its 9 taps in the ring kernel's order), folded into gv when its MMAs retire: 24 accumulator registers instead of
            // the ring kernel's 96, which the reduce accumulators leave no room for (two sub-blocks in flight in alternating
            // register sets make ptxas serialise the chain, C7511).  The per-column arithmetic is the ring kernel's.
            float gv[32];
            auto grouped_issue = [&](int k, float* dk, float* ek) {
                wgmma_fence();
#pragma unroll
                for (int r = 0; r < 3; ++r) {
#pragma unroll
                    for (int s = 0; s < 3; ++s) {
                        const uint32_t ah = smid + (uint32_t)(((8 * wg + r) * BT_HW + s) * 128 + k * 32);
                        const uint64_t bd = gmma_desc_sw32(swg + (uint32_t)(c * BT_WG_CHUNK + r * BT_WG_ROW + s * 4096 + k * 1024));
                        const uint32_t f0 = (r == 0 && s == 0) ? 0u : 1u;
                        wgmma_bf16<32>(dk, desc_sw128_sbo(ah, BT_MID_SBO), bd, f0);                         // [a_hi*b_hi | a_hi*b_lo]
                        if (split) wgmma_bf16<16>(ek, desc_sw128_sbo(ah + BT_HPLANE, BT_MID_SBO), bd, f0);  // a_lo*b_hi
                    }
                }
                wgmma_commit();
            };
            auto grouped_fold = [&](int k, const float* dk, const float* ek) {   // the fold of k_gconv3x3_ring
#pragma unroll
                for (int q = 0; q < 8; ++q) gv[8 * k + q] = dk[q] + (split ? dk[8 + q] + ek[q] : dk[8 + q]);
            };
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                grouped_issue(k, dg, eg);
                wgmma_wait<0>();
                grouped_fold(k, dg, eg);
            }
            epi_bar(3);                                           // both warpgroups are done with the mid chunk
            {
                const uint32_t row0 = smid + (uint32_t)(frow * 128 + 2 * fcol);     // pixel frow + 8 is 1024 B further
                const int fswz = frow & 7;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b2 + c * 64 + 8 * j + fcol));
                    float v[4] = {gv[4 * j] + bb.x, gv[4 * j + 1] + bb.y, gv[4 * j + 2] + bb.x, gv[4 * j + 3] + bb.y};
#pragma unroll
                    for (int i = 0; i < 4; ++i) v[i] = fmaxf(v[i], 0.f);
                    const uint32_t a0 = row0 + (uint32_t)((j ^ fswz) << 4);
                    sts_b32(a0, pack_bf16(v[0], v[1])); sts_b32(a0 + 1024, pack_bf16(v[2], v[3]));
                    if (split) {
                        sts_b32(a0 + BT_TPLANE, pack_bf16(bf16_rest(v[0]), bf16_rest(v[1])));
                        sts_b32(a0 + BT_TPLANE + 1024, pack_bf16(bf16_rest(v[2]), bf16_rest(v[3])));
                    }
                }
            }
            fence_async_smem();
            epi_bar(4);
            // ---- 3. reduce: this chunk's 64 K rows of W3, accumulated across the chunks
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t ah = smid + (uint32_t)(wg * 64 * 128 + k * 32);
                const uint64_t b = gmma_desc_sw128(sw3 + c * BT_W3_CHUNK + k * 32);
                const uint32_t f = (c == 0 && k == 0) ? 0u : 1u;
                wgmma_bf16<128>(rd, gmma_desc_sw128(ah), b, f);                          // [a_hi*b_hi | a_hi*b_lo]
                if (split) wgmma_bf16<64>(re, gmma_desc_sw128(ah + BT_TPLANE), b, f);    // a_lo*b_hi
            }
            wgmma_commit();
            wgmma_wait<0>();
        }
        // ---- epilogue: fold, bias3, residual (x at the tile's interior), ReLU
        float y[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) y[i] = rd[i] + (split ? rd[i + 32] + re[i] : rd[i + 32]);
        uint32_t xa[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int px = frow + 8 * h;
            xa[h] = sx + (uint32_t)((((px >> 3) + 1) * BT_HW + (px & 7) + 1) * 128);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b3 + 8 * j + fcol));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float v0 = y[4 * j + 2 * h] + bb.x, v1 = y[4 * j + 2 * h + 1] + bb.y;
                const uint32_t rh = lds_b32(sw_slot(xa[h], j) + 2 * fcol);
                v0 += bf16_lo_f(rh); v1 += bf16_hi_f(rh);
                if (split) {
                    const uint32_t rl = lds_b32(sw_slot(xa[h] + BT_HPLANE, j) + 2 * fcol);
                    v0 += bf16_lo_f(rl); v1 += bf16_hi_f(rl);
                }
                y[4 * j + 2 * h] = fmaxf(v0, 0.f); y[4 * j + 2 * h + 1] = fmaxf(v1, 0.f);
            }
        }
        epi_bar(5);                       // both warpgroups are done with the x tile and their reduce MMAs have read the g chunk
        if (is_store && tile + (int)gridDim.x < p.tiles) load_x(tile + (int)gridDim.x);
        {
            const uint32_t row0 = smid + (uint32_t)(frow * 128 + 2 * fcol);
            const int fswz = frow & 7;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint32_t a0 = row0 + (uint32_t)((j ^ fswz) << 4);
                sts_b32(a0, pack_bf16(y[4 * j], y[4 * j + 1])); sts_b32(a0 + 1024, pack_bf16(y[4 * j + 2], y[4 * j + 3]));
                if (split) {
                    sts_b32(a0 + BT_TPLANE, pack_bf16(bf16_rest(y[4 * j]), bf16_rest(y[4 * j + 1])));
                    sts_b32(a0 + BT_TPLANE + 1024, pack_bf16(bf16_rest(y[4 * j + 2]), bf16_rest(y[4 * j + 3])));
                }
            }
        }
        fence_async_smem();
        epi_bar(6);
        if (is_store) {                                           // out-of-image pixels are clipped by the TMA unit
            tma_store_5d(&tmO, smid, 0, w0, h0, img, 0);
            bulk_commit();
        }
    }
    if (is_store) bulk_wait_all();
}

}  // namespace

extern "C" int heal_bottleneck_tc(const void* x, size_t x_plane_stride, int N, int H, int W, int C, int x_cstride,
                                  const void* w1, const float* b1, const void* w2_diag, const float* b2, const void* w3,
                                  const float* b3, int planes, int w_planes, void* out, size_t out_plane_stride, int out_cstride,
                                  int out_coffset, void* stream_) {
    if (!x || !w1 || !b1 || !w2_diag || !b2 || !w3 || !b3 || !out || N < 1 || H < 1 || W < 1) return HEAL_ERR_ARG;
    if (planes != 1 && planes != 2) return HEAL_ERR_ARG;
    if (C != BT_C || w_planes != 2) return HEAL_ERR_UNSUPPORTED;
    if ((x_cstride & 7) || x_cstride < C || (out_cstride & 7) || (out_coffset & 7) || out_coffset + C > out_cstride) return HEAL_ERR_UNSUPPORTED;
    PFN_tmEncodeTiled enc = get_encode();
    if (!enc) return HEAL_ERR_DRIVER;
    const cuuint32_t P = (cuuint32_t)planes;
    CUtensorMap tmX, tmW1, tmWg, tmW3, tmO;
    CUresult r;
    {
        cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N, (cuuint64_t)planes};
        cuuint64_t st[4] = {(cuuint64_t)x_cstride * 2, (cuuint64_t)W * x_cstride * 2, (cuuint64_t)H * W * x_cstride * 2,
                            (cuuint64_t)x_plane_stride * 2};
        if (planes == 1) st[3] = st[2] * N;
        cuuint32_t box[5] = {64u, (cuuint32_t)BT_HW, (cuuint32_t)(BT_TH + 2), 1u, P};
        cuuint32_t es[5] = {1, 1, 1, 1, 1};
        r = enc(&tmX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(x), dims, st, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
    }
    {
        cuuint64_t st[4] = {(cuuint64_t)out_cstride * 2, (cuuint64_t)W * out_cstride * 2, (cuuint64_t)H * W * out_cstride * 2,
                            (cuuint64_t)out_plane_stride * 2};
        if (planes == 1) st[3] = st[2] * N;
        cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N, (cuuint64_t)planes};
        cuuint32_t box[5] = {64u, (cuuint32_t)BT_TW, (cuuint32_t)BT_TH, 1u, P};
        cuuint32_t es[5] = {1, 1, 1, 1, 1};
        r = enc(&tmO, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)((__nv_bfloat16*)out + out_coffset), dims, st, box, es,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
    }
    {
        cuuint32_t es[5] = {1, 1, 1, 1, 1};
        // W1: [plane][width rows][C] -> smem [plane][width rows][128 B]
        cuuint64_t d1[3] = {(cuuint64_t)C, (cuuint64_t)BT_WIDTH, 2};
        cuuint64_t s1[2] = {(cuuint64_t)C * 2, (cuuint64_t)BT_WIDTH * C * 2};
        cuuint32_t bx1[3] = {64u, (cuuint32_t)BT_WIDTH, 2u};
        r = enc(&tmW1, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(w1), d1, s1, bx1, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
        // W3: [plane][C rows][width] -> per 64-channel K block, smem [plane][C rows][128 B]
        cuuint64_t d3[3] = {(cuuint64_t)BT_WIDTH, (cuuint64_t)C, 2};
        cuuint64_t s3[2] = {(cuuint64_t)BT_WIDTH * 2, (cuuint64_t)C * BT_WIDTH * 2};
        cuuint32_t bx3[3] = {64u, (cuuint32_t)C, 2u};
        r = enc(&tmW3, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(w3), d3, s3, bx3, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
        // grouped 3x3 diagonal sub-blocks: [plane][9 taps * width rows][16] -> per kernel row, smem [3 taps][4 sub-blocks][plane][16][32 B]
        // (the map of the ring kernel)
        cuuint64_t dg[5] = {16, 16, 2, (cuuint64_t)BT_WIDTH / 16, 9};
        cuuint64_t sg[4] = {32, (cuuint64_t)9 * BT_WIDTH * 32, 512, (cuuint64_t)BT_WIDTH * 32};
        cuuint32_t bxg[5] = {16u, 16u, 2u, 4u, 3u};
        r = enc(&tmWg, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(w2_diag), dg, sg, bxg, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
    }
    BtP p;
    p.N = N; p.H = H; p.W = W;
    p.tiles_w = (W + BT_TW - 1) / BT_TW; p.tiles_h = (H + BT_TH - 1) / BT_TH;
    p.tiles = N * p.tiles_h * p.tiles_w;
    p.planes = planes; p.pdl = 1;
    p.b1 = b1; p.b2 = b2; p.b3 = b3;
    const size_t smem = bt_smem_bytes(planes);
    if (smem > 227 * 1024) return HEAL_ERR_UNSUPPORTED;
    static size_t attr_set[HEAL_MAX_DEVICES] = {};
    if (!heal_ensure_dyn_smem(k_bottleneck_tc, 227 * 1024, attr_set)) return HEAL_ERR_LAUNCH;
    const int grid = p.tiles < HEAL_NUM_SMS ? p.tiles : HEAL_NUM_SMS;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(BT_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream_;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, k_bottleneck_tc, tmX, tmW1, tmWg, tmW3, tmO, p);
    heal_launch_counter_add(1);
    return e == cudaSuccess ? HEAL_OK : HEAL_ERR_LAUNCH;
}
