// Grouped 3x3 convolution (stride 1, pad 1; the ResNeXt bottleneck conv2, resblock.py:102-122 with groups = 32) as a ROW RING
// on the Hopper tensor cores (wgmma): every input row is fetched from L2 ONCE and the weights ONCE per CTA.
//
// Why: the tile-per-CTA kernel (k_conv2d_tc<64,*,1>, halo mode) pulls each 130-pixel input row through the L2->SM crossbar
// three times (once per kernel row) and the 36 KB of packed weights once per 128-pixel tile -- about 4x the input size at the
// 256x256 level -- with only a few 45 KB stages in flight, and was bound by that latency rather than by MMA issue (profiled on
// the B200 build; not re-profiled on the H100).
//
// Here a CTA owns a vertical strip: (image, 128-pixel column tile, 64-channel block) x a range of rows.  Shared memory holds
//   * a ring of R input rows, each [plane][130 pixels][64 channels] bf16 as written by one 5-D TMA box (128B swizzle; rows
//     outside the image are zero-filled by the TMA unit = the convolution padding),
//   * the 9 x 4 packed 16x16 diagonal weight sub-blocks of the channel block (hi and lo planes), loaded once,
//   * one output staging tile for the TMA store.
// Output row h needs ring rows h-1, h, h+1: the three horizontal taps are row-shifted descriptors of the same ring row (the
// swizzle is a function of the absolute shared-memory address), so one new row per output row is all that is loaded.
// Precision and MMA forms are those of conv2d_tc.cu: a_hi x [b_hi | b_lo] as one N = 32 MMA plus a_lo x b_hi as an N = 16 MMA
// into separate registers per 16-channel sub-block and tap, fp32 accumulation in registers, folded in the same order.  Roles:
// warpgroup 0 = TMA producer (warp 0); warpgroups 1 and 2 = the M = 64 wgmma of one half of the row tile each, then the
// epilogue of their half straight from the accumulator fragment (bias, ReLU, hi/lo split into the swizzled staging tile), one
// TMA tensor store per row.
#include <cuda.h>
#include "common.cuh"
#include "tc_prims.cuh"
#include "conv_ring.cuh"

namespace {

constexpr int RG_THREADS = 384;
constexpr int RG_TW = 128;                          // output pixels per row tile = MMA M
constexpr int RG_ROW_PLANE = (RG_TW + 2) * 128;     // one plane of one ring row: 130 pixels x 64 channels bf16
constexpr int RG_STG_PLANE = RG_TW * 128;           // one plane of the output staging tile
constexpr int RG_MAX_SLOTS = 8;
constexpr int RG_SMEM_LIMIT = 227 * 1024;

__host__ __device__ inline int rg_slot_bytes(int planes) { return (planes * RG_ROW_PLANE + 1023) & ~1023; }
__host__ __device__ inline int rg_wrow_bytes(int wplanes) { return 3 * 4 * wplanes * 512; }   // one kernel row: [3 taps][4 sub-blocks][plane][16][32 B]
// output staging tile
__host__ __device__ inline int rg_stg_bytes(int planes) { return planes * RG_STG_PLANE; }

__global__ void __launch_bounds__(RG_THREADS, 1)
k_gconv3x3_ring(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmO, const RingP p, const int slots) {
    // strip / segment of this CTA
    const int CB = p.C / 64, WT = p.W / RG_TW;
    const int seg = blockIdx.x % p.segs;
    int strip = blockIdx.x / p.segs;
    const int cb = strip % CB; strip /= CB;
    const int wt = strip % WT; const int img = strip / WT;
    const int h_begin = seg * p.seg_rows;
    const int rows = min(p.seg_rows, p.H - h_begin);
    if (rows <= 0) return;
    const int w0 = wt * RG_TW;

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uintptr_t raw_addr = reinterpret_cast<uintptr_t>(smem_raw);
    asm volatile("" : "+l"(raw_addr));                    // keep shared-memory addresses run-time values (see conv2d_tc.cu)
    uint8_t* smem = reinterpret_cast<uint8_t*>(raw_addr);
    if (smem_u32(smem) & 1023u) __trap();
    const int slot_bytes = rg_slot_bytes(p.planes);
    const int wrow_bytes = rg_wrow_bytes(p.wplanes);
    const int stg_bytes = rg_stg_bytes(p.planes);
    const uint32_t ring = smem_u32(smem);
    const uint32_t wbase = ring + (uint32_t)(slots * slot_bytes);
    const uint32_t stg = wbase + (uint32_t)(3 * wrow_bytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)slots * slot_bytes + 3 * wrow_bytes + stg_bytes);
    // bars: full[8], empty[8], wfull
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + RG_MAX_SLOTS), bar_w = smem_u32(bars + 2 * RG_MAX_SLOTS);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < RG_MAX_SLOTS; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }   // 8 consumer warps
        mbar_init(bar_w, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const bool split = (p.planes == 2), wsplit = (p.wplanes == 2);
    // programmatic dependent launch: the barrier init above overlapped the previous kernel's tail; nothing it produced has
    // been touched yet
    if (p.pdl) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }

    if (warp < 4) {
        regs_dec<40>();
        // ============================== TMA producer (warp 0) =====================
        if (warp == 0) {
            if (elect_one()) {
                mbar_expect_tx(bar_w, (uint32_t)(3 * wrow_bytes));
                for (int r = 0; r < 3; ++r) tma_load_5d(wbase + r * wrow_bytes, &tmB, bar_w, 0, 0, 0, cb * 4, r * 3);
            }
            __syncwarp();
            const int n_in = rows + 2;                       // input rows h_begin-1 .. h_begin+rows
            for (int j = 0; j < n_in; ++j) {
                const int slot = j % slots, use = j / slots;
                mbar_wait(bar_empty + 8 * slot, (uint32_t)((use & 1) ^ 1));
                if (elect_one()) {
                    mbar_expect_tx(bar_full + 8 * slot, (uint32_t)(p.planes * RG_ROW_PLANE));
                    tma_load_5d(ring + slot * slot_bytes, &tmA, bar_full + 8 * slot, cb * 64, w0 - 1, h_begin - 1 + j, img, 0);
                }
                __syncwarp();
            }
        }
    } else {
        // ============================== consumers: wgmma + epilogue ===============
        regs_inc<232>();
        const int wg = (warp >> 2) - 1;                 // MMAs: pixels [64 wg, 64 wg + 64) of the row tile
        // accumulator fragment of this thread (tc_prims.cuh): pixels frow and frow + 8, channels 8 j + fcol, +1 of every 8-channel
        // group j; both pixels have the 128B-swizzle phase fswz in the staging tile
        const int ft = threadIdx.x & 127;
        const int frow = 64 * wg + 16 * (ft >> 5) + ((ft & 31) >> 2), fcol = 2 * (ft & 3);
        const int fswz = (ft >> 2) & 7;
        const uint32_t row0 = stg + (uint32_t)(frow * 128 + 2 * fcol);      // pixel frow + 8 is 1024 B further
        float2 bv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
            bv[j] = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + cb * 64 + 8 * j + fcol)) : make_float2(0.f, 0.f);
        const uint32_t tap_bytes = (uint32_t)(4 * p.wplanes * 512), sub_bytes = (uint32_t)(p.wplanes * 512);
        float d[64], e[32];                              // e: a_lo*b_hi (or a_hi*b_hi with one weight plane) in registers of its own
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) e[i] = 0.f;
        mbar_wait(bar_w, 0);
        int waited = 0;
        for (int t = 0; t < rows; ++t) {
            while (waited < t + 3) { mbar_wait(bar_full + 8 * (waited % slots), (uint32_t)((waited / slots) & 1)); ++waited; }
            wgmma_fence();
            for (int r = 0; r < 3; ++r) {
                const uint32_t sa = ring + (uint32_t)(((t + r) % slots) * slot_bytes) + (uint32_t)(wg * 64 * 128);
#pragma unroll
                for (int s = 0; s < 3; ++s) {
                    const uint32_t ah = sa + s * 128, al = ah + RG_ROW_PLANE;      // tap s = rows [s, s+128) of the 130-row tile
                    const uint32_t bs = wbase + r * wrow_bytes + s * tap_bytes;
                    const uint32_t f0 = (r == 0 && s == 0) ? 0u : 1u;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const uint64_t a_hi = gmma_desc_sw128(ah + k * 32);
                        const uint64_t bd = gmma_desc_sw32(bs + k * sub_bytes);
                        if (wsplit) {
                            wgmma_bf16<32>(d + 16 * k, a_hi, bd, f0);                                    // [a_hi*b_hi | a_hi*b_lo]
                            if (split) wgmma_bf16<16>(e + 8 * k, gmma_desc_sw128(al + k * 32), bd, f0);  // a_lo*b_hi
                        } else {
                            wgmma_bf16<16>(e + 8 * k, a_hi, bd, f0);     // e: every MMA on a register array has one shape
                        }
                    }
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8 * (t % slots));    // input row h-1 is not needed by any later output row
            if (wsplit) {          // [main16 | aux16] per sub-block + a_lo*b_hi -> 64 logical columns (the fold of k_conv2d_tc)
#pragma unroll
                for (int k = 0; k < 4; ++k)
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                        d[8 * k + q] = d[16 * k + q] + (split ? d[16 * k + 8 + q] + e[8 * k + q] : d[16 * k + 8 + q]);
            } else {
#pragma unroll
                for (int i = 0; i < 32; ++i) d[i] = e[i];
            }
            // the previous row's TMA store has finished reading the staging tile
            if (warp == 4 && lane == 0) bulk_wait_read<0>();
            epi_bar(1);
            // bias, ReLU, hi/lo split straight from the fragment into its swizzled slots of the staging tile
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float v[4] = {d[4 * j] + bv[j].x, d[4 * j + 1] + bv[j].y, d[4 * j + 2] + bv[j].x, d[4 * j + 3] + bv[j].y};
                if (p.relu) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) v[i] = fmaxf(v[i], 0.f);
                }
                const uint32_t a0 = row0 + (uint32_t)((j ^ fswz) << 4);
                sts_b32(a0, pack_bf16(v[0], v[1])); sts_b32(a0 + 1024, pack_bf16(v[2], v[3]));
                if (split) {
                    sts_b32(a0 + RG_STG_PLANE, pack_bf16(bf16_rest(v[0]), bf16_rest(v[1])));
                    sts_b32(a0 + RG_STG_PLANE + 1024, pack_bf16(bf16_rest(v[2]), bf16_rest(v[3])));
                }
            }
            fence_async_smem();
            epi_bar(2);
            if (warp == 4 && lane == 0) {
                tma_store_5d(&tmO, stg, cb * 64, w0, h_begin + t, img, 0);
                bulk_commit();
            }
        }
        if (warp == 4 && lane == 0) bulk_wait_all();     // the last tile has left shared memory
    }
}

}  // namespace

int heal_conv3x3_ring_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, RingP p, cudaStream_t st) {
    if ((p.W % RG_TW) || (p.C % 64) || p.N < 1 || p.H < 1) return HEAL_ERR_UNSUPPORTED;
    const int slot_bytes = rg_slot_bytes(p.planes), w_bytes = 3 * rg_wrow_bytes(p.wplanes), stg_bytes = rg_stg_bytes(p.planes);
    int slots = (RG_SMEM_LIMIT - w_bytes - stg_bytes - 512) / slot_bytes;
    if (slots > RG_MAX_SLOTS) slots = RG_MAX_SLOTS;
    if (slots < 4) return HEAL_ERR_UNSUPPORTED;
    const size_t smem = (size_t)slots * slot_bytes + w_bytes + stg_bytes + 512;
    // strips x row segments: one wave of CTAs when the strips alone do not fill the SMs
    const int strips = p.N * (p.W / RG_TW) * (p.C / 64);
    int segs = strips >= HEAL_NUM_SMS ? 1 : HEAL_NUM_SMS / strips;
    if (segs > p.H / 4) segs = p.H / 4 > 0 ? p.H / 4 : 1;
    p.seg_rows = (p.H + segs - 1) / segs;
    p.segs = (p.H + p.seg_rows - 1) / p.seg_rows;
    static size_t attr_set[HEAL_MAX_DEVICES] = {};
    if (!heal_ensure_dyn_smem(k_gconv3x3_ring, RG_SMEM_LIMIT, attr_set)) return HEAL_ERR_LAUNCH;
    if (p.pdl) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(strips * p.segs); cfg.blockDim = dim3(RG_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        cudaError_t e = cudaLaunchKernelEx(&cfg, k_gconv3x3_ring, tmA, tmB, tmO, p, slots);
        heal_launch_counter_add(1);
        return e == cudaSuccess ? HEAL_OK : HEAL_ERR_LAUNCH;
    }
    k_gconv3x3_ring<<<strips * p.segs, RG_THREADS, smem, st>>>(tmA, tmB, tmO, p, slots);
    return heal_check_launch();
}
