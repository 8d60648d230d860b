// Implicit-GEMM 2-D convolution on the Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers),
// operands staged by TMA (cp.async.bulk.tensor) with the 128-byte swizzle, warp-specialised and persistent.
//
// Replaces the dense convolutions of the BEV backbones / ResNeXt pyramid / shrink header
// (reference: resblock.py:48-64,102-122; base_bev_backbone.py:40-86; base_bev_backbone_resnet.py:54-85;
//  downsample_conv.py:16-27) with BN folded, and ReLU / residual / bias in the epilogue.
//
// Precision ("split-bf16", fp32-equivalent): an fp32 value x is stored as two bf16 planes hi = bf16(x),
// lo = bf16(x - hi) (16 mantissa bits).  A product a*b is evaluated as a_hi*b_hi + a_hi*b_lo + a_lo*b_hi
// with fp32 accumulation: three wgmma per K step into the same accumulator, relative
// error ~2^-16 per product, which keeps 70 stacked layers inside the 1e-3 fp32 parity tolerance that plain
// bf16 / tf32 tensor-core math cannot meet.  With planes == 1 the same kernel is a plain bf16 conv.
//
// GEMM view: M = output pixels (tile = TH x TW = 128 pixels of one image), N = output channels,
// K = taps x Cin in blocks of 64 channels.  A tile for tap (r,s) is ONE 5-D TMA box of the activation
// tensor {C, W, H, N, plane} at (c0, w0+s-pad, h0+r-pad, n, 0); out-of-bounds elements are zero-filled
// by the TMA unit, which implements the convolution padding.  B tiles come from the packed weights
// {Cin, taps*CoutPad, plane}.
//
// Roles (384 threads): warpgroup 0 = TMA producer (warp 0 loops as a converged warp and issues under elect.sync; its
// registers are handed to the consumers with setmaxnreg), warpgroups 1 and 2 = consumers: each runs the M = 64 wgmma of one
// half of the 128-pixel tile, then applies bias / residual / ReLU / hi-lo split to its accumulator fragment in place and
// writes it to the fragment's positions of a swizzled smem staging tile -> one cp.async.bulk.tensor store per 64-channel
// chunk (fp32 / transposed-conv / narrow outputs are stored from the fragment straight to global memory).
// The producer keeps STAGES k-blocks in flight, so the next tile's operands arrive while the consumers run the epilogue.
// Modes: stride 2 through TMA element strides; grouped 3x3 as 16-channel sub-block MMAs on block-diagonal 64-channel
// tiles; "halo" (3x3, stride 1, N = 64, one-row tiles or grouped two-row tiles): one activation box of TH rows x TW+2 pixels per
// kernel ROW, the three horizontal taps are row-shifted descriptors of the same smem tile (3x less L2->smem activation traffic);
// "A-row ring" (3x3, stride 1, N = 128, one-row tiles): the same row reuse with the A rows in a ring of their own and weight-only
// stages, K ordered (channel block, kernel row, kernel column).
// HEAL_TC_* environment switches are measurement hooks (profiles/tc_experiment.py), not product paths.
#include <cuda.h>
#include <stdlib.h>
#include "common.cuh"
#include "tc_prims.cuh"
#include "conv_ring.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int TC_THREADS = 384;      // warpgroup 0 TMA (warp 0), warpgroups 1 and 2 wgmma + epilogue
constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;                 // bf16 elements = 128 B = one swizzle row
constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;   // 16 KiB per plane

struct TcP {
    int N, Ho, Wo, Cout;          // output grid (conv resolution) and real output channels
    int taps_w, taps, pad;        // kw, kh*kw, padding
    int stride;                   // conv stride (TMA element stride on W and H)
    int blockdiag;                // grouped conv as block-diagonal 64x64 channel blocks: n-tile nt reads channel block nt only
    int bdiag;                    // block-diagonal weights arrive packed: only the four 16x16 diagonal sub-blocks ([16 rows][32 B], 32B swizzle)
    int kc_blocks;                // Cin / 64
    int TH, TW, tiles_h, tiles_w; // pixel tile and tile grid per image
    int m_tiles, n_tiles;
    int planes;                   // ACTIVATION planes: 1 = bf16, 2 = split-bf16 (fp32-equivalent)
    int wplanes;                  // WEIGHT planes: 2 = split weights (hi + lo).  planes 1 + wplanes 2 = the 'bf16' engine mode:
                                  // bf16 activations x un-rounded (16-mantissa-bit) weights, a_hi x [b_hi | b_lo]
    int coutp;                    // padded Cout rows per tap in the weight matrix (multiple of BLOCK_N)
    int relu;                     // epilogue activation: 0 none, 1 ReLU, 2 GELU (erf)
    int up;                       // transposed conv (k == stride == up): n-tile -> (i,j) sub-position
    int pdl;                      // launched with programmatic stream serialization
    int bo_mode;                  // experiment: base-offset convention of the halo descriptors
    int halo;                     // 3x3 stride-1, TH <= 2: ONE activation load per kernel ROW (TH x (TW+2) pixels) serves the 3 horizontal taps
    int arow;                     // dense 3x3 stride-1, BLOCK_N = 128, TH == 1: K order (channel block, kernel row, kernel column); one
                                  // A row of TW+2 pixels per (channel block, kernel row) in a ring of 2 serves the 3 columns' k-blocks
    int tma_out;                  // epilogue drains through shared memory + TMA tensor store (tmO valid)
    int res_tma;                  // STG >= 2: the residual chunk is TMA-loaded into the staging buffer one chunk ahead (tmR valid)
    int dbg;                      // HEAL_TC_DBG experiment bits (timing only, results invalid): 1 no stores, 2 no B loads, 4 no A loads, 8 no residual loads (TMA-store epilogue), 16 no MMAs
    const float* bias;            // [Cout]
    // residual (optional): split planes or fp32
    const __nv_bfloat16* res_split; size_t res_plane; const float* res_f32; int res_cs, res_co;
    // outputs (either or both)
    __nv_bfloat16* out_split; size_t out_plane; int out_cs, out_co;
    float* out_f32; int out32_cs, out32_co;
};

// STG = number of 64-channel output staging buffers in shared memory (0: the epilogue stores straight to global memory;
// >0: it writes the swizzled tile to smem and one elected thread issues a TMA tensor store, so every global write is a
// full coalesced line and the drain is asynchronous).
// GELU: the exact-erf GELU epilogue (ConvNeXt pwconv1) lives in its OWN instantiations: this kernel is sensitive to code size
// (an erff call inside every instantiation's epilogue cost the ReLU paths ~4 % of the C2 frame, A/B on the bench)
// GROUPED (p.blockdiag): the grouped conv's MMA shapes are their own instantiations too, so that each one issues a single
// set of wgmma shapes on its accumulator registers (mixed shapes on the same registers make ptxas serialise the chain).
template <int BLOCK_N, int STAGES, int STG, bool GELU = false, bool GROUPED = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv2d_tc(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR, const TcP p) {
    // 1024 B alignment for the 128B swizzle atoms: requested from the toolchain (no slack bytes to round up inside -- the halo
    // configuration needs all 227 KiB) and checked once.  The pointer is laundered through an empty asm so
    // that shared-memory addresses stay run-time values: with compile-time-constant addresses ptxas emitted a slower kernel
    // (an A/B on the B200 build).
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uintptr_t raw_addr = reinterpret_cast<uintptr_t>(smem_raw);
    asm volatile("" : "+l"(raw_addr));
    uint8_t* smem = reinterpret_cast<uint8_t*>(raw_addr);
    if (smem_u32(smem) & 1023u) __trap();
    // weight bytes per (tap, plane) in a stage: a BLOCK_N x 64 tile, or (grouped, packed) the four 16x16 diagonal sub-blocks
    const int B_TILE_BYTES = p.bdiag ? (BLOCK_N / 16) * 512 : BLOCK_N * BLOCK_K * 2;
    // halo mode: A = [plane][TH][TW+2 rows][128 B] (padded to 1 KiB), B = [plane][3 taps][BLOCK_N rows][128 B]
    const int halo_a_plane = p.TH * (p.TW + 2) * 128;
    const int halo_a_bytes = (p.planes * halo_a_plane + 1023) & ~1023;
    // A-row ring mode: the stages hold B only; the A rows (halo layout, TH == 1) sit in a ring of 2 after the staging buffers
    const int stage_bytes = p.halo ? (halo_a_bytes + p.wplanes * 3 * B_TILE_BYTES)
                          : p.arow ? p.wplanes * B_TILE_BYTES : (p.planes * A_TILE_BYTES + p.wplanes * B_TILE_BYTES);
    const int stg_bytes = p.planes * A_TILE_BYTES;                        // one staging buffer: [plane][128 rows][128 B]
    uint8_t* stg = smem + (size_t)STAGES * stage_bytes;                   // 1024-aligned (stage_bytes is a multiple of 1024)
    uint8_t* aring = stg + (size_t)STG * stg_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(aring + (p.arow ? 2 * halo_a_bytes : 0));
    // bars: full[STAGES], empty[STAGES], residual_full[3], a_full[2], a_empty[2]
    const uint32_t bar_res = smem_u32(bars + 2 * STAGES);
    const uint32_t bar_afull = smem_u32(bars + 2 * STAGES + 3), bar_aempty = smem_u32(bars + 2 * STAGES + 5);
    const uint32_t smem_base = smem_u32(smem), aring_base = smem_u32(aring);
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + STAGES);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // Split-bf16 products a_hi*b_hi + a_hi*b_lo + a_lo*b_hi.  For BLOCK_N <= 64 the hi and lo weight planes sit next to each other
    // in shared memory, so ONE MMA with N' = 2N computes a_hi x [b_hi | b_lo] (main | aux accumulator columns) and a second
    // N-wide MMA computes a_lo x b_hi into registers of its own: 2 tensor-core instructions and 2 reads of the A slice per K
    // step instead of 3.  The consumers fold main + (aux + a_lo x b_hi) before the epilogue.  BLOCK_N = 128 keeps 3 MMAs (N' = 256 would need 128 accumulator
    // registers per thread).
    constexpr bool NCAT = (BLOCK_N <= 64);
    constexpr int NACC = NCAT ? 2 * BLOCK_N : BLOCK_N;            // accumulator columns per tile half

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }   // 8 consumer warps
        for (int a = 0; a < 3; ++a) mbar_init(bar_res + 8 * a, 1);
        for (int a = 0; a < 2; ++a) { mbar_init(bar_afull + 8 * a, 1); mbar_init(bar_aempty + 8 * a, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // Programmatic dependent launch: everything above (barrier init) overlapped the tail of the previous
    // kernel in the stream / graph; from here on we touch memory it produced, so wait for it, and let the next kernel start
    // its own prologue as soon as our CTAs begin to drain.
    if (p.pdl) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }

    const int total_tiles = p.m_tiles * p.n_tiles;
    const int kcn = p.blockdiag ? 1 : p.kc_blocks;      // channel blocks per tap visited by one tile
    const int kblocks = (p.halo ? 3 : p.taps) * kcn;    // halo mode: one k-block per kernel ROW (3 taps each)

    if (warp < 4) {
        regs_dec<40>();
        // ============================== TMA producer: warp 0 (whole warp loops, one elected lane issues) ==
        if (warp == 0) {
            int stage = 0; uint32_t phase = 0;
            int ast = 0; uint32_t aphase = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int nt = tile % p.n_tiles, mt = tile / p.n_tiles;
                const int tw_i = mt % p.tiles_w; const int t2 = mt / p.tiles_w;
                const int th_i = t2 % p.tiles_h; const int img = t2 / p.tiles_h;
                const int h0 = th_i * p.TH, w0 = tw_i * p.TW;
                for (int kb = 0; kb < kblocks; ++kb) {
                    if (p.arow) {
                        // k-block = (channel block, kernel row r, kernel column s): at s == 0 the TW+2 pixels of input row h0+r-1
                        // go to the A ring, then every k-block brings its tap's weight tile
                        const int kc = kb / 9, tap = kb % 9, r = tap / 3, s = tap % 3;
                        if (s == 0) {
                            mbar_wait(bar_aempty + 8 * ast, aphase ^ 1);
                            if (elect_one()) {
                                mbar_expect_tx(bar_afull + 8 * ast, (uint32_t)(p.planes * halo_a_plane));
                                tma_load_5d(aring_base + ast * halo_a_bytes, &tmA, bar_afull + 8 * ast, kc * BLOCK_K, w0 - 1, h0 + r - 1, img, 0);
                            }
                            __syncwarp();
                        }
                        mbar_wait(bar_empty + 8 * stage, phase ^ 1);
                        if (elect_one()) {
                            mbar_expect_tx(bar_full + 8 * stage, (uint32_t)(p.wplanes * B_TILE_BYTES));
                            tma_load_3d(smem_base + stage * stage_bytes, &tmB, bar_full + 8 * stage, kc * BLOCK_K, tap * p.coutp + nt * BLOCK_N, 0);
                        }
                        __syncwarp();
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                        if (s == 2 && ++ast == 2) { ast = 0; aphase ^= 1; }
                        continue;
                    }
                    const int tap = kb / kcn, kc = p.blockdiag ? nt : kb % kcn;
                    const int r = tap / p.taps_w, s = tap % p.taps_w;
                    mbar_wait(bar_empty + 8 * stage, phase ^ 1);
                    if (p.halo) {
                        // k-block = (kernel row tap, channel block): pixels [w0-1, w0+TW] of input rows [h0+tap-1, h0+tap-1+TH), and the
                        // 3 taps' weights
                        const uint32_t sa = smem_base + stage * stage_bytes, sb = sa + halo_a_bytes;
                        if (elect_one()) {
                            mbar_expect_tx(bar_full + 8 * stage, (uint32_t)(p.planes * halo_a_plane + p.wplanes * 3 * B_TILE_BYTES));
                            tma_load_5d(sa, &tmA, bar_full + 8 * stage, kc * BLOCK_K, w0 - 1, h0 + tap - 1, img, 0);
                            // B lands as [tap][plane][rows] (dense) or [tap][16-row sub-block][plane][16 rows] (block-diagonal)
                            if (p.blockdiag) tma_load_5d(sb, &tmB, bar_full + 8 * stage, 0, 0, 0, nt * (BLOCK_N / 16), tap * 3);
                            else tma_load_4d(sb, &tmB, bar_full + 8 * stage, kc * BLOCK_K, nt * BLOCK_N, 0, tap * 3);
                        }
                        __syncwarp();
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                        continue;
                    }
                    const uint32_t sa = smem_base + stage * stage_bytes;
                    const uint32_t sb = sa + p.planes * A_TILE_BYTES;
                    const bool ldA = !(p.dbg & 4), ldB = !(p.dbg & 2);
                    if (elect_one()) {
                        mbar_expect_tx(bar_full + 8 * stage, (uint32_t)((ldA ? p.planes * A_TILE_BYTES : 0) + (ldB ? p.wplanes * B_TILE_BYTES : 0)));
                        if (ldA) tma_load_5d(sa, &tmA, bar_full + 8 * stage, kc * BLOCK_K, w0 * p.stride + s - p.pad, h0 * p.stride + r - p.pad, img, 0);
                        if (ldB) {
                            if (p.blockdiag) tma_load_4d(sb, &tmB, bar_full + 8 * stage, 0, 0, 0, (tap * p.coutp + nt * BLOCK_N) / 16);   // [sub-block][plane][16 rows]
                            else tma_load_3d(sb, &tmB, bar_full + 8 * stage, kc * BLOCK_K, tap * p.coutp + nt * BLOCK_N, 0);                // [plane][rows]
                        }
                    }
                    __syncwarp();
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ============================== consumers (warpgroups 1 and 2): wgmma, then the epilogue ==
        regs_inc<232>();
        const int wg = (warp >> 2) - 1;                 // tile rows [64 wg, 64 wg + 64)
        // This thread's part of the accumulator fragment (tc_prims.cuh): rows frow and frow + 8 of the tile, columns 8 j + fcol
        // and 8 j + fcol + 1 of every 8-column group j, in d[4 j .. 4 j + 3].  Both rows have the same 128B-swizzle phase fswz.
        const int ft = threadIdx.x & 127;
        const int frow = 64 * wg + 16 * (ft >> 5) + ((ft & 31) >> 2), fcol = 2 * (ft & 3);
        const int fswz = (ft >> 2) & 7;
        int stg_count = 0;
        const bool split = (p.planes == 2);                      // activations carry a lo plane
        const bool wsplit = (p.wplanes == 2);                    // weights carry a lo plane
        const int sub_bytes = p.wplanes * 2048;                  // smem bytes per 16-channel diagonal sub-block: [plane][16 rows][128 B]
        const uint32_t a_plane = (p.halo || p.arow) ? (uint32_t)halo_a_plane : (uint32_t)A_TILE_BYTES;
        const int ntap = p.halo ? 3 : 1;
        // first A row of this warpgroup's 64 pixels: tile pixel 64 wg, i.e. tile row 64 wg / TW, column 64 wg % TW; a halo tile's
        // rows are TW + 2 pixels long (TH == 2: warpgroup wg owns tile row wg)
        const uint32_t a_row0 = (p.halo || p.arow) ? (uint32_t)((64 * wg / p.TW) * (p.TW + 2) + (64 * wg) % p.TW) : (uint32_t)(64 * wg);
        int stage = 0; uint32_t phase = 0;
        int ast = 0; uint32_t aphase = 0;                       // A-row ring slot and parity (p.arow)
        float d[NACC / 2];
        float e[NCAT ? BLOCK_N / 2 : 1];                        // NCAT: a_lo*b_hi, or a_hi*b_hi with one weight plane
#pragma unroll
        for (int i = 0; i < NACC / 2; ++i) d[i] = 0.f;
#pragma unroll
        for (int i = 0; i < (NCAT ? BLOCK_N / 2 : 1); ++i) e[i] = 0.f;
        // All k-blocks of one tile into d (this warpgroup's 64 rows); afterwards d[0, BLOCK_N / 2) is the fragment of the
        // BLOCK_N logical columns (main + (aux + a_lo*b_hi)).  With NCAT every MMA shape has a register array of its own (the
        // N = BLOCK_N ones write e, not the first half of d): in-flight MMAs of different N on overlapping registers make ptxas
        // serialise the whole wgmma chain.
        auto mma_tile = [&]() {
            int prev = -1, prev_a = -1;
            for (int kb = 0; kb < kblocks; ++kb) {
                // A-row ring: kernel column tc of the row in ring slot ast (waited for at its first column)
                const int tc = p.arow ? kb % 3 : 0;
                if (p.arow && tc == 0) mbar_wait(bar_afull + 8 * ast, aphase);
                mbar_wait(bar_full + 8 * stage, phase);
                // A: [plane][rows][128 B]; halo mode: tap s reads rows [a_row0 + s, a_row0 + s + 64) of the TH x (TW+2)-row tile
                // (start address + s*128 B); A-row ring: the same with s = tc, in the ring slot; B alone fills the stage
                const uint32_t sa = p.arow ? aring_base + ast * halo_a_bytes + tc * 128 : smem_base + stage * stage_bytes;
                const uint32_t sb = p.arow ? smem_base + stage * stage_bytes
                                           : sa + (p.halo ? (uint32_t)halo_a_bytes : (uint32_t)(p.planes * A_TILE_BYTES));
                wgmma_fence();
                if (!(p.dbg & 16))
                for (int s = 0; s < ntap; ++s) {
                    const uint32_t ah = sa + (a_row0 + (uint32_t)s) * 128u, al = ah + a_plane;
                    const uint32_t bs = sb + s * p.wplanes * B_TILE_BYTES;
#pragma unroll
                    for (int k = 0; k < BLOCK_K / 16; ++k) {
                        const uint64_t a_hi = gmma_desc_sw128_off(ah + k * 32, p.bo_mode), a_lo = gmma_desc_sw128_off(al + k * 32, p.bo_mode);
                        if constexpr (GROUPED) {
                            if constexpr (BLOCK_N == 64) {
                                // Grouped conv: channels-per-group divides 16, so output channels [16k,16k+16) of this 64-block depend
                                // only on input channels [16k,16k+16): one M64 x N16 x K16 product per 16-channel sub-block, into
                                // its own accumulator registers d[16k ..] ([main16 | aux16]) and e[8k ..], or d[8k ..].
                                // sub-block k: [plane][16 rows] of 128 B rows at K offset k*16 elements, or packed 32 B rows
                                const uint32_t bk = p.bdiag ? bs + k * p.wplanes * 512 : bs + k * sub_bytes + k * 32;
                                const uint64_t bd = p.bdiag ? gmma_desc_sw32(bk) : gmma_desc_sw128(bk);
                                const uint32_t f0 = (kb == 0 && s == 0) ? 0u : 1u;
                                if (wsplit) {
                                    wgmma_bf16<32>(d + 16 * k, a_hi, bd, f0);               // [a_hi*b_hi | a_hi*b_lo]
                                    if (split) wgmma_bf16<16>(e + 8 * k, a_lo, bd, f0);     // a_lo*b_hi
                                } else {
                                    wgmma_bf16<16>(e + 8 * k, a_hi, bd, f0);
                                }
                            }
                        } else {
                            const uint32_t first = (kb == 0 && s == 0 && k == 0) ? 0u : 1u;
                            const uint64_t b_hi = gmma_desc_sw128(bs + k * 32);
                            if (!wsplit) {
                                if constexpr (NCAT) wgmma_bf16<BLOCK_N>(e, a_hi, b_hi, first);
                                else wgmma_bf16<BLOCK_N>(d, a_hi, b_hi, first);
                            } else if constexpr (NCAT) {
                                wgmma_bf16<2 * BLOCK_N>(d, a_hi, b_hi, first);               // [a_hi*b_hi | a_hi*b_lo]
                                if (split) wgmma_bf16<BLOCK_N>(e, a_lo, b_hi, first);        // a_lo*b_hi
                            } else {
                                const uint64_t b_lo = gmma_desc_sw128(bs + B_TILE_BYTES + k * 32);
                                wgmma_bf16<BLOCK_N>(d, a_hi, b_lo, first);
                                if (split) wgmma_bf16<BLOCK_N>(d, a_lo, b_hi, 1u);
                                wgmma_bf16<BLOCK_N>(d, a_hi, b_hi, 1u);
                            }
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();                                   // the previous k-block's MMAs have retired: free its stage
                if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
                if (prev_a >= 0 && lane == 0) mbar_arrive(bar_aempty + 8 * prev_a);   // the row's last column has retired
                prev = stage;
                prev_a = -1;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
                if (tc == 2) {
                    prev_a = ast;
                    if (++ast == 2) { ast = 0; aphase ^= 1; }
                }
            }
            wgmma_wait<0>();
            if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
            if (prev_a >= 0 && lane == 0) mbar_arrive(bar_aempty + 8 * prev_a);
            if constexpr (NCAT) {
                if (!wsplit) {
#pragma unroll
                    for (int i = 0; i < BLOCK_N / 2; ++i) d[i] = e[i];
                } else if constexpr (GROUPED && BLOCK_N == 64) {   // the same fold as k_gconv3x3_ring (the two kernels agree bit for bit)
#pragma unroll
                    for (int k = 0; k < 4; ++k)
#pragma unroll
                        for (int q = 0; q < 8; ++q)
                            d[8 * k + q] = d[16 * k + q] + (split ? d[16 * k + 8 + q] + e[8 * k + q] : d[16 * k + 8 + q]);
                } else {
#pragma unroll
                    for (int i = 0; i < BLOCK_N / 2; ++i) d[i] += split ? d[i + BLOCK_N / 2] + e[i] : d[i + BLOCK_N / 2];
                }
            }
        };
        // compiled only into the instantiations with at least two staging buffers (the ones dispatched with a residual)
        constexpr bool RES_TMA_OK = (STG >= 2);
        const bool res_tma = RES_TMA_OK && p.res_tma && !(p.dbg & 8);
        // residual chunk i+1 lands in staging buffer (i+1) % STG while chunk i is processed; the epilogue then adds it IN PLACE
        // (the fragment's own swizzled slots, which it overwrites with the output) -- fully coalesced, no global loads per thread.
        auto res_tma_issue = [&](int tile_, int c64_, int buf_) {
            const int nt_ = tile_ % p.n_tiles, mt_ = tile_ / p.n_tiles;
            const int tw_ = mt_ % p.tiles_w; const int t2_ = mt_ / p.tiles_w;
            const int th_ = t2_ % p.tiles_h; const int img_ = t2_ / p.tiles_h;
            mbar_expect_tx(bar_res + 8 * buf_, (uint32_t)stg_bytes);
            tma_load_5d(smem_u32(stg) + buf_ * stg_bytes, &tmR, bar_res + 8 * buf_, (nt_ * BLOCK_N) % p.coutp + c64_ * 64, tw_ * p.TW, th_ * p.TH, img_, 0);
        };
        if (res_tma && warp == 4 && lane == 0 && (int)blockIdx.x < total_tiles) res_tma_issue(blockIdx.x, 0, 0);
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int nt = tile % p.n_tiles, mt = tile / p.n_tiles;
            const int tw_i = mt % p.tiles_w; const int t2 = mt / p.tiles_w;
            const int th_i = t2 % p.tiles_h; const int img = t2 / p.tiles_h;
            const int n_glob = nt * BLOCK_N;
            const int q = n_glob / p.coutp, ch0 = n_glob % p.coutp;   // q = sub-position of a transposed conv (0 otherwise)
            const int ui = q / p.up, uj = q % p.up;
            // the fragment's two rows: in range, and the output pixel's linear index
            bool valid[2]; size_t pix[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = frow + 8 * h;
                const int oh = th_i * p.TH + r / p.TW, ow = tw_i * p.TW + r % p.TW;
                valid[h] = (oh < p.Ho) && (ow < p.Wo);
                pix[h] = ((size_t)img * (p.Ho * p.up) + (size_t)(oh * p.up + ui)) * (size_t)(p.Wo * p.up) + (size_t)(ow * p.up + uj);
            }
            mma_tile();
            if constexpr (STG > 0 && BLOCK_N >= 64) {
              if (p.tma_out) {
                const uint32_t stg_base = smem_u32(stg);
#pragma unroll
                for (int c64 = 0; c64 < BLOCK_N / 64; ++c64) {
                    const int b = stg_count % STG;
                    // tma_out needs Cout % 64 == 0, so a chunk is wholly inside Cout or wholly past it (the last n-tile of
                    // Cout = 192, 320, ... against coutp = 256, 384, ...).  A dead chunk reads no bias or residual (both are
                    // [Cout] / Cout-wide in global memory) but is still staged and stored, clipped by the TMA unit, so the
                    // buffer rotation and the residual barrier parity stay the same for every chunk.
                    const bool live = ch0 + 64 * c64 < p.Cout;
                    // the chunk's bias pairs, requested before the waits (the shared-memory stores below are compiler barriers)
                    float2 bb[8];
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj)
                        bb[jj] = (p.bias && live) ? __ldg(reinterpret_cast<const float2*>(p.bias + ch0 + 64 * c64 + 8 * jj + fcol)) : make_float2(0.f, 0.f);
                    if (res_tma) {
                        // (A') the store that last used buffer (i+1) % STG has been read out -> request residual(i+1) into it, then wait
                        // for residual(i) in buffer b (STG == 3: a full chunk of lead; STG == 2: the lead is the chunk minus the store drain)
                        if (warp == 4 && lane == 0) {
                            bulk_wait_read<(STG >= 2 ? STG - 2 : 0)>();
                            int ntile = tile, nc = c64 + 1;
                            if (nc == BLOCK_N / 64) { nc = 0; ntile = tile + (int)gridDim.x; }
                            if (ntile < total_tiles) res_tma_issue(ntile, nc, (stg_count + 1) % STG);
                        }
                        mbar_wait(bar_res + 8 * b, (uint32_t)((stg_count / STG) & 1));
                    } else {
                        // (A) buffer b is free once at most STG-1 store groups are still reading shared memory
                        if (warp == 4 && lane == 0) bulk_wait_read<STG - 1>();
                        epi_bar(1);
                    }
                    // (B) this thread's 2 rows x 16 columns of the 64-column chunk, straight from the fragment: bias, residual (read
                    // from the staging buffer at the fragment's swizzled slots), activation, hi/lo split, written back to the same
                    // slots (bank-conflict free: the 8 rows of a warp have 8 different swizzle phases).
                    const uint32_t row0 = stg_base + b * stg_bytes + frow * 128 + 2 * fcol;   // row frow + 8 is 1024 B further
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const int j = c64 * 8 + jj;
                        const int c = ch0 + 8 * j + fcol;
                        const uint32_t a0 = row0 + (uint32_t)((jj ^ fswz) << 4);
                        float v[4] = {d[4 * j] + bb[jj].x, d[4 * j + 1] + bb[jj].y, d[4 * j + 2] + bb[jj].x, d[4 * j + 3] + bb[jj].y};
                        if (res_tma) {
                            // residual pairs [hi row0, hi row0 + 8, lo row0, lo row0 + 8]
                            const uint32_t rs[4] = {lds_b32(a0), lds_b32(a0 + 1024), split ? lds_b32(a0 + A_TILE_BYTES) : 0u,
                                                    split ? lds_b32(a0 + A_TILE_BYTES + 1024) : 0u};
#pragma unroll
                            for (int h = 0; h < 2; ++h) { v[2 * h] += bf16_lo_f(rs[h]); v[2 * h + 1] += bf16_hi_f(rs[h]); }
                            if (split) {
#pragma unroll
                                for (int h = 0; h < 2; ++h) { v[2 * h] += bf16_lo_f(rs[2 + h]); v[2 * h + 1] += bf16_hi_f(rs[2 + h]); }
                            }
                        } else if (p.res_f32 && live && !(p.dbg & 8)) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                if (valid[h]) {
                                    const float* rp = p.res_f32 + pix[h] * p.res_cs + p.res_co + c;
                                    v[2 * h] += __ldg(rp); v[2 * h + 1] += __ldg(rp + 1);
                                }
                            }
                        }
                        if constexpr (GELU) {
#pragma unroll
                            for (int i = 0; i < 4; ++i) v[i] = heal_act_fn(v[i], 2);
                        } else if (p.relu) {
#pragma unroll
                            for (int i = 0; i < 4; ++i) v[i] = fmaxf(v[i], 0.f);
                        }
                        sts_b32(a0, pack_bf16(v[0], v[1])); sts_b32(a0 + 1024, pack_bf16(v[2], v[3]));
                        if (split) {
                            sts_b32(a0 + A_TILE_BYTES, pack_bf16(bf16_rest(v[0]), bf16_rest(v[1])));
                            sts_b32(a0 + A_TILE_BYTES + 1024, pack_bf16(bf16_rest(v[2]), bf16_rest(v[3])));
                        }
                    }
                    fence_async_smem();
                    epi_bar(2);
                    // (C) one thread drains the buffer with a TMA tensor store (out-of-range pixels are clipped by the unit)
                    if (warp == 4 && lane == 0 && !(p.dbg & 1)) {
                        tma_store_5d(&tmO, stg_base + b * stg_bytes, ch0 + c64 * 64, tw_i * p.TW, th_i * p.TH, img, 0);
                        bulk_commit();
                    }
                    ++stg_count;
                }
                continue;
              }
            }
            // direct stores (fp32 outputs, transposed convs, N = 16 / 32, Cout % 64 != 0): each thread writes its fragment's
            // column pairs of its two rows
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
                const int c = ch0 + 8 * j + fcol;
                if (c >= p.Cout) continue;
                const bool two = c + 1 < p.Cout;
                const float b0 = p.bias ? __ldg(p.bias + c) : 0.f, b1 = (two && p.bias) ? __ldg(p.bias + c + 1) : 0.f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!valid[h]) continue;
                    float v0 = d[4 * j + 2 * h] + b0, v1 = d[4 * j + 2 * h + 1] + b1;
                    if (p.res_split) {
                        const __nv_bfloat16* rp = p.res_split + pix[h] * p.res_cs + p.res_co + c;
                        v0 += __bfloat162float(rp[0]);
                        if (two) v1 += __bfloat162float(rp[1]);
                        if (split) {
                            v0 += __bfloat162float(rp[p.res_plane]);
                            if (two) v1 += __bfloat162float(rp[p.res_plane + 1]);
                        }
                    } else if (p.res_f32) {
                        const float* rp = p.res_f32 + pix[h] * p.res_cs + p.res_co + c;
                        v0 += __ldg(rp);
                        if (two) v1 += __ldg(rp + 1);
                    }
                    if constexpr (GELU) {
                        v0 = heal_act_fn(v0, 2); v1 = heal_act_fn(v1, 2);
                    } else if (p.relu) {
                        v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);
                    }
                    if (p.out_split && !((p.dbg & 1) && v0 != 1.2345e30f)) {
                        __nv_bfloat16* op = p.out_split + pix[h] * p.out_cs + p.out_co + c;
                        if (two && !((p.out_cs | p.out_co | p.out_plane) & 1)) {
                            *reinterpret_cast<uint32_t*>(op) = pack_bf16(v0, v1);
                            if (split) *reinterpret_cast<uint32_t*>(op + p.out_plane) = pack_bf16(bf16_rest(v0), bf16_rest(v1));
                        } else {
                            op[0] = __float2bfloat16_rn(v0);
                            if (split) op[p.out_plane] = __float2bfloat16_rn(bf16_rest(v0));
                            if (two) {
                                op[1] = __float2bfloat16_rn(v1);
                                if (split) op[p.out_plane + 1] = __float2bfloat16_rn(bf16_rest(v1));
                            }
                        }
                    }
                    if (p.out_f32 && !((p.dbg & 1) && v0 != 1.2345e30f)) {
                        float* op = p.out_f32 + pix[h] * p.out32_cs + p.out32_co + c;
                        if (two && !((p.out32_cs | p.out32_co) & 1)) {
                            *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
                        } else {
                            op[0] = v0;
                            if (two) op[1] = v1;
                        }
                    }
                }
            }
        }
        if (STG > 0 && warp == 4 && lane == 0) bulk_wait_all();     // all output tiles have left shared memory
        (void)stg_count;
    }
}

// HEAL_TC_* measurement hooks (profiles/tc_experiment.py), read once per process instead of six getenv calls per launch.
struct TcEnv {
    int dbg, pdl, halo, bo, tma_store, res_tma, ring, l2promo;
    TcEnv() {
        auto geti = [](const char* n, int dflt) { const char* e = getenv(n); return e ? atoi(e) : dflt; };
        dbg = geti("HEAL_TC_DBG", 0); pdl = geti("HEAL_TC_PDL", 1); halo = geti("HEAL_TC_HALO", 1); bo = geti("HEAL_TC_BO", 0);
        tma_store = geti("HEAL_TC_TMA_STORE", 1); res_tma = geti("HEAL_TC_RES_TMA", 1); ring = geti("HEAL_TC_RING", 1); l2promo = geti("HEAL_TC_L2PROMO", 128);
    }
};
const TcEnv& tc_env() { static const TcEnv e; return e; }

template <int BLOCK_N, int STAGES, int STG, bool GELU = false, bool GROUPED = false>
int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const CUtensorMap& tmR, const TcP& p_in, cudaStream_t st) {
    TcP p = p_in;
    p.res_tma = (STG >= 2 && p.tma_out && p.res_split && p_in.res_tma) ? 1 : 0;
    const size_t b_tile = p.bdiag ? (size_t)(BLOCK_N / 16) * 512 : (size_t)BLOCK_N * BLOCK_K * 2;
    size_t stage_bytes = (size_t)p.planes * A_TILE_BYTES + (size_t)p.wplanes * b_tile;
    const size_t halo_a = ((size_t)p.planes * p.TH * (p.TW + 2) * 128 + 1023) & ~(size_t)1023;
    if (p.halo) stage_bytes = halo_a + (size_t)p.wplanes * 3 * b_tile;
    if (p.arow) stage_bytes = (size_t)p.wplanes * b_tile;
    size_t smem = (size_t)STAGES * stage_bytes + (size_t)STG * p.planes * A_TILE_BYTES + (p.arow ? 2 * halo_a : 0) + 256;
    if (smem > 227 * 1024) return HEAL_ERR_UNSUPPORTED;
    if (p.tma_out && p.res_split && !p.res_tma) return HEAL_ERR_UNSUPPORTED;
    if ((p.blockdiag != 0) != GROUPED || (GROUPED && BLOCK_N != 64)) return HEAL_ERR_UNSUPPORTED;    // the staging epilogue adds a split residual only from TMA loads
    static size_t attr_set[HEAL_MAX_DEVICES] = {};
    if (!heal_ensure_dyn_smem(k_conv2d_tc<BLOCK_N, STAGES, STG, GELU, GROUPED>, 227 * 1024, attr_set)) return HEAL_ERR_LAUNCH;
    int total = p.m_tiles * p.n_tiles;
    int grid = total < HEAL_NUM_SMS ? total : HEAL_NUM_SMS;
    if (grid < 1) return HEAL_ERR_UNSUPPORTED;
    if (p.pdl) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        cudaError_t e = cudaLaunchKernelEx(&cfg, k_conv2d_tc<BLOCK_N, STAGES, STG, GELU, GROUPED>, tmA, tmB, tmO, tmR, p);
        heal_launch_counter_add(1);
        return e == cudaSuccess ? HEAL_OK : HEAL_ERR_LAUNCH;
    }
    k_conv2d_tc<BLOCK_N, STAGES, STG, GELU, GROUPED><<<grid, TC_THREADS, smem, st>>>(tmA, tmB, tmO, tmR, p);
    return heal_check_launch();
}

// 64 output channels per tile: halo tiles with unpacked weights have 81 KiB stages, every other one at most 48 KiB
template <bool GROUPED>
int launch_tc64(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const CUtensorMap& tmR, const TcP& p, cudaStream_t st) {
    const bool big = p.halo && !p.bdiag;
    if (!p.tma_out) return big ? launch_tc<64, 2, 0, false, GROUPED>(tmA, tmB, tmO, tmR, p, st) : launch_tc<64, 4, 0, false, GROUPED>(tmA, tmB, tmO, tmR, p, st);
    return big ? launch_tc<64, 2, 2, false, GROUPED>(tmA, tmB, tmO, tmR, p, st) : launch_tc<64, 3, 2, false, GROUPED>(tmA, tmB, tmO, tmR, p, st);
}

}  // namespace

extern "C" int heal_conv2d_tc(const void* in_split, size_t in_plane_stride, int N, int H, int W, int Cin, int in_cstride, int in_coffset,
                              const void* w_packed, const void* w_diag, int w_rows, int coutp, const float* bias,
                              int kh, int kw, int stride, int pad, int blockdiag, int planes, int w_planes,
                              const void* res_split, size_t res_plane_stride, const float* res_f32, int res_cstride, int res_coffset,
                              void* out_split, size_t out_plane_stride, int out_cstride, int out_coffset,
                              float* out_f32, int out32_cstride, int out32_coffset,
                              int Ho, int Wo, int Cout, int upsample, int relu, void* stream_) {
    if (!in_split || !w_packed || (!out_split && !out_f32)) return HEAL_ERR_ARG;
    if (planes != 1 && planes != 2) return HEAL_ERR_ARG;
    if (w_planes != 1 && w_planes != 2) return HEAL_ERR_ARG;
    if (planes == 2 && w_planes != 2) return HEAL_ERR_UNSUPPORTED;
    if ((Cin % BLOCK_K) || (in_cstride & 7) || (in_coffset & 7) || upsample < 1) return HEAL_ERR_UNSUPPORTED;
    if (stride < 1 || stride > 2) return HEAL_ERR_UNSUPPORTED;
    if (Ho != (H + 2 * pad - kh) / stride + 1 || Wo != (W + 2 * pad - kw) / stride + 1) return HEAL_ERR_ARG;
    if (blockdiag && (upsample > 1 || coutp != Cin || (coutp % 64))) return HEAL_ERR_UNSUPPORTED;
    if (upsample > 1 && (kh != 1 || kw != 1)) return HEAL_ERR_UNSUPPORTED;
    const int taps = kh * kw;
    const int block_n = blockdiag ? 64 : (coutp >= 128 ? 128 : coutp);
    if (!(block_n == 16 || block_n == 32 || block_n == 64 || block_n == 128) || (coutp % block_n)) return HEAL_ERR_UNSUPPORTED;
    if (w_rows != (upsample > 1 ? upsample * upsample : taps) * coutp) return HEAL_ERR_ARG;
    PFN_tmEncodeTiled enc = get_encode();
    if (!enc) return HEAL_ERR_DRIVER;

    TcP p;
    p.res_tma = 0; p.bdiag = 0;
    p.N = N; p.Ho = Ho; p.Wo = Wo; p.Cout = Cout;
    p.taps_w = kw; p.taps = taps; p.pad = pad; p.kc_blocks = Cin / BLOCK_K;
    int tw = 128; while (tw > Wo && tw > 8) tw >>= 1;
    p.TW = tw; p.TH = BLOCK_M / tw;
    p.tiles_w = (Wo + p.TW - 1) / p.TW; p.tiles_h = (Ho + p.TH - 1) / p.TH;
    p.m_tiles = N * p.tiles_h * p.tiles_w;
    p.n_tiles = w_rows / taps / block_n;
    p.stride = stride; p.blockdiag = blockdiag;
    if (upsample > 1) p.n_tiles = w_rows / block_n;
    p.planes = planes; p.wplanes = w_planes; p.coutp = coutp; p.relu = relu; p.up = upsample; p.bias = bias;
    const TcEnv& env = tc_env();
    p.dbg = env.dbg; p.pdl = env.pdl;
    p.res_split = (const __nv_bfloat16*)res_split; p.res_plane = res_plane_stride; p.res_f32 = res_f32;
    p.res_cs = res_cstride; p.res_co = res_coffset;
    p.out_split = (__nv_bfloat16*)out_split; p.out_plane = out_plane_stride; p.out_cs = out_cstride; p.out_co = out_coffset;
    p.out_f32 = out_f32; p.out32_cs = out32_cstride; p.out32_co = out32_coffset;

    {
        const bool want = env.halo != 0;
        p.bo_mode = env.bo;
        // Two-row tiles (64-wide maps) only for the grouped convs: their k-block order is the same with or without halo loads
        // (bit-identical), and with packed diagonal weights their 45 KiB halo stages keep three stages.  A dense halo stage is
        // 81 KiB (two stages), and no dense 64-wide layer of the product has been measured to gain from that trade.
        const bool rows_ok = p.TH == 1 || (p.TH == 2 && blockdiag);
        p.halo = (want && kh == 3 && kw == 3 && stride == 1 && pad == 1 && rows_ok && block_n == 64 && upsample == 1) ? 1 : 0;
        // 128-wide dense 3x3 (the shrink header): three taps' B tiles do not fit a stage next to an A row, so the A rows get a
        // ring of their own and each (tap, channel block) k-block brings only its B tile.  Only where it was measured faster:
        // long K (Cin >= 256) and three weight stages (no split residual, which needs two staging buffers and leaves two).
        p.arow = (want && kh == 3 && kw == 3 && stride == 1 && pad == 1 && p.TH == 1 && block_n == 128 && !blockdiag && upsample == 1 &&
                  relu != 2 && Cin >= 256 && !res_split) ? 1 : 0;
    }
    // L2 promotion of the activation / residual loads (HEAL_TC_L2PROMO=256: experiment)
    const CUtensorMapL2promotion act_promo = env.l2promo == 256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
    CUtensorMap tmA, tmB;
    {
        cuuint64_t dims[5] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N, (cuuint64_t)planes};
        cuuint64_t strides[4] = {(cuuint64_t)in_cstride * 2, (cuuint64_t)W * in_cstride * 2, (cuuint64_t)H * W * in_cstride * 2,
                                 (cuuint64_t)in_plane_stride * 2};
        cuuint32_t box[5] = {(cuuint32_t)BLOCK_K, (cuuint32_t)(p.TW * stride), (cuuint32_t)(p.TH * stride), 1u, (cuuint32_t)planes};
        if (p.halo || p.arow) box[1] = (cuuint32_t)(p.TW + 2);
        cuuint32_t es[5] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1, 1};
        void* base = (void*)((const __nv_bfloat16*)in_split + in_coffset);
        if (planes == 1) { strides[3] = strides[2] * N; }
        CUresult r = enc(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, act_promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
    }
    {
        // packed weights in global memory: [plane][taps * coutp rows][wk] bf16.  The box order decides the shared-memory layout:
        // hi and lo planes of the same rows must be adjacent for the N-concatenated MMAs (see NCAT in the kernel).
        const cuuint64_t wk = blockdiag ? 64 : Cin;      // K extent of the packed weight matrix
        const cuuint64_t row_b = wk * 2, plane_b = (cuuint64_t)w_rows * wk * 2;
        const cuuint32_t pl = (cuuint32_t)w_planes;
        cuuint32_t es[5] = {1, 1, 1, 1, 1};
        CUresult r;
        p.bdiag = (blockdiag && w_diag) ? 1 : 0;
        if (p.bdiag) {
            // packed diagonal sub-blocks in global memory: [plane][taps * coutp rows][16] bf16 (32 B rows) -> a quarter of the bytes
            const cuuint64_t pb = (cuuint64_t)w_rows * 32;
            if (p.halo) {                   // smem [3 taps][4 sub-blocks][plane][16 rows][32 B]
                cuuint64_t d[5] = {16, 16, (cuuint64_t)w_planes, (cuuint64_t)coutp / 16, (cuuint64_t)taps};
                cuuint64_t st[4] = {32, pb, 512, (cuuint64_t)coutp * 32};
                cuuint32_t b[5] = {16u, 16u, pl, (cuuint32_t)block_n / 16, 3u};
                r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)w_diag, d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            } else {                        // smem [4 sub-blocks][plane][16 rows][32 B]
                cuuint64_t d[4] = {16, 16, (cuuint64_t)w_planes, (cuuint64_t)w_rows / 16};
                cuuint64_t st[3] = {32, pb, 512};
                cuuint32_t b[4] = {16u, 16u, pl, (cuuint32_t)block_n / 16};
                r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)w_diag, d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            }
        } else if (blockdiag && p.halo) {   // smem [3 taps][4 sub-blocks][plane][16 rows]
            cuuint64_t d[5] = {wk, 16, (cuuint64_t)w_planes, (cuuint64_t)coutp / 16, (cuuint64_t)taps};
            cuuint64_t st[4] = {row_b, plane_b, 16 * row_b, (cuuint64_t)coutp * row_b};
            cuuint32_t b[5] = {(cuuint32_t)BLOCK_K, 16u, pl, (cuuint32_t)block_n / 16, 3u};
            r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)w_packed, d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        } else if (blockdiag) {             // smem [4 sub-blocks][plane][16 rows]
            cuuint64_t d[4] = {wk, 16, (cuuint64_t)w_planes, (cuuint64_t)w_rows / 16};
            cuuint64_t st[3] = {row_b, plane_b, 16 * row_b};
            cuuint32_t b[4] = {(cuuint32_t)BLOCK_K, 16u, pl, (cuuint32_t)block_n / 16};
            r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)w_packed, d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        } else if (p.halo) {                // smem [3 taps][plane][block_n rows]: one box brings the 3 horizontal taps of a kernel row
            cuuint64_t d[4] = {wk, (cuuint64_t)coutp, (cuuint64_t)w_planes, (cuuint64_t)taps};
            cuuint64_t st[3] = {row_b, plane_b, (cuuint64_t)coutp * row_b};
            cuuint32_t b[4] = {(cuuint32_t)BLOCK_K, (cuuint32_t)block_n, pl, 3u};
            r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)w_packed, d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        } else {                            // smem [plane][block_n rows]
            cuuint64_t d[3] = {wk, (cuuint64_t)w_rows, (cuuint64_t)w_planes};
            cuuint64_t st[2] = {row_b, plane_b};
            cuuint32_t b[3] = {(cuuint32_t)BLOCK_K, (cuuint32_t)block_n, pl};
            r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)w_packed, d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        }
        if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
    }
    // output tensor map for the TMA-store epilogue (split / bf16 output at conv resolution, 64-channel boxes)
    CUtensorMap tmO = tmA;
    p.tma_out = 0;
    {
        const bool want = env.tma_store != 0;
        if (want && out_split && upsample == 1 && block_n >= 64 && (Cout % 64) == 0 && !(out_cstride & 7) && !(out_coffset & 7) &&
            (!res_split || (!(res_cstride & 7) && !(res_coffset & 7)))) {
            cuuint64_t dims[5] = {(cuuint64_t)Cout, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)N, (cuuint64_t)planes};
            cuuint64_t strides[4] = {(cuuint64_t)out_cstride * 2, (cuuint64_t)Wo * out_cstride * 2, (cuuint64_t)Ho * Wo * out_cstride * 2,
                                     (cuuint64_t)out_plane_stride * 2};
            if (planes == 1) strides[3] = strides[2] * N;
            cuuint32_t box[5] = {(cuuint32_t)BLOCK_K, (cuuint32_t)p.TW, (cuuint32_t)p.TH, 1u, (cuuint32_t)planes};
            cuuint32_t es[5] = {1, 1, 1, 1, 1};
            void* base = (void*)((__nv_bfloat16*)out_split + out_coffset);
            CUresult r = enc(&tmO, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, act_promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
            p.tma_out = out_f32 ? 0 : 1;
        }
    }
    // residual tensor map (same boxes as the output map): the residual chunk is TMA-loaded into the output staging buffer
    CUtensorMap tmR = tmO;
    bool res_tma_ok = false;
    {
        const bool want = env.res_tma != 0;
        if (want && p.tma_out && res_split) {
            cuuint64_t dims[5] = {(cuuint64_t)Cout, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)N, (cuuint64_t)planes};
            cuuint64_t strides[4] = {(cuuint64_t)res_cstride * 2, (cuuint64_t)Wo * res_cstride * 2, (cuuint64_t)Ho * Wo * res_cstride * 2,
                                     (cuuint64_t)res_plane_stride * 2};
            if (planes == 1) strides[3] = strides[2] * N;
            cuuint32_t box[5] = {(cuuint32_t)BLOCK_K, (cuuint32_t)p.TW, (cuuint32_t)p.TH, 1u, (cuuint32_t)planes};
            cuuint32_t es[5] = {1, 1, 1, 1, 1};
            void* base = (void*)((const __nv_bfloat16*)res_split + res_coffset);
            CUresult r = enc(&tmR, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, act_promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) return HEAL_ERR_DRIVER;
            res_tma_ok = true;
            p.res_tma = 1;
        }
    }
    // the TMA-store epilogue adds a split residual from a TMA-loaded copy in its staging buffer; otherwise the direct stores do
    if (p.tma_out && res_split && !res_tma_ok) p.tma_out = 0;
    cudaStream_t st = (cudaStream_t)stream_;
    const int kblocks = (blockdiag ? 1 : p.kc_blocks) * taps;
    // grouped 3x3 on maps at least 128 pixels wide: the row-ring kernel (conv3x3_ring.cu) reads every input row and the weights
    // once per CTA instead of three times / once per tile; it shares the three tensor maps built above
    if (env.ring && p.halo && p.bdiag && p.tma_out && !res_split && !res_f32 && (Wo % 128) == 0 && relu != 2 && Cin == Cout &&
        coutp == Cout && !p.dbg) {
        RingP rp;
        rp.N = N; rp.H = Ho; rp.W = Wo; rp.C = Cout; rp.planes = planes; rp.wplanes = w_planes; rp.relu = relu; rp.bias = bias;
        rp.segs = 1; rp.seg_rows = Ho; rp.pdl = env.pdl;
        return heal_conv3x3_ring_launch(tmA, tmB, tmO, rp, st);
    }
    if (relu == 2) {        // GELU: 1x1 / 3x3 convs with >= 128 output channels and no residual (ConvNeXt pwconv1: dim -> 4 dim)
        if (block_n != 128 || res_split || res_f32) return HEAL_ERR_UNSUPPORTED;
        if (!p.tma_out) return launch_tc<128, 3, 0, true>(tmA, tmB, tmO, tmR, p, st);
        return kblocks <= 4 ? launch_tc<128, 2, 2, true>(tmA, tmB, tmO, tmR, p, st) : launch_tc<128, 3, 1, true>(tmA, tmB, tmO, tmR, p, st);
    }
    // Configurations (stages, staging buffers) are sized to the 227 KiB of shared memory per block (split operands; planes == 1
    // needs less).  A split residual needs two staging buffers (STG >= 2): the next chunk's residual is loaded into one while the
    // other is drained.  Long-K layers get three stages; short-K layers are bound by the output stream and get two staging
    // buffers instead.
    switch (block_n) {
        case 16: return launch_tc<16, 4, 0>(tmA, tmB, tmO, tmR, p, st);
        case 32: return launch_tc<32, 4, 0>(tmA, tmB, tmO, tmR, p, st);
        case 64:
            return blockdiag ? launch_tc64<true>(tmA, tmB, tmO, tmR, p, st) : launch_tc64<false>(tmA, tmB, tmO, tmR, p, st);
        default:                                                       // 64 KiB stages
            if (!p.tma_out) return launch_tc<128, 3, 0>(tmA, tmB, tmO, tmR, p, st);
            if (res_tma_ok || kblocks <= 4) return launch_tc<128, 2, 2>(tmA, tmB, tmO, tmR, p, st);
            return launch_tc<128, 3, 1>(tmA, tmB, tmO, tmR, p, st);
    }
}
