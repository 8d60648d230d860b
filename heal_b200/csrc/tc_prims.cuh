// wgmma / TMA / mbarrier primitives shared by the tensor-core kernels (conv2d_tc.cu, conv3x3_ring.cu, spconv_tc.cu).
// Inline PTX for sm_90a; every helper is a thin wrapper around ONE instruction (or a bounded wait loop).
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (reported as a launch failure) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();
    }
}

__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1, int c2, int c3, int c4) {
    asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
                 " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
                 " [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
                 " [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// K-major, 128B-swizzled shared-memory matrix descriptor (sm_90 wgmma): rows of 128 B, 8-row groups 1024 B apart.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);          // start address (16 B units)
    d |= (uint64_t)1 << 16;                           // leading byte offset (unused for swizzled K-major) = 1
    d |= (uint64_t)(1024 >> 4) << 32;                 // stride byte offset: 8 rows * 128 B
    d |= (uint64_t)1 << 62;                           // SWIZZLE_128B
    return d;
}

// K-major, 32B-swizzled descriptor (rows of 32 B = 16 bf16, 8-row groups 256 B apart): the packed diagonal weight sub-blocks.
__device__ __forceinline__ uint64_t gmma_desc_sw32(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(256 >> 4) << 32;
    d |= (uint64_t)3 << 62;                           // SWIZZLE_32B
    return d;
}

// Same, for a start address that is only 128 B aligned (a ROW offset inside a TMA-written swizzled tile).  mode 0: base offset
// 0 (the swizzle is taken from the absolute shared-memory address, as the TMA unit writes it); mode 1: base offset = the row
// phase of the start address (HEAL_TC_BO=1, kept to check the convention on a new part).
__device__ __forceinline__ uint64_t gmma_desc_sw128_off(uint32_t saddr, int mode) {
    uint32_t ph = (saddr >> 7) & 7;
    uint32_t bo = (mode == 0) ? 0u : ph;
    return gmma_desc_sw128(saddr) | ((uint64_t)bo << 49);
}

// Warpgroup MMA, D(64 x N, fp32 registers) (+)= A(64 x 16, smem) * B(16 x N, smem), both operands K-major bf16.
// accum == 0 overwrites D (first K step of a tile).  Fragment of thread t of the warpgroup: register i holds
// row 16*(t/32) + (t%32)/4 + 8*((i%4)/2), column 8*(i/4) + 2*(t%4) + i%2.
__device__ __forceinline__ void wgmma_n16(float* d, uint64_t a, uint64_t b, uint32_t accum) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %10, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(a), "l"(b), "r"(accum));
}
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t a, uint64_t b, uint32_t accum) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a), "l"(b), "r"(accum));
}
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t a, uint64_t b, uint32_t accum) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(accum));
}
__device__ __forceinline__ void wgmma_n128(float* d, uint64_t a, uint64_t b, uint32_t accum) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a), "l"(b), "r"(accum));
}
template <int N>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t a, uint64_t b, uint32_t accum) {
    static_assert(N == 16 || N == 32 || N == 64 || N == 128, "wgmma N");
    if constexpr (N == 16) wgmma_n16(d, a, b, accum);
    else if constexpr (N == 32) wgmma_n32(d, a, b, accum);
    else if constexpr (N == 64) wgmma_n64(d, a, b, accum);
    else wgmma_n128(d, a, b, accum);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Accumulator transposition through shared memory (spconv_tc.cu).  Its epilogue works one output ROW per thread (32 consecutive channels),
// the wgmma fragment spreads a row over 4 lanes; a chunk of SW (16, 32 or 64) columns of the 128-row tile goes through an
// fp32 scratch [128 rows][SW] whose 16-byte slots are XOR-swizzled by row (conflict-free row reads).
template <int SW>
__device__ __forceinline__ uint32_t scratch_addr(uint32_t base, int row, int col) {
    constexpr int SWZ = (SW / 4 < 8 ? SW / 4 : 8) - 1;
    return base + (uint32_t)(row * SW * 4) + (uint32_t)((((col >> 2) ^ (row & SWZ)) << 4) + (col & 3) * 4);
}
// columns [c0, c0 + SW) of the 64 x (2 * NR) fragment L (rows row0 .. row0 + 63 of the tile) -> scratch
template <int NR, int SW>
__device__ __forceinline__ void frag_to_scratch(const float* L, uint32_t base, int row0, int c0) {
    const int t = threadIdx.x & 127;
    const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
    for (int i = 0; i < NR; i += 2) {
        const int col = 8 * (i >> 2) + 2 * (t & 3) - c0;
        if (col >= 0 && col < SW) {
            const int rr = r + 8 * ((i & 3) >> 1);
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(scratch_addr<SW>(base, rr, col)), "f"(L[i]), "f"(L[i + 1]) : "memory");
        }
    }
}
// N (multiple of 4) consecutive fp32 of one scratch row, starting at chunk column col -> raw bits
template <int SW, int N>
__device__ __forceinline__ void scratch_row(uint32_t base, int row, int col, uint32_t* raw) {
#pragma unroll
    for (int j = 0; j < N; j += 4) {
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(raw[j]), "=r"(raw[j + 1]), "=r"(raw[j + 2]), "=r"(raw[j + 3]) : "r"(scratch_addr<SW>(base, row, col + j)) : "memory");
    }
}

// One lane of a converged warp; the compiler keeps code under this predicate on the uniform datapath (the TMA
// instructions take uniform-register operands: issuing them from an `if (lane == 0)` region costs an ELECT + branch loop
// per instruction).
__device__ __forceinline__ uint32_t elect_one() {
    uint32_t pred = 0;
    asm volatile("{\n .reg .b32 rx;\n .reg .pred px;\n elect.sync rx|px, 0xffffffff;\n @px mov.s32 %0, 1;\n}" : "+r"(pred));
    return pred;
}

__device__ __forceinline__ void tma_store_5d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3, int c4) {
    asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier over the 256 threads of the two consumer warpgroups
__device__ __forceinline__ void epi_bar(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
}
// the two halves of a packed bf16 pair (low half = lower address) as fp32
__device__ __forceinline__ float bf16_lo_f(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi_f(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
// what the bf16 rounding of v leaves: the lo plane of the split-bf16 pair (hi = bf16(v), lo = bf16(v - hi))
__device__ __forceinline__ float bf16_rest(float v) { return v - __bfloat162float(__float2bfloat16_rn(v)); }
__device__ __forceinline__ uint32_t lds_b32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_b32(uint32_t a, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

// 16-byte Ampere-style async copy global -> shared; src_bytes = 0 zero-fills the destination (used for gather rows that miss)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

typedef CUresult (*PFN_tmEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_tmEncodeTiled get_encode() {
    static PFN_tmEncodeTiled fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = (PFN_tmEncodeTiled)f;
    }
    return fn;
}

}  // namespace
