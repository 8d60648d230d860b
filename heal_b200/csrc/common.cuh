// Common device/host helpers for the heal_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <math.h>

#define HEAL_OK 0
#define HEAL_ERR_ARG (-1)
#define HEAL_ERR_WORKSPACE (-2)
#define HEAL_ERR_LAUNCH (-3)
#define HEAL_ERR_UNSUPPORTED (-4)
#define HEAL_ERR_DRIVER (-5)

#define HEAL_NUM_SMS 132  // H100 SXM

// process-wide count of kernels this library has launched (bench.py reports it as gpu_launches)
extern "C" void heal_launch_counter_add(int n);

static inline int heal_check_launch(int kernels_launched = 1) {
    cudaError_t e = cudaGetLastError();
    heal_launch_counter_add(kernels_launched);
    return e == cudaSuccess ? HEAL_OK : HEAL_ERR_LAUNCH;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: remember the largest value set per device ordinal
// (a process that drives several GPUs must set it on each of them).
#define HEAL_MAX_DEVICES 64
template <typename K>
static inline bool heal_ensure_dyn_smem(K kernel, size_t bytes, size_t (&set_for_device)[HEAL_MAX_DEVICES]) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return false;
    const bool tracked = dev >= 0 && dev < HEAL_MAX_DEVICES;
    if (tracked && set_for_device[dev] >= bytes) return true;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) return false;
    if (tracked) set_for_device[dev] = bytes;
    return true;
}

static inline size_t heal_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bump allocator over a caller-provided workspace; no internal allocation anywhere in the library.
struct HealArena {
    char* base;
    size_t cap;
    size_t off;
    __host__ HealArena(void* p, size_t bytes) : base((char*)p), cap(bytes), off(0) {}
    template <typename T>
    __host__ T* take(size_t n) {
        off = heal_align_up(off, 256);
        T* r = (T*)(base + off);
        off += n * sizeof(T);
        return r;
    }
    __host__ bool ok() const { return base != nullptr && off <= cap; }
};

__device__ __forceinline__ float4 ldg_f4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void stg_f4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// epilogue activation selector shared by the conv kernels: 0 none, 1 ReLU, 2 GELU (exact, erf form: torch.nn.GELU() default)
__device__ __forceinline__ float heal_act_fn(float v, int mode) {
    if (mode == 1) return fmaxf(v, 0.f);
    if (mode == 2) return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_min_i(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---- activation views: fp32, bf16 (one plane) or split-bf16 (hi + lo planes), channels-last ----------
// Mirrors heal_act_t of include/heal_b200.h.
struct ActV {
    void* p;
    int fmt;        // 0 = f32, 1 = bf16, 2 = split-bf16
    int cs, co;     // pixel stride / first channel (elements)
    size_t plane;   // elements between hi and lo plane (fmt 2)
};

__device__ __forceinline__ float4 bf16x4_to_f4(uint2 u) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
    float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ uint2 f4_to_bf16x4(float4 v) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&a); u.y = *reinterpret_cast<uint32_t*>(&b);
    return u;
}
// 4 consecutive channels starting at channel c (multiple of 4) of pixel `pix`
__device__ __forceinline__ float4 act_load4(const ActV& a, size_t pix, int c) {
    size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (a.fmt == 0) return __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.p) + idx));
    const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(a.p) + idx;
    float4 v = bf16x4_to_f4(__ldg(reinterpret_cast<const uint2*>(b)));
    if (a.fmt == 2) {
        float4 l = bf16x4_to_f4(__ldg(reinterpret_cast<const uint2*>(b + a.plane)));
        v.x += l.x; v.y += l.y; v.z += l.z; v.w += l.w;
    }
    return v;
}
__device__ __forceinline__ void act_store4(const ActV& a, size_t pix, int c, float4 v) {
    size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (a.fmt == 0) { *reinterpret_cast<float4*>(reinterpret_cast<float*>(a.p) + idx) = v; return; }
    __nv_bfloat16* b = reinterpret_cast<__nv_bfloat16*>(a.p) + idx;
    uint2 h = f4_to_bf16x4(v);
    *reinterpret_cast<uint2*>(b) = h;
    if (a.fmt == 2) {
        float4 hf = bf16x4_to_f4(h);
        *reinterpret_cast<uint2*>(b + a.plane) = f4_to_bf16x4(make_float4(v.x - hf.x, v.y - hf.y, v.z - hf.z, v.w - hf.w));
    }
}
__device__ __forceinline__ float act_load1(const ActV& a, size_t pix, int c) {
    size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (a.fmt == 0) return __ldg(reinterpret_cast<const float*>(a.p) + idx);
    const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(a.p) + idx;
    float v = __bfloat162float(b[0]);
    if (a.fmt == 2) v += __bfloat162float(b[a.plane]);
    return v;
}
__device__ __forceinline__ void act_store1(const ActV& a, size_t pix, int c, float v) {
    size_t idx = pix * (size_t)a.cs + (size_t)(a.co + c);
    if (a.fmt == 0) { reinterpret_cast<float*>(a.p)[idx] = v; return; }
    __nv_bfloat16* b = reinterpret_cast<__nv_bfloat16*>(a.p) + idx;
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    b[0] = h;
    if (a.fmt == 2) b[a.plane] = __float2bfloat16_rn(v - __bfloat162float(h));
}
