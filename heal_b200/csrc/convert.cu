// fp32 <-> bf16 / split-bf16 activation conversion (boundary plumbing of the tensor-core path).
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {
__global__ void k_act_convert(ActV src, ActV dst, size_t npix, int chunks) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = npix * (size_t)chunks;
    for (; i < total; i += (size_t)gridDim.x * blockDim.x) {
        size_t pix = i / chunks;
        int c = (int)(i % chunks) * 4;
        act_store4(dst, pix, c, act_load4(src, pix, c));
    }
}
__global__ void k_act_convert_scalar(ActV src, ActV dst, size_t npix, int channels) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = npix * (size_t)channels;
    for (; i < total; i += (size_t)gridDim.x * blockDim.x) {
        size_t pix = i / channels;
        int c = (int)(i % channels);
        act_store1(dst, pix, c, act_load1(src, pix, c));
    }
}
}  // namespace

// act_load4 / act_store4 move 4 channels at once: every 4-channel group starts 16 B-aligned in fp32 and 8 B-aligned in each bf16
// plane, so the base pointer as well as the channel stride, offset and (split) plane stride.
static inline bool aligned4(const heal_act_t* a) {
    const uintptr_t need = a->fmt == 0 ? 15 : 7;
    return ((uintptr_t)a->data & need) == 0 && (a->cstride & 3) == 0 && (a->coffset & 3) == 0 &&
           (a->fmt != 2 || (a->plane_stride & 3) == 0);
}

extern "C" int heal_act_convert(const heal_act_t* src, const heal_act_t* dst, size_t num_pixels, int channels, void* stream_) {
    if (!src || !dst) return HEAL_ERR_ARG;
    if (num_pixels == 0) return HEAL_OK;            // an empty map may have no storage (a null data pointer)
    if (!src->data || !dst->data) return HEAL_ERR_ARG;
    const bool vec = (channels & 3) == 0 && aligned4(src) && aligned4(dst);
    ActV s, d;
    s.p = src->data; s.fmt = src->fmt; s.cs = src->cstride; s.co = src->coffset; s.plane = src->plane_stride;
    d.p = dst->data; d.fmt = dst->fmt; d.cs = dst->cstride; d.co = dst->coffset; d.plane = dst->plane_stride;
    size_t total = vec ? num_pixels * (size_t)(channels / 4) : num_pixels * (size_t)channels;
    size_t blocks = (total + 255) / 256;
    size_t cap = (size_t)HEAL_NUM_SMS * 16;
    unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
    if (vec) k_act_convert<<<grid, 256, 0, (cudaStream_t)stream_>>>(s, d, num_pixels, channels / 4);
    else k_act_convert_scalar<<<grid, 256, 0, (cudaStream_t)stream_>>>(s, d, num_pixels, channels);
    return heal_check_launch();
}
