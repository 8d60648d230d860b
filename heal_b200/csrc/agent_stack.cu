// Agent assembly of a heterogeneous scene: every modality's per-agent maps, center-cropped or zero-padded to the scene grid
// (torchvision CenterCrop), written in scene order into one (n_agents, H, W, C) map in one launch.
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {
// Everything the kernel reads besides the maps travels in its parameters: nothing is copied to the device, so the launch
// captures into a CUDA graph.
struct StackParams {
    ActV src[HEAL_AGENT_STACK_MAX_SOURCES];
    int sh[HEAL_AGENT_STACK_MAX_SOURCES], sw[HEAL_AGENT_STACK_MAX_SOURCES];      // source height / width
    int top[HEAL_AGENT_STACK_MAX_SOURCES], left[HEAL_AGENT_STACK_MAX_SOURCES];   // source pixel of output (0, 0); < 0 = padding
    short agent_src[HEAL_AGENT_STACK_MAX_AGENTS], agent_img[HEAL_AGENT_STACK_MAX_AGENTS];
    ActV dst;
    int H, W;
};

// source pixel of output pixel `pix`, or -1 where the output is zero padding
__device__ __forceinline__ long long stack_source(const StackParams& p, size_t pix, int& s) {
    const size_t hw = (size_t)p.H * p.W;
    const int a = (int)(pix / hw);
    const int r = (int)(pix - (size_t)a * hw);
    const int y = r / p.W, x = r - (r / p.W) * p.W;
    s = p.agent_src[a];
    const int sy = y + p.top[s], sx = x + p.left[s];
    if (sy < 0 || sy >= p.sh[s] || sx < 0 || sx >= p.sw[s]) return -1;
    return ((long long)p.agent_img[a] * p.sh[s] + sy) * p.sw[s] + sx;
}

__global__ void k_agent_stack(const __grid_constant__ StackParams p, size_t npix, int chunks) {
    const size_t total = npix * (size_t)chunks;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / chunks;
        const int c = (int)(i % chunks) * 4;
        int s;
        const long long sp = stack_source(p, pix, s);
        act_store4(p.dst, pix, c, sp < 0 ? make_float4(0.f, 0.f, 0.f, 0.f) : act_load4(p.src[s], (size_t)sp, c));
    }
}

__global__ void k_agent_stack_scalar(const __grid_constant__ StackParams p, size_t npix, int channels) {
    const size_t total = npix * (size_t)channels;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / channels;
        const int c = (int)(i % channels);
        int s;
        const long long sp = stack_source(p, pix, s);
        act_store1(p.dst, pix, c, sp < 0 ? 0.f : act_load1(p.src[s], (size_t)sp, c));
    }
}
}  // namespace

// the vector rule of heal_act_convert: 16 B (fp32) or 8 B (bf16 / split) data pointers, channel stride, offset and split plane
// stride multiples of 4
static inline bool aligned4(const heal_act_t* a) {
    const uintptr_t need = a->fmt == 0 ? 15 : 7;
    return ((uintptr_t)a->data & need) == 0 && (a->cstride & 3) == 0 && (a->coffset & 3) == 0 &&
           (a->fmt != 2 || (a->plane_stride & 3) == 0);
}

static inline bool valid_view(const heal_act_t* a, int channels) {
    return a->data && a->fmt >= 0 && a->fmt <= 2 && a->coffset >= 0 && a->cstride >= a->coffset + channels;
}

// torchvision CenterCrop offset: int(round((s - t) / 2.0)), Python's round (halves to even); a negative offset is the
// zero padding (t - s) // 2 that CenterCrop puts before the map when t > s
static inline int center_offset(int s, int t) {
    if (t > s) return -((t - s) / 2);
    const int d = s - t, q = d / 2;
    return (d & 1) && (q & 1) ? q + 1 : q;
}

static inline ActV act_v(const heal_act_t* a) {
    ActV v;
    v.p = a->data; v.fmt = a->fmt; v.cs = a->cstride; v.co = a->coffset; v.plane = a->plane_stride;
    return v;
}

extern "C" int heal_agent_stack(const heal_stack_source_t* sources_host, int num_sources, const int* agent_source_host,
                                const int* agent_image_host, int num_agents, int channels, const heal_act_t* dst, int H, int W,
                                void* stream_) {
    if (!sources_host || !agent_source_host || !agent_image_host || !dst) return HEAL_ERR_ARG;
    if (num_sources < 1 || num_agents < 1 || channels < 1 || H < 1 || W < 1) return HEAL_ERR_ARG;
    if (num_sources > HEAL_AGENT_STACK_MAX_SOURCES || num_agents > HEAL_AGENT_STACK_MAX_AGENTS) return HEAL_ERR_UNSUPPORTED;
    if (!valid_view(dst, channels)) return HEAL_ERR_ARG;
    StackParams p;
    bool vec = (channels & 3) == 0 && aligned4(dst);
    for (int s = 0; s < num_sources; ++s) {
        const heal_stack_source_t& src = sources_host[s];
        if (!valid_view(&src.map, channels) || src.images < 1 || src.height < 1 || src.width < 1) return HEAL_ERR_ARG;
        if (!src.center_crop && (src.height != H || src.width != W)) return HEAL_ERR_ARG;
        vec = vec && aligned4(&src.map);
        p.src[s] = act_v(&src.map);
        p.sh[s] = src.height;
        p.sw[s] = src.width;
        p.top[s] = center_offset(src.height, H);
        p.left[s] = center_offset(src.width, W);
    }
    for (int a = 0; a < num_agents; ++a) {
        const int s = agent_source_host[a], i = agent_image_host[a];
        if (s < 0 || s >= num_sources || i < 0 || i >= sources_host[s].images) return HEAL_ERR_ARG;
        p.agent_src[a] = (short)s;
        p.agent_img[a] = (short)i;
    }
    p.dst = act_v(dst);
    p.H = H;
    p.W = W;
    const size_t npix = (size_t)num_agents * H * W;
    const size_t total = vec ? npix * (size_t)(channels / 4) : npix * (size_t)channels;
    const size_t blocks = (total + 255) / 256, cap = (size_t)HEAL_NUM_SMS * 16;
    const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
    if (vec) k_agent_stack<<<grid, 256, 0, (cudaStream_t)stream_>>>(p, npix, channels / 4);
    else k_agent_stack_scalar<<<grid, 256, 0, (cudaStream_t)stream_>>>(p, npix, channels);
    return heal_check_launch();
}
