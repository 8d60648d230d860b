// Detection post-processing on the GPU (SURVEY.md 8f rank 1): the reference does this on the host after a D2H copy of the heads
// (torch masked_select + a shapely polygon loop over the top-1000 boxes).
// Reference: opencood/data_utils/post_processor/voxel_postprocessor.py:245-405 (post_process), :408-453 (delta_to_boxes3d);
//            opencood/utils/box_utils.py:152-204 (boxes_to_corners_3d), :278-316 (project_box3d), :693-738 (nms_rotated),
//            :840-890 (remove_large_pred_bbx / remove_bbx_abnormal_z), :384-421 (mask_boxes_outside_range_numpy);
//            opencood/utils/common_utils.py:104-113 (limit_period), :230-270 (compute_iou / convert_format).
// Pipeline (all on the caller's stream, no host sync; the counts stay on the device):
//   k_decode      one thread per anchor (late entry point: blockIdx.y = cav, its 4x4 transform read on the device): sigmoid, score threshold, delta decode, direction-bin fix, 8 corners, ego projection,
//                 size / z filters -> sort key (score or -1) + the 24 corner floats
//   cub radix sort (descending, stable) of (key, anchor index): the reference's `scores.argsort()[::-1][:top]`
//   k_gather_top  the `top` best: corners, score, the 2-D polygon (corners 0..3, x/y) made counter-clockwise, its area (fp64)
//   k_iou_mask    64 x 64 tiles of the upper triangle: convex-quad intersection by Sutherland-Hodgman clipping in fp64
//                 (the same operation order as oracle/postprocess.py), bit j of word (i, j/64) = IoU(i, j) > threshold
//   k_nms_finish  one warp: greedy scan in score order (lane w owns word w of the removed set), then the 8-corners-in-range mask,
//                 ordered compaction of the survivors into the output
// Traps kept: remove_large_pred_bbx takes its "z length" from the y column and only tests it for truthiness (box_utils.py:862-867);
// IoU is compared as float32; a zero-area union gives NaN and never suppresses.
// Order: descending score, then ascending candidate slot (cav * H*W*A + (h*W + w)*A + a) on ties -- the stable sort's order.
// Where the kernel and torch differ by design (NaN logits only): a NaN direction logit never wins the argmax scan (a NaN in bin 0
// keeps bin 0), and a NaN IoU logit counts as IoU 0 (fmaxf(NaN, 0) = 0, score * 1/16) where torch's clamp would give a NaN score.
#include <cub/cub.cuh>

#include "common.cuh"
#include "quad_iou.cuh"
#include "../../include/heal_b200.h"

namespace {

struct DecP {
    ActV cls, reg, dir, iou;       // (1,H,W,A) logits, (1,H,W,7A) deltas, (1,H,W,A*bins) or null, (1,H,W,A) IoU logits or null -- fp32 channels-last
    int base;                      // first candidate slot of this cav (late fusion: the cavs' anchors are concatenated in cav order)
    const float* anchors;          // (H,W,A,7)
    int H, W, A, bins, hwl;
    float thr, dir_offset;
    float T[12];                   // rows 0..2 of the 4x4 cav -> ego transform (host-given; used when Tdev is null)
    const float* Tdev;             // or: device (gridDim.y, 4, 4) row-major transforms, cav = blockIdx.y, heads (gridDim.y, H, W, .)
    float* keys; int* vals; float* cand;    // per anchor: sort key, index, 24 corner floats
    int* counters;                 // [0] above the score threshold, [1] after the size / z filters
};

__device__ __forceinline__ float ldf(const ActV& a, size_t pix, int c) {
    return __ldg(reinterpret_cast<const float*>(a.p) + pix * (size_t)a.cs + (size_t)(a.co + c));
}

__global__ void __launch_bounds__(256)
k_decode(DecP p) {
    const int n = p.H * p.W * p.A;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int cav = blockIdx.y;
    const int a = i % p.A; const size_t pix = (size_t)cav * p.H * p.W + (size_t)(i / p.A);
    const int slot = p.base + cav * n + i;
    float T[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) T[k] = p.Tdev ? __ldg(p.Tdev + (size_t)cav * 16 + k) : p.T[k];
    p.vals[slot] = slot;
    float key = -1.f;
    const float prob = 1.f / (1.f + expf(-ldf(p.cls, pix, a)));
    if (prob > p.thr) {
        atomicAdd(p.counters + 0, 1);
        const float* an = p.anchors + (size_t)i * 7;
        float d[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) d[k] = ldf(p.reg, pix, a * 7 + k);
        const float ad = sqrtf(an[4] * an[4] + an[5] * an[5]);
        float b[7];
        b[0] = d[0] * ad + an[0];
        b[1] = d[1] * ad + an[1];
        b[2] = d[2] * an[3] + an[2];
        b[3] = expf(d[3]) * an[3];
        b[4] = expf(d[4]) * an[4];
        b[5] = expf(d[5]) * an[5];
        b[6] = d[6] + an[6];
        if (p.dir.p) {
            int lab = 0; float best = ldf(p.dir, pix, a * p.bins);
            for (int q = 1; q < p.bins; ++q) { float v = ldf(p.dir, pix, a * p.bins + q); if (v > best) { best = v; lab = q; } }
            const float period = (float)(2.0 * 3.14159265358979323846 / (double)p.bins);
            const float twopi = (float)(2.0 * 3.14159265358979323846);
            const float v = b[6] - p.dir_offset;
            const float rot = v - floorf(v / period + 0.f) * period;
            const float y2 = rot + p.dir_offset + period * (float)lab;
            b[6] = y2 - floorf(y2 / twopi + 0.5f) * twopi;
        }
        // corners: 'hwl' boxes are [x y z h w l yaw] -> dims (l, w, h); template order of boxes_to_corners_3d
        const float dx = p.hwl ? b[5] : b[3], dy = b[4], dz = p.hwl ? b[3] : b[5];
        const float ca = cosf(b[6]), sa = sinf(b[6]);
        const float sx[8] = {1, 1, -1, -1, 1, 1, -1, -1}, sy[8] = {-1, 1, 1, -1, -1, 1, 1, -1}, sz[8] = {-1, -1, -1, -1, 1, 1, 1, 1};
        float c[24];
        float xmin = INFINITY, xmax = -INFINITY, ymin = INFINITY, ymax = -INFINITY, zmin = INFINITY, zmax = -INFINITY;
        bool has_nan = false;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float lx = dx * (sx[k] * 0.5f), ly = dy * (sy[k] * 0.5f), lz = dz * (sz[k] * 0.5f);
            const float x = lx * ca + ly * (-sa) + b[0], y = lx * sa + ly * ca + b[1], z = lz + b[2];
            const float X = T[0] * x + T[1] * y + T[2] * z + T[3];
            const float Y = T[4] * x + T[5] * y + T[6] * z + T[7];
            const float Z = T[8] * x + T[9] * y + T[10] * z + T[11];
            c[3 * k] = X; c[3 * k + 1] = Y; c[3 * k + 2] = Z;
            xmin = fminf(xmin, X); xmax = fmaxf(xmax, X); ymin = fminf(ymin, Y); ymax = fmaxf(ymax, Y);
            zmin = fminf(zmin, Z); zmax = fmaxf(zmax, Z);
            has_nan = has_nan || isnan(X) || isnan(Y) || isnan(Z);
        }
        // fminf / fmaxf skip a NaN, torch's max / min return it: a box with a NaN corner (a NaN yaw or size delta) has NaN
        // lengths in the reference and fails every filter there, so it is dropped here too
        const float xl = xmax - xmin, yl = ymax - ymin;
        const bool keep = !has_nan && (xl <= 6.f) && (yl <= 6.f) && (yl != 0.f) && (zmin >= -3.f) && (zmax <= 1.f);
        if (keep) {
            atomicAdd(p.counters + 1, 1);
            key = prob;
            if (p.iou.p) {     // voxel_postprocessor.py:343-347: score *= ((clamp(sigmoid(iou), 0, 1) + 1) / 2) ^ 4
                float q = 1.f / (1.f + expf(-ldf(p.iou, pix, a)));
                q = (fminf(fmaxf(q, 0.f), 1.f) + 1.f) * 0.5f;
                key = prob * powf(q, 4.f);
            }
            float* o = p.cand + (size_t)slot * 24;
#pragma unroll
            for (int k = 0; k < 24; ++k) o[k] = c[k];
        }
    }
    p.keys[slot] = key;
}

// top rows: [24 corner floats]; poly rows: 8 doubles (ccw x0 y0 .. x3 y3) + area
__global__ void k_gather_top(const float* __restrict__ keys_sorted, const int* __restrict__ vals_sorted, const float* __restrict__ cand,
                             const int* __restrict__ counters, int top, float* __restrict__ top_c, float* __restrict__ top_s,
                             double* __restrict__ poly, float lx, float ly, float lz, float hx, float hy, float hz, int use_range,
                             unsigned char* __restrict__ inrange) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(counters[1], top);
    if (r >= n) return;
    const float* src = cand + (size_t)vals_sorted[r] * 24;
    float c[24];
#pragma unroll
    for (int k = 0; k < 24; ++k) { c[k] = src[k]; top_c[(size_t)r * 24 + k] = c[k]; }
    top_s[r] = keys_sorted[r];
    bool in = true;                       // mask_boxes_outside_range_numpy: all 8 corners inside [min, max] on x, y and z
    if (use_range) {
#pragma unroll
        for (int k = 0; k < 8; ++k)
            in = in && (c[3 * k] >= lx) && (c[3 * k] <= hx) && (c[3 * k + 1] >= ly) && (c[3 * k + 1] <= hy) && (c[3 * k + 2] >= lz) && (c[3 * k + 2] <= hz);
    }
    inrange[r] = in ? 1 : 0;
    quad_ccw(c, poly + (size_t)r * 9);
}

__global__ void __launch_bounds__(64)
k_iou_mask(const double* __restrict__ poly, const int* __restrict__ counters, int top, float thr, int words,
           unsigned long long* __restrict__ mask) {
    const int n = min(counters[1], top);
    const int row0 = blockIdx.y * 64, col0 = blockIdx.x * 64;
    if (row0 >= n || col0 >= n || blockIdx.x < blockIdx.y) return;      // upper triangle only
    __shared__ double sq[64 * 9];
    const int cols = min(64, n - col0);
    for (int k = threadIdx.x; k < cols * 9; k += 64) sq[k] = poly[(size_t)col0 * 9 + k];
    __syncthreads();
    const int i = row0 + threadIdx.x;
    if (i >= n) return;
    double P[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) P[k] = poly[(size_t)i * 9 + k];
    const double pminx = fmin(fmin(P[0], P[2]), fmin(P[4], P[6])), pmaxx = fmax(fmax(P[0], P[2]), fmax(P[4], P[6]));
    const double pminy = fmin(fmin(P[1], P[3]), fmin(P[5], P[7])), pmaxy = fmax(fmax(P[1], P[3]), fmax(P[5], P[7]));
    unsigned long long bits = 0ull;
    for (int jj = 0; jj < cols; ++jj) {
        const int j = col0 + jj;
        if (j <= i) continue;
        const double* Q = sq + jj * 9;
        // disjoint bounding boxes: the clip would come back empty (IoU 0, or NaN for two zero-area boxes) -> never above the threshold
        if (pmaxx < fmin(fmin(Q[0], Q[2]), fmin(Q[4], Q[6])) || fmax(fmax(Q[0], Q[2]), fmax(Q[4], Q[6])) < pminx ||
            pmaxy < fmin(fmin(Q[1], Q[3]), fmin(Q[5], Q[7])) || fmax(fmax(Q[1], Q[3]), fmax(Q[5], Q[7])) < pminy) continue;
        const double inter = quad_intersection(P, sq + jj * 9);
        const double uni = P[8] + sq[jj * 9 + 8] - inter;
        const float iou = (float)(inter / uni);              // NaN for a zero-area union: never suppresses
        if (iou > thr) bits |= 1ull << jj;
    }
    mask[(size_t)i * words + blockIdx.x] = bits;
}

// One block: all threads stage the suppression matrix (top x words x 8 B <= 128 KiB for top = 1000) and the in-range flags in shared
// memory, then warp 0 does the greedy scan from there and lists the survivors that are also in range; k_emit copies them in
// parallel.  (Reading the mask row and the corners of every kept box straight from global memory inside the scan costs two
// dependent global-memory loads per box on the serial path.)
__global__ void __launch_bounds__(1024)
k_nms_finish(const unsigned long long* __restrict__ mask, const unsigned char* __restrict__ inrange, const int* __restrict__ counters,
             int top, int words, int* __restrict__ keep_idx, int* __restrict__ count_out) {
    extern __shared__ unsigned long long smask[];
    const int n = min(counters[1], top);
    unsigned char* srange = reinterpret_cast<unsigned char*>(smask + (size_t)top * words);
    for (int k = threadIdx.x; k < n * words; k += blockDim.x) smask[k] = mask[k];
    for (int k = threadIdx.x; k < n; k += blockDim.x) srange[k] = inrange[k];
    __syncthreads();
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    unsigned long long removed = 0ull;        // lane w owns bits [64w, 64w+64)
    int kept = 0;
    for (int i = 0; i < n; ++i) {
        const int w = i >> 6;
        const unsigned long long mine = __shfl_sync(0xffffffffu, removed, w);
        if ((mine >> (i & 63)) & 1ull) continue;
        // box i survives the NMS: it suppresses its overlaps whether or not it passes the range mask applied afterwards
        if (lane < words && lane >= w) removed |= smask[(size_t)i * words + lane];
        if (srange[i]) {
            if (lane == 0) keep_idx[kept] = i;
            ++kept;
        }
    }
    if (lane == 0) *count_out = kept;
}

__global__ void k_emit(const int* __restrict__ keep_idx, const int* __restrict__ count, const float* __restrict__ top_c,
                       const float* __restrict__ top_s, float* __restrict__ boxes_out, float* __restrict__ scores_out) {
    const int r = blockIdx.x;
    if (r >= *count) return;
    const int i = keep_idx[r];
    if (threadIdx.x < 24) boxes_out[(size_t)r * 24 + threadIdx.x] = top_c[(size_t)i * 24 + threadIdx.x];
    if (threadIdx.x == 24) scores_out[r] = top_s[i];
}

inline ActV to_view(const heal_act_t* a) {
    ActV v;
    v.p = a->data; v.fmt = a->fmt; v.cs = a->cstride; v.co = a->coffset; v.plane = a->plane_stride;
    return v;
}

struct WsLayout {
    size_t keys_in, keys_out, vals_in, vals_out, cand, counters, top_c, top_s, poly, mask, inrange, keep, cub, total, cub_bytes;
    int words;
};

WsLayout layout(int n, int top) {
    WsLayout L;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t o = 0;
    L.keys_in = o; o = al(o + (size_t)n * 4);
    L.keys_out = o; o = al(o + (size_t)n * 4);
    L.vals_in = o; o = al(o + (size_t)n * 4);
    L.vals_out = o; o = al(o + (size_t)n * 4);
    L.cand = o; o = al(o + (size_t)n * 24 * 4);
    L.counters = o; o = al(o + 16);
    L.top_c = o; o = al(o + (size_t)top * 24 * 4);
    L.top_s = o; o = al(o + (size_t)top * 4);
    L.poly = o; o = al(o + (size_t)top * 9 * 8);
    L.words = (top + 63) / 64;
    L.mask = o; o = al(o + (size_t)top * L.words * 8);
    L.inrange = o; o = al(o + (size_t)top);
    L.keep = o; o = al(o + (size_t)top * 4);
    size_t cb = 0;
    cub::DeviceRadixSort::SortPairsDescending(nullptr, cb, (const float*)nullptr, (float*)nullptr, (const int*)nullptr, (int*)nullptr, n);
    L.cub_bytes = cb;
    L.cub = o; o = al(o + cb);
    L.total = o;
    return L;
}

// The chain after the decode, shared by the multi and the late entry points: sort -> k_gather_top -> k_iou_mask -> k_nms_finish
// -> k_emit (+ the stats copy).  `p` holds the workspace pointers the decode filled.
int sort_nms_emit(const WsLayout& L, uint8_t* ws, const DecP& p, int n, int top, const float* range6_host, float nms_threshold,
                  float* boxes_out, float* scores_out, int* count_out, int* stats_out, cudaStream_t st) {
    size_t cb = L.cub_bytes;
    if (cub::DeviceRadixSort::SortPairsDescending(ws + L.cub, cb, (const float*)p.keys, (float*)(ws + L.keys_out), (const int*)p.vals,
                                                  (int*)(ws + L.vals_out), n, 0, 32, st) != cudaSuccess) return HEAL_ERR_LAUNCH;
    const float* r = range6_host;
    const float rl[6] = {r ? r[0] : 0.f, r ? r[1] : 0.f, r ? r[2] : 0.f, r ? r[3] : 0.f, r ? r[4] : 0.f, r ? r[5] : 0.f};
    k_gather_top<<<(top + 127) / 128, 128, 0, st>>>((const float*)(ws + L.keys_out), (const int*)(ws + L.vals_out), p.cand, p.counters, top,
                                                    (float*)(ws + L.top_c), (float*)(ws + L.top_s), (double*)(ws + L.poly),
                                                    rl[0], rl[1], rl[2], rl[3], rl[4], rl[5], r ? 1 : 0, (unsigned char*)(ws + L.inrange));
    dim3 g((top + 63) / 64, (top + 63) / 64);
    k_iou_mask<<<g, 64, 0, st>>>((const double*)(ws + L.poly), p.counters, top, nms_threshold, L.words, (unsigned long long*)(ws + L.mask));
    const size_t nms_smem = (size_t)top * L.words * 8 + (((size_t)top + 15) & ~(size_t)15);
    static size_t nms_attr[HEAL_MAX_DEVICES] = {};
    if (!heal_ensure_dyn_smem(k_nms_finish, nms_smem, nms_attr)) return HEAL_ERR_LAUNCH;
    k_nms_finish<<<1, 1024, nms_smem, st>>>((const unsigned long long*)(ws + L.mask), (const unsigned char*)(ws + L.inrange), p.counters, top,
                                            L.words, (int*)(ws + L.keep), count_out);
    k_emit<<<top, 32, 0, st>>>((const int*)(ws + L.keep), count_out, (const float*)(ws + L.top_c), (const float*)(ws + L.top_s),
                               boxes_out, scores_out);
    if (stats_out) cudaMemcpyAsync(stats_out, p.counters, 8, cudaMemcpyDeviceToDevice, st);
    return HEAL_OK;
}

}  // namespace

extern "C" size_t heal_postprocess_workspace(int H, int W, int anchors_per_cell, int top) {
    if (H < 1 || W < 1 || anchors_per_cell < 1 || top < 1) return 0;
    return layout(H * W * anchors_per_cell, top).total;
}

extern "C" int heal_box_decode_nms_multi(const heal_cav_heads_t* cavs_host, int n_cav, int H, int W, int anchors_per_cell,
                                         float score_threshold, float dir_offset, int num_bins, int order_hwl, float nms_threshold,
                                         int top, const float* range6_host, float* boxes_out, float* scores_out, int* count_out,
                                         int* stats_out, void* workspace, size_t workspace_bytes, void* stream_) {
    if (!cavs_host || n_cav < 1 || n_cav > 16 || !boxes_out || !scores_out || !count_out || !workspace) return HEAL_ERR_ARG;
    if (H < 1 || W < 1 || anchors_per_cell < 1 || top < 1 || top > 1320 || num_bins < 1) return HEAL_ERR_ARG;   // mask must fit 227 KiB of smem
    const int n1 = H * W * anchors_per_cell;
    const long long nt = (long long)n1 * n_cav;
    if (nt >= (1LL << 30)) return HEAL_ERR_UNSUPPORTED;
    const int n = (int)nt;
    const WsLayout L = layout(n, top);
    if (workspace_bytes < L.total) return HEAL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    uint8_t* ws = (uint8_t*)workspace;
    DecP p;
    p.H = H; p.W = W; p.A = anchors_per_cell; p.bins = num_bins; p.hwl = order_hwl ? 1 : 0;
    p.thr = score_threshold; p.dir_offset = dir_offset;
    p.keys = (float*)(ws + L.keys_in); p.vals = (int*)(ws + L.vals_in); p.cand = (float*)(ws + L.cand);
    p.counters = (int*)(ws + L.counters);
    p.Tdev = nullptr;
    cudaMemsetAsync(p.counters, 0, 16, st);
    cudaMemsetAsync(ws + L.mask, 0, (size_t)top * L.words * 8, st);
    for (int c = 0; c < n_cav; ++c) {
        const heal_cav_heads_t& h = cavs_host[c];
        if (!h.cls || !h.cls->data || !h.reg || !h.reg->data || !h.anchors || !h.transform4x4_host) return HEAL_ERR_ARG;
        if (h.cls->fmt != 0 || h.reg->fmt != 0 || (h.dir && h.dir->data && h.dir->fmt != 0) || (h.iou && h.iou->data && h.iou->fmt != 0))
            return HEAL_ERR_UNSUPPORTED;
        p.cls = to_view(h.cls); p.reg = to_view(h.reg);
        if (h.dir && h.dir->data) p.dir = to_view(h.dir); else { p.dir = p.cls; p.dir.p = nullptr; }
        if (h.iou && h.iou->data) p.iou = to_view(h.iou); else { p.iou = p.cls; p.iou.p = nullptr; }
        p.anchors = h.anchors; p.base = c * n1;
        for (int k = 0; k < 12; ++k) p.T[k] = h.transform4x4_host[k];
        k_decode<<<(n1 + 255) / 256, 256, 0, st>>>(p);
    }
    const int rc = sort_nms_emit(L, ws, p, n, top, range6_host, nms_threshold, boxes_out, scores_out, count_out, stats_out, st);
    if (rc != HEAL_OK) return rc;
    return heal_check_launch(4 + n_cav);
}

extern "C" int heal_box_decode_nms_late(const heal_act_t* cls, const heal_act_t* reg, const heal_act_t* dir, const float* anchors,
                                        const float* transforms_dev, int n_cav, int H, int W, int anchors_per_cell,
                                        float score_threshold, float dir_offset, int num_bins, int order_hwl, float nms_threshold,
                                        int top, const float* range6_host, float* boxes_out, float* scores_out, int* count_out,
                                        int* stats_out, void* workspace, size_t workspace_bytes, void* stream_) {
    if (n_cav < 1 || n_cav > 16 || !cls || !cls->data || !reg || !reg->data || !anchors || !transforms_dev) return HEAL_ERR_ARG;
    if (!boxes_out || !scores_out || !count_out || !workspace) return HEAL_ERR_ARG;
    if (H < 1 || W < 1 || anchors_per_cell < 1 || top < 1 || top > 1320 || num_bins < 1) return HEAL_ERR_ARG;
    if (cls->fmt != 0 || reg->fmt != 0 || (dir && dir->data && dir->fmt != 0)) return HEAL_ERR_UNSUPPORTED;
    const int n1 = H * W * anchors_per_cell;
    const long long nt = (long long)n1 * n_cav;
    if (nt >= (1LL << 30)) return HEAL_ERR_UNSUPPORTED;
    const int n = (int)nt;
    const WsLayout L = layout(n, top);
    if (workspace_bytes < L.total) return HEAL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    uint8_t* ws = (uint8_t*)workspace;
    DecP p;
    p.H = H; p.W = W; p.A = anchors_per_cell; p.bins = num_bins; p.hwl = order_hwl ? 1 : 0;
    p.thr = score_threshold; p.dir_offset = dir_offset;
    p.keys = (float*)(ws + L.keys_in); p.vals = (int*)(ws + L.vals_in); p.cand = (float*)(ws + L.cand);
    p.counters = (int*)(ws + L.counters);
    p.cls = to_view(cls); p.reg = to_view(reg);
    if (dir && dir->data) p.dir = to_view(dir); else { p.dir = p.cls; p.dir.p = nullptr; }
    p.iou = p.cls; p.iou.p = nullptr;
    p.anchors = anchors; p.base = 0; p.Tdev = transforms_dev;
    cudaMemsetAsync(p.counters, 0, 16, st);
    cudaMemsetAsync(ws + L.mask, 0, (size_t)top * L.words * 8, st);
    k_decode<<<dim3((n1 + 255) / 256, n_cav), 256, 0, st>>>(p);
    const int rc = sort_nms_emit(L, ws, p, n, top, range6_host, nms_threshold, boxes_out, scores_out, count_out, stats_out, st);
    if (rc != HEAL_OK) return rc;
    return heal_check_launch(5);
}

extern "C" int heal_box_decode_nms(const heal_act_t* cls, const heal_act_t* reg, const heal_act_t* dir, const float* anchors,
                                   int H, int W, int anchors_per_cell, float score_threshold, float dir_offset, int num_bins,
                                   const float* transform4x4_host, int order_hwl, float nms_threshold, int top,
                                   const float* range6_host, float* boxes_out, float* scores_out, int* count_out, int* stats_out,
                                   void* workspace, size_t workspace_bytes, void* stream_) {
    heal_cav_heads_t h;
    h.cls = cls; h.reg = reg; h.dir = dir; h.iou = nullptr; h.anchors = anchors; h.transform4x4_host = transform4x4_host;
    return heal_box_decode_nms_multi(&h, 1, H, W, anchors_per_cell, score_threshold, dir_offset, num_bins, order_hwl, nms_threshold, top,
                                     range6_host, boxes_out, scores_out, count_out, stats_out, workspace, workspace_bytes, stream_);
}
