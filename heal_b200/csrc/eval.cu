// Detection evaluation on the GPU: the true / false-positive matching the reference runs on the host once per frame and IoU threshold
// after post_process (opencood/tools/inference.py:171-185 -> opencood/utils/eval_utils.py:40-92 caluclate_tp_fp, with
// common_utils.py:230-270 compute_iou / convert_format: a shapely polygon loop over every detection and every unmatched GT).
// Pipeline (the caller's stream, no host sync):
//   k_polys  one thread per box (dets, then GTs): corners 0..3 (x, y) in fp64, made counter-clockwise, and the area (quad_iou.cuh)
//   k_rank   one thread per det: its place in descending score order, ties by ascending index (a stable sort; NaN scores last,
//            where np.argsort(-score) puts them) -> the permutation and the sorted scores
//   k_iou    one thread per (sorted det, GT): IoU = inter / (area_det + area_gt - inter) in fp64 with the det clipped against the
//            GT's edges, rounded once to fp32 (compute_iou's np.array(..., dtype=np.float32)); a zero union sets status bit 0
//            where the reference raises ZeroDivisionError
//   k_match  one warp per threshold, all thresholds at once: the greedy pass in score order (eval_utils.py:74-87).  Each det
//            reduces the max IoU and its first argmax over the GTs not yet taken; it is a TP unless no GT remains or max < thr in
//            fp32 (NumPy 2 casts the Python threshold to the array's float32), and a TP takes its argmax GT.
// Two entry points share these kernels.  heal_eval_tp_fp takes K and G from the host and sizes everything by them.
// heal_eval_tp_fp_counted reads K and G from device ints (e.g. the box count heal_box_decode_nms writes), so it can follow the
// post-processing in one captured graph: grids, workspace and output strides follow host capacities, every kernel reads the
// live counts and leaves the rows and columns beyond them alone, and a count above its capacity sets HEAL_EVAL_OVER_CAPACITY
// (k_polys) and makes every kernel return.
#include "common.cuh"
#include "quad_iou.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int kMaxBoxes = 4096;
constexpr int kMaxThr = 8;

struct Thresholds { float v[kMaxThr]; };

// The frame's sizes.  k_dev / g_dev NULL: the live counts are k / g (== kcap / gcap).  Else the live counts are *k_dev / *g_dev,
// read on the device, and kcap / gcap size the grids, the poly rows and the strides of the IoU matrix and of the flags.
struct Counts { const int* k_dev; const int* g_dev; int k, g, kcap, gcap; };

// the live (K, G); false when a device count lies outside [0, capacity] (nothing is then computed)
__device__ __forceinline__ bool live(const Counts& c, int& K, int& G) {
    K = c.k_dev ? __ldg(c.k_dev) : c.k;
    G = c.g_dev ? __ldg(c.g_dev) : c.g;
    return K >= 0 && K <= c.kcap && G >= 0 && G <= c.gcap;
}

// poly rows: 8 doubles (ccw x0 y0 .. x3 y3) + area; rows 0..kcap-1 the dets, kcap..kcap+gcap-1 the GTs
__global__ void k_polys(const float* __restrict__ det, const float* __restrict__ gt, Counts c, double* __restrict__ poly,
                        int* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int K, G;
    if (!live(c, K, G)) {
        if (i == 0) atomicOr(status, HEAL_EVAL_OVER_CAPACITY);
        return;
    }
    if (i < c.kcap ? i >= K : i - c.kcap >= G) return;
    quad_ccw(i < c.kcap ? det + (size_t)i * 24 : gt + (size_t)(i - c.kcap) * 24, poly + (size_t)i * 9);
}

// a ranks before b: descending score, NaN last, ties by ascending index
__device__ __forceinline__ bool ranks_before(float a, int ia, float b, int ib) {
    if (isnan(a)) return isnan(b) && ia < ib;
    if (isnan(b)) return true;
    return a > b || (a == b && ia < ib);
}

__global__ void __launch_bounds__(256)
k_rank(const float* __restrict__ scores, Counts c, int* __restrict__ perm, float* __restrict__ sorted_scores) {
    __shared__ float ss[1024];
    int K, G;
    if (!live(c, K, G)) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const float s = i < K ? scores[i] : 0.f;
    int rank = 0;
    for (int j0 = 0; j0 < K; j0 += 1024) {
        const int n = min(1024, K - j0);
        __syncthreads();
        for (int k = threadIdx.x; k < n; k += blockDim.x) ss[k] = scores[j0 + k];
        __syncthreads();
        if (i < K)
            for (int k = 0; k < n; ++k) rank += ranks_before(ss[k], j0 + k, s, i) ? 1 : 0;
    }
    if (i < K) { perm[rank] = i; sorted_scores[rank] = s; }
}

// row r of iou (stride gcap) = sorted det r against every GT
__global__ void __launch_bounds__(128)
k_iou(const double* __restrict__ poly, const int* __restrict__ perm, Counts c, float* __restrict__ iou, int* __restrict__ status) {
    int K, G;
    if (!live(c, K, G)) return;
    const int r = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= K || j >= G) return;
    double P[9], Q[9];
    const double* p = poly + (size_t)perm[r] * 9;
    const double* q = poly + (size_t)(c.kcap + j) * 9;
#pragma unroll
    for (int k = 0; k < 9; ++k) { P[k] = p[k]; Q[k] = q[k]; }
    const double inter = quad_bbox_disjoint(P, Q) ? 0.0 : quad_intersection(P, Q);
    const double uni = P[8] + Q[8] - inter;           // QuadPolygon.union: self.area + o.area - intersection, self = the det
    if (uni == 0.0) atomicOr(status, HEAL_EVAL_ZERO_UNION);
    iou[(size_t)r * c.gcap + j] = (float)(inter / uni);
}

// one warp per threshold (blockIdx.x); `taken` marks the GTs matched so far.  NaN IoUs (zero unions, reported in the status word)
// never win the max.  Flags of threshold t at tp[t * kcap ..].
__global__ void __launch_bounds__(32)
k_match(const float* __restrict__ iou, Counts c, Thresholds thr, unsigned char* __restrict__ tp) {
    __shared__ unsigned char taken[kMaxBoxes];
    int K, G;
    if (!live(c, K, G)) return;
    const int t = blockIdx.x, lane = threadIdx.x;
    for (int j = lane; j < G; j += 32) taken[j] = 0;
    __syncwarp();
    const float th = thr.v[t];
    int left = G;
    for (int r = 0; r < K; ++r) {
        unsigned char flag = 0;
        if (left > 0) {
            const float* row = iou + (size_t)r * c.gcap;
            float best = -INFINITY;
            int arg = 0x7fffffff;
#pragma unroll 4
            for (int j = lane; j < G; j += 32) {
                const float v = row[j];
                if (!taken[j] && v > best) { best = v; arg = j; }     // ascending j: the first maximum of this lane
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
                if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }   // np.argmax: the lowest index of the maxima
            }
            if (best >= th) {                           // not (np.max(ious) < iou_thresh) in fp32
                flag = 1;
                if (lane == 0) taken[arg] = 1;
                --left;
            }
            __syncwarp();
        }
        if (lane == 0) tp[(size_t)t * c.kcap + r] = flag;
    }
}

struct WsLayout { size_t poly, perm, iou, total; };

WsLayout layout(int K, int G) {
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    WsLayout L;
    size_t o = 0;
    L.poly = o; o = al(o + (size_t)(K + G) * 9 * 8);
    L.perm = o; o = al(o + (size_t)K * 4);
    L.iou = o; o = al(o + (size_t)K * G * 4);
    L.total = o > 0 ? o : 256;
    return L;
}

// the thresholds of a call -> the kernel argument; false for a count outside [1, 8] or a threshold that is not > 0 (NaN included)
bool thresholds(const float* thresholds_host, int n_thr, Thresholds& thr) {
    if (n_thr < 1 || n_thr > kMaxThr || !thresholds_host) return false;
    for (int t = 0; t < kMaxThr; ++t) thr.v[t] = 0.f;
    for (int t = 0; t < n_thr; ++t) {
        if (!(thresholds_host[t] > 0.f)) return false;
        thr.v[t] = thresholds_host[t];
    }
    return true;
}

// the kernels over kcap >= 1 dets and gcap GTs (k_iou only when gcap > 0); status_out cleared first
int launch(const float* det_corners, const float* det_scores, const float* gt_corners, const Counts& c, const Thresholds& thr,
           int n_thr, float* sorted_scores_out, unsigned char* tp_out, int* status_out, void* ws, cudaStream_t st) {
    const WsLayout L = layout(c.kcap, c.gcap);
    uint8_t* w = (uint8_t*)ws;
    double* poly = (double*)(w + L.poly);
    int* perm = (int*)(w + L.perm);
    float* iou = (float*)(w + L.iou);
    k_polys<<<(c.kcap + c.gcap + 127) / 128, 128, 0, st>>>(det_corners, gt_corners, c, poly, status_out);
    k_rank<<<(c.kcap + 255) / 256, 256, 0, st>>>(det_scores, c, perm, sorted_scores_out);
    if (c.gcap > 0) k_iou<<<dim3((c.gcap + 127) / 128, c.kcap), 128, 0, st>>>(poly, perm, c, iou, status_out);
    k_match<<<n_thr, 32, 0, st>>>(iou, c, thr, tp_out);
    return heal_check_launch(c.gcap > 0 ? 4 : 3);
}

}  // namespace

extern "C" size_t heal_eval_workspace(int K, int G) {
    if (K < 0 || G < 0) return 0;
    return layout(K, G).total;
}

extern "C" int heal_eval_tp_fp(const float* det_corners, const float* det_scores, int K, const float* gt_corners, int G,
                               const float* thresholds_host, int n_thr, float* sorted_scores_out, unsigned char* tp_out,
                               int* status_out, void* ws, size_t ws_bytes, void* stream_) {
    Thresholds thr;
    if (K < 0 || K > kMaxBoxes || G < 0 || G > kMaxBoxes || !thresholds(thresholds_host, n_thr, thr) || !status_out)
        return HEAL_ERR_ARG;
    if (K > 0 && (!det_corners || !det_scores || !sorted_scores_out || !tp_out)) return HEAL_ERR_ARG;
    if (G > 0 && !gt_corners) return HEAL_ERR_ARG;
    if (!ws || ws_bytes < layout(K, G).total) return HEAL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    if (cudaMemsetAsync(status_out, 0, sizeof(int), st) != cudaSuccess) return HEAL_ERR_LAUNCH;
    if (K == 0) return HEAL_OK;
    const Counts c{nullptr, nullptr, K, G, K, G};
    return launch(det_corners, det_scores, gt_corners, c, thr, n_thr, sorted_scores_out, tp_out, status_out, ws, st);
}

extern "C" int heal_eval_tp_fp_counted(const float* det_corners, const float* det_scores, const int* det_count, int K_cap,
                                       const float* gt_corners, const int* gt_count, int G_cap, const float* thresholds_host,
                                       int n_thr, float* sorted_scores_out, unsigned char* tp_out, int* status_out, void* ws,
                                       size_t ws_bytes, void* stream_) {
    Thresholds thr;
    if (K_cap < 1 || K_cap > kMaxBoxes || G_cap < 1 || G_cap > kMaxBoxes || !thresholds(thresholds_host, n_thr, thr))
        return HEAL_ERR_ARG;
    if (!det_corners || !det_scores || !det_count || !gt_corners || !gt_count || !sorted_scores_out || !tp_out || !status_out)
        return HEAL_ERR_ARG;
    if (!ws || ws_bytes < layout(K_cap, G_cap).total) return HEAL_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    if (cudaMemsetAsync(status_out, 0, sizeof(int), st) != cudaSuccess) return HEAL_ERR_LAUNCH;
    const Counts c{det_count, gt_count, 0, 0, K_cap, G_cap};
    return launch(det_corners, det_scores, gt_corners, c, thr, n_thr, sorted_scores_out, tp_out, status_out, ws, st);
}
