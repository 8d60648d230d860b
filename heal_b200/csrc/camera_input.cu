// Camera input of Lift-Splat-Shoot at inference: raw uint8 RGB frames -> Pillow's resize (antialiased bicubic, 8-bit fixed point)
// -> crop (black outside the resized frame) -> ToTensor + Normalize(ImageNet mean / std), bit for bit
// (opencood/utils/camera_utils.py:62-91 `img_transform`, :120-125 `normalize_img`).
//   k_camera_input    one CTA per (output tile of 32 rows x 64 columns, image): the horizontal pass of the source rows the tile needs
//                     into a uint8 shared tile, then the vertical pass, the normalisation and the store, in either output layout
// The crop is folded into the coefficient tables the host builds (heal_b200/data_utils/camera_input.py): entry i of the column
// table describes column crop_left + i of the resized frame, with its first source column, its tap count (0 when the column lies
// outside the resized frame) and its int32 taps; the row table likewise.  An axis that keeps its size has one tap of 1 << 22 per
// entry, which reproduces the pass Pillow skips.  Integer sums, IEEE division: no atomics, the same bits on every run.
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr int TH = 32, TW = 64, THREADS = 256;
constexpr int PREC = 22;                                // Pillow's PRECISION_BITS for 8-bit images

__device__ __forceinline__ int clip8(int acc) {
    const int v = acc >> PREC;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// torchvision ToTensor (u / 255) then Normalize ((x - mean) / std), each step rounded to fp32
__device__ __forceinline__ float normalize(int u, int c) {
    const float mean = c == 0 ? 0.485f : (c == 1 ? 0.456f : 0.406f);
    const float std_ = c == 0 ? 0.229f : (c == 1 ? 0.224f : 0.225f);
    return (__int2float_rn(u) / 255.f - mean) / std_;
}

struct CamP {
    const uint8_t* frames;                   // (n_img, H0, W0, 3)
    const int* xtab; const int* ytab;        // (fW, 2 + xk), (fH, 2 + yk): start, count, taps
    float* out;
    int H0, W0, xk, yk, fH, fW, span, layout;
};

__global__ void __launch_bounds__(THREADS) k_camera_input(CamP p) {
    extern __shared__ uint8_t hs[];         // [rows r0 .. r1)[TW][3]: the horizontal pass of the source rows the tile needs
    const int img = blockIdx.z, y0 = blockIdx.y * TH, x0 = blockIdx.x * TW;
    const int th = min(TH, p.fH - y0), tw = min(TW, p.fW - x0);
    const int xs = 2 + p.xk, ys = 2 + p.yk;
    // the rows inside the resized frame are contiguous and their windows move monotonically, so the tile needs
    // [first row's start, last row's start + count)
    int first = -1, last = -1;
    for (int y = 0; y < th; ++y)
        if (__ldg(p.ytab + (size_t)(y0 + y) * ys + 1) > 0) { if (first < 0) first = y; last = y; }
    int r0 = 0, nr = 0;
    if (first >= 0) {
        r0 = __ldg(p.ytab + (size_t)(y0 + first) * ys);
        nr = __ldg(p.ytab + (size_t)(y0 + last) * ys) + __ldg(p.ytab + (size_t)(y0 + last) * ys + 1) - r0;
    }
    const bool fits = nr <= p.span;          // the host sizes `span` from the same tables; a table that breaks it gives NaN, not a stray read
    if (fits) {
        const uint8_t* src = p.frames + (size_t)img * p.H0 * p.W0 * 3;
        for (int i = threadIdx.x; i < nr * TW; i += THREADS) {
            const int r = i / TW, x = i - r * TW;
            int a0 = 1 << (PREC - 1), a1 = a0, a2 = a0;
            if (x < tw) {
                const int* t = p.xtab + (size_t)(x0 + x) * xs;
                const int n = __ldg(t + 1);
                const uint8_t* s = src + ((size_t)(r0 + r) * p.W0 + __ldg(t)) * 3;
                for (int k = 0; k < n; ++k) {
                    const int w = __ldg(t + 2 + k);
                    a0 += (int)__ldg(s + 3 * k) * w;
                    a1 += (int)__ldg(s + 3 * k + 1) * w;
                    a2 += (int)__ldg(s + 3 * k + 2) * w;
                }
            }
            hs[3 * i] = (uint8_t)clip8(a0); hs[3 * i + 1] = (uint8_t)clip8(a1); hs[3 * i + 2] = (uint8_t)clip8(a2);
        }
    }
    __syncthreads();
    auto value = [&](int c, int y, int x) -> float {
        if (!fits) return __int_as_float(0x7fc00000);
        const int* ty = p.ytab + (size_t)(y0 + y) * ys;
        const int* tx = p.xtab + (size_t)(x0 + x) * xs;
        const int n = __ldg(ty + 1);
        int u = 0;                                       // black outside the resized frame
        if (n > 0 && __ldg(tx + 1) > 0) {
            const uint8_t* h = hs + ((__ldg(ty) - r0) * TW + x) * 3 + c;
            int acc = 1 << (PREC - 1);
            for (int k = 0; k < n; ++k) acc += (int)h[k * TW * 3] * __ldg(ty + 2 + k);
            u = clip8(acc);
        }
        return normalize(u, c);
    };
    if (p.layout == 0) {
        // (n_img, 3, fH, fW) fp32: consecutive threads store consecutive columns
        for (int i = threadIdx.x; i < 3 * TH * TW; i += THREADS) {
            const int x = i % TW, y = (i / TW) % TH, c = i / (TW * TH);
            if (y >= th || x >= tw) continue;
            p.out[(((size_t)img * 3 + c) * p.fH + y0 + y) * p.fW + x0 + x] = value(c, y, x);
        }
    } else {
        // (n_img, fH/4, fW/4, 64) fp32, channel c*16 + dy*4 + dx, c == 3 zero: consecutive threads store consecutive channels
        const int H4 = p.fH / 4, W4 = p.fW / 4;
        for (int i = threadIdx.x; i < (TH / 4) * (TW / 4) * 64; i += THREADS) {
            const int ch = i & 63, X = (i >> 6) % (TW / 4), Y = (i >> 6) / (TW / 4);
            const int c = ch >> 4, y = 4 * Y + ((ch >> 2) & 3), x = 4 * X + (ch & 3);
            if (y >= th || x >= tw) continue;
            p.out[(((size_t)img * H4 + y0 / 4 + Y) * W4 + x0 / 4 + X) * 64 + ch] = c == 3 ? 0.f : value(c, y, x);
        }
    }
}

size_t g_smem_set[HEAL_MAX_DEVICES];

}  // namespace

extern "C" int heal_camera_input(const uint8_t* frames, int n_img, int H0, int W0, const int* col_table, int col_taps,
                                 const int* row_table, int row_taps, int fH, int fW, int span_rows, int layout, float* out,
                                 void* stream_) {
    if (!frames || !col_table || !row_table || !out || n_img < 1 || H0 < 1 || W0 < 1 || col_taps < 1 || row_taps < 1 || fH < 1 ||
        fW < 1 || span_rows < 1)
        return HEAL_ERR_ARG;
    if ((layout != 0 && layout != 1) || (layout == 1 && ((fH % 8) || (fW % 8))) || n_img > 65535) return HEAL_ERR_UNSUPPORTED;
    const size_t smem = (size_t)span_rows * TW * 3;
    if (smem > 227 * 1024) return HEAL_ERR_UNSUPPORTED;
    if (smem > 48 * 1024 && !heal_ensure_dyn_smem(k_camera_input, smem, g_smem_set)) return HEAL_ERR_DRIVER;
    CamP p;
    p.frames = frames; p.xtab = col_table; p.ytab = row_table; p.out = out;
    p.H0 = H0; p.W0 = W0; p.xk = col_taps; p.yk = row_taps; p.fH = fH; p.fW = fW; p.span = span_rows; p.layout = layout;
    const dim3 grid((fW + TW - 1) / TW, (fH + TH - 1) / TH, n_img);
    k_camera_input<<<grid, THREADS, smem, (cudaStream_t)stream_>>>(p);
    return heal_check_launch();
}
