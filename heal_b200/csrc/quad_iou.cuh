// fp64 convex-quad geometry shared by the rotated NMS (postprocess.cu) and the TP / FP matching (eval.cu): the reference's shapely
// Polygon of a box's corners 0..3 (x, y) (common_utils.py:255-270 convert_format), its area and the area of the intersection of two
// such polygons.  The operation order is the one of oracle/postprocess.py:QuadPolygon (Sutherland-Hodgman clipping).
#pragma once
#include <math.h>

// corners 0..3 (x, y) of one (8, 3) fp32 box -> o[0..7] = x0 y0 .. x3 y3 counter-clockwise (a clockwise quad is reversed, as the
// stand-in's p[::-1]), o[8] = its area |sum / 2|
static __device__ __forceinline__ void quad_ccw(const float* c, double* o) {
    double x[4], y[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { x[k] = (double)c[3 * k]; y[k] = (double)c[3 * k + 1]; }
    double a2 = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) a2 += x[k] * y[(k + 1) & 3] - y[k] * x[(k + 1) & 3];
    if (a2 < 0.0) {                       // clockwise -> reverse (oracle: p[::-1])
#pragma unroll
        for (int k = 0; k < 4; ++k) { o[2 * k] = x[3 - k]; o[2 * k + 1] = y[3 - k]; }
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) { o[2 * k] = x[k]; o[2 * k + 1] = y[k]; }
    }
    o[8] = fabs(0.5 * a2);
}

static __device__ __forceinline__ double poly_area2(const double* px, const double* py, int n) {
    double s = 0.0;
    for (int k = 0; k < n; ++k) { const int k1 = (k + 1 == n) ? 0 : k + 1; s += px[k] * py[k1] - py[k] * px[k1]; }
    return s;
}

// intersection area of two counter-clockwise convex quads: clip P against the 4 directed edges of Q (keep the left side)
static __device__ double quad_intersection(const double* P, const double* Q) {
    double ax[10], ay[10], bx[10], by[10];
    int n = 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) { ax[k] = P[2 * k]; ay[k] = P[2 * k + 1]; }
    for (int e = 0; e < 4; ++e) {
        const double qx = Q[2 * e], qy = Q[2 * e + 1];
        const double ex = Q[2 * ((e + 1) & 3)] - qx, ey = Q[2 * ((e + 1) & 3) + 1] - qy;
        int m = 0;
        for (int k = 0; k < n; ++k) {
            const int k1 = (k + 1 == n) ? 0 : k + 1;
            const double sp = ex * (ay[k] - qy) - ey * (ax[k] - qx);
            const double sq = ex * (ay[k1] - qy) - ey * (ax[k1] - qx);
            if (sp >= 0.0) { bx[m] = ax[k]; by[m] = ay[k]; ++m; }
            if ((sp > 0.0 && sq < 0.0) || (sp < 0.0 && sq > 0.0)) {
                const double t = sp / (sp - sq);
                bx[m] = ax[k] + t * (ax[k1] - ax[k]); by[m] = ay[k] + t * (ay[k1] - ay[k]); ++m;
            }
        }
        n = m;
        if (n < 3) return 0.0;
        for (int k = 0; k < n; ++k) { ax[k] = bx[k]; ay[k] = by[k]; }
    }
    return fabs(0.5 * poly_area2(ax, ay, n));
}

// the axis-aligned bounding boxes of two ccw quads (as quad_ccw writes them) do not touch: the clip would come back empty
static __device__ __forceinline__ bool quad_bbox_disjoint(const double* P, const double* Q) {
    const double pminx = fmin(fmin(P[0], P[2]), fmin(P[4], P[6])), pmaxx = fmax(fmax(P[0], P[2]), fmax(P[4], P[6]));
    const double pminy = fmin(fmin(P[1], P[3]), fmin(P[5], P[7])), pmaxy = fmax(fmax(P[1], P[3]), fmax(P[5], P[7]));
    return pmaxx < fmin(fmin(Q[0], Q[2]), fmin(Q[4], Q[6])) || fmax(fmax(Q[0], Q[2]), fmax(Q[4], Q[6])) < pminx ||
           pmaxy < fmin(fmin(Q[1], Q[3]), fmin(Q[5], Q[7])) || fmax(fmax(Q[1], Q[3]), fmax(Q[5], Q[7])) < pminy;
}
