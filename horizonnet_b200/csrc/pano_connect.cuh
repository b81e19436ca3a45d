// misc/panostretch.pano_connect_points on the device, shared by layout_eval.cu and layout_cuboid.cu: the column range a
// wall samples and its boundary row at one sampled column, with numpy's dtypes (the corner steps in T, the corners'
// dtype; the per-column steps in float64), and the np.interp both files run over the sorted samples.  Both files are
// compiled without FMA contraction (build.py).
#pragma once

namespace hn {
namespace pano {

constexpr int W = 1024, H = 512;
constexpr double PI = 3.141592653589793;

// transcendental functions of numpy's float32 / float64 scalars (float32: the float64 result rounded, as layout.cu)
__device__ __forceinline__ float tan_(float v) { return (float)tan((double)v); }
__device__ __forceinline__ float sin_(float v) { return (float)sin((double)v); }
__device__ __forceinline__ float cos_(float v) { return (float)cos((double)v); }
__device__ __forceinline__ double tan_(double v) { return tan(v); }
__device__ __forceinline__ double sin_(double v) { return sin(v); }
__device__ __forceinline__ double cos_(double v) { return cos(v); }

// pano_connect_points' column range of the wall p1 -> p2 (in T, the corners' dtype); false for a vertical wall
template <typename T>
__device__ bool wall_range(T ax, T bx, long long& s, long long& e) {
    if (ax == bx) return false;
    T ps, pe;
    if (fabs((double)(ax - bx)) < W / 2.0) { ps = ceil(fmin(ax, bx)); pe = floor(fmax(ax, bx)); }
    else { ps = ceil(fmax(ax, bx)); pe = floor(fmin(ax, bx) + (T)W); }
    s = (long long)ps;
    e = (long long)pe;                               // np.arange(ps, pe + 1): integers s .. e
    return true;
}

// pano_connect_points' row at sampled column c of the wall (ax, ay) -> (bx, by) on the plane z
template <typename T>
__device__ double wall_row(T ax, T ay, T bx, T by, int c, double z) {
    const T pi = (T)PI;
    const T u1 = ((ax + (T)0.5) / (T)W - (T)0.5) * (T)2 * pi, v1 = ((ay + (T)0.5) / (T)H - (T)0.5) * pi;
    const T u2 = ((bx + (T)0.5) / (T)W - (T)0.5) * (T)2 * pi, v2 = ((by + (T)0.5) / (T)H - (T)0.5) * pi;
    const T c1 = (T)z / tan_(v1), c2 = (T)z / tan_(v2);
    const T x1 = c1 * cos_(u1), y1 = c1 * sin_(u1), x2 = c2 * cos_(u2), y2 = c2 * sin_(u2);
    const T vx = x2 - x1, vy = y2 - y1;
    const double us = (((double)c + 0.5) / W - 0.5) * 2 * PI;
    const double t = tan(us);
    const double ps = (t * (double)x1 - (double)y1) / ((double)vy - t * (double)vx);
    const double qx = (double)x1 + ps * (double)vx, qy = (double)y1 + ps * (double)vy;
    const double cs = sqrt(qx * qx + qy * qy);
    return (atan2(z, cs) / PI + 0.5) * H - 0.5;
}

// np.interp(x, xp, fp) at one x for sorted xp[0..n) (n >= 1), with numpy's arithmetic and its NaN fallbacks
__device__ __forceinline__ double interp(const double* xp, const double* fp, int n, double x) {
    int lo = -1, hi = n - 1;                         // the last j with xp[j] <= x
    while (lo < hi) {
        const int m = (lo + hi + 1) >> 1;
        if (xp[m] <= x) lo = m; else hi = m - 1;
    }
    if (lo < 0) return fp[0];
    if (lo == n - 1 || xp[lo] == x) return fp[lo];
    const double slope = (fp[lo + 1] - fp[lo]) / (xp[lo + 1] - xp[lo]);
    double r = slope * (x - xp[lo]) + fp[lo];
    if (isnan(r)) {
        r = slope * (x - xp[lo + 1]) + fp[lo + 1];
        if (isnan(r) && fp[lo] == fp[lo + 1]) r = fp[lo];
    }
    return r;
}

}  // namespace pano
}  // namespace hn
