// Validity of a closed float32 polygon ring, the definition layout.cu and layout_eval.cu both use where the reference asks
// shapely's Polygon(...).is_valid (DESIGN.md section 8).  A ring is valid when, evaluated in float64 on the float32
// vertices (the including file is compiled without FMA contraction):
//   * after dropping each vertex equal to its predecessor (cyclically), at least 3 vertices remain;
//   * no vertex folds its two edges back over each other (collinear, opposite directions);
//   * no two non-adjacent edges intersect or touch.
#pragma once

namespace hn {
namespace ring {

__device__ inline double orient(const float* a, const float* b, const float* c) {
    return ((double)b[0] - a[0]) * ((double)c[1] - a[1]) - ((double)b[1] - a[1]) * ((double)c[0] - a[0]);
}
__device__ inline bool on_box(const float* a, const float* b, const float* c) {
    return fminf(a[0], b[0]) <= c[0] && c[0] <= fmaxf(a[0], b[0]) && fminf(a[1], b[1]) <= c[1] && c[1] <= fmaxf(a[1], b[1]);
}
__device__ inline bool segments_meet(const float* a, const float* b, const float* c, const float* d) {
    const double o1 = orient(a, b, c), o2 = orient(a, b, d), o3 = orient(c, d, a), o4 = orient(c, d, b);
    if (((o1 > 0 && o2 < 0) || (o1 < 0 && o2 > 0)) && ((o3 > 0 && o4 < 0) || (o3 < 0 && o4 > 0))) return true;
    return (o1 == 0 && on_box(a, b, c)) || (o2 == 0 && on_box(a, b, d)) || (o3 == 0 && on_box(c, d, a)) ||
           (o4 == 0 && on_box(c, d, b));
}

// Block-wide test of the ring r[0..n), n <= CAP, with NT threads (all of them call it).  The ring is compacted in place
// (repeated vertices dropped); scan[NT] and *flag are shared scratch.
template <int NT, int CAP>
__device__ bool is_simple(float (*r)[2], int n, int* scan, int* flag) {
    constexpr int PER = (CAP + NT - 1) / NT;
    int keep[PER], cnt = 0;
    float kx[PER], ky[PER];
    for (int k = 0; k < PER; ++k) {
        const int i = threadIdx.x * PER + k;
        keep[k] = 0;
        if (i < n) {
            const int p = (i - 1 + n) % n;
            keep[k] = !(r[i][0] == r[p][0] && r[i][1] == r[p][1]);
            kx[k] = r[i][0];
            ky[k] = r[i][1];
        }
        cnt += keep[k];
    }
    scan[threadIdx.x] = cnt;                                     // inclusive prefix over the threads' counts
    __syncthreads();
    for (int o = 1; o < NT; o <<= 1) {
        const int t = threadIdx.x >= o ? scan[threadIdx.x - o] : 0;
        __syncthreads();
        scan[threadIdx.x] += t;
        __syncthreads();
    }
    int o = scan[threadIdx.x] - cnt;
    const int m = scan[NT - 1];
    __syncthreads();
    for (int k = 0; k < PER; ++k) if (keep[k]) { r[o][0] = kx[k]; r[o][1] = ky[k]; ++o; }
    if (threadIdx.x == 0) *flag = 0;
    __syncthreads();
    if (m < 3) return false;
    for (int i = threadIdx.x; i < m; i += NT) {                  // no fold-back at a vertex
        const float* a = r[(i - 1 + m) % m];
        const float* b = r[i];
        const float* c = r[(i + 1) % m];
        const double d1x = (double)b[0] - a[0], d1y = (double)b[1] - a[1], d2x = (double)c[0] - b[0], d2y = (double)c[1] - b[1];
        if (d1x * d2y - d1y * d2x == 0 && d1x * d2x + d1y * d2y < 0) *flag = 1;
    }
    const long long pairs = (long long)m * m;                    // no two non-adjacent edges meet
    bool met = false;
    for (long long t = threadIdx.x; t < pairs && !met; t += NT) {
        const int i = (int)(t / m), j = (int)(t % m);
        if (j < i + 2 || (i == 0 && j == m - 1)) continue;
        met = segments_meet(r[i], r[(i + 1) % m], r[j], r[(j + 1) % m]);
    }
    if (met) *flag = 1;
    __syncthreads();
    return *flag == 0;
}

}  // namespace ring
}  // namespace hn
