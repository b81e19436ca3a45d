// dataset.cor_2_1d on the device, shared by layout_eval.cu (the depth renders of eval_general) and targets.cu (the y_bon
// training target): one CTA of BT threads turns one boundary's corners into its 1024 boundary angles -- every wall
// sampled per column (pano_connect_points), the first point of each x in argsort order of xs +- ys / ys.max()
// (sort_xy_filter_unique), the periodic np.interp to 1024 columns, the conversion to angles.  Sort ties keep
// concatenation order (DESIGN.md section 9).  Both files are compiled without FMA contraction (build.py).
#pragma once
#include "pano_connect.cuh"

namespace hn {
namespace c21d {

constexpr int W = 1024, H = 512;
constexpr int MAXC = 1024;                 // corners per boundary (max_rows <= 2048)
constexpr int SLOTS = W + 2 * MAXC;        // one candidate per column + both points of every vertical wall
constexpr int PMAX = 4096;                 // power of two >= SLOTS
constexpr int BT = 512, CPT = W / BT;      // threads per boundary CTA; columns (and walls) per thread
constexpr double PI = 3.141592653589793;
using pano::wall_range;
using pano::wall_row;

struct BSmem {
    float px[MAXC], py[MAXC];                        // this boundary's corners (exact in float32 in both modes)
    long long pstart[MAXC], pend[MAXC];              // per wall: the sampled column range (empty when pstart > pend)
    signed char vert[MAXC];                          // per wall: p1[0] == p2[0], two float32 points instead
    int off[MAXC];                                   // per wall: index of its first point in the concatenation
    double ex[SLOTS + 2], ek[SLOTS + 2], ey[SLOTS + 2];
    int eidx[SLOTS];
    int perm[PMAX];
    double xp[SLOTS], fp[SLOTS];
    int scan[BT];
    double dred[BT / 32];
    double ymax;
};

// slot order for the argsort + np.unique: valid slots first, then by x, key, concatenation index
__device__ inline bool slot_less(const BSmem& s, int i, int j, int nslot) {
    const bool vi = i < nslot && s.eidx[i] >= 0, vj = j < nslot && s.eidx[j] >= 0;
    if (vi != vj) return vi;
    if (!vi) return i < j;
    if (s.ex[i] != s.ex[j]) return s.ex[i] < s.ex[j];
    if (s.ek[i] != s.ek[j]) return s.ek[i] < s.ek[j];
    return s.eidx[i] < s.eidx[j];
}
// order of the unique points for np.interp's period: by x % 1024, then by position (a stable sort)
__device__ inline bool mod_less(const BSmem& s, int i, int j, int n) {
    if ((i < n) != (j < n)) return i < n;
    if (i >= n) return i < j;
    if (s.xp[i] != s.xp[j]) return s.xp[i] < s.xp[j];
    return i < j;
}

template <bool MOD>
__device__ void sort_perm(BSmem& s, int n) {
    int p = 1;
    while (p < n) p <<= 1;
    for (int i = threadIdx.x; i < p; i += BT) s.perm[i] = i;
    __syncthreads();
    for (int k = 2; k <= p; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < p; i += BT) {
                const int l = i ^ j;
                if (l > i) {
                    const bool up = (i & k) == 0;
                    const int a = s.perm[i], b = s.perm[l];
                    const bool gt = MOD ? mod_less(s, b, a, n) : slot_less(s, b, a, n);
                    if (gt == up) { s.perm[i] = b; s.perm[l] = a; }
                }
            }
            __syncthreads();
        }
}

__device__ inline int bscan(BSmem& s, int v) {       // exclusive prefix; the total in s.scan[BT - 1] afterwards
    s.scan[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < BT; o <<= 1) {
        const int t = threadIdx.x >= o ? s.scan[threadIdx.x - o] : 0;
        __syncthreads();
        s.scan[threadIdx.x] += t;
        __syncthreads();
    }
    return s.scan[threadIdx.x] - v;
}

// cor_2_1d of one boundary: s.px / s.py hold its nw corners (T: the corners' dtype, float32 or train.py's int64 box as
// float64).  v_out[W] receives the angles; *flag_out = 1 when no wall samples a column (v_out NaN: ys.max() raises) or
// the boundary crosses the horizon (layout_2_depth's assertions), else 0.
template <typename T>
__device__ void boundary(BSmem& s, int nw, bool floor_b, double* v_out, int* flag_out) {
    const double z = floor_b ? 50.0 : -50.0;
    const double sgn = floor_b ? -1.0 : 1.0;         // y_small_first: ceiling True, floor False
    // walls 2t, 2t + 1 of thread t: column ranges and point counts
    int cnt[CPT] = {0, 0};
    bool any_wall = false;
    for (int k = 0; k < CPT; ++k) {
        const int w = CPT * threadIdx.x + k;
        if (w >= nw) continue;
        const int q = (w + 1) % nw;
        long long a, e;
        if (wall_range<T>((T)s.px[w], (T)s.px[q], a, e)) {
            s.pstart[w] = a;
            s.pend[w] = e;
            cnt[k] = e >= a ? (int)min(e - a + 1, (long long)W) : 0;
            s.vert[w] = 0;
            any_wall = true;
        } else {
            s.pstart[w] = 1;
            s.pend[w] = 0;
            s.vert[w] = 1;
            cnt[k] = 2;
        }
    }
    const bool f64_keys = __syncthreads_or(any_wall);    // all walls vertical: xs, ys stay float32 (np.array of float32)
    const int o0 = bscan(s, cnt[0] + cnt[1]);
    s.off[CPT * threadIdx.x] = o0;
    s.off[CPT * threadIdx.x + 1] = o0 + cnt[0];
    __syncthreads();
    // per column c = t + k BT: the point of each wall sampling it; vertical walls add their two corners as float32 points
    // pass 1: ys.max()
    double ym = -INFINITY;
    for (int k = 0; k < CPT; ++k) {
        const int c = threadIdx.x + k * BT;
        for (int i = 0; i < nw; ++i) {
            const int q = (i + 1) % nw;
            if (s.pstart[i] > s.pend[i]) {
                if (s.vert[i] && c == 0) ym = fmax(ym, fmax((double)s.py[i], (double)s.py[q]));
                continue;
            }
            const long long j = s.pstart[i] + (((c - s.pstart[i]) % W) + W) % W;
            if (j > s.pend[i]) continue;
            ym = fmax(ym, wall_row<T>((T)s.px[i], (T)s.py[i], (T)s.px[q], (T)s.py[q], c, z));
        }
    }
    for (int o = 16; o; o >>= 1) ym = fmax(ym, __shfl_xor_sync(0xffffffffu, ym, o));
    if ((threadIdx.x & 31) == 0) s.dred[threadIdx.x >> 5] = ym;
    __syncthreads();
    if (threadIdx.x == 0) {
        double m = -INFINITY;
        for (int i = 0; i < BT / 32; ++i) m = fmax(m, s.dred[i]);
        s.ymax = m;
    }
    __syncthreads();
    const double ymax = s.ymax;
    // pass 2: the candidate of each column (the smallest key, then the first in concatenation order)
    for (int k = 0; k < CPT; ++k) {
        const int c = threadIdx.x + k * BT;
        double bk = 0, by = 0;
        int bi = -1;
        for (int i = 0; i < nw; ++i) {
            if (s.pstart[i] > s.pend[i]) continue;
            const long long j = s.pstart[i] + (((c - s.pstart[i]) % W) + W) % W;
            if (j > s.pend[i]) continue;
            const int q = (i + 1) % nw;
            const double y = wall_row<T>((T)s.px[i], (T)s.py[i], (T)s.px[q], (T)s.py[q], c, z);
            const double key = (double)c + y / ymax * sgn;
            const int idx = s.off[i] + (int)(j - s.pstart[i]);
            if (bi < 0 || key < bk || (key == bk && idx < bi)) { bk = key; by = y; bi = idx; }
        }
        s.ex[c] = (double)c;
        s.ek[c] = bk;
        s.ey[c] = by;
        s.eidx[c] = bi;
    }
    for (int j = threadIdx.x; j < 2 * MAXC; j += BT) {
        const int i = j >> 1, slot = W + j;
        s.eidx[slot] = -1;
        if (i < nw && s.vert[i]) {
            const int q = (j & 1) ? (i + 1) % nw : i;
            const float x = s.px[q], y = s.py[q];
            s.ex[slot] = x;
            s.ey[slot] = y;
            s.ek[slot] = f64_keys ? (double)x + (double)y / ymax * sgn : (double)(x + y / (float)ymax * (float)sgn);
            s.eidx[slot] = s.off[i] + (j & 1);
        }
    }
    __syncthreads();
    // argsort + np.unique(return_index): the first slot of each x
    sort_perm<false>(s, SLOTS);
    int keep[PMAX / BT], nk = 0;
    for (int k = 0; k < PMAX / BT; ++k) {
        const int i = threadIdx.x * (PMAX / BT) + k;
        const int a = s.perm[i];
        keep[k] = a < SLOTS && s.eidx[a] >= 0 && (i == 0 || s.ex[s.perm[i - 1]] != s.ex[a]);
        nk += keep[k];
    }
    int o = bscan(s, nk);
    const int n_u = s.scan[BT - 1];
    __syncthreads();
    for (int k = 0; k < PMAX / BT; ++k)
        if (keep[k]) {
            const int a = s.perm[threadIdx.x * (PMAX / BT) + k];
            double m = fmod(s.ex[a], (double)W);             // numpy's float remainder: the sign of the divisor
            if (m != 0) { if (m < 0) m += W; } else m = 0.0;
            s.xp[o] = m;
            s.fp[o] = s.ey[a];
            ++o;
        }
    __syncthreads();
    if (n_u == 0) {                                      // no sample: ys.max() raises ValueError
        for (int c = threadIdx.x; c < W; c += BT) v_out[c] = NAN;
        if (threadIdx.x == 0) *flag_out = 1;
        return;
    }
    // np.interp(arange(W), xs, ys, period=W): sort by x % W (stably), pad one point on each side
    sort_perm<true>(s, n_u);
    for (int i = threadIdx.x; i < n_u; i += BT) { s.ex[i + 1] = s.xp[s.perm[i]]; s.ey[i + 1] = s.fp[s.perm[i]]; }
    if (threadIdx.x == 0) {
        s.ex[0] = s.xp[s.perm[n_u - 1]] - W;
        s.ey[0] = s.fp[s.perm[n_u - 1]];
        s.ex[n_u + 1] = s.xp[s.perm[0]] + W;
        s.ey[n_u + 1] = s.fp[s.perm[0]];
    }
    __syncthreads();
    const int n = n_u + 2;
    bool bad = false;
    for (int c = threadIdx.x; c < W; c += BT) {
        const double x = (double)c;
        const double r = pano::interp(s.ex, s.ey, n, x);
        const double v = ((r + 0.5) / H - 0.5) * PI;
        v_out[c] = v;
        bad |= floor_b ? v < 0 : v > 0;                  // layout_2_depth's two assertions
    }
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) *flag_out = bad ? 1 : 0;
}

}  // namespace c21d
}  // namespace hn
