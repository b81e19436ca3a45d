// Room-layout evaluation on the device (reference eval_general.py:14-122, test_general and layout_2_depth, with
// dataset.cor_2_1d and misc/panostretch.pano_connect_points): for B (dt, gt) corner-list pairs, the 2D IoU, 3D IoU,
// depth RMSE and delta_1 (DESIGN.md section 9).  Four launches:
//   bound_kernel   one CTA per (pair, boundary): cor_2_1d of the dt / gt ceiling / floor -- every wall sampled per column
//                  (pano_connect_points), the first point of each x in argsort order of xs +- ys / ys.max()
//                  (sort_xy_filter_unique), the periodic np.interp to 1024 columns, the conversion to angles;
//   iou_kernel     one CTA per pair: the column checks, the floor rings (np_coor2xy), their validity (ring.cuh), the
//                  shoelace areas, the intersection area by Green's theorem, the get_z1 heights;
//   depth_kernel   a grid of row blocks per pair: the float32 depth of both layouts per pixel (layout_2_depth), reduced
//                  to sum (gt - dt)^2, sum gt^2, the delta_1 count and the zero-depth flags, never stored unless asked;
//   final_kernel   one thread per pair: the assertions of layout_2_depth, RMSE, delta_1, the status.
// Every step keeps numpy's dtype: the corners are float32 (dt scaled by (1024, 512) in float32), so the per-corner steps
// run in float32 and the per-column ones in float64; train.py's fallback box is int64, and for it every step is float64.
// This file is compiled without FMA contraction (build.py) so the float64 steps round like numpy's.
#include "hn_common.cuh"
#include "pano_connect.cuh"
#include "ring.cuh"

namespace hn {

namespace {

constexpr int W = 1024, H = 512;
constexpr int MAXC = 1024;                 // corners per boundary (max_rows <= 2048)
constexpr int SLOTS = W + 2 * MAXC;        // one candidate per column + both points of every vertical wall
constexpr int PMAX = 4096;                 // power of two >= SLOTS
constexpr int BT = 512, CPT = W / BT;      // bound_kernel threads; columns (and walls) per thread
constexpr int IT = 256;                    // iou_kernel threads
constexpr int DT_ = 256, RB = 16, NBLK = H / RB;   // depth_kernel threads, rows per CTA, CTAs per pair
constexpr double PI = 3.141592653589793;
using pano::tan_;
using pano::sin_;
using pano::cos_;
using pano::wall_range;
using pano::wall_row;
enum { ST_OK = 0, ST_DT_INVALID = 1, ST_SKIP = 2, ST_ERR_GT_DEPTH = 3, ST_ERR_COLUMNS = 4, ST_ERR_RING = 5 };

struct Part {
    double sd, sg;                         // sum (gt - dt)^2, sum gt^2 (each term float32)
    int cnt, zero;                         // delta_1 count; bit 0: a dt depth is 0, bit 1: a gt depth is 0
};

struct Pairs {                             // the inputs of one launch
    const float* dt;
    const int* dt_rows;
    const int* dt_status;                  // NULL, or hn_layout_postproc statuses: 2..5 scores train.py's fallback box
    const float* gt;
    const int* gt_rows;
    int dt_max_rows, gt_max_rows;          // row capacity of each dt / gt corner list
};

__device__ bool use_fallback(const Pairs& p, int b) {
    if (!p.dt_status) return false;
    const int s = p.dt_status[b];
    return s >= 2 && s <= 5;
}
__device__ int rows_of(const Pairs& p, int b, int gt) {
    if (!gt && use_fallback(p, b)) return 8;
    return gt ? p.gt_rows[b] : p.dt_rows[b];
}
// corner `row` of the pair's dt (gt = 0) or gt (gt = 1), in pixels: float32 values, or the fallback's integers
__device__ void corner(const Pairs& p, int b, int gt, int row, double& x, double& y) {
    if (!gt && use_fallback(p, b)) {       // train.py:310-313: [k//2 * 1024, 256 - ((k%2)*2 - 1) * 120]
        x = (double)(row / 2 * 1024);
        y = (double)(256 - ((row % 2) * 2 - 1) * 120);
        return;
    }
    const float* c = gt ? p.gt + ((size_t)b * p.gt_max_rows + row) * 2 : p.dt + ((size_t)b * p.dt_max_rows + row) * 2;
    if (gt) { x = c[0]; y = c[1]; }
    else { x = c[0] * 1024.f; y = c[1] * 512.f; }   // eval_general.py:157-158, train.py:307-308, float32
}

// --------------------------------------------------------------------------------------------- cor_2_1d
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
__device__ bool slot_less(const BSmem& s, int i, int j, int nslot) {
    const bool vi = i < nslot && s.eidx[i] >= 0, vj = j < nslot && s.eidx[j] >= 0;
    if (vi != vj) return vi;
    if (!vi) return i < j;
    if (s.ex[i] != s.ex[j]) return s.ex[i] < s.ex[j];
    if (s.ek[i] != s.ek[j]) return s.ek[i] < s.ek[j];
    return s.eidx[i] < s.eidx[j];
}
// order of the unique points for np.interp's period: by x % 1024, then by position (a stable sort)
__device__ bool mod_less(const BSmem& s, int i, int j, int n) {
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

__device__ int bscan(BSmem& s, int v) {              // exclusive prefix; the total in s.scan[BT - 1] afterwards
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

__global__ void __launch_bounds__(BT, 1) bound_kernel(Pairs p, double* __restrict__ v, int* __restrict__ flags) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    BSmem& s = *reinterpret_cast<BSmem*>(smem_raw);
    const int b = blockIdx.y, which = blockIdx.x;        // 0 dt ceiling, 1 dt floor, 2 gt ceiling, 3 gt floor
    const int gt = which >> 1, fl = which & 1;
    const int rows = rows_of(p, b, gt);
    if (rows <= 0 || rows > (gt ? p.gt_max_rows : max(p.dt_max_rows, 8)) || (rows & 1)) return;   // an error status; iou_kernel sets it
    const int nw = rows / 2;
    const bool f64 = !gt && use_fallback(p, b);
    for (int i = threadIdx.x; i < nw; i += BT) {
        double x, y;
        corner(p, b, gt, 2 * i + fl, x, y);
        s.px[i] = (float)x;
        s.py[i] = (float)y;
    }
    __syncthreads();
    double* out = v + ((size_t)b * 4 + which) * W;
    int* flag = flags + (size_t)b * 4 + which;
    if (f64) boundary<double>(s, nw, fl, out, flag);
    else boundary<float>(s, nw, fl, out, flag);
}

// --------------------------------------------------------------------------------------------- IoU
struct ISmem {
    double x[2][MAXC], y[2][MAXC];                   // floor xy of dt (0) and gt (1)
    double cz[2][MAXC];                              // get_z1 per corner
    float ring[MAXC][2];
    int scan[IT];
    int flag;
    double red[IT / 32];
    double bd;
    int status;
};

__device__ double isum(ISmem& s, double v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s.red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int i = 0; i < IT / 32; ++i) t += s.red[i];
        s.bd = t;
    }
    __syncthreads();
    return s.bd;
}

// np_coor2xy(floor, z=-1.6, 1024, 512, floorW=1, floorH=1) and get_z1(floor y, ceiling y, -1.6, 512) of one corner
template <typename T>
__device__ void floor_corner(double fx, double fy, double cy, double& x, double& y, double& z1) {
    const T pi = (T)PI, ch = (T)-1.6;
    const T u = (((T)fx + (T)0.5) / (T)W - (T)0.5) * (T)2 * pi;
    const T v = -((((T)fy + (T)0.5) / (T)H - (T)0.5) * pi);
    const T v1 = -((((T)cy + (T)0.5) / (T)H - (T)0.5) * pi);
    const T c = ch / tan_(v);
    x = (double)(c * sin_(u) + (T)0.0);
    y = (double)(-c * cos_(u) + (T)0.0);
    z1 = (double)(c * tan_(v1));
}

__device__ double cross(double ax, double ay, double bx, double by) { return ax * by - ay * bx; }

__device__ __forceinline__ bool inside(const double* qx, const double* qy, int nq, double mx, double my) {   // even-odd rule
    bool in = false;
    for (int j = 0; j < nq; ++j) {
        const int k = (j + 1) % nq;
        if ((qy[j] > my) != (qy[k] > my) && mx < (qx[k] - qx[j]) * (my - qy[j]) / (qy[k] - qy[j]) + qx[j]) in = !in;
    }
    return in;
}

// Twice the signed-area contribution of edge i of polygon P (orientation sign sp) to the intersection with Q (sign sq):
// the pieces of the edge inside Q; a piece on an edge of Q counts when both run the same way (after orienting both
// counter-clockwise) and `own` (P's pass counts shared pieces, Q's does not), and never when they run opposite ways.
__device__ __forceinline__ double edge_part(const double* px, const double* py, int np, int i, double sp, const double* qx,
                            const double* qy, int nq, double sq, bool own) {
    const int i2 = (i + 1) % np;
    const double ax = px[i], ay = py[i], bx = px[i2], by = py[i2];
    const double dx = bx - ax, dy = by - ay, dd = dx * dx + dy * dy;
    if (dd == 0) return 0;
    double total = 0, t0 = 0;
    double x0 = ax, y0 = ay;
    for (int guard = 0; guard < 4 * nq + 4 && t0 < 1; ++guard) {
        double t1 = 1;                                   // the next breakpoint after t0
        for (int j = 0; j < nq; ++j) {
            const int k = (j + 1) % nq;
            const double cx = qx[j] - ax, cy = qy[j] - ay, fx = qx[k] - qx[j], fy = qy[k] - qy[j];
            const double den = cross(dx, dy, fx, fy);
            if (den == 0) {
                if (cross(cx, cy, dx, dy) != 0) continue;
                const double tc = (cx * dx + cy * dy) / dd, te = ((qx[k] - ax) * dx + (qy[k] - ay) * dy) / dd;
                if (tc > t0 && tc < t1) t1 = tc;
                if (te > t0 && te < t1) t1 = te;
            } else {
                const double t = cross(cx, cy, fx, fy) / den, u = cross(cx, cy, dx, dy) / den;
                if (u >= 0 && u <= 1 && t > t0 && t < t1) t1 = t;
            }
        }
        const double tm = 0.5 * (t0 + t1);
        int shared = 0;
        for (int j = 0; j < nq && !shared; ++j) {
            const int k = (j + 1) % nq;
            const double cx = qx[j] - ax, cy = qy[j] - ay, fx = qx[k] - qx[j], fy = qy[k] - qy[j];
            if (cross(dx, dy, fx, fy) != 0 || cross(cx, cy, dx, dy) != 0) continue;
            const double tc = (cx * dx + cy * dy) / dd, te = ((qx[k] - ax) * dx + (qy[k] - ay) * dy) / dd;
            if (fmin(tc, te) < tm && tm < fmax(tc, te)) shared = (dx * fx + dy * fy) * sp * sq > 0 ? 1 : -1;
        }
        const double x1 = t1 >= 1 ? bx : ax + t1 * dx, y1 = t1 >= 1 ? by : ay + t1 * dy;
        const bool in = shared ? (own && shared > 0) : inside(qx, qy, nq, ax + tm * dx, ay + tm * dy);
        if (in) total += cross(x0, y0, x1, y1);
        t0 = t1;
        x0 = x1;
        y0 = y1;
    }
    return total * sp;
}

__device__ bool columns_differ(const Pairs& p, int b, int gt, int rows) {
    bool bad = false;
    for (int i = threadIdx.x; i < rows / 2; i += IT) {
        double cx, cy, fx, fy;
        corner(p, b, gt, 2 * i, cx, cy);
        corner(p, b, gt, 2 * i + 1, fx, fy);
        bad |= cx != fx;
    }
    return __syncthreads_or(bad);
}

__global__ void __launch_bounds__(IT, 1) iou_kernel(Pairs p, double* __restrict__ iou2d, double* __restrict__ iou3d,
                                                 int* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ISmem& s = *reinterpret_cast<ISmem*>(smem_raw);
    const int b = blockIdx.x;
    const int rows[2] = {rows_of(p, b, 0), rows_of(p, b, 1)};
    const int cap[2] = {max(p.dt_max_rows, 8), p.gt_max_rows};
    int st = ST_OK;
    for (int g = 0; g < 2 && st == ST_OK; ++g) {         // eval_general.py:61-62, dt first
        if (rows[g] < 0 || rows[g] > cap[g] || (rows[g] & 1)) st = ST_ERR_COLUMNS;
        else if (columns_differ(p, b, g, rows[g])) st = ST_ERR_COLUMNS;
    }
    if (st == ST_OK && (rows[0] < 6 || rows[1] < 6)) st = ST_ERR_RING;      // shapely: a ring needs 3 corners
    double a2 = NAN, a3 = NAN;
    if (st == ST_OK) {
        const bool f64 = use_fallback(p, b);
        for (int g = 0; g < 2; ++g)
            for (int i = threadIdx.x; i < rows[g] / 2; i += IT) {
                double cx, cy, fx, fy;
                corner(p, b, g, 2 * i, cx, cy);
                corner(p, b, g, 2 * i + 1, fx, fy);
                if (g == 0 && f64) floor_corner<double>(fx, fy, cy, s.x[g][i], s.y[g][i], s.cz[g][i]);
                else floor_corner<float>(fx, fy, cy, s.x[g][i], s.y[g][i], s.cz[g][i]);
            }
        __syncthreads();
        bool valid[2];
        for (int g = 1; g >= 0; --g) {
            const int n = rows[g] / 2;
            for (int i = threadIdx.x; i < n; i += IT) { s.ring[i][0] = (float)s.x[g][i]; s.ring[i][1] = (float)s.y[g][i]; }
            __syncthreads();
            valid[g] = ring::is_simple<IT, MAXC>(s.ring, n, s.scan, &s.flag);
            __syncthreads();
        }
        if (!valid[1]) st = ST_SKIP;                                        // eval_general.py:71-73
        else if (!valid[0]) { st = ST_DT_INVALID; a2 = 0; a3 = 0; }         // the except branches of :76-95
        else {
            const int nd = rows[0] / 2, ng = rows[1] / 2;
            double ad = 0, ag = 0;
            for (int i = threadIdx.x; i < nd; i += IT) ad += cross(s.x[0][i], s.y[0][i], s.x[0][(i + 1) % nd], s.y[0][(i + 1) % nd]);
            for (int i = threadIdx.x; i < ng; i += IT) ag += cross(s.x[1][i], s.y[1][i], s.x[1][(i + 1) % ng], s.y[1][(i + 1) % ng]);
            ad = isum(s, ad);
            ag = isum(s, ag);
            const double sd = ad < 0 ? -1.0 : 1.0, sg = ag < 0 ? -1.0 : 1.0;
            double it = 0;
            for (int i = threadIdx.x; i < nd + ng; i += IT)
                it += i < nd ? edge_part(s.x[0], s.y[0], nd, i, sd, s.x[1], s.y[1], ng, sg, true)
                             : edge_part(s.x[1], s.y[1], ng, i - nd, sg, s.x[0], s.y[0], nd, sd, false);
            const double area_dt = fabs(ad) / 2, area_gt = fabs(ag) / 2, inter = isum(s, it) / 2;
            a2 = inter / (area_gt + area_dt - inter);
            double zs[2];
            for (int g = 0; g < 2; ++g) {
                double t = 0;
                for (int i = threadIdx.x; i < rows[g] / 2; i += IT) t += s.cz[g][i];
                zs[g] = isum(s, t) / (rows[g] / 2);
            }
            // h = |mean(z1) - ch|, float32 unless the dt is the int64 fallback
            const double h_dt = f64 ? fabs(zs[0] + 1.6) : (double)fabsf((float)zs[0] - (float)-1.6);
            const double h_gt = (double)fabsf((float)zs[1] - (float)-1.6);
            const double i3 = inter * fmin(h_dt, h_gt), p3 = area_dt * h_dt, g3 = area_gt * h_gt;
            a3 = i3 / (p3 + g3 - i3);
        }
    }
    if (threadIdx.x == 0) {
        iou2d[b] = a2;
        iou3d[b] = a3;
        status[b] = st;
    }
}

// --------------------------------------------------------------------------------------------- depth
__device__ float depth_px(double vs, double sv, double cv, double vc, double vf, double cs, double ceil_h) {
    if (vs < vc) return (float)fabs(ceil_h / sv);        // ceil_mask is assigned last: it wins over floor_mask
    if (vs > vf) return (float)fabs(1.6 / sv);
    return (float)fabs(cs / cv);
}

__global__ void __launch_bounds__(DT_) depth_kernel(const double* __restrict__ v, const int* __restrict__ status,
                                                    Part* __restrict__ parts, float* __restrict__ depth_out) {
    __shared__ double red[2][DT_ / 32];
    __shared__ int redi[2][DT_ / 32];
    const int b = blockIdx.y, r0 = blockIdx.x * RB;
    const int st = status[b];
    if (st != ST_OK && st != ST_DT_INVALID && st != ST_SKIP) return;   // SKIP: the maps only, for depth_out
    constexpr int PER = W / DT_;
    double vc[2][PER], vf[2][PER], cs[2][PER], chh[2][PER];
    for (int m = 0; m < 2; ++m)
        for (int k = 0; k < PER; ++k) {
            const int c = threadIdx.x + k * DT_;
            vc[m][k] = v[((size_t)b * 4 + 2 * m) * W + c];
            vf[m][k] = v[((size_t)b * 4 + 2 * m + 1) * W + c];
            cs[m][k] = 1.6 / tan(vf[m][k]);
            chh[m][k] = fabs(cs[m][k] * tan(vc[m][k]));
        }
    double sd = 0, sg = 0;
    int cnt = 0, zero = 0;
    for (int r = r0; r < r0 + RB; ++r) {
        const double vs = (((double)r + 0.5) / H - 0.5) * PI, sv = sin(vs), cv = cos(vs);
        for (int k = 0; k < PER; ++k) {
            const int c = threadIdx.x + k * DT_;
            const float d = depth_px(vs, sv, cv, vc[0][k], vf[0][k], cs[0][k], chh[0][k]);
            const float g = depth_px(vs, sv, cv, vc[1][k], vf[1][k], cs[1][k], chh[1][k]);
            const float e = g - d;
            sd += (double)(e * e);
            sg += (double)(g * g);
            cnt += (g / d < 1.25f) && (d / g < 1.25f);   // max(gt/dt, dt/gt) < 1.25, NaN compares false
            zero |= (d == 0.f ? 1 : 0) | (g == 0.f ? 2 : 0);
            if (depth_out) {
                depth_out[(((size_t)b * 2 + 0) * H + r) * W + c] = d;
                depth_out[(((size_t)b * 2 + 1) * H + r) * W + c] = g;
            }
        }
    }
    for (int o = 16; o; o >>= 1) {
        sd += __shfl_xor_sync(0xffffffffu, sd, o);
        sg += __shfl_xor_sync(0xffffffffu, sg, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        zero |= __shfl_xor_sync(0xffffffffu, zero, o);
    }
    if ((threadIdx.x & 31) == 0) {
        red[0][threadIdx.x >> 5] = sd;
        red[1][threadIdx.x >> 5] = sg;
        redi[0][threadIdx.x >> 5] = cnt;
        redi[1][threadIdx.x >> 5] = zero;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        Part q{0, 0, 0, 0};
        for (int i = 0; i < DT_ / 32; ++i) { q.sd += red[0][i]; q.sg += red[1][i]; q.cnt += redi[0][i]; q.zero |= redi[1][i]; }
        parts[(size_t)b * NBLK + blockIdx.x] = q;
    }
}

__global__ void final_kernel(int B, const int* __restrict__ flags, const Part* __restrict__ parts, int* __restrict__ status,
                             double* __restrict__ iou2d, double* __restrict__ iou3d, double* __restrict__ rmse,
                             double* __restrict__ delta_1, int* __restrict__ dt_zero) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    int st = status[b];
    double r = NAN, d1 = NAN;
    int dz = 0;
    if (st == ST_OK || st == ST_DT_INVALID || st == ST_SKIP) {
        Part q{0, 0, 0, 0};
        for (int i = 0; i < NBLK; ++i) {
            const Part t = parts[(size_t)b * NBLK + i];
            q.sd += t.sd; q.sg += t.sg; q.cnt += t.cnt; q.zero |= t.zero;
        }
        const int* f = flags + (size_t)b * 4;
        const double n = (double)H * W;
        dz = f[0] || f[1] || (q.zero & 1);               // layout_2_depth(dt) raises: its depth is all zeros
        if (st == ST_SKIP) {
                                                          // not scored: the reference returns before the depth
        } else if (f[2] || f[3] || (q.zero & 2)) {        // layout_2_depth(gt) raises
            st = ST_ERR_GT_DEPTH;
            iou2d[b] = NAN;
            iou3d[b] = NAN;
        } else if (dz) {
            r = sqrt(q.sg / n);
            d1 = 0.0;
        } else {
            r = sqrt(q.sd / n);
            d1 = q.cnt / n;
        }
    }
    status[b] = st;
    rmse[b] = r;
    delta_1[b] = d1;
    dt_zero[b] = dz;
}

__global__ void zero_dt_kernel(const int* __restrict__ dt_zero, float* __restrict__ depth_out) {
    const int b = blockIdx.y;
    if (!dt_zero[b]) return;
    float* d = depth_out + (size_t)b * 2 * H * W + (size_t)blockIdx.x * RB * W;
    for (int i = threadIdx.x; i < RB * W; i += blockDim.x) d[i] = 0.f;
}

}  // namespace

int layout_eval_general(const float* dt, const int* dt_rows, const int* dt_status, int dt_max_rows, const float* gt,
                        const int* gt_rows, int gt_max_rows, int B, double* iou2d, double* iou3d, double* rmse, double* delta_1, int* status,
                        float* depth_out, cudaStream_t st) {
    static int configured = -1;
    int dev = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    if (configured != dev) {
        HN_CUDA_OK(cudaFuncSetAttribute(bound_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BSmem)));
        HN_CUDA_OK(cudaFuncSetAttribute(iou_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ISmem)));
        configured = dev;
    }
    const Pairs p{dt, dt_rows, dt_status, gt, gt_rows, dt_max_rows, gt_max_rows};
    const size_t v_bytes = (size_t)B * 4 * W * sizeof(double), part_bytes = (size_t)B * NBLK * sizeof(Part);
    const size_t bytes = v_bytes + part_bytes + (size_t)B * 5 * sizeof(int);
    unsigned char* ws = nullptr;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ws), bytes, st));
    double* v = reinterpret_cast<double*>(ws);
    Part* parts = reinterpret_cast<Part*>(ws + v_bytes);
    int* flags = reinterpret_cast<int*>(ws + v_bytes + part_bytes);
    int* dt_zero = flags + (size_t)B * 4;
    bound_kernel<<<dim3(4, B), BT, sizeof(BSmem), st>>>(p, v, flags);
    HN_LAUNCH_OK();
    iou_kernel<<<B, IT, sizeof(ISmem), st>>>(p, iou2d, iou3d, status);
    HN_LAUNCH_OK();
    depth_kernel<<<dim3(NBLK, B), DT_, 0, st>>>(v, status, parts, depth_out);
    HN_LAUNCH_OK();
    final_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, flags, parts, status, iou2d, iou3d, rmse, delta_1, dt_zero);
    HN_LAUNCH_OK();
    if (depth_out) {
        zero_dt_kernel<<<dim3(NBLK, B), 256, 0, st>>>(dt_zero, depth_out);
        HN_LAUNCH_OK();
    }
    HN_CUDA_OK(cudaFreeAsync(ws, st));
    return 0;
}

}  // namespace hn
