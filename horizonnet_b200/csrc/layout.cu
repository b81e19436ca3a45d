// Room-layout post-processing on the device (reference inference.py:95-141 and the misc/post_proc.py functions it
// calls): from the TTA outputs y_bon_pix [2][1024] / y_cor [1024] of one panorama to its corner list cor_id, one CTA per
// panorama.  Steps, each following numpy's dtype at that point (DESIGN.md section 8):
//   z1       np_refine_by_fix_z: float32 per column, numpy's linear-interpolation 25/75 percentiles of a block sort,
//            the mean of the values between them summed in numpy's pairwise order; tol = |0.16 z1 / 1.6| in float32;
//   peaks    find_N_peaks: wrap-mode maximum over r_px columns (offsets -(r_px/2) .. r_px-1-r_px/2, scipy's placement of
//            an even window), > min_v; top 4 by value with ties to the lower column, in column order;
//   walls    gen_ww in float64: column -> wall group (get_gpid), floor-plane projection (np_coor2xy), vote per group and
//            axis (block sort + the first longest run within tol covering 40 %, or the median), gen_ww_cuboid or the
//            gen_ww_general loop (a block argmax picks the wall, thread 0 decides, the block shifts the wall list);
//   validity the general result's float32 ring xy2d must be a simple polygon (ring.cuh), else a cuboid fit on the top-4 peaks with
//            min_v 0 replaces it (status HN_LAYOUT_FALLBACK);
//   output   np_xy2coor, the roll to the smallest ceiling column, infer_coory, cor_id rows normalised by W and H.
// This file is compiled without FMA contraction (build.py) so the float64 steps round like numpy's.
#include "hn_common.cuh"
#include "ring.cuh"

namespace hn {

namespace {

constexpr int W = 1024, H = 512, NT = 512, NWARP = NT / 32;
constexpr int WMAX = 2 * W;              // gen_ww_general inserts at most one wall per wall it starts from
constexpr double PI = 3.141592653589793;
enum { ST_OK = 0, ST_FALLBACK = 1, ST_GROUPS = 2, ST_VOTE = 3, ST_RING = 4, ST_OVERFLOW = 5 };

struct Smem {
    float ceil_row[W], floor_row[W], ycor[W];
    float zf[W], zs[W];                  // per-column z1 and its sorted copy / compacted selection
    double xy[2][W];
    double sbuf[W];                      // one group's values of one axis, sorted
    int peaks[W];
    short gid[W];
    int scan[NT];
    // wall list (struct of arrays)
    double wval[WMAX], wscore[WMAX], wu0[WMAX], wu1[WMAX];
    short wgroup[WMAX];
    signed char waxis[WMAX], wpend[WMAX];
    float ring[WMAX][2];
    // reductions and broadcasts
    double red_d[NWARP];
    int red_i[NWARP], red_j[NWARP];
    double bd;
    int bi, bj;
    int n_peaks, n_walls, status, flag;
    int op, at;
    double new_val[2];
    int new_axis[2];
};

// ---------------------------------------------------------------------------------------------- block primitives
__device__ double block_sum(Smem& s, double v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s.red_d[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int w = 0; w < NWARP; ++w) t += s.red_d[w];
        s.bd = t;
    }
    __syncthreads();
    return s.bd;
}

// Largest key, the smallest index among equal keys (index < 0: no candidate).  Result in s.bd / s.bi.
__device__ void block_argmax(Smem& s, double key, int idx) {
    for (int o = 16; o; o >>= 1) {
        const double k2 = __shfl_xor_sync(0xffffffffu, key, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, idx, o);
        if (i2 >= 0 && (idx < 0 || k2 > key || (k2 == key && i2 < idx))) { key = k2; idx = i2; }
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { s.red_d[threadIdx.x >> 5] = key; s.red_i[threadIdx.x >> 5] = idx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double k = 0;
        int b = -1;
        for (int w = 0; w < NWARP; ++w) {
            const int i2 = s.red_i[w];
            if (i2 >= 0 && (b < 0 || s.red_d[w] > k || (s.red_d[w] == k && i2 < b))) { k = s.red_d[w]; b = i2; }
        }
        s.bd = k;
        s.bi = b;
    }
    __syncthreads();
}

// Exclusive prefix over the threads' counts; returns this thread's offset, total in s.bi.
__device__ int block_scan(Smem& s, int v) {
    s.scan[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < NT; o <<= 1) {
        const int t = threadIdx.x >= o ? s.scan[threadIdx.x - o] : 0;
        __syncthreads();
        s.scan[threadIdx.x] += t;
        __syncthreads();
    }
    const int incl = s.scan[threadIdx.x];
    if (threadIdx.x == NT - 1) s.bi = incl;
    __syncthreads();
    return incl - v;
}

template <typename T>
__device__ void block_sort(T* a, int n, T pad) {          // ascending bitonic sort of a[0..n), n <= W
    int p = 1;
    while (p < n) p <<= 1;
    for (int i = n + threadIdx.x; i < p; i += NT) a[i] = pad;
    __syncthreads();
    for (int k = 2; k <= p; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < p; i += NT) {
                const int l = i ^ j;
                if (l > i) {
                    const bool up = (i & k) == 0;
                    const T x = a[i], y = a[l];
                    if ((x > y) == up) { a[i] = y; a[l] = x; }
                }
            }
            __syncthreads();
        }
}

// numpy's float32 pairwise summation (add.reduce over a contiguous array), on one thread
__device__ float pairwise_block(const float* a, int n) {
    if (n < 8) {
        float r = 0.f;
        for (int i = 0; i < n; ++i) r += a[i];
        return r;
    }
    float r[8];
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; ++j) r[j] += a[i + j];
    float res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i];
    return res;
}

template <int D>
__device__ float pairwise_sum(const float* a, int n) {
    if (n <= 128) return pairwise_block(a, n);
    int n2 = n / 2;
    n2 -= n2 % 8;
    return pairwise_sum<D - 1>(a, n2) + pairwise_sum<D - 1>(a + n2, n - n2);
}
template <>
__device__ float pairwise_sum<0>(const float* a, int n) { return pairwise_block(a, n); }

// ---------------------------------------------------------------------------------------------- geometry (float64)
__device__ double col_to_u(double x) { return ((x + 0.5) / W - 0.5) * 2.0 * PI; }
__device__ double row_to_v(double y) { return -((y + 0.5) / H - 0.5) * PI; }
__device__ double y_from_x(double x, double u) { const double c = (x - W / 2.0 + 0.5) / sin(u); return -c * cos(u) + H / 2.0 - 0.5; }
__device__ double x_from_y(double y, double u) { const double c = -(y - H / 2.0 + 0.5) / cos(u); return c * sin(u) + W / 2.0 - 0.5; }
__device__ void xy_to_coor(double cx, double cy, double& col, double& row) {
    const double x = cx - W / 2.0 + 0.5, y = cy - H / 2.0 + 0.5;
    const double u = atan2(x, -y), v = atan(50.0 / sqrt(x * x + y * y));
    col = (u / (2.0 * PI) + 0.5) * W - 0.5;
    row = (-v / PI + 0.5) * H - 0.5;
}
__device__ double floor_row(double ceil_row, float z1) {       // infer_coory with h = z1 - z0
    const float zz = 50.f + (z1 - 50.f);
    const double c0 = 50.0 / tan(row_to_v(ceil_row));
    return (-atan2((double)zz, c0) / PI + 0.5) * H - 0.5;
}

// ---------------------------------------------------------------------------------------------- steps
__device__ float refine_z1(Smem& s) {
    const float pif = (float)PI;
    for (int i = threadIdx.x; i < W; i += NT) {
        const float v0 = -((s.ceil_row[i] + 0.5f) / (float)H - 0.5f) * pif;
        const float v1 = -((s.floor_row[i] + 0.5f) / (float)H - 0.5f) * pif;
        const float c0 = 50.f / (float)tan((double)v0);
        const float z = c0 * (float)tan((double)v1);
        s.zf[i] = z;
        s.zs[i] = z;
    }
    __syncthreads();
    block_sort(s.zs, W, __int_as_float(0x7f800000));
    // numpy 'linear' percentile: index q (n-1) / 100, lerp between the neighbours, from the upper one when t >= 0.5
    const float a0 = s.zs[255], b0 = s.zs[256], a1 = s.zs[767], b1 = s.zs[768];
    const float lo = (float)((double)b0 - (double)(b0 - a0) * 0.25);
    const float hi = (float)((double)a1 + (double)(b1 - a1) * 0.25);
    __syncthreads();
    // compact the selection in column order, then numpy's pairwise sum on one thread
    int cnt = 0;
    for (int k = 0; k < 2; ++k) { const float z = s.zf[2 * threadIdx.x + k]; cnt += (lo <= z && z <= hi); }
    const int off = block_scan(s, cnt);
    const int total = s.bi;
    int o = off;
    for (int k = 0; k < 2; ++k) { const float z = s.zf[2 * threadIdx.x + k]; if (lo <= z && z <= hi) s.zs[o++] = z; }
    __syncthreads();
    if (threadIdx.x == 0) s.bd = (double)(pairwise_sum<4>(s.zs, total) / (float)total);
    __syncthreads();
    return (float)s.bd;
}

// Peaks into s.peaks / s.n_peaks; column -> group into s.gid.
__device__ void find_peaks(Smem& s, int r_px, float min_v, int top_n) {
    const int lo = -(r_px / 2);
    int flag[2], cnt = 0;
    for (int k = 0; k < 2; ++k) {
        const int i = 2 * threadIdx.x + k;
        const float v = s.ycor[i];
        float m = v;
        for (int d = lo; d < lo + r_px; ++d) m = fmaxf(m, s.ycor[(i + d + W) & (W - 1)]);
        flag[k] = (m == v) && (v > min_v);
        cnt += flag[k];
    }
    int o = block_scan(s, cnt);
    const int n = s.bi;
    for (int k = 0; k < 2; ++k) if (flag[k]) s.peaks[o++] = 2 * threadIdx.x + k;
    __syncthreads();
    if (threadIdx.x == 0) {
        int np = n;
        if (top_n > 0 && n > top_n) {
            int best[8];
            for (int t = 0; t < top_n; ++t) {            // t-th largest value; the lower column on ties
                int b = -1;
                for (int i = 0; i < n; ++i) {
                    bool used = false;
                    for (int u = 0; u < t; ++u) used |= best[u] == i;
                    if (used) continue;
                    if (b < 0 || s.ycor[s.peaks[i]] > s.ycor[s.peaks[b]]) b = i;
                }
                best[t] = b;
            }
            for (int a = 1; a < top_n; ++a)               // back to column order
                for (int b = a; b > 0 && best[b] < best[b - 1]; --b) { const int t = best[b]; best[b] = best[b - 1]; best[b - 1] = t; }
            for (int t = 0; t < top_n; ++t) s.peaks[t] = s.peaks[best[t]];
            np = top_n;
        }
        s.n_peaks = np;
    }
    __syncthreads();
    const int np = s.n_peaks;
    for (int i = threadIdx.x; i < W; i += NT) {           // number of peaks <= i; the last group wraps to 0
        int a = 0, b = np;
        while (a < b) { const int m = (a + b) >> 1; if (s.peaks[m] <= i) a = m + 1; else b = m; }
        s.gid[i] = (short)(a == np ? 0 : a);
    }
    __syncthreads();
}

// vote() of one group and axis: fit, run fraction, mean |v - fit|; false when the reference's assert fails.
__device__ bool vote(Smem& s, int g, int axis, float tol, double& fit, double& frac, double& l1) {
    int cnt = 0;
    for (int k = 0; k < 2; ++k) cnt += s.gid[2 * threadIdx.x + k] == g;
    int o = block_scan(s, cnt);
    const int n = s.bi;
    for (int k = 0; k < 2; ++k) if (s.gid[2 * threadIdx.x + k] == g) s.sbuf[o++] = s.xy[axis][2 * threadIdx.x + k];
    __syncthreads();
    block_sort(s.sbuf, n, (double)__longlong_as_double(0x7ff0000000000000ll));
    const double dtol = (double)tol;
    bool ok = true;
    // longest run [i, j] of the sorted values with (s_j - s_i) + 1e-9 <= tol (j > i) covering at least 40 %
    double key = -1.0;
    int best = -1;
    if (!((double)n < dtol)) {
        for (int i = threadIdx.x; i < n; i += NT) {
            int a = i, b = n - 1;                        // last j with s_j - s_i + 1e-9 <= tol (j = i always qualifies)
            while (a < b) {
                const int m = (a + b + 1) >> 1;
                if ((s.sbuf[m] - s.sbuf[i]) + 1e-9 <= dtol) a = m; else b = m - 1;
            }
            const double span = (double)(a - i + 1);
            if (span >= n * 0.4 && (best < 0 || span > key)) { key = span; best = i; }
        }
    }
    block_argmax(s, key, best);
    const int row = s.bi;
    int col = 0;
    if (row >= 0) col = row + (int)s.bd - 1;
    if (row < 0) {
        fit = (n & 1) ? s.sbuf[n / 2] : (s.sbuf[n / 2 - 1] + s.sbuf[n / 2]) / 2.0;
        frac = 0.0;
    } else {
        if (col <= row) ok = false;
        double t = 0;
        for (int i = row + threadIdx.x; i <= col; i += NT) t += s.sbuf[i];
        fit = block_sum(s, t) / (double)(col - row + 1);
        frac = (double)(col - row + 1) / (double)n;
    }
    double t = 0;
    for (int i = threadIdx.x; i < n; i += NT) t += fabs(s.sbuf[i] - fit);
    l1 = block_sum(s, t) / (double)n;
    return ok;
}

// One wall per group: the axis whose vote wins (score, -l1) lexicographically.
__device__ bool pick_walls(Smem& s, int groups, float tol) {
    for (int g = 0; g < groups; ++g) {
        double fx, sx, lx, fy, sy, ly;
        if (!vote(s, g, 0, tol, fx, sx, lx)) return false;
        if (!vote(s, g, 1, tol, fy, sy, ly)) return false;
        if (threadIdx.x == 0) {
            const bool x = sx > sy || (sx == sy && -lx > -ly);
            s.waxis[g] = x ? 0 : 1;
            s.wval[g] = x ? fx : fy;
            s.wscore[g] = x ? sx : sy;
            s.wgroup[g] = (short)g;
            s.wpend[g] = 1;
            const int np = s.n_peaks;
            s.wu0[g] = col_to_u((double)s.peaks[(g - 1 + np) % np]);
            s.wu1[g] = col_to_u((double)s.peaks[g]);
        }
        __syncthreads();
    }
    return true;
}

__device__ void make_wall(Smem& s, int i, int axis, double val) {
    s.waxis[i] = (signed char)axis; s.wval[i] = val; s.wscore[i] = 0.0; s.wgroup[i] = -1; s.wpend[i] = 0;
    s.wu0[i] = -1.0; s.wu1[i] = -1.0;
}

// Moves walls [from, n) one place up (the block cooperates; n < WMAX).
__device__ void shift_walls(Smem& s, int from, int n) {
    constexpr int PER = WMAX / NT;
    double v[PER], sc[PER], u0[PER], u1[PER];
    short gr[PER];
    signed char ax[PER], pe[PER];
    for (int k = 0; k < PER; ++k) {
        const int i = from + threadIdx.x + k * NT;
        if (i < n) { v[k] = s.wval[i]; sc[k] = s.wscore[i]; u0[k] = s.wu0[i]; u1[k] = s.wu1[i]; gr[k] = s.wgroup[i]; ax[k] = s.waxis[i]; pe[k] = s.wpend[i]; }
    }
    __syncthreads();
    for (int k = 0; k < PER; ++k) {
        const int i = from + threadIdx.x + k * NT;
        if (i < n) { s.wval[i + 1] = v[k]; s.wscore[i + 1] = sc[k]; s.wu0[i + 1] = u0[k]; s.wu1[i + 1] = u1[k]; s.wgroup[i + 1] = gr[k]; s.waxis[i + 1] = ax[k]; s.wpend[i + 1] = pe[k]; }
    }
    __syncthreads();
}

enum { OP_NONE = 0, OP_INSERT = 1, OP_REPLACE = 2, OP_TURN = 3, OP_DONE = 4, OP_FULL = 5 };

// gen_ww_general's loop over the walls in s.w* (s.n_walls of them): status ST_OK or ST_OVERFLOW.
__device__ int general_loop(Smem& s) {
    for (int iter = 0; iter < 4 * WMAX; ++iter) {
        const int n = s.n_walls;
        double key = 0;
        int idx = -1;
        for (int i = threadIdx.x; i < n; i += NT)
            if (s.wpend[i] && (idx < 0 || s.wscore[i] > key)) { key = s.wscore[i]; idx = i; }
        block_argmax(s, key, idx);
        if (threadIdx.x == 0) {
            const int cur = s.bi;
            s.op = OP_NONE;
            if (cur < 0) {
                s.op = OP_DONE;
            } else {
                s.wpend[cur] = 0;
                const int p = (cur - 1 + n) % n, q = (cur + 1) % n;
                const int und = s.wpend[p] + s.wpend[q];
                const int ax = s.waxis[cur];
                if (und == 1) {
                    if ((!s.wpend[p] && s.waxis[p] == ax) || (!s.wpend[q] && s.waxis[q] == ax)) {
                        if (s.wscore[cur] >= -1.0) {               // decide it after its other neighbour
                            s.wpend[cur] = 1;
                            s.wscore[cur] -= 100.0;
                        } else {
                            const int src = !s.wpend[p] ? p : q;
                            const double u = !s.wpend[p] ? s.wu1[p] : s.wu0[q];
                            s.at = !s.wpend[p] ? cur : q;
                            s.new_axis[0] = s.waxis[src] == 0 ? 1 : 0;
                            s.new_val[0] = s.waxis[src] == 0 ? y_from_x(s.wval[src], u) : x_from_y(s.wval[src], u);
                            s.op = n < WMAX ? OP_INSERT : OP_FULL;
                        }
                    }
                } else if (und == 0) {
                    if (s.waxis[p] == s.waxis[q]) {
                        if (ax == s.waxis[p]) { s.waxis[cur] = (signed char)(ax ^ 1); s.at = cur; s.op = OP_TURN; }
                    } else {
                        s.new_axis[0] = s.waxis[q];
                        s.new_axis[1] = s.waxis[p];
                        if (s.waxis[p] == 0) {
                            s.new_val[0] = y_from_x(s.wval[p], s.wu1[p]);
                            s.new_val[1] = x_from_y(s.wval[q], s.wu0[q]);
                        } else {
                            s.new_val[0] = x_from_y(s.wval[p], s.wu1[p]);
                            s.new_val[1] = y_from_x(s.wval[q], s.wu0[q]);
                        }
                        s.at = cur;
                        s.op = n < WMAX ? OP_REPLACE : OP_FULL;
                    }
                }
            }
        }
        __syncthreads();
        const int op = s.op, at = s.at;
        if (op == OP_DONE) return ST_OK;
        if (op == OP_FULL) return ST_OVERFLOW;
        if (op == OP_INSERT) {
            shift_walls(s, at, n);
            if (threadIdx.x == 0) { make_wall(s, at, s.new_axis[0], s.new_val[0]); s.n_walls = n + 1; }
        } else if (op == OP_REPLACE) {
            shift_walls(s, at + 1, n);
            if (threadIdx.x == 0) {
                make_wall(s, at, s.new_axis[0], s.new_val[0]);
                make_wall(s, at + 1, s.new_axis[1], s.new_val[1]);
                s.n_walls = n + 1;
            }
        } else if (op == OP_TURN) {                               // three parallel walls: the middle one turns
            const int g = s.wgroup[at], ax = s.waxis[at];
            double t = 0;
            int c = 0;
            for (int i = threadIdx.x; i < W; i += NT) if (s.gid[i] == g) { t += s.xy[ax][i]; ++c; }
            const double sum = block_sum(s, t);
            const double cnt = block_sum(s, (double)c);
            if (threadIdx.x == 0) s.wval[at] = sum / cnt;
        }
        __syncthreads();
    }
    return ST_OVERFLOW;
}

// gen_ww on the current peaks: walls in s.w*, status ST_OK / ST_GROUPS / ST_VOTE / ST_OVERFLOW.
__device__ int fit_walls(Smem& s, int r_px, float min_v, bool cuboid, float tol) {
    find_peaks(s, r_px, min_v, cuboid ? 4 : 0);
    const int np = s.n_peaks;
    const int groups = np > 0 ? np : 1;
    if (cuboid ? groups != 4 : np != groups) return ST_GROUPS;
    if (!pick_walls(s, groups, tol)) return ST_VOTE;
    if (threadIdx.x == 0) s.n_walls = groups;
    __syncthreads();
    if (cuboid) {
        if (threadIdx.x == 0) {
            double bal[2] = {0.0, 0.0};
            for (int j = 0; j < 4; ++j) bal[j & 1] += s.waxis[j] == 0 ? s.wscore[j] : -s.wscore[j];
            const int first = bal[0] > bal[1] ? 0 : 1;
            for (int j = 0; j < 4; ++j) s.waxis[j] = (signed char)(first ^ (j & 1));
        }
        __syncthreads();
        return ST_OK;
    }
    return general_loop(s);
}

// The float32 ring xy2d of the walls (inference.py:115-119) is a simple polygon (DESIGN.md section 8).
__device__ bool ring_is_simple(Smem& s) {
    const int n = s.n_walls;
    // ring[i]: coordinate axis_i = val_i, then coordinate axis_{i-1} = val_{i-1} (the later write wins)
    for (int i = threadIdx.x; i < n; i += NT) {
        const int p = (i - 1 + n) % n;
        const float vi = (float)s.wval[i], vp = (float)s.wval[p];
        s.ring[i][0] = s.waxis[p] == 0 ? vp : (s.waxis[i] == 0 ? vi : 0.f);
        s.ring[i][1] = s.waxis[p] == 1 ? vp : (s.waxis[i] == 1 ? vi : 0.f);
    }
    __syncthreads();
    return ring::is_simple<NT, WMAX>(s.ring, n, s.scan, &s.flag);
}

__global__ void __launch_bounds__(NT, 1)
layout_kernel(const float* __restrict__ y_bon_pix, const float* __restrict__ y_cor, int r_px, float min_v, int force_cuboid,
              int force_raw, int max_rows, float* __restrict__ cor_id, int* __restrict__ n_rows, float* __restrict__ z0_out,
              float* __restrict__ z1_out, int* __restrict__ status_out, int* __restrict__ peaks_out,
              int* __restrict__ n_peaks_out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem& s = *reinterpret_cast<Smem*>(smem_raw);
    const int b = blockIdx.x;
    for (int i = threadIdx.x; i < W; i += NT) {
        s.ceil_row[i] = y_bon_pix[(size_t)b * 2 * W + i];
        s.floor_row[i] = y_bon_pix[(size_t)b * 2 * W + W + i];
        s.ycor[i] = y_cor[(size_t)b * W + i];
    }
    __syncthreads();
    const float z1 = refine_z1(s);
    const float tol = fabsf(0.16f * z1 / 1.6f);
    for (int i = threadIdx.x; i < W; i += NT) {                  // np_coor2xy of (column, ceiling row) on z = 50
        const double u = col_to_u((double)i);
        const double c = 50.0 / tan(row_to_v((double)s.ceil_row[i]));
        s.xy[0][i] = c * sin(u) + W / 2.0 - 0.5;
        s.xy[1][i] = -c * cos(u) + H / 2.0 - 0.5;
    }
    __syncthreads();
    float* out = cor_id + (size_t)b * max_rows * 2;
    int st = ST_OK, rows = 0;
    if (force_raw) {
        if (2 * W > max_rows) {
            st = ST_OVERFLOW;
        } else {
            rows = 2 * W;
            for (int j = threadIdx.x; j < W; j += NT) {
                const double r = (double)s.ceil_row[j];
                out[4 * j + 0] = (float)j / (float)W;
                out[4 * j + 1] = (float)r / (float)H;
                out[4 * j + 2] = (float)j / (float)W;
                out[4 * j + 3] = (float)floor_row(r, z1) / (float)H;
            }
        }
        if (threadIdx.x == 0) s.n_peaks = 0;
        __syncthreads();
    } else {
        st = fit_walls(s, r_px, min_v, force_cuboid != 0, tol);
        if (st == ST_OK && !force_cuboid) {
            if (s.n_walls < 3) st = ST_RING;                     // shapely: a ring needs at least 4 coordinates
            else if (!ring_is_simple(s)) {
                st = fit_walls(s, r_px, 0.f, true, tol);
                if (st == ST_OK) st = ST_FALLBACK;
            }
        }
        const int n = s.n_walls;
        if ((st == ST_OK || st == ST_FALLBACK) && 2 * n > max_rows) st = ST_OVERFLOW;
        if (st == ST_OK || st == ST_FALLBACK) {
            // the even-indexed corner with the smallest column leads (np.roll by -2 argmin)
            double key = 0;
            int idx = -1;
            for (int j = 2 * threadIdx.x; j < n; j += 2 * NT) {
                const int nj = (j + 1) % n;
                const double cx = s.waxis[j] == 1 ? s.wval[nj] : s.wval[j], cy = s.waxis[j] == 1 ? s.wval[j] : s.wval[nj];
                double col, row;
                xy_to_coor(cx, cy, col, row);
                if (idx < 0 || -col > key) { key = -col; idx = j / 2; }
            }
            block_argmax(s, key, idx);
            const int shift = 2 * s.bi;
            rows = 2 * n;
            for (int j = threadIdx.x; j < n; j += NT) {
                const int nj = (j + 1) % n;
                const double cx = s.waxis[j] == 1 ? s.wval[nj] : s.wval[j], cy = s.waxis[j] == 1 ? s.wval[j] : s.wval[nj];
                double col, row;
                xy_to_coor(cx, cy, col, row);
                const int pos = ((j - shift) % n + n) % n;
                out[4 * pos + 0] = (float)col / (float)W;
                out[4 * pos + 1] = (float)row / (float)H;
                out[4 * pos + 2] = (float)col / (float)W;
                out[4 * pos + 3] = (float)floor_row(row, z1) / (float)H;
            }
        }
    }
    for (int i = rows * 2 + threadIdx.x; i < max_rows * 2; i += NT) out[i] = 0.f;
    const int np = (st == ST_GROUPS || st == ST_VOTE || st == ST_OK || st == ST_FALLBACK || st == ST_RING) ? s.n_peaks : 0;
    if (peaks_out)
        for (int i = threadIdx.x; i < W; i += NT) peaks_out[(size_t)b * W + i] = i < np ? s.peaks[i] : -1;
    if (threadIdx.x == 0) {
        n_rows[b] = rows;
        z0_out[b] = 50.f;
        z1_out[b] = z1;
        status_out[b] = st;
        if (n_peaks_out) n_peaks_out[b] = np;
    }
}

}  // namespace

int layout_postproc(const float* y_bon_pix, const float* y_cor, int B, int r_px, float min_v, int force_cuboid, int force_raw,
                    int max_rows, float* cor_id, int* n_rows, float* z0, float* z1, int* status, int* peaks, int* n_peaks,
                    cudaStream_t st) {
    const int smem = (int)sizeof(Smem);
    static int configured = -1;
    int dev = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    if (configured != dev) {
        HN_CUDA_OK(cudaFuncSetAttribute(layout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = dev;
    }
    layout_kernel<<<B, NT, smem, st>>>(y_bon_pix, y_cor, r_px, min_v, force_cuboid, force_raw, max_rows, cor_id, n_rows, z0,
                                       z1, status, peaks, n_peaks);
    HN_LAUNCH_OK();
    return 0;
}

}  // namespace hn
