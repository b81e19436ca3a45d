// Cuboid-layout evaluation on the device (reference eval_cuboid.py:13-145, test and eval_3diou, with
// misc/panostretch.pano_connect_points and misc/post_proc.infer_coory): for B (dt, gt) pairs of 8-row corner lists, the
// corner error, the pixel error of the ceiling / wall / floor labels and the 3D IoU (DESIGN.md section 10).
// Three launches:
//   bound_kernel  one CTA per (pair, boundary): the dt ceiling, gt ceiling and gt floor of gen_reg_from_xy -- each wall
//                 sampled per column (pano_connect_points), the points sorted by x % 1024 then x then concatenation
//                 order (two stable argsorts), the periodic np.interp to 1024 columns; the dt floor by infer_coory;
//   pe_kernel     one CTA per pair, a thread per column: the corner error, the rounded marks of both label surfaces
//                 and the count of pixels whose label differs, never storing a surface; the statuses up to PE;
//   iou_kernel    one warp per pair: the 24 oriented planes of each room (xyzlst2halfspaces) and the volumes of the
//                 dt room, the gt room and both, each by clipping a box face by face (Sutherland-Hodgman plus a cap
//                 polygon on every cutting plane); the 3D IoU and the last status.
// Every step keeps numpy's dtype: the corners are float32 (dt scaled by (1024, 512) in float32), so the per-corner steps
// run in float32 and the per-column and 3D ones in float64.  This file is compiled without FMA contraction (build.py).
#include "hn_common.cuh"
#include "pano_connect.cuh"

namespace hn {

namespace {

using pano::W;
using pano::H;
using pano::PI;
using pano::tan_;
using pano::sin_;
using pano::cos_;

constexpr int ROWS = 8;                       // the reference's cuboid: 4 corners, ceiling / floor rows alternating
constexpr int WALL_PTS = W / 2 + 1;           // a wall samples at most 513 columns (pano_connect_points' two ranges)
constexpr int NPT = 4 * WALL_PTS;             // points of one boundary
constexpr int PMAX = 4096;                    // power of two >= NPT
constexpr int BT = 1024;                      // bound_kernel / pe_kernel threads: one per column
constexpr int MAXF = 56, MAXV = 56;           // faces of a clipped box (6 + 48 cuts) and vertices per face
constexpr int MAXCAP = 256;                   // points on one cutting plane
constexpr int ONBUF = 24;                     // points on the cutting plane per lane and plane
constexpr double ON_PLANE = 1e-10;            // |distance| <= ON_PLANE * scale: on the plane
constexpr double FLAT_VOLUME = 1e-9;          // volume <= FLAT_VOLUME * scale^3: flat, refused
constexpr int NBOX = 3;                       // starting boxes of 16 * 64^k * scale (k = 0..2): further is unbounded
enum { ST_OK = 0, ST_ERR_ROWS = 1, ST_ERR_INDEX = 2, ST_ERR_COLUMNS = 3, ST_ERR_HULL = 4, ST_DT_FAILED = 5 };

struct Pairs {                                // the inputs of one launch
    const float* dt;
    const int* dt_rows;
    const int* dt_status;                     // NULL, or hn_layout_postproc statuses: 2..5 have no cuboid
    const double* z0;                         // float64 z0 / z1 per pair (NULL: the float32 ones)
    const double* z1;
    const float* z0f;
    const float* z1f;
    const float* gt;
    const int* gt_rows;
    int dt_max_rows, gt_max_rows;
};

__device__ bool dt_failed(const Pairs& p, int b) {
    if (!p.dt_status) return false;
    const int s = p.dt_status[b];
    return s >= 2 && s <= 5;
}
__device__ bool rows_ok(const Pairs& p, int b) { return p.dt_rows[b] == ROWS && p.gt_rows[b] == ROWS; }
__device__ double z0_of(const Pairs& p, int b) { return p.z0 ? p.z0[b] : (double)p.z0f[b]; }
__device__ double z1_of(const Pairs& p, int b) { return p.z1 ? p.z1[b] : (double)p.z1f[b]; }

// corner `row` of the pair's dt (gt = 0) or gt (gt = 1) in pixels, float32
__device__ void corner(const Pairs& p, int b, int gt, int row, float& x, float& y) {
    if (gt) {
        const float* c = p.gt + ((size_t)b * p.gt_max_rows + row) * 2;
        x = c[0];
        y = c[1];
    } else {                                  // eval_cuboid.py:192-194, float32
        const float* c = p.dt + ((size_t)b * p.dt_max_rows + row) * 2;
        x = c[0] * (float)W;
        y = c[1] * (float)H;
    }
}

// --------------------------------------------------------------------------------------------- gen_reg_from_xy
struct BSmem {
    float px[4], py[4];
    long long s[4], e[4];
    int off[5];
    int vert[4];
    double xm[NPT], xr[NPT], y[NPT];          // per point: x % 1024, x, row (concatenation order)
    int perm[PMAX];
    double ex[NPT + 2], ey[NPT + 2];          // sorted, padded by one point on each side (np.interp's period)
};

__device__ bool point_less(const BSmem& s, int i, int j, int n) {
    if ((i < n) != (j < n)) return i < n;
    if (i >= n) return i < j;
    if (s.xm[i] != s.xm[j]) return s.xm[i] < s.xm[j];
    if (s.xr[i] != s.xr[j]) return s.xr[i] < s.xr[j];
    return i < j;
}

__global__ void __launch_bounds__(BT, 1) bound_kernel(Pairs p, double* __restrict__ v) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    BSmem& s = *reinterpret_cast<BSmem*>(smem_raw);
    const int b = blockIdx.y, which = blockIdx.x;     // 0 dt ceiling, 1 gt ceiling, 2 gt floor
    if (dt_failed(p, b) || !rows_ok(p, b)) return;   // pe_kernel sets the status
    const int gt = which > 0, fl = which == 2;
    const double z0 = z0_of(p, b);
    const double z = fl ? z0 : -z0;                    // eval_cuboid.py:110-122
    if (threadIdx.x < 4) corner(p, b, gt, 2 * threadIdx.x + fl, s.px[threadIdx.x], s.py[threadIdx.x]);
    __syncthreads();
    if (threadIdx.x == 0) {
        int o = 0;
        for (int w = 0; w < 4; ++w) {
            const int q = (w + 1) & 3;
            long long a = 1, e = 0;
            int cnt;
            const bool finite = isfinite(s.px[w]) && isfinite(s.px[q]);
            if (finite && pano::wall_range<float>(s.px[w], s.px[q], a, e)) {
                cnt = e >= a ? (int)min(e - a + 1, (long long)WALL_PTS) : 0;
                s.vert[w] = 0;
            } else {                           // vertical (a non-finite column: pe_kernel refuses the pair)
                cnt = 2;
                s.vert[w] = 1;
            }
            s.s[w] = a;
            s.e[w] = e;
            s.off[w] = o;
            o += cnt;
        }
        s.off[4] = o;
    }
    __syncthreads();
    const int n = s.off[4];
    double* out = v + (size_t)b * 4 * W;
    if (n == 0) {                              // no wall samples a column: np.interp has no point, no row to mark
        if (which == 0) out[threadIdx.x] = out[W + threadIdx.x] = NAN;
        else out[(which + 1) * W + threadIdx.x] = NAN;
        return;
    }
    for (int i = threadIdx.x; i < n; i += BT) {
        int w = 0;
        while (i >= s.off[w + 1]) ++w;
        const int q = (w + 1) & 3, k = i - s.off[w];
        double x, y;
        if (s.vert[w]) {                       // pano_connect_points returns both corners, float32
            x = k ? s.px[q] : s.px[w];
            y = k ? s.py[q] : s.py[w];
        } else {
            const int c = (int)(((s.s[w] + k) % W + W) % W);
            x = (double)c;
            y = pano::wall_row<float>(s.px[w], s.py[w], s.px[q], s.py[q], c, z);
        }
        double m = fmod(x, (double)W);         // numpy's float remainder: the sign of the divisor
        if (m != 0) { if (m < 0) m += W; } else m = 0.0;
        s.xm[i] = m;
        s.xr[i] = x;
        s.y[i] = y;
    }
    for (int i = threadIdx.x; i < PMAX; i += BT) s.perm[i] = i;
    __syncthreads();
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    for (int k = 2; k <= np2; k <<= 1)          // bitonic sort of the point indices
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < np2; i += BT) {
                const int l = i ^ j;
                if (l > i) {
                    const bool up = (i & k) == 0;
                    const int a = s.perm[i], c = s.perm[l];
                    if (point_less(s, c, a, n) == up) { s.perm[i] = c; s.perm[l] = a; }
                }
            }
            __syncthreads();
        }
    for (int i = threadIdx.x; i < n; i += BT) { s.ex[i + 1] = s.xm[s.perm[i]]; s.ey[i + 1] = s.y[s.perm[i]]; }
    if (threadIdx.x == 0) {
        s.ex[0] = s.xm[s.perm[n - 1]] - W;
        s.ey[0] = s.y[s.perm[n - 1]];
        s.ex[n + 1] = s.xm[s.perm[0]] + W;
        s.ey[n + 1] = s.y[s.perm[0]];
    }
    __syncthreads();
    const int c = threadIdx.x, m = n + 2;
    const double x = (double)c;
    const double r = pano::interp(s.ex, s.ey, m, x);   // np.interp
    if (which == 0) {
        out[c] = r;
        // post_proc.infer_coory(y0_dt, z1 - z0, z0), float64
        const double h = z1_of(p, b) - z0;
        const double v0 = -((r + 0.5) / H - 0.5) * PI;
        const double c0 = z0 / tan(v0);
        const double v1 = atan2(z0 + h, c0);
        out[W + c] = (-v1 / PI + 0.5) * H - 0.5;
    } else {
        out[(which + 1) * W + c] = r;
    }
}

// --------------------------------------------------------------------------------------------- CE, PE
__device__ int mark(double r, bool& bad) {     // np.round(r).astype(int) as a row index of a 512-row array
    const double q = rint(r);
    if (!(q >= -H && q < H)) { bad = true; return 0; }
    const int i = (int)q;
    return i < 0 ? i + H : i;
}

__global__ void __launch_bounds__(BT) pe_kernel(Pairs p, const double* __restrict__ v, double* __restrict__ ce,
                                                double* __restrict__ pe, int* __restrict__ status) {
    __shared__ int red[BT / 32];
    __shared__ int flag;
    const int b = blockIdx.x, c = threadIdx.x;
    if (dt_failed(p, b) || !rows_ok(p, b)) {
        if (c == 0) status[b] = dt_failed(p, b) ? ST_DT_FAILED : ST_ERR_ROWS;
        return;
    }
    if (c == 0) flag = 0;
    __syncthreads();
    const double* q = v + (size_t)b * 4 * W;
    bool bad = false;
    const int a0 = mark(q[c], bad), a1 = mark(q[W + c], bad), g0 = mark(q[2 * W + c], bad), g1 = mark(q[3 * W + c], bad);
    if (c < 12) {                               // a non-finite column of a boundary corner: no row to mark
        float x, y;
        corner(p, b, c >= 4, c < 4 ? 2 * c : (c < 8 ? 2 * (c - 4) : 2 * (c - 8) + 1), x, y);
        bad |= !isfinite(x);
    }
    // label(r) = number of marks at rows <= r (cumsum of a 0/1 column: two equal marks are one)
    int diff = 0;
    for (int r = 0; r < H; ++r) {
        const int ld = (r >= a0) + (a1 != a0 && r >= a1), lg = (r >= g0) + (g1 != g0 && r >= g1);
        diff += ld != lg;
    }
    for (int o = 16; o; o >>= 1) diff += __shfl_xor_sync(0xffffffffu, diff, o);
    if ((c & 31) == 0) red[c >> 5] = diff;
    if (bad) atomicOr(&flag, 1);
    __syncthreads();
    if (c == 0) {
        long long cnt = 0;
        for (int i = 0; i < BT / 32; ++i) cnt += red[i];
        // CE: float32 up to the mean (numpy's pairwise sum of 8), float64 after (eval_cuboid.py:102-103)
        float d[ROWS];
        for (int i = 0; i < ROWS; ++i) {
            float dx, dy, gx, gy;
            corner(p, b, 0, i, dx, dy);
            corner(p, b, 1, i, gx, gy);
            const float ex = gx - dx, ey = gy - dy;
            d[i] = sqrtf(ex * ex + ey * ey);
        }
        const float sum = ((d[0] + d[1]) + (d[2] + d[3])) + ((d[4] + d[5]) + (d[6] + d[7]));
        const float mse = sum / (float)ROWS;
        ce[b] = (double)(100.f * mse) / sqrt((double)(W * W + H * H));
        pe[b] = (double)(100 * cnt) / (double)(H * W);
        int st = flag ? ST_ERR_INDEX : ST_OK;
        for (int i = 0; i < 4 && st == ST_OK; ++i) {      // eval_3diou's assertions, dt first
            float cx, cy, fx, fy;
            for (int g = 0; g < 2; ++g) {
                corner(p, b, g, 2 * i, cx, cy);
                corner(p, b, g, 2 * i + 1, fx, fy);
                if (cx != fx) st = ST_ERR_COLUMNS;
            }
        }
        status[b] = st;
    }
}

// --------------------------------------------------------------------------------------------- 3D IoU
struct V3 {
    double x, y, z;
};

struct ISmem {
    double pl[48][4];                          // the dt planes, then the gt planes: n.x + d <= 0
    V3 f[MAXF][MAXV];                          // faces of the clipped polyhedron, counter-clockwise from outside
    int nv[MAXF];                              // vertices per face (0: clipped away)
    int lab[MAXF];                             // 0..5: a face of the starting box
    V3 tmp[32][MAXV];                          // one lane's clipped face
    V3 on[32][ONBUF];                          // one lane's points on the cutting plane
    V3 cap[MAXCAP];
    double ang[MAXCAP];
    int ord[MAXCAP];
    int nf, ncap, overflow;
};

__device__ double side(const double* h, const V3& v) { return ((h[0] * v.x + h[1] * v.y) + h[2] * v.z) + h[3]; }

// eval_3diou.py:58-77 for corner i of one room: float64 floor and ceiling points (np_coor2xy with floorW = floorH = 1)
__device__ void room_corner(const Pairs& p, int b, int gt, int i, V3& fl, V3& cl) {
    float fx, fy, cx, cy;
    corner(p, b, gt, 2 * i + 1, fx, fy);
    corner(p, b, gt, 2 * i, cx, cy);
    const float pi = (float)PI, ch = -1.6f;
    const float u = ((fx + 0.5f) / (float)W - 0.5f) * 2.f * pi;
    const float v = -(((fy + 0.5f) / (float)H - 0.5f) * pi);
    const float c = ch / tan_(v);
    const float x = c * sin_(u) + 0.5f - 0.5f, y = -c * cos_(u) + 0.5f - 0.5f;   // + floorW / 2 - 0.5 in float32
    fl = V3{(double)x, (double)y, -1.6};
    const double r = sqrt((double)x * (double)x + (double)y * (double)y);
    const float v2 = -(((cy + 0.5f) / (float)H - 0.5f) * pi);
    cl = V3{(double)x, (double)y, r * (double)tan_(v2)};
}

// tri2halfspace: the plane of the triangle, oriented so that the origin is inside
__device__ void tri(const V3& pa, const V3& pb, const V3& q, double* h) {
    const double a0 = pa.x - q.x, a1 = pa.y - q.y, a2 = pa.z - q.z, b0 = pb.x - q.x, b1 = pb.y - q.y, b2 = pb.z - q.z;
    double n0 = a1 * b2 - a2 * b1, n1 = a2 * b0 - a0 * b2, n2 = a0 * b1 - a1 * b0;   // np.cross
    if ((-n0 * q.x + -n1 * q.y) + -n2 * q.z > 0) { n0 = -n0; n1 = -n1; n2 = -n2; }
    h[0] = n0;
    h[1] = n1;
    h[2] = n2;
    h[3] = (-n0 * q.x + -n1 * q.y) + -n2 * q.z;
}

// Clip the polyhedron in s by the plane h (warp-wide); the faces' vertex counts are <= MAXV - 1 before the cut.
__device__ void clip(ISmem& s, const double* h, int label, double eps) {
    const int lane = threadIdx.x;
    if (h[0] == 0 && h[1] == 0 && h[2] == 0) return;            // a zero normal: no-op
    const double tol = eps * sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
    const int nf = s.nf;
    bool out = false;
    for (int f = lane; f < nf; f += 32)
        for (int i = 0; i < s.nv[f]; ++i) out |= side(h, s.f[f][i]) > tol;
    if (!__any_sync(0xffffffffu, out)) return;
    int non = 0;
    for (int f = lane; f < nf; f += 32) {
        const int k = s.nv[f];
        int m = 0;
        for (int i = 0; i < k; ++i) {
            const V3 a = s.f[f][i], bb = s.f[f][(i + 1) % k];
            const double sa = side(h, a), sb = side(h, bb);
            const int ca = sa > tol ? 1 : (sa < -tol ? -1 : 0), cb = sb > tol ? 1 : (sb < -tol ? -1 : 0);
            if (ca <= 0) {
                s.tmp[lane][m++] = a;
                if (ca == 0) { if (non < ONBUF) s.on[lane][non] = a; ++non; }
            }
            if (ca * cb < 0) {                  // the crossing, from the inside end: both faces of the edge agree
                const V3 u = ca < 0 ? a : bb, w = ca < 0 ? bb : a;
                const double su = ca < 0 ? sa : sb, sw = ca < 0 ? sb : sa;
                const double t = su / (su - sw);
                const V3 x{u.x + t * (w.x - u.x), u.y + t * (w.y - u.y), u.z + t * (w.z - u.z)};
                s.tmp[lane][m++] = x;
                if (non < ONBUF) s.on[lane][non] = x;
                ++non;
            }
        }
        if (m > MAXV - 1) { s.overflow = 1; m = 0; }
        for (int i = 0; i < m; ++i) s.f[f][i] = s.tmp[lane][i];
        s.nv[f] = m >= 3 ? m : 0;
    }
    if (non > ONBUF) { s.overflow = 1; non = ONBUF; }
    int off = non;                              // the points on the plane in lane order
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, off, o);
        if (lane >= o) off += t;
    }
    const int total = __shfl_sync(0xffffffffu, off, 31);
    off -= non;
    if (total > MAXCAP) { if (lane == 0) s.overflow = 1; __syncwarp(); return; }
    for (int i = 0; i < non; ++i) s.cap[off + i] = s.on[lane][i];
    __syncwarp();
    if (total < 3 || nf >= MAXF) { if (lane == 0 && total >= 3) s.overflow = 1; __syncwarp(); return; }
    // the cap: the points ordered counter-clockwise about the outward normal h[0..2]
    const double n0 = h[0], n1 = h[1], n2 = h[2];
    const double a0 = fabs(n0), a1 = fabs(n1), a2 = fabs(n2);
    const int ax = (a0 <= a1 && a0 <= a2) ? 0 : (a1 <= a2 ? 1 : 2);
    const double e0 = ax == 0, e1 = ax == 1, e2 = ax == 2;
    const double u0 = n1 * e2 - n2 * e1, u1 = n2 * e0 - n0 * e2, u2 = n0 * e1 - n1 * e0;        // n x e
    const double w0 = n1 * u2 - n2 * u1, w1 = n2 * u0 - n0 * u2, w2 = n0 * u1 - n1 * u0;        // n x (n x e)
    double cx = 0, cy = 0, cz = 0;
    for (int i = 0; i < total; ++i) { cx += s.cap[i].x; cy += s.cap[i].y; cz += s.cap[i].z; }
    cx /= total;
    cy /= total;
    cz /= total;
    for (int i = lane; i < total; i += 32) {
        const double dx = s.cap[i].x - cx, dy = s.cap[i].y - cy, dz = s.cap[i].z - cz;
        s.ang[i] = atan2(dx * w0 + dy * w1 + dz * w2, dx * u0 + dy * u1 + dz * u2);
    }
    __syncwarp();
    if (lane == 0) {
        for (int i = 0; i < total; ++i) {       // insertion sort by (angle, index)
            int j = i;
            while (j > 0 && s.ang[s.ord[j - 1]] > s.ang[i]) { s.ord[j] = s.ord[j - 1]; --j; }
            s.ord[j] = i;
        }
        const int g = nf;
        int k = 0;
        for (int i = 0; i < total; ++i) {       // each point comes from both faces of its edge: keep one
            const V3 q = s.cap[s.ord[i]];
            if (k && q.x == s.f[g][k - 1].x && q.y == s.f[g][k - 1].y && q.z == s.f[g][k - 1].z) continue;
            if (k == MAXV - 1) { s.overflow = 1; break; }
            s.f[g][k++] = q;
        }
        if (k > 1 && s.f[g][k - 1].x == s.f[g][0].x && s.f[g][k - 1].y == s.f[g][0].y && s.f[g][k - 1].z == s.f[g][0].z) --k;
        if (k >= 3) {
            s.nv[g] = k;
            s.lab[g] = label;
            s.nf = nf + 1;
        }
    }
    __syncwarp();
}

// Volume of the intersection of planes pl[first .. first + count) (warp-wide); touch: the result meets the box.
__device__ double region_volume(ISmem& s, int first, int count, double R, bool& touch) {
    const int lane = threadIdx.x;
    double vol = 0;
    double L = 16.0 * R;
    for (int stage = 0; stage < NBOX; ++stage, L *= 64.0) {
        if (lane == 0) {
            const double m = -L, q = L;
            const double bx[6][4][3] = {{{q, m, m}, {q, q, m}, {q, q, q}, {q, m, q}}, {{m, m, m}, {m, m, q}, {m, q, q}, {m, q, m}},
                                        {{m, q, m}, {m, q, q}, {q, q, q}, {q, q, m}}, {{m, m, m}, {q, m, m}, {q, m, q}, {m, m, q}},
                                        {{m, m, q}, {q, m, q}, {q, q, q}, {m, q, q}}, {{m, m, m}, {m, q, m}, {q, q, m}, {q, m, m}}};
            for (int f = 0; f < 6; ++f) {
                for (int i = 0; i < 4; ++i) s.f[f][i] = V3{bx[f][i][0], bx[f][i][1], bx[f][i][2]};
                s.nv[f] = 4;
                s.lab[f] = f;
            }
            s.nf = 6;
        }
        __syncwarp();
        for (int i = 0; i < count; ++i) clip(s, s.pl[first + i], 6 + i, ON_PLANE * R);
        bool t = false;
        double v = 0;
        for (int f = lane; f < s.nf; f += 32) {
            const int k = s.nv[f];
            if (k && s.lab[f] < 6) t = true;
            for (int i = 1; i + 1 < k; ++i) {   // triangle fans around the origin
                const V3 a = s.f[f][0], p1 = s.f[f][i], p2 = s.f[f][i + 1];
                v += a.x * (p1.y * p2.z - p1.z * p2.y) + a.y * (p1.z * p2.x - p1.x * p2.z) + a.z * (p1.x * p2.y - p1.y * p2.x);
            }
        }
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        touch = __any_sync(0xffffffffu, t);
        vol = v / 6;
        __syncwarp();
        if (!touch) break;
    }
    return vol;
}

__global__ void __launch_bounds__(32) iou_kernel(Pairs p, double* __restrict__ ce, double* __restrict__ pe,
                                                double* __restrict__ iou3d, int* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ISmem& s = *reinterpret_cast<ISmem*>(smem_raw);
    const int b = blockIdx.x, lane = threadIdx.x;
    int st = status[b];
    double iou = NAN;
    if (st == ST_OK) {
        V3 fl[2][4], cl[2][4];
        double R = 0;
        bool finite = true;
        for (int g = 0; g < 2; ++g)
            for (int i = 0; i < 4; ++i) {
                room_corner(p, b, g, i, fl[g][i], cl[g][i]);
                const double c[6] = {fl[g][i].x, fl[g][i].y, fl[g][i].z, cl[g][i].x, cl[g][i].y, cl[g][i].z};
                for (int k = 0; k < 6; ++k) { finite &= isfinite(c[k]); R = fmax(R, fabs(c[k])); }
            }
        R += 1.0;
        if (lane == 0) {
            for (int g = 0; g < 2; ++g)          // xyzlst2halfspaces, 6 planes per corner
                for (int i = 0; i < 4; ++i) {
                    const int a = (i + 3) & 3, n = (i + 1) & 3;
                    double* h = s.pl[g * 24 + i * 6];
                    tri(fl[g][a], fl[g][n], fl[g][i], h);
                    tri(fl[g][a], cl[g][i], fl[g][i], h + 4);
                    tri(cl[g][i], fl[g][n], fl[g][i], h + 8);
                    tri(cl[g][a], cl[g][n], cl[g][i], h + 12);
                    tri(cl[g][a], fl[g][i], cl[g][i], h + 16);
                    tri(fl[g][i], cl[g][n], cl[g][i], h + 20);
                }
            s.overflow = 0;
        }
        __syncwarp();
        bool through = false;                    // a plane through the origin: qhull's feasible point is not inside
        for (int i = 0; i < 48; ++i)
            through |= s.pl[i][3] == 0 && (s.pl[i][0] != 0 || s.pl[i][1] != 0 || s.pl[i][2] != 0);
        st = ST_ERR_HULL;
        if (finite && !through) {
            bool t_dt, t_gt, t_in;
            const double v_dt = region_volume(s, 0, 24, R, t_dt);
            const double v_gt = region_volume(s, 24, 24, R, t_gt);
            if (!t_dt && !t_gt) {
                const double v_in = region_volume(s, 0, 48, R, t_in);
                const double flat = FLAT_VOLUME * R * R * R;
                if (!s.overflow && fmin(v_dt, fmin(v_gt, v_in)) > flat) {
                    iou = 100 * v_in / (v_dt + v_gt - v_in);
                    st = ST_OK;
                }
            }
        }
    }
    if (lane == 0) {
        if (st != ST_OK) {
            ce[b] = NAN;
            pe[b] = NAN;
        }
        iou3d[b] = iou;
        status[b] = st;
    }
}

}  // namespace

int layout_eval_cuboid(const float* dt, const int* dt_rows, const int* dt_status, int dt_max_rows, const double* z0,
                       const double* z1, const float* z0f, const float* z1f, const float* gt, const int* gt_rows,
                       int gt_max_rows, int B, double* ce, double* pe, double* iou3d, int* status, cudaStream_t st) {
    static int configured = -1;
    int dev = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    if (configured != dev) {
        HN_CUDA_OK(cudaFuncSetAttribute(bound_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BSmem)));
        HN_CUDA_OK(cudaFuncSetAttribute(iou_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ISmem)));
        configured = dev;
    }
    const Pairs p{dt, dt_rows, dt_status, z0, z1, z0f, z1f, gt, gt_rows, dt_max_rows, gt_max_rows};
    double* v = nullptr;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&v), (size_t)B * 4 * W * sizeof(double), st));
    bound_kernel<<<dim3(3, B), BT, sizeof(BSmem), st>>>(p, v);
    HN_LAUNCH_OK();
    pe_kernel<<<B, BT, 0, st>>>(p, v, ce, pe, status);
    HN_LAUNCH_OK();
    iou_kernel<<<B, 32, sizeof(ISmem), st>>>(p, ce, pe, iou3d, status);
    HN_LAUNCH_OK();
    HN_CUDA_OK(cudaFreeAsync(v, st));
    return 0;
}

}  // namespace hn
