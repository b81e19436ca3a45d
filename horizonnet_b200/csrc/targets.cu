// Training targets on the device (reference dataset.py:56-67, 84-120, the label half of PanoCorBonDataset.__getitem__,
// with cor_2_1d and find_occlusion): for N samples, y_bon [N][2][1024] and y_cor [N][1][1024] float32, the flipped and
// rolled corners and the per-corner occlusion flags (DESIGN.md section 11).  Three launches:
//   occ_kernel    one CTA per sample: find_occlusion of the ceiling corners of cor0 (an exact segment-intersection
//                 predicate on their float32 floor-plane points), the flip / roll of the stretched corners, and y_cor
//                 (the circular L1 distance of every column to the nearest non-occluded corner, p_base ** distance);
//   bon_kernel    one CTA per (sample, boundary): cor_2_1d of the stretched corners (cor_2_1d.cuh), then np.flip and
//                 np.roll of the finished row;
//   final_kernel  one CTA per sample: the status in the reference's order, NaN targets for a failed sample.
// Every step keeps numpy's dtype: the corners are float32, so the per-corner steps run in float32, the per-column ones in
// float64.  This file is compiled without FMA contraction (build.py) so the float64 steps round like numpy's.
#include "hn_common.cuh"
#include "cor_2_1d.cuh"
#include "pano_connect.cuh"

namespace hn {

namespace {

constexpr int W = 1024;
constexpr int OT = 256;                    // occ_kernel / final_kernel threads
using c21d::BT;
using c21d::BSmem;
using c21d::MAXC;
using pano::tan_;
using pano::sin_;
using pano::cos_;
enum { ST_OK = 0, ST_ROWS = 1, ST_CORNERS = 2, ST_BOUNDARY = 3, ST_OCCLUDED = 4 };

struct Samples {                           // the inputs of one call
    const float* cor0;                     // [N][max_rows][2] corners as read (rolled), for the occlusion test
    const float* cor;                      // [N][max_rows][2] the same corners after stretch
    const int* rows;
    const int* flip;
    const int* dx;                         // np.roll shift; < 0: no roll
    int max_rows;
};

__device__ int rows_status(const Samples& p, int n) {
    const int r = p.rows[n];
    if (r <= 0 || r > p.max_rows || (r & 1)) return ST_ROWS;
    if (r < 6) return ST_CORNERS;          // the polyline of the other ceiling corners has < 2 points: shapely refuses it
    return ST_OK;
}

// ---------------------------------------------------------------------------------------------- exact orientation
// Every coordinate is a float32, so each product of two coordinates is exact in float64; an orientation is a sum of
// such products and its sign is read off a nonoverlapping expansion of the sum (Shewchuk's Grow-Expansion).
__device__ __forceinline__ void two_sum(double a, double b, double& s, double& e) {
    s = a + b;
    const double bv = s - a, av = s - bv;
    e = (a - av) + (b - bv);
}

template <int N>
__device__ int sum_sign(const double (&t)[N]) {
    double e[N];
    int m = 0;
    for (int k = 0; k < N; ++k) {
        double q = t[k];
        for (int i = 0; i < m; ++i) {
            double s, r;
            two_sum(q, e[i], s, r);
            e[i] = r;
            q = s;
        }
        e[m++] = q;
    }
    for (int i = N - 1; i >= 0; --i)
        if (e[i] != 0) return e[i] > 0 ? 1 : -1;
    return 0;
}

// sign of (b - a) x (c - a)
__device__ int orient(float ax, float ay, float bx, float by, float cx, float cy) {
    const double t[6] = {(double)bx * cy, -((double)bx * ay), -((double)ax * cy), -((double)by * cx), (double)by * ax,
                         (double)ay * cx};
    return sum_sign(t);
}

// c lies in the bounding box of a, b (for c collinear with them: on the closed segment)
__device__ bool in_box(float ax, float ay, float bx, float by, float cx, float cy) {
    return fminf(ax, bx) <= cx && cx <= fmaxf(ax, bx) && fminf(ay, by) <= cy && cy <= fmaxf(ay, by);
}

// the closed segments (0, 0) - (px, py) and (ax, ay) - (bx, by) meet (GEOS intersects: touching counts)
__device__ bool ray_meets(float px, float py, float ax, float ay, float bx, float by) {
    const int d1 = orient(ax, ay, bx, by, 0.f, 0.f), d2 = orient(ax, ay, bx, by, px, py);
    const int d3 = orient(0.f, 0.f, px, py, ax, ay), d4 = orient(0.f, 0.f, px, py, bx, by);
    if (d1 * d2 < 0 && d3 * d4 < 0) return true;
    if (d1 == 0 && in_box(ax, ay, bx, by, 0.f, 0.f)) return true;
    if (d2 == 0 && in_box(ax, ay, bx, by, px, py)) return true;
    if (d3 == 0 && in_box(0.f, 0.f, px, py, ax, ay)) return true;
    if (d4 == 0 && in_box(0.f, 0.f, px, py, bx, by)) return true;
    return false;
}

// ---------------------------------------------------------------------------------------------- occlusion + y_cor
__global__ void __launch_bounds__(OT) occ_kernel(Samples p, double p_base, float* __restrict__ y_cor,
                                                 float* __restrict__ cor_out, int* __restrict__ occ_out,
                                                 int* __restrict__ part) {
    __shared__ float qx[MAXC], qy[MAXC];               // ceiling corners on the z = -50 plane (find_occlusion)
    __shared__ float cx[2 * MAXC];                     // x of every row after flip and roll
    __shared__ unsigned char occ[MAXC];
    const int n = blockIdx.x;
    int st = rows_status(p, n);
    if (st != ST_OK) {
        if (threadIdx.x == 0) part[n] = st;
        return;
    }
    const int rows = p.rows[n], nc = rows / 2;
    const float* c0 = p.cor0 + (size_t)n * p.max_rows * 2;
    const float* c1 = p.cor + (size_t)n * p.max_rows * 2;
    const float pi = (float)c21d::PI;
    for (int i = threadIdx.x; i < nc; i += OT) {       // coorx2u, coory2v, uv2xy(z=-50) in float32
        const float x = c0[4 * i], y = c0[4 * i + 1];
        const float u = ((x + 0.5f) / 1024.f - 0.5f) * 2.f * pi, v = ((y + 0.5f) / 512.f - 0.5f) * pi;
        const float c = -50.f / tan_(v);
        qx[i] = c * cos_(u);
        qy[i] = c * sin_(u);
    }
    const int f = p.flip[n], d = p.dx[n];
    for (int r = threadIdx.x; r < rows; r += OT) {     // dataset.py:91, 98 in float32
        float x = c1[2 * r];
        if (f) x = 1023.f - x;
        if (d >= 0) {
            float m = fmodf(x + (float)d, 1024.f);      // numpy's float remainder: the sign of the divisor
            if (m != 0) { if (m < 0) m += 1024.f; } else m = 0.f;
            x = m;
        }
        cx[r] = x;
        if (cor_out) {
            cor_out[((size_t)n * p.max_rows + r) * 2] = x;
            cor_out[((size_t)n * p.max_rows + r) * 2 + 1] = c1[2 * r + 1];
        }
    }
    __syncthreads();
    bool any_seen = false;
    for (int i = threadIdx.x; i < nc; i += OT) {       // the ray to corner i against the polyline i+1 .. n-1, 0 .. i-1
        bool o = false;
        for (int k = 0; k + 2 < nc && !o; ++k) {
            const int a = (i + 1 + k) % nc, b = (i + 2 + k) % nc;
            o = ray_meets(qx[i], qy[i], qx[a], qy[a], qx[b], qy[b]);
        }
        occ[i] = o;
        any_seen |= !o;
        if (occ_out) {
            occ_out[(size_t)n * p.max_rows + 2 * i] = o;
            occ_out[(size_t)n * p.max_rows + 2 * i + 1] = o;
        }
    }
    any_seen = __syncthreads_or(any_seen);
    if (!any_seen) {                                   // dist.min(0) of no corner raises
        if (threadIdx.x == 0) part[n] = ST_OCCLUDED;
        return;
    }
    for (int c = threadIdx.x; c < W; c += OT) {        // dataset.py:107-120 in float64
        double best = INFINITY;
        for (int r = 0; r < rows; ++r) {
            if (occ[r >> 1]) continue;
            const double x = cx[r], j = (double)c;
            best = fmin(best, fmin(fabs(x - j), fmin(fabs(x - (j + W)), fabs(x - (j - W)))));
        }
        y_cor[(size_t)n * W + c] = (float)pow(p_base, best);
    }
    if (threadIdx.x == 0) part[n] = ST_OK;
}

// ---------------------------------------------------------------------------------------------- y_bon
__global__ void __launch_bounds__(BT, 1) bon_kernel(Samples p, float* __restrict__ y_bon, int* __restrict__ empty) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    BSmem& s = *reinterpret_cast<BSmem*>(smem_raw);
    double* v = reinterpret_cast<double*>(smem_raw + sizeof(BSmem));
    __shared__ int flag;
    const int n = blockIdx.y, fl = blockIdx.x;        // 0 ceiling, 1 floor
    if (rows_status(p, n) != ST_OK) return;            // final_kernel reports it
    const int nw = p.rows[n] / 2;
    const float* c1 = p.cor + (size_t)n * p.max_rows * 2;
    bool any = false;
    for (int i = threadIdx.x; i < nw; i += BT) {
        s.px[i] = c1[2 * (2 * i + fl)];
        s.py[i] = c1[2 * (2 * i + fl) + 1];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nw; i += BT) {       // a vertical wall adds two points, any other its column range
        long long a, e;
        any |= !pano::wall_range<float>(s.px[i], s.px[(i + 1) % nw], a, e) || e >= a;
    }
    any = __syncthreads_or(any);
    if (threadIdx.x == 0) empty[2 * n + fl] = !any;
    if (!any) return;                                  // ys.max() of no sample raises
    c21d::boundary<float>(s, nw, fl, v, &flag);
    const int f = p.flip[n], d = p.dx[n];
    for (int j = threadIdx.x; j < W; j += BT) {        // np.flip, then np.roll by dx
        int k = d >= 0 ? ((j - d) % W + W) % W : j;
        if (f) k = W - 1 - k;
        y_bon[((size_t)n * 2 + fl) * W + j] = (float)v[k];
    }
}

__global__ void __launch_bounds__(OT) final_kernel(const Samples p, const int* __restrict__ part,
                                                   const int* __restrict__ empty, float* __restrict__ y_bon,
                                                   float* __restrict__ y_cor, int* __restrict__ status) {
    const int n = blockIdx.x;
    int st = part[n];
    if ((st == ST_OK || st == ST_OCCLUDED) && (empty[2 * n] || empty[2 * n + 1])) st = ST_BOUNDARY;
    if (st != ST_OK)
        for (int c = threadIdx.x; c < W; c += OT) {
            y_bon[((size_t)n * 2) * W + c] = NAN;
            y_bon[((size_t)n * 2 + 1) * W + c] = NAN;
            y_cor[(size_t)n * W + c] = NAN;
        }
    if (threadIdx.x == 0) status[n] = st;
}

}  // namespace

int train_targets(const float* cor0, const float* cor, const int* rows, const int* flip, const int* dx, int N, int max_rows,
                  double p_base, float* y_bon, float* y_cor, float* cor_out, int* occlusion, int* status, cudaStream_t st) {
    static int configured = -1;
    int dev = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    const int bon_smem = (int)(sizeof(BSmem) + W * sizeof(double));
    if (configured != dev) {
        HN_CUDA_OK(cudaFuncSetAttribute(bon_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bon_smem));
        configured = dev;
    }
    const Samples p{cor0, cor, rows, flip, dx, max_rows};
    int* ws = nullptr;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ws), (size_t)N * 3 * sizeof(int), st));
    int* part = ws;
    int* empty = ws + N;
    occ_kernel<<<N, OT, 0, st>>>(p, p_base, y_cor, cor_out, occlusion, part);
    HN_LAUNCH_OK();
    bon_kernel<<<dim3(2, N), BT, bon_smem, st>>>(p, y_bon, empty);
    HN_LAUNCH_OK();
    final_kernel<<<N, OT, 0, st>>>(p, part, empty, y_bon, y_cor, status);
    HN_LAUNCH_OK();
    HN_CUDA_OK(cudaFreeAsync(ws, st));
    return 0;
}

}  // namespace hn
