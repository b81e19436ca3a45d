// Bidirectional LSTM recurrence on thread-block clusters (reference model.py:222-227 nn.LSTM, h0 = c0 = 0,
// gate order i,f,g,o; c' = s(f)c + s(i)tanh(g), h' = s(o)tanh(c')).
//
// Every step needs h_{t-1} of all 512 units.  Exchanged through L2 between CTAs, the store -> fence -> flag -> poll ->
// TMA chain costs about 4.9 us per step and is the whole step time (ncu).  Here one CLUSTER of 16 CTAs owns
// (direction, 8 batch columns) completely, so the per-step all-to-all stays inside the cluster's distributed shared
// memory (~0.1 us latency) and clusters never talk to each other:
//   cluster = 16 CTAs x 32 hidden units;  CTA = 32 units x 4 gates = 128 rows of W_hh
//   W_hh    = fp16 hi plane as mma.sync A fragments in REGISTERS (128 per thread) for the whole sequence,
//             fp16 lo plane as ready-made fragments in SHARED MEMORY (128 KB, written once, read back 32 registers
//             at a time, lane-contiguous so that every read is conflict-free); per-row power-of-two scale
//             (11 + 11 significant bits)
//   step    = D[128 rows x 8 cols] = W[128 x 512] h[512 x 8]: three products Whi*hhi + Whi*hlo + Wlo*hhi with
//             mma.sync.m16n8k16, K split over the 8 warps, partial sums reduced through shared memory in two halves
//             of 64 rows (gates i, f, then g, o: the partial-sum block is 17 KB instead of 33 KB); thread
//             (column = warp, unit = lane) finishes one cell in fp32, writes the fp32 output and the fp16 hi/lo planes
//             of 256*h into a 1152-byte staging block; one thread then bulk-copies that block into the receive
//             buffer of all 16 CTAs of the cluster (cp.async.bulk shared::cta -> shared::cluster), each copy
//             completing on the destination's mbarrier.  Receive / staging buffers are double-buffered by step
//             parity; a peer can only send h_{t+1} after it has received this CTA's h_t, which makes that safe
//             without any further handshake.
//   groups  = one or two column groups of 8 per cluster, interleaved step by step (each group has its own exchange
//             buffers and barriers): while one group's h is in flight between the CTAs the other group's MMAs run.
//             Two groups per cluster when one group each would not fit in one wave of co-resident clusters (see
//             lstm_plan): the batch-32 recurrence then takes 4 clusters = 64 of the 132 SMs and leaves the
//             rest to the next batch's encoder.  Clusters beyond what the device co-schedules run in a later wave.
//   grid    = 2 directions x ceil(B/8) clusters, or 2 directions x ceil(B/16) with two groups per cluster.
#include <cuda_fp16.h>
#include <cstdlib>
#include "hn_common.cuh"
#include "ptx.cuh"

namespace hn {

namespace {

constexpr int HID = 512;
constexpr int CL = 16;                  // CTAs per cluster (non-portable size)
constexpr int UNITS = HID / CL;         // 32 hidden units per CTA
constexpr int NCOL = 8;                 // batch columns per cluster = N of the MMA
constexpr int NT = 256;                 // 8 warps
constexpr float H_SCALE = 256.f;        // h planes carry 256*h (|h| < 1): lo stays in fp16's normal range
constexpr int COLP = 144;               // bytes per column of an exchange block: 64 B hi + 64 B lo + 16 B pad (bank spread)
constexpr int BLK = NCOL * COLP;        // 1152 B: one CTA's h of one step (32 units x 8 columns, hi + lo)
constexpr int PROWS = 64;               // rows of W_hh per partial-sum half (two gates)
constexpr int PCOL = PROWS + 4;         // floats per column of a partial-sum block: 64 rows + 4 pad (bank spread)

constexpr int MAXG = 2;                                        // column groups interleaved by one cluster
constexpr int SM_RECV = 0;                                     // [MAXG][2 parity][16 source CTAs][BLK]
constexpr int SM_STAGE = SM_RECV + MAXG * 2 * CL * BLK;        // [MAXG][2 parity][BLK]
constexpr int SM_PART = SM_STAGE + MAXG * 2 * BLK;             // [8 warps][NCOL][PCOL] fp32 (init: [8 warps][128] row maxima)
constexpr int SM_WLO = SM_PART + 8 * NCOL * PCOL * 4;          // W_hh lo fragments [8 warps][128 registers][32 lanes]
constexpr int SM_BAR = SM_WLO + 8 * 128 * 32 * 4;              // full[MAXG][2]
constexpr int SM_TOTAL = SM_BAR + 64;
static_assert(SM_RECV % 16 == 0 && SM_STAGE % 16 == 0 && SM_PART % 16 == 0 && SM_WLO % 16 == 0 && SM_BAR % 8 == 0,
              "alignment");
static_assert(SM_TOTAL <= 227 * 1024, "shared memory per block");
static_assert(8 * 128 <= 8 * NCOL * PCOL, "init row maxima fit the partial-sum block");

struct ClArgs {
    const float* xproj;      // [T][B][4096]  (dir*2048 + gate*512 + unit), bias already added
    const float* w_hh[2];    // [2048][512] per direction (PyTorch layout, row = gate*512 + unit)
    float* out;              // [T][B][1024]  (dir*512 + unit)
    int T, B, ngroups;      // ngroups = ceil(B / 8) column groups
    int gpc;                // column groups per cluster (1 or 2)
};

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float lo_elem, float hi_elem) {
    const __half2 h = __floats2half2_rn(lo_elem, hi_elem);
    return *reinterpret_cast<const uint32_t*>(&h);
}
// power-of-two scale that puts max|w| of a row into (2^13, 2^14]
__device__ __forceinline__ float row_scale(float absmax) {
    if (!(absmax > 0.f) || !isfinite(absmax)) return 1.f;
    int e;
    frexpf(16384.f / absmax, &e);
    return ldexpf(1.f, e - 1);
}

__global__ void __launch_bounds__(NT, 1) lstm_cluster_kernel(const ClArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM_BAR);    // [MAXG][2]: h of (group, step parity) arrived from all 16 CTAs
    float* part = reinterpret_cast<float*>(smem + SM_PART);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int gid = lane >> 2, tig = lane & 3;
    const uint32_t rank = cl_rank();
    const int cid = blockIdx.x / CL;
    const int dir = cid % 2;
    const int g_first = (cid / 2) * a.gpc;                              // first column group of this cluster
    const int ng = min(a.gpc, a.ngroups - g_first);                     // column groups this cluster interleaves (1 or 2)
    const int tstep = dir ? -1 : 1;
    const int t_first = dir ? a.T - 1 : 0;

    if (tid == 0) {
        for (int i = 0; i < MAXG * 2; ++i) mbar_init(full_bar + i, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }

    // ---- W_hh slice -> fp16 hi (registers) / lo (shared memory) A fragments.  Warp w owns k in [64w, 64w + 64); local row
    // lr = gate*32 + unit = 16m + 8rs + gid.  Fragment register (rs + 2hf): row 16m + 8rs + gid, k = 64w + 16kt + 2tig + 8hf (+1).
    uint32_t a_hi[8][4][4];
    float* rowbuf = part;                                  // [8 warps][128 rows] during init
#pragma unroll
    for (int m = 0; m < 8; ++m)
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            const int lr = 16 * m + 8 * rs + gid;
            const float* wrow = a.w_hh[dir] + (size_t)((lr >> 5) * HID + rank * UNITS + (lr & 31)) * HID;
            float mx = 0.f;
#pragma unroll
            for (int kt = 0; kt < 4; ++kt)
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    const float2 v = __ldg(reinterpret_cast<const float2*>(wrow + 64 * warp + 16 * kt + tig * 2 + 8 * hf));
                    mx = fmaxf(mx, fmaxf(fabsf(v.x), fabsf(v.y)));
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            if (tig == 0) rowbuf[warp * 128 + lr] = mx;
        }
    __syncthreads();
    // this thread's lo fragments: register (m*4 + kt)*4 + i at wlo[((m*4 + kt)*4 + i) * 32]
    uint32_t* wlo = reinterpret_cast<uint32_t*>(smem + SM_WLO) + warp * 128 * 32 + lane;
    // the cell this thread finishes every step: column `warp`, unit `lane`
    float unscale[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        float mx = 0.f;
        for (int w8 = 0; w8 < 8; ++w8) mx = fmaxf(mx, rowbuf[w8 * 128 + g * 32 + lane]);
        unscale[g] = 1.f / (row_scale(mx) * H_SCALE);
    }
#pragma unroll
    for (int m = 0; m < 8; ++m) {
        float sc[2];
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            float mx = 0.f;
            for (int w8 = 0; w8 < 8; ++w8) mx = fmaxf(mx, rowbuf[w8 * 128 + 16 * m + 8 * rs + gid]);
            sc[rs] = row_scale(mx);
        }
#pragma unroll
        for (int kt = 0; kt < 4; ++kt) {
            uint32_t lo[4];
#pragma unroll
            for (int rs = 0; rs < 2; ++rs) {
                const int lr = 16 * m + 8 * rs + gid;
                const float* wrow = a.w_hh[dir] + (size_t)((lr >> 5) * HID + rank * UNITS + (lr & 31)) * HID;
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    const float2 v = __ldg(reinterpret_cast<const float2*>(wrow + 64 * warp + 16 * kt + tig * 2 + 8 * hf));
                    const float s0 = v.x * sc[rs], s1 = v.y * sc[rs];
                    const __half2 h = __floats2half2_rn(s0, s1);
                    const float2 b = __half22float2(h);
                    a_hi[m][kt][rs + 2 * hf] = *reinterpret_cast<const uint32_t*>(&h);
                    lo[rs + 2 * hf] = pack_h2(s0 - b.x, s1 - b.y);
                }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) wlo[((m * 4 + kt) * 4 + i) * 32] = lo[i];
        }
    }
    if (tid == 0 && a.T >= 2)
        for (int g2 = 0; g2 < ng; ++g2) mbar_expect_tx(full_bar + g2 * 2 + 0, (uint32_t)(CL * BLK));     // h_0 will arrive here
    __syncthreads();          // rowbuf (aliases the partial sums) is dead from here on
    cl_sync();                // every CTA of the cluster has its barriers initialised and armed

    float c_state[MAXG] = {};
    const int col = warp;                              // this thread's cell: (column `warp`, unit `lane`) of each group

    for (int step = 0; step < a.T; ++step) {
        const int t = t_first + step * tstep;
#pragma unroll
        for (int g2 = 0; g2 < MAXG; ++g2) {
            if (g2 >= ng) break;
            const int col0 = (g_first + g2) * NCOL;
            const int nb = min(NCOL, a.B - col0);                  // valid columns of this group
            float xp[4];
            {
                const float* xb = a.xproj + ((size_t)t * a.B + col0 + min(col, nb - 1)) * 4096 + dir * 2048 + rank * UNITS + lane;
#pragma unroll
                for (int g = 0; g < 4; ++g) xp[g] = __ldg(xb + g * HID);
            }
            float sum[4] = {0.f, 0.f, 0.f, 0.f};
            if (step > 0) {
                const int par = (step - 1) & 1;
                mbar_wait(full_bar + g2 * 2 + par, ((step - 1) >> 1) & 1);
                const uint8_t* rb = smem + SM_RECV + (g2 * 2 + par) * (CL * BLK);
                float* pw = part + warp * (NCOL * PCOL);
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {                   // rows [64 hh, 64 hh + 64): gates 2 hh, 2 hh + 1
                    float v[2][2][4];                              // [mp][mm][fragment element]: this warp's partial sums
#pragma unroll
                    for (int mq = 0; mq < 2; ++mq) {               // two m-tiles per tensor-memory read
                        const int mp = 2 * hh + mq;
                        uint32_t al[32];
#pragma unroll
                        for (int i = 0; i < 32; ++i) al[i] = wlo[(mp * 32 + i) * 32];
                        // six independent accumulators (2 m-tiles x 3 products): consecutive MMAs never depend on each other
                        float d[2][3][4];
#pragma unroll
                        for (int mm = 0; mm < 2; ++mm)
#pragma unroll
                            for (int pr = 0; pr < 3; ++pr)
#pragma unroll
                                for (int e = 0; e < 4; ++e) d[mm][pr][e] = 0.f;
#pragma unroll
                        for (int kt = 0; kt < 4; ++kt) {
                            // B fragments: k = 64*warp + 16*kt + 2*tig (+8) -> source CTA k/32, unit k%32; column gid
                            const uint8_t* hb = rb + (2 * warp + (kt >> 1)) * BLK + gid * COLP + ((kt & 1) * 16 + tig * 2) * 2;
                            const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(hb);
                            const uint32_t bh1 = *reinterpret_cast<const uint32_t*>(hb + 16);
                            const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(hb + 64);
                            const uint32_t bl1 = *reinterpret_cast<const uint32_t*>(hb + 64 + 16);
#pragma unroll
                            for (int mm = 0; mm < 2; ++mm) {
                                const int m = mp * 2 + mm;
                                const uint32_t alo[4] = {al[(mm * 4 + kt) * 4 + 0], al[(mm * 4 + kt) * 4 + 1],
                                                         al[(mm * 4 + kt) * 4 + 2], al[(mm * 4 + kt) * 4 + 3]};
                                mma16816(d[mm][0], a_hi[m][kt], bh0, bh1);
                                mma16816(d[mm][1], a_hi[m][kt], bl0, bl1);
                                mma16816(d[mm][2], alo, bh0, bh1);
                            }
                        }
#pragma unroll
                        for (int mm = 0; mm < 2; ++mm)
#pragma unroll
                            for (int e = 0; e < 4; ++e) v[mq][mm][e] = d[mm][0][e] + (d[mm][1][e] + d[mm][2][e]);
                    }
                    if (hh) __syncthreads();                       // every thread has read the first half
                    // partial sums of this warp's k-range: part[warp][column][row - 64 hh]
#pragma unroll
                    for (int mq = 0; mq < 2; ++mq)
#pragma unroll
                        for (int mm = 0; mm < 2; ++mm) {
                            const int r = 16 * (2 * mq + mm) + gid;
                            pw[(tig * 2) * PCOL + r] = v[mq][mm][0];
                            pw[(tig * 2 + 1) * PCOL + r] = v[mq][mm][1];
                            pw[(tig * 2) * PCOL + r + 8] = v[mq][mm][2];
                            pw[(tig * 2 + 1) * PCOL + r + 8] = v[mq][mm][3];
                        }
                    __syncthreads();
                    // ((p0 + p1) + ...) + p7 over the 8 warps' k-ranges, for the two gates of this half
#pragma unroll
                    for (int gq = 0; gq < 2; ++gq)
#pragma unroll
                        for (int w8 = 0; w8 < 8; ++w8) sum[2 * hh + gq] += part[(w8 * NCOL + col) * PCOL + gq * 32 + lane];
                }
            }
            float pre[4];
#pragma unroll
            for (int g = 0; g < 4; ++g) pre[g] = fmaf(sum[g], unscale[g], xp[g]);
            const float c_new = sigmoidf_(pre[1]) * c_state[g2] + sigmoidf_(pre[0]) * tanhf(pre[2]);
            c_state[g2] = c_new;
            const float h_new = sigmoidf_(pre[3]) * tanhf(c_new);
            if (col < nb) a.out[((size_t)t * a.B + col0 + col) * 1024 + dir * HID + rank * UNITS + lane] = h_new;
            {
                // exchange planes of 256*h for the next step's MMAs
                const float hs = h_new * H_SCALE;
                const __half hh = __float2half_rn(hs);
                __half* sg = reinterpret_cast<__half*>(smem + SM_STAGE + (g2 * 2 + (step & 1)) * BLK + col * COLP) + lane;
                sg[0] = hh;
                sg[32] = __float2half_rn(hs - __half2float(hh));
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> bulk-copy engine
            __syncthreads();       // staging block complete; all reads of the partial sums / receive buffer are done
            if (tid == 0 && step + 1 < a.T) {
                if (step + 2 < a.T) mbar_expect_tx(full_bar + g2 * 2 + ((step + 1) & 1), (uint32_t)(CL * BLK));   // arm for h_{step+1}
                const uint32_t dst = smem_u32(smem + SM_RECV + (g2 * 2 + (step & 1)) * (CL * BLK) + rank * BLK);
                const uint32_t bar = smem_u32(full_bar + g2 * 2 + (step & 1));
                const uint8_t* src = smem + SM_STAGE + (g2 * 2 + (step & 1)) * BLK;
#pragma unroll 1
                for (uint32_t p = 0; p < (uint32_t)CL; ++p) cl_bulk_copy(cl_map(dst, p), src, BLK, cl_map(bar, p));
            }
        }
    }
    cl_sync();     // nobody leaves while a peer's copy may still read this CTA's staging block
}

}  // namespace

// How many of the recurrence's 16-CTA clusters the current device co-schedules (cudaOccupancyMaxActiveClusters, cached
// per device); -1 on error.
static int lstm_max_clusters() {
    // function attributes are per device: set them on every call (cheap); the occupancy answer is cached per device
    int dev = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    cudaError_t e = cudaFuncSetAttribute(lstm_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(lstm_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        return fail("lstm_layer: the 16-CTA recurrence clusters are not supported on device " + std::to_string(dev) + ": " +
                    cudaGetErrorString(e));
    }
    static int cached[64];
    static bool cached_init = false;
    if (!cached_init) { for (int i = 0; i < 64; ++i) cached[i] = -1; cached_init = true; }
    int max_clusters = (dev >= 0 && dev < 64) ? cached[dev] : -1;
    if (max_clusters < 0) {
        max_clusters = 0;
        cudaLaunchConfig_t q = {};
        q.gridDim = dim3(2 * 4 * CL);
        q.blockDim = dim3(NT);
        q.dynamicSmemBytes = SM_TOTAL;
        cudaLaunchAttribute qa[1];
        qa[0].id = cudaLaunchAttributeClusterDimension;
        qa[0].val.clusterDim.x = CL; qa[0].val.clusterDim.y = 1; qa[0].val.clusterDim.z = 1;
        q.attrs = qa; q.numAttrs = 1;
        int n = 0;
        if (cudaOccupancyMaxActiveClusters(&n, lstm_cluster_kernel, &q) == cudaSuccess) max_clusters = n;
        (void)cudaGetLastError();
        if (dev >= 0 && dev < 64) cached[dev] = max_clusters;
        if (const char* e = getenv("HN_LSTM_VERBOSE"))
            if (atoi(e)) fprintf(stderr, "lstm_cluster: device %d: max active 16-CTA clusters = %d\n", dev, max_clusters);
    }
    return max_clusters;
}

int lstm_plan(int T, int B, int max_clusters, int plan[7]) {
    HN_CHECK(T >= 1 && B >= 1, "lstm_plan: T and B must be positive");
    if (max_clusters <= 0 && (max_clusters = lstm_max_clusters()) < 0) return -1;
    if (max_clusters < 2)
        return fail("lstm_layer: not supported: the device co-schedules " + std::to_string(max_clusters) +
                    " of the recurrence's 16-CTA clusters, 2 are needed");
    const int ngroups = (B + NCOL - 1) / NCOL;
    // One group per cluster when every cluster fits in one wave: a second group makes a cluster about 1.7x slower
    // (T = 256, kernel time on an H100 at 700 W: 0.71 ms with one group per cluster, 1.20 ms with two).  Two groups
    // per cluster when one group each would need a second wave: batch 32 on the 7 co-resident clusters of that H100
    // then runs on 4 clusters in one wave instead of 8 in two, and leaves 68 SMs to the other stream.
    const int gpc = (2 * ngroups <= max_clusters) ? 1 : MAXG;
    const int per_dir = (ngroups + gpc - 1) / gpc;
    plan[0] = max_clusters;
    plan[1] = ngroups;
    plan[2] = gpc;
    plan[3] = 2 * per_dir;
    plan[4] = ngroups - (per_dir - 1) * gpc;
    plan[5] = B - (ngroups - 1) * NCOL;
    plan[6] = (plan[3] + max_clusters - 1) / max_clusters;
    return 0;
}

// One LSTM layer, both directions, on 16-CTA clusters; xproj [T][B][4096], out [T][B][1024].  Returns 0 on success,
// -1 on error, including a device that cannot co-schedule two such clusters.
int lstm_layer(const float* xproj, const float* w_hh_fwd, const float* w_hh_bwd, float* out, int T, int B,
               cudaStream_t st) {
    int plan[7];
    if (lstm_plan(T, B, 0, plan)) return -1;          // also sets the kernel's function attributes on this device
    ClArgs a;
    a.xproj = xproj; a.w_hh[0] = w_hh_fwd; a.w_hh[1] = w_hh_bwd; a.out = out;
    a.T = T; a.B = B; a.ngroups = plan[1];
    a.gpc = plan[2];
    const int nclusters = plan[3];
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nclusters * CL);
    cfg.blockDim = dim3(NT);
    cfg.dynamicSmemBytes = SM_TOTAL;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    HN_CUDA_OK(cudaLaunchKernelEx(&cfg, lstm_cluster_kernel, a));
    HN_LAUNCH_OK();
    return 0;
}

}  // namespace hn
