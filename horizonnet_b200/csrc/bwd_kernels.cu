// Backward-pass kernels of the training step (SURVEY 8 row f1; reference train.py:272-281 `loss.backward()` through
// model.py:254-281).  First correct path: fp32 CUDA-core kernels over the same halo-NHWC activations as the fp32
// inference path; the data gradient of every convolution reuses the forward implicit-GEMM kernel (conv_f32.cu) on the
// zero-dilated output gradient with flipped weights, so only the weight gradient needs a kernel of its own.
//   conv_wgrad_f32      dW[co][(dy,dx,ci)] = sum_pixels dz[p][co] * im2col(in)[p][(dy,dx,ci)]   (split over pixels, atomics)
//   conv_dgrad_f32      d_in (+)= conv(dilate(dz), flip(W))                                     (conv_f32 does the work)
//   bn_*                train / frozen BatchNorm2d forward-apply, backward reduce + apply (ReLU and identity fused)
//   maxpool_bwd, ghc_to_sequence_bwd, head_bwd_*, lstm_* (gate recompute scan, one backward launch per time step)
// Parity target: torch.autograd on the CPU oracle (tests/test_gpu_parity.py, relative tolerance in the tests).
#include <cstdlib>

#include "hn_common.cuh"
#include "conv_tc.cuh"
#include "bwd_kernels.cuh"

namespace hn {
namespace {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

// ------------------------------------------------------------------------------------------------ weight gradient
struct WgradArgs {
    const float* in;      // forward input, halo-NHWC
    const float* dz;      // gradient of the raw conv output, halo-NHWC (interior read only)
    float* dw;            // [Cout][K] (OHWI), accumulated atomically
    int B, H, Wp, Cin;
    int Ho, Wo, Wop, Cout, out_halo;
    int kh, kw, sh, sw, ph, woff;
    int M, K, m_per_slice;
};

// CTA: 64 output channels x 64 k columns, loop over its pixel slice in chunks of 16.  256 threads, 4 x 4 per thread.
template <bool VEC>
__global__ void __launch_bounds__(256) conv_wgrad_kernel(const WgradArgs a) {
    __shared__ __align__(16) float Zs[16][64 + 4];
    __shared__ __align__(16) float As[16][64 + 4];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int k0 = blockIdx.x * 64, co0 = blockIdx.y * 64;
    const int m_begin = blockIdx.z * a.m_per_slice;
    const int m_end = min(a.M, m_begin + a.m_per_slice);
    // loader coordinates: row lm of the chunk, 4 consecutive columns starting at lc
    const int lm = tid >> 4, lc = (tid & 15) * 4;
    // the 4 k columns this thread loads: (tap, ci) decomposition is fixed for the whole kernel
    int k_ci[4], k_dy[4], k_dx[4];
    bool k_ok[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int k = k0 + lc + j;
        k_ok[j] = k < a.K;
        const int tap = k_ok[j] ? k / a.Cin : 0;
        k_ci[j] = k_ok[j] ? k - tap * a.Cin : 0;
        k_dy[j] = tap / a.kw;
        k_dx[j] = tap - k_dy[j] * a.kw;
    }
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int mc = m_begin; mc < m_end; mc += 16) {
        const int m = mc + lm;
        float4 zv = make_float4(0.f, 0.f, 0.f, 0.f), av = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m < m_end) {
            const int wo = m % a.Wo;
            const int t = m / a.Wo;
            const int ho = t % a.Ho;
            const int b = t / a.Ho;
            const size_t zrow = (((size_t)b * a.Ho + ho) * a.Wop + wo + a.out_halo) * a.Cout;
            if (co0 + lc + 3 < a.Cout) {
                zv = __ldg(reinterpret_cast<const float4*>(a.dz + zrow + co0 + lc));
            } else {
                float* zp = &zv.x;
                for (int j = 0; j < 4; ++j) if (co0 + lc + j < a.Cout) zp[j] = __ldg(a.dz + zrow + co0 + lc + j);
            }
            if (VEC) {
                // Cin % 4 == 0: the 4 columns share a tap and are 4 consecutive channels
                if (k_ok[0]) {
                    const int hi = ho * a.sh - a.ph + k_dy[0];
                    if (hi >= 0 && hi < a.H) {
                        const size_t arow = (((size_t)b * a.H + hi) * a.Wp + wo * a.sw + a.woff + k_dx[0]) * a.Cin;
                        av = __ldg(reinterpret_cast<const float4*>(a.in + arow + k_ci[0]));
                    }
                }
            } else {
                float* ap = &av.x;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (!k_ok[j]) continue;
                    const int hi = ho * a.sh - a.ph + k_dy[j];
                    if (hi < 0 || hi >= a.H) continue;
                    ap[j] = __ldg(a.in + (((size_t)b * a.H + hi) * a.Wp + wo * a.sw + a.woff + k_dx[j]) * a.Cin + k_ci[j]);
                }
            }
        }
        __syncthreads();
        *reinterpret_cast<float4*>(&Zs[lm][lc]) = zv;
        *reinterpret_cast<float4*>(&As[lm][lc]) = av;
        __syncthreads();
#pragma unroll
        for (int mm = 0; mm < 16; ++mm) {
            const float4 z4 = *reinterpret_cast<const float4*>(&Zs[mm][ty * 4]);
            const float4 a4 = *reinterpret_cast<const float4*>(&As[mm][tx * 4]);
            const float zz[4] = {z4.x, z4.y, z4.z, z4.w};
            const float aa[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(zz[i], aa[j], acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int co = co0 + ty * 4 + i;
        if (co >= a.Cout) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + tx * 4 + j;
            if (k < a.K) atomicAdd(a.dw + (size_t)co * a.K + k, acc[i][j]);
        }
    }
}

// Same product on a 128 x 128 tile with 8 x 8 accumulators per thread and a double-buffered, register-prefetched pixel
// loop (Cin % 4 == 0, Cout >= 128, K >= 128): 4 LDS.128 per 64 FMAs instead of 2 per 16.  Each thread owns rows
// {ty*4.., 64+ty*4..} and columns {tx*4.., 64+tx*4..} so that every LDS.128 of a quarter-warp is contiguous.
__global__ void __launch_bounds__(256, 2) conv_wgrad128_kernel(const WgradArgs a) {
    __shared__ __align__(16) float Zs[2][16][128];
    __shared__ __align__(16) float As[2][16][128];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int k0 = blockIdx.x * 128, co0 = blockIdx.y * 128;
    const int m_begin = blockIdx.z * a.m_per_slice;
    const int m_end = min(a.M, m_begin + a.m_per_slice);
    const int lm = tid >> 4, lc = (tid & 15) * 4;
    int k_ci[2], k_dy[2], k_dx[2];
    bool k_ok[2];
#pragma unroll
    for (int g = 0; g < 2; ++g) {
        const int k = k0 + lc + 64 * g;
        k_ok[g] = k < a.K;
        const int tap = k_ok[g] ? k / a.Cin : 0;
        k_ci[g] = k_ok[g] ? k - tap * a.Cin : 0;
        k_dy[g] = tap / a.kw;
        k_dx[g] = tap - k_dy[g] * a.kw;
    }
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    float4 zr[2], ar[2];
    auto load = [&](int mc) {
        const int m = mc + lm;
        zr[0] = zr[1] = ar[0] = ar[1] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m >= m_end) return;
        const int wo = m % a.Wo;
        const int t = m / a.Wo;
        const int ho = t % a.Ho;
        const int b = t / a.Ho;
        const size_t zrow = (((size_t)b * a.Ho + ho) * a.Wop + wo + a.out_halo) * a.Cout;
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            if (co0 + lc + 64 * g + 3 < a.Cout) zr[g] = __ldg(reinterpret_cast<const float4*>(a.dz + zrow + co0 + lc + 64 * g));
            if (k_ok[g]) {
                const int hi = ho * a.sh - a.ph + k_dy[g];
                if (hi >= 0 && hi < a.H)
                    ar[g] = __ldg(reinterpret_cast<const float4*>(
                        a.in + (((size_t)b * a.H + hi) * a.Wp + wo * a.sw + a.woff + k_dx[g]) * a.Cin + k_ci[g]));
            }
        }
    };
    auto store = [&](int buf) {
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            *reinterpret_cast<float4*>(&Zs[buf][lm][lc + 64 * g]) = zr[g];
            *reinterpret_cast<float4*>(&As[buf][lm][lc + 64 * g]) = ar[g];
        }
    };
    load(m_begin);
    store(0);
    __syncthreads();
    int buf = 0;
    for (int mc = m_begin; mc < m_end; mc += 16, buf ^= 1) {
        const bool more = mc + 16 < m_end;
        if (more) load(mc + 16);
#pragma unroll
        for (int mm = 0; mm < 16; ++mm) {
            float zz[8], aa[8];
#pragma unroll
            for (int g = 0; g < 2; ++g) {
                const float4 z4 = *reinterpret_cast<const float4*>(&Zs[buf][mm][ty * 4 + 64 * g]);
                const float4 a4 = *reinterpret_cast<const float4*>(&As[buf][mm][tx * 4 + 64 * g]);
                zz[4 * g] = z4.x; zz[4 * g + 1] = z4.y; zz[4 * g + 2] = z4.z; zz[4 * g + 3] = z4.w;
                aa[4 * g] = a4.x; aa[4 * g + 1] = a4.y; aa[4 * g + 2] = a4.z; aa[4 * g + 3] = a4.w;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(zz[i], aa[j], acc[i][j]);
        }
        if (more) store(buf ^ 1);
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int co = co0 + ty * 4 + (i & 3) + 64 * (i >> 2);
        if (co >= a.Cout) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = k0 + tx * 4 + (j & 3) + 64 * (j >> 2);
            if (k < a.K) atomicAdd(a.dw + (size_t)co * a.K + k, acc[i][j]);
        }
    }
}

// [Cout][kh][kw][Cin] -> [Cout][Cin][kh][kw] (the reference's nn.Conv2d.weight layout)
__global__ void ohwi_to_oihw_kernel(const float* __restrict__ in, float* __restrict__ out, int Cout, int Cin, int kh,
                                    int kw) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)Cout * Cin * kh * kw;
    if (i >= total) return;
    const int dx = (int)(i % kw);
    size_t t = i / kw;
    const int dy = (int)(t % kh); t /= kh;
    const int ci = (int)(t % Cin);
    const int co = (int)(t / Cin);
    out[i] = in[(((size_t)co * kh + dy) * kw + dx) * Cin + ci];
}

// ------------------------------------------------------------------------------------------------ data gradient
// OIHW -> conv_f32 packing [K' = (dy', dx', co)][N = ci] of the flipped, transposed kernel:
//   Wd[(dy'*kw + dx')*Cout + co][ci] = W[co][ci][kh-1-dy'][kw-1-dx']
__global__ void pack_dgrad_weight_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int Cin, int kh,
                                         int kw) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)Cout * Cin * kh * kw;
    if (i >= total) return;
    const int ci = (int)(i % Cin);
    size_t t = i / Cin;
    const int co = (int)(t % Cout); t /= Cout;
    const int dx = (int)(t % kw);
    const int dy = (int)(t / kw);
    out[i] = w[(((size_t)co * Cin + ci) * kh + (kh - 1 - dy)) * kw + (kw - 1 - dx)];
}

// zero-insertion: out[b][ho*sh][wo*sw + 1][c] = dz[b][ho][wo + halo][c], everything else 0, halo columns = circular wrap
__global__ void dilate_kernel(const float* __restrict__ dz, float* __restrict__ out, int B, int Ho, int Wo, int in_halo,
                              int H, int W, int C, int sh, int sw) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;     // over out elements / 4
    const int C4 = C / 4;
    const size_t total = (size_t)B * H * (W + 2) * C4;
    if (i >= total) return;
    const int c4 = (int)(i % C4);
    size_t t = i / C4;
    const int wp = (int)(t % (W + 2)); t /= (W + 2);
    const int h = (int)(t % H);
    const int b = (int)(t / H);
    int w = wp - 1;
    if (w < 0) w += W; else if (w >= W) w -= W;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (h % sh == 0 && w % sw == 0) {
        const int ho = h / sh, wo = w / sw;
        if (ho < Ho && wo < Wo)
            v = __ldg(reinterpret_cast<const float4*>(dz + (((size_t)b * Ho + ho) * (Wo + 2 * in_halo) + wo + in_halo) * C) + c4);
    }
    reinterpret_cast<float4*>(out)[i] = v;
}

// ------------------------------------------------------------------------------------------------ BatchNorm
// statistics of the raw conv output -> everything the forward apply and the backward need, per channel:
//   bn[0..C) scale = gamma*invstd, [C..2C) shift, [2C..3C) mean, [3C..4C) invstd ; running stats moved (train only)
__global__ void bn_finalize_full_kernel(const double* __restrict__ sums, double count, const float* __restrict__ gamma,
                                        const float* __restrict__ beta, const float* __restrict__ bias,
                                        float* __restrict__ running_mean, float* __restrict__ running_var, double factor,
                                        int train, float* __restrict__ bn, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C) return;
    double mean, var;
    if (train) {
        mean = sums[i] / count;
        var = sums[C + i] / count - mean * mean;
        if (var < 0.0) var = 0.0;
    } else {                        // frozen module: running statistics (the conv bias is not part of them)
        mean = (double)running_mean[i] - (bias ? (double)bias[i] : 0.0);
        var = (double)running_var[i];
    }
    const double invstd = 1.0 / sqrt(var + 1e-5);
    const double s = (double)gamma[i] * invstd;
    // `mean` is the mean of z = conv + bias in train mode; in frozen mode it was shifted so that the same
    // formula y = (z - mean_z) * s + beta holds with z = conv + bias
    const double mean_z = train ? mean : mean + (bias ? (double)bias[i] : 0.0);
    bn[i] = (float)s;
    bn[C + i] = (float)((double)beta[i] - mean_z * s);
    bn[2 * C + i] = (float)mean_z;
    bn[3 * C + i] = (float)invstd;
    if (train && factor >= 0.0) {
        const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
        running_mean[i] = (float)((1.0 - factor) * (double)running_mean[i] + factor * mean);
        running_var[i] = (float)((1.0 - factor) * (double)running_var[i] + factor * unbiased);
    }
}

// y = relu?(z*scale + shift (+ res)); interior pixels + the two circular halo columns.  One thread = 4 channels.
__device__ __forceinline__ void store_planes4(unsigned short* __restrict__ planes, size_t plane, size_t o, const float4 v) {
    const float f[4] = {v.x, v.y, v.z, v.w};
    unsigned short h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split_scaled(f[j], h[j], l[j]);
    *reinterpret_cast<uint2*>(planes + o) = make_uint2((unsigned)h[0] | ((unsigned)h[1] << 16), (unsigned)h[2] | ((unsigned)h[3] << 16));
    *reinterpret_cast<uint2*>(planes + plane + o) = make_uint2((unsigned)l[0] | ((unsigned)l[1] << 16), (unsigned)l[2] | ((unsigned)l[3] << 16));
}

// planes != nullptr: also the fp16 hi/lo plane pair of y (the tensor-core conv kernel's operand format, conv_tc.cuh)
__global__ void bn_apply_fwd_kernel(const float* __restrict__ z, const float* __restrict__ bn, const float* __restrict__ res,
                                    float* __restrict__ y, unsigned short* __restrict__ planes, int B, int H, int W, int C,
                                    int relu) {
    const int C4 = C / 4;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)B * H * W * C4;
    if (i >= total) return;
    const int c4 = (int)(i % C4);
    size_t t = i / C4;
    const int w = (int)(t % W);
    const size_t bh = t / W;
    const size_t o = (bh * (W + 2) + w + 1) * C + c4 * 4;
    const float4 zv = *reinterpret_cast<const float4*>(z + o);
    const float4 sc = __ldg(reinterpret_cast<const float4*>(bn) + c4);
    const float4 sf = __ldg(reinterpret_cast<const float4*>(bn + C) + c4);
    float4 v = make_float4(fmaf(zv.x, sc.x, sf.x), fmaf(zv.y, sc.y, sf.y), fmaf(zv.z, sc.z, sf.z), fmaf(zv.w, sc.w, sf.w));
    if (res) {
        const float4 r = *reinterpret_cast<const float4*>(res + o);
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    const size_t oh1 = (bh * (W + 2) + W + 1) * C + c4 * 4, oh0 = (bh * (W + 2)) * C + c4 * 4;
    *reinterpret_cast<float4*>(y + o) = v;
    if (w == 0) *reinterpret_cast<float4*>(y + oh1) = v;
    if (w == W - 1) *reinterpret_cast<float4*>(y + oh0) = v;
    if (planes) {
        const size_t plane = (size_t)B * H * (W + 2) * C;
        store_planes4(planes, plane, o, v);
        if (w == 0) store_planes4(planes, plane, oh1, v);
        if (w == W - 1) store_planes4(planes, plane, oh0, v);
    }
}

// sums[c] = sum g, sums[C+c] = sum g * xhat, g = dy * (relu ? y > 0 : 1), xhat = (z - mean) * invstd
// Block = CL4 channel-quad lanes x (256 / CL4) pixel lanes, rows walked with 32-bit arithmetic, 16-byte loads (same
// layout as bn_stats_kernel in train_fwd.cu; the sums stay fp64 per element).
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ z,
                     const float* __restrict__ bn, int rows, int W, int C, int relu, int CL4, double* __restrict__ sums) {
    __shared__ double sh[256][8];
    const int cl = threadIdx.x % CL4, pl = threadIdx.x / CL4, PL = 256 / CL4;
    const int c4 = blockIdx.x * CL4 + cl;
    const bool active = c4 * 4 < C;
    double a[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (active) {
        const float4 mean = __ldg(reinterpret_cast<const float4*>(bn + 2 * C) + c4);
        const float4 invstd = __ldg(reinterpret_cast<const float4*>(bn + 3 * C) + c4);
        const float mm[4] = {mean.x, mean.y, mean.z, mean.w}, iv[4] = {invstd.x, invstd.y, invstd.z, invstd.w};
        for (int row = blockIdx.y; row < rows; row += gridDim.y) {
            const size_t base = ((size_t)row * (W + 2) + 1) * C + (size_t)c4 * 4;
            for (int w = pl; w < W; w += PL) {
                const size_t i = base + (size_t)w * C;
                const float4 dv = *reinterpret_cast<const float4*>(dy + i);
                const float4 zv = *reinterpret_cast<const float4*>(z + i);
                float g[4] = {dv.x, dv.y, dv.z, dv.w};
                const float zz[4] = {zv.x, zv.y, zv.z, zv.w};
                if (relu) {
                    const float4 yv = *reinterpret_cast<const float4*>(y + i);
                    const float yy[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
                    for (int j = 0; j < 4; ++j) if (!(yy[j] > 0.f)) g[j] = 0.f;
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    a[j] += (double)g[j];
                    a[4 + j] += (double)g[j] * (double)((zz[j] - mm[j]) * iv[j]);
                }
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sh[threadIdx.x][j] = a[j];
    __syncthreads();
    if (pl == 0 && active) {
        for (int k = 1; k < PL; ++k)
#pragma unroll
            for (int j = 0; j < 8; ++j) a[j] += sh[k * CL4 + cl][j];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            atomicAdd(sums + c4 * 4 + j, a[j]);
            atomicAdd(sums + C + c4 * 4 + j, a[4 + j]);
        }
    }
}

// Per channel, once: the two means the apply pass subtracts (as floats: mf[c] = s1/N, mf[C+c] = s2/N) and the
// parameter gradients dgamma = s2, dbeta = s1, dbias = (frozen) scale * s1 | (train) 0.  (The first version divided
// the fp64 sums in every thread of the apply pass: 8 double divisions per 4 outputs.)
__global__ void bn_bwd_means_kernel(const double* __restrict__ sums, double count, const float* __restrict__ bn, int train,
                                    float* __restrict__ mf, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                    float* __restrict__ dbias, int C) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    mf[c] = (float)(sums[c] / count);
    mf[C + c] = (float)(sums[C + c] / count);
    if (dgamma) dgamma[c] = (float)sums[C + c];
    if (dbeta) dbeta[c] = (float)sums[c];
    if (dbias) dbias[c] = train ? 0.f : (float)((double)bn[c] * sums[c]);
}

// dz = scale * (g - s1/N - xhat * s2/N)  (train)   |   scale * g  (frozen);  dres += g;  dz gets circular halo columns.
__global__ void bn_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ z,
                                    const float* __restrict__ bn, const float* __restrict__ mf, int train, int relu,
                                    float* __restrict__ dz, float* __restrict__ dres, unsigned total, int W, int C) {
    const unsigned C4 = (unsigned)C / 4;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const unsigned c4 = i % C4;
    const unsigned t = i / C4;
    const unsigned w = t % (unsigned)W;
    const size_t bh = t / (unsigned)W;
    const size_t o = (bh * (W + 2) + w + 1) * C + c4 * 4;
    const float4 dv = *reinterpret_cast<const float4*>(dy + o);
    float g[4] = {dv.x, dv.y, dv.z, dv.w};
    if (relu) {
        const float4 yv = *reinterpret_cast<const float4*>(y + o);
        const float yy[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) if (!(yy[j] > 0.f)) g[j] = 0.f;
    }
    if (dres) {
        float4 r = *reinterpret_cast<float4*>(dres + o);
        r.x += g[0]; r.y += g[1]; r.z += g[2]; r.w += g[3];
        *reinterpret_cast<float4*>(dres + o) = r;
    }
    const float4 sc4 = __ldg(reinterpret_cast<const float4*>(bn) + c4);
    const float sc[4] = {sc4.x, sc4.y, sc4.z, sc4.w};
    float out[4];
    if (train) {
        const float4 zv = *reinterpret_cast<const float4*>(z + o);
        const float4 mean4 = __ldg(reinterpret_cast<const float4*>(bn + 2 * C) + c4);
        const float4 inv4 = __ldg(reinterpret_cast<const float4*>(bn + 3 * C) + c4);
        const float4 m14 = __ldg(reinterpret_cast<const float4*>(mf) + c4);
        const float4 m24 = __ldg(reinterpret_cast<const float4*>(mf + C) + c4);
        const float zz[4] = {zv.x, zv.y, zv.z, zv.w}, mm[4] = {mean4.x, mean4.y, mean4.z, mean4.w};
        const float iv[4] = {inv4.x, inv4.y, inv4.z, inv4.w};
        const float m1[4] = {m14.x, m14.y, m14.z, m14.w}, m2[4] = {m24.x, m24.y, m24.z, m24.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float xhat = (zz[j] - mm[j]) * iv[j];
            out[j] = sc[j] * (g[j] - m1[j] - xhat * m2[j]);
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) out[j] = sc[j] * g[j];
    }
    const float4 ov = make_float4(out[0], out[1], out[2], out[3]);
    *reinterpret_cast<float4*>(dz + o) = ov;
    if (w == 0) *reinterpret_cast<float4*>(dz + (bh * (W + 2) + W + 1) * C + c4 * 4) = ov;
    if (w == (unsigned)W - 1) *reinterpret_cast<float4*>(dz + (bh * (W + 2)) * C + c4 * 4) = ov;
}

// ------------------------------------------------------------------------------------------------ pooling / tail / head
// MaxPool2d(3, 2, 1) backward (model.py:76; -inf padding on both axes): the gradient of an output goes to the first
// maximum of its window in scan order (torch's rule; ties only happen between ReLU zeros, whose gradient dies anyway).
__global__ void maxpool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dp, float* __restrict__ dx,
                                   int B, int H, int W, int C, int Ho, int Wo) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)B * Ho * Wo * C;
    if (i >= total) return;
    const int c = (int)(i % C);
    size_t t = i / C;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float best = -INFINITY;
    size_t arg = 0;
    bool found = false;
    for (int dy = 0; dy < 3; ++dy) {
        const int h = ho * 2 - 1 + dy;
        if (h < 0 || h >= H) continue;
        for (int dxx = 0; dxx < 3; ++dxx) {
            const int w = wo * 2 - 1 + dxx;
            if (w < 0 || w >= W) continue;
            const size_t o = (((size_t)b * H + h) * (W + 2) + w + 1) * C + c;
            const float v = x[o];
            if (!found || v > best) { best = v; arg = o; found = true; }
        }
    }
    const float g = dp[(((size_t)b * Ho + ho) * (Wo + 2) + wo + 1) * C + c];
    if (found && g != 0.f) atomicAdd(dx + arg, g);
}

struct GhcDst {
    float* p[4];
    int H[4], W[4], C[4], chan_off[4];
    int lg;                   // log2 of the sequence width (1024 or 256)
};

// adjoint of ghc_to_sequence_kernel (tail.cu): scatter d seq[t][b][ch] to the two source columns it interpolated
__global__ void ghc_to_sequence_bwd_kernel(const float* __restrict__ dseq, const GhcDst s, int B) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = ((size_t)256 * B) << s.lg;
    if (i >= total) return;
    const int ch = (int)(i & ((1u << s.lg) - 1));
    const int b = (int)((i >> s.lg) % B);
    const int t = (int)((i >> s.lg) / B);
    int sc = 3;
    if (ch < s.chan_off[1]) sc = 0; else if (ch < s.chan_off[2]) sc = 1; else if (ch < s.chan_off[3]) sc = 2;
    const int H = s.H[sc], W = s.W[sc], C = s.C[sc];
    const int local = ch - s.chan_off[sc];
    const int c = local / H, h = local - c * H;
    const int f = 256 / W;
    const float pos = ((float)t + 0.5f) / (float)f + 0.5f;
    const int i0 = (int)floorf(pos);
    const float l1 = pos - (float)i0;
    const float l0 = 1.f - l1;
    const float d = dseq[i];
    // halo coordinate wp <-> interior column (wp - 1) mod W; the gradient lands on the interior copy
    int w0 = i0 - 1, w1 = min(i0 + 1, W + 1) - 1;
    if (w0 < 0) w0 += W; else if (w0 >= W) w0 -= W;
    if (w1 < 0) w1 += W; else if (w1 >= W) w1 -= W;
    const size_t row = ((size_t)b * H + h) * (W + 2);
    if (l0 != 0.f) atomicAdd(s.p[sc] + (row + w0 + 1) * C + c, l0 * d);
    if (l1 != 0.f) atomicAdd(s.p[sc] + (row + w1 + 1) * C + c, l1 * d);
}

// d[t][b][o] from (dbon [B][2][1024], dcor [B][1][1024]); o = s*4 + k, column t*4 + k (model.py:267-269, 278-279)
__device__ __forceinline__ float head_grad(const float* __restrict__ dbon, const float* __restrict__ dcor, int t, int b,
                                           int o) {
    const int s = o >> 2, k = o & 3;
    return s == 0 ? dcor[(size_t)b * 1024 + t * 4 + k] : dbon[((size_t)b * 2 + (s - 1)) * 1024 + t * 4 + k];
}

// d rnn[t][b][j] = sum_o d[t][b][o] * W[o][j]      (K inputs per row: 1024 bi-LSTM head, 512 last MLP layer)
template <int K>
__global__ void head_bwd_input_kernel(const float* __restrict__ dbon, const float* __restrict__ dcor,
                                      const float* __restrict__ w, float* __restrict__ drnn, int T, int B) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)T * B * K;
    if (i >= total) return;
    const int j = (int)(i % K);
    const int row = (int)(i / K);
    const int t = row / B, b = row - t * B;
    float acc = 0.f;
#pragma unroll
    for (int o = 0; o < 12; ++o) acc = fmaf(head_grad(dbon, dcor, t, b, o), __ldg(w + o * K + j), acc);
    drnn[i] = acc;
}

// dW[o][j] += sum_{t,b} d[t][b][o] * rnn[t][b][j];  db[o] += sum d   (grid: (K / 256, 12, row splits), 256 threads = 256 j;
// every block sums its rows in fp64 and adds the partial sum to the zeroed outputs)
template <int K>
__global__ void head_bwd_weight_kernel(const float* __restrict__ dbon, const float* __restrict__ dcor,
                                       const float* __restrict__ rnn, float* __restrict__ dw, float* __restrict__ db, int T,
                                       int B) {
    const int o = blockIdx.y;
    const int j = blockIdx.x * 256 + threadIdx.x;
    const int rows = T * B, per = (rows + gridDim.z - 1) / gridDim.z;
    const int r0 = blockIdx.z * per, r1 = min(rows, r0 + per);
    double acc = 0.0, accb = 0.0;
    for (int row = r0; row < r1; ++row) {
        const int t = row / B, b = row - t * B;
        const float d = head_grad(dbon, dcor, t, b, o);
        acc += (double)d * (double)rnn[(size_t)row * K + j];
        accb += (double)d;
    }
    atomicAdd(dw + o * K + j, (float)acc);
    if (j == 0) atomicAdd(db + o, (float)accb);
}

// dx[i] = 0 where the ReLU output y[i] was not positive (the gradient of relu at its input)
__global__ void relu_bwd_inplace_kernel(float* __restrict__ dx, const float* __restrict__ y, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && !(y[i] > 0.f)) dx[i] = 0.f;
}

// out[c] = sum_r x[r][c]      (grid over column chunks of 256 x row splits; atomics)
__global__ void col_sum_kernel(const float* __restrict__ x, size_t rows, int cols, float* __restrict__ out) {
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c >= cols) return;
    double acc = 0.0;
    for (size_t r = blockIdx.y; r < rows; r += gridDim.y) acc += (double)x[r * cols + c];
    atomicAdd(out + c, (float)acc);
}

// ------------------------------------------------------------------------------------------------ LSTM
// hprev[dir][t][b][j] = hout[t -/+ 1][b][dir*512 + j] (0 at the start of the direction);
// xpd[dir][t][b][n] = xp[t][b][dir*2048 + n]
__global__ void lstm_gather_kernel(const float* __restrict__ hout, const float* __restrict__ xp, float* __restrict__ hprev,
                                   float* __restrict__ xpd, int T, int B) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t nx = (size_t)2 * T * B * 2048;
    if (i < nx) {
        const int n = (int)(i % 2048);
        size_t t = i / 2048;
        const int b = (int)(t % B); t /= B;
        const int tt = (int)(t % T);
        const int dir = (int)(t / T);
        xpd[i] = xp[((size_t)tt * B + b) * 4096 + dir * 2048 + n];
    }
    const size_t nh = (size_t)2 * T * B * 512;
    if (i < nh) {
        const int j = (int)(i % 512);
        size_t t = i / 512;
        const int b = (int)(t % B); t /= B;
        const int tt = (int)(t % T);
        const int dir = (int)(t / T);
        const int tp = dir == 0 ? tt - 1 : tt + 1;
        hprev[i] = (tp < 0 || tp >= T) ? 0.f : hout[((size_t)tp * B + b) * 1024 + dir * 512 + j];
    }
}

// gates (pre-activation, [dir][t][b][i|f|g|o]) -> activated in place; cell[dir][t][b][j] = c_t.  Thread = (dir, b, j).
__global__ void lstm_cell_scan_kernel(float* __restrict__ gates, float* __restrict__ cell, int T, int B) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * B * 512) return;
    const int j = i % 512;
    const int b = (i / 512) % B;
    const int dir = i / (512 * B);
    float c = 0.f;
    for (int s = 0; s < T; ++s) {
        const int t = dir == 0 ? s : T - 1 - s;
        float* g = gates + (((size_t)dir * T + t) * B + b) * 2048;
        const float ig = sigmoidf_(g[j]), fg = sigmoidf_(g[512 + j]), gg = tanhf(g[1024 + j]), og = sigmoidf_(g[1536 + j]);
        c = fg * c + ig * gg;
        g[j] = ig; g[512 + j] = fg; g[1024 + j] = gg; g[1536 + j] = og;
        cell[(((size_t)dir * T + t) * B + b) * 512 + j] = c;
    }
}

// One backward time step of both directions.  Block = 8 hidden units of one direction, one per warp: first
// dh[b][j] = dout[t][b][dir*512+j] + sum_n dG_prev[b][n] * W_hh[n][j] (W_hh^T rows and dG rows are read as coalesced
// float4 streams, warp-shuffle reduction), then the gate gradients of step t for those units.
struct LstmBwdArgs {
    const float* dout;      // [T][B][1024]
    const float* gates;     // [2][T][B][2048] activated
    const float* cell;      // [2][T][B][512]
    const float* whh_t[2];  // W_hh^T: [512][2048]
    float* dgates;          // [2][T][B][2048]
    float* dc;              // [2][B][512] carry
    int T, B, step;
};

__global__ void __launch_bounds__(256) lstm_bwd_step_kernel(const LstmBwdArgs a) {
    const int dir = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + warp;                      // one hidden unit per warp, 8 per block
    // reverse of the forward order: forward dir walks t = 0..T-1, so its backward starts at T-1
    const int t = dir == 0 ? a.T - 1 - a.step : a.step;
    const int tprev_bwd = dir == 0 ? t + 1 : t - 1;          // the step processed just before this one
    const int tprev_fwd = dir == 0 ? t - 1 : t + 1;          // c_{t-1} in forward order
    const float4* w = reinterpret_cast<const float4*>(a.whh_t[dir] + (size_t)j * 2048);
    for (int b0 = 0; b0 < a.B; b0 += 8) {
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = 0.f;
        if (a.step > 0) {
            const float* dg = a.dgates + (((size_t)dir * a.T + tprev_bwd) * a.B) * 2048;
#pragma unroll 4
            for (int i = lane; i < 512; i += 32) {              // 512 float4 = 2048 gate rows
                const float4 wv = __ldg(w + i);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    if (b0 + q < a.B) {
                        const float4 g = *reinterpret_cast<const float4*>(dg + (size_t)(b0 + q) * 2048 + i * 4);
                        acc[q] = fmaf(g.x, wv.x, fmaf(g.y, wv.y, fmaf(g.z, wv.z, fmaf(g.w, wv.w, acc[q]))));
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < 8; ++q)
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], off);
        }
        // lanes 0..7 finish one (b, j) cell each
        const int b = b0 + lane;
        if (lane < 8 && b < a.B) {
            float dh = 0.f;
#pragma unroll
            for (int q = 0; q < 8; ++q) if (q == lane) dh = acc[q];
            dh += a.dout[((size_t)t * a.B + b) * 1024 + dir * 512 + j];
            const float* g = a.gates + (((size_t)dir * a.T + t) * a.B + b) * 2048;
            const float ig = g[j], fg = g[512 + j], gg = g[1024 + j], og = g[1536 + j];
            const float c = a.cell[(((size_t)dir * a.T + t) * a.B + b) * 512 + j];
            const float cprev = (tprev_fwd < 0 || tprev_fwd >= a.T)
                                    ? 0.f : a.cell[(((size_t)dir * a.T + tprev_fwd) * a.B + b) * 512 + j];
            const float tc = tanhf(c);
            float* dcp = a.dc + ((size_t)dir * a.B + b) * 512 + j;
            const float dcar = a.step > 0 ? *dcp : 0.f;
            const float dc = dcar + dh * og * (1.f - tc * tc);
            float* o = a.dgates + (((size_t)dir * a.T + t) * a.B + b) * 2048;
            o[j] = dc * gg * ig * (1.f - ig);
            o[512 + j] = dc * cprev * fg * (1.f - fg);
            o[1024 + j] = dc * ig * (1.f - gg * gg);
            o[1536 + j] = dh * tc * og * (1.f - og);
            *dcp = dc * fg;
        }
    }
}

// The same recurrence as ONE cooperative launch: every warp keeps its W_hh^T row in registers for all T steps, the steps
// are separated by a grid barrier (arrival counter + bounded spin; a time-out raises *error_flag and lets the kernel
// run out instead of hanging).  dG of the previous step is read with ld.global.cg (written by other CTAs of this launch).
// STAGED (B <= 16): the block copies that step's dG [B][2048] of its direction into shared memory once and its 8 warps
// read it from there (ncu launch list: the eight warps each streaming the same 64 KB from L2 made a step cost 12 us).
template <bool STAGED>
__global__ void __launch_bounds__(256) lstm_bwd_persistent_kernel(const LstmBwdArgs a, unsigned int* __restrict__ barrier,
                                                                  int* __restrict__ error_flag) {
    extern __shared__ float4 sdg[];                        // STAGED: [B][512] float4
    const int dir = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + warp;
    const unsigned int nblocks = gridDim.x * gridDim.y;
    float4 wreg[16];
    {
        const float4* w = reinterpret_cast<const float4*>((dir == 0 ? a.whh_t[0] : a.whh_t[1]) + (size_t)j * 2048);
#pragma unroll
        for (int i = 0; i < 16; ++i) wreg[i] = __ldg(w + lane + 32 * i);
    }
    bool dead = false;
    for (int step = 0; step < a.T; ++step) {
        const int t = dir == 0 ? a.T - 1 - step : step;
        const int tprev_bwd = dir == 0 ? t + 1 : t - 1;
        const int tprev_fwd = dir == 0 ? t - 1 : t + 1;
        if (STAGED && step > 0) {
            const float4* dg4 = reinterpret_cast<const float4*>(a.dgates + (((size_t)dir * a.T + tprev_bwd) * a.B) * 2048);
            for (int i = threadIdx.x; i < a.B * 512; i += 256) sdg[i] = __ldcg(dg4 + i);
            __syncthreads();                               // (the grid barrier's __syncthreads separates this from the last reads)
        }
        for (int b0 = 0; b0 < a.B; b0 += 8) {
            float acc[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] = 0.f;
            if (step > 0) {
                const float* dg = a.dgates + (((size_t)dir * a.T + tprev_bwd) * a.B) * 2048;
#pragma unroll
                for (int i = 0; i < 16; ++i) {
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        if (b0 + q < a.B) {
                            const float4 g = STAGED ? sdg[(b0 + q) * 512 + lane + 32 * i]
                                                    : __ldcg(reinterpret_cast<const float4*>(dg + (size_t)(b0 + q) * 2048) + lane + 32 * i);
                            acc[q] = fmaf(g.x, wreg[i].x, fmaf(g.y, wreg[i].y, fmaf(g.z, wreg[i].z, fmaf(g.w, wreg[i].w, acc[q]))));
                        }
                    }
                }
#pragma unroll
                for (int q = 0; q < 8; ++q)
#pragma unroll
                    for (int off = 16; off > 0; off >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], off);
            }
            const int b = b0 + lane;
            if (lane < 8 && b < a.B) {
                float dh = 0.f;
#pragma unroll
                for (int q = 0; q < 8; ++q) if (q == lane) dh = acc[q];
                dh += a.dout[((size_t)t * a.B + b) * 1024 + dir * 512 + j];
                const float* g = a.gates + (((size_t)dir * a.T + t) * a.B + b) * 2048;
                const float ig = g[j], fg = g[512 + j], gg = g[1024 + j], og = g[1536 + j];
                const float c = a.cell[(((size_t)dir * a.T + t) * a.B + b) * 512 + j];
                const float cprev = (tprev_fwd < 0 || tprev_fwd >= a.T)
                                        ? 0.f : a.cell[(((size_t)dir * a.T + tprev_fwd) * a.B + b) * 512 + j];
                const float tc = tanhf(c);
                float* dcp = a.dc + ((size_t)dir * a.B + b) * 512 + j;
                const float dcar = step > 0 ? *dcp : 0.f;
                const float dc = dcar + dh * og * (1.f - tc * tc);
                float* o = a.dgates + (((size_t)dir * a.T + t) * a.B + b) * 2048;
                o[j] = dc * gg * ig * (1.f - ig);
                o[512 + j] = dc * cprev * fg * (1.f - fg);
                o[1024 + j] = dc * ig * (1.f - gg * gg);
                o[1536 + j] = dh * tc * og * (1.f - og);
                *dcp = dc * fg;
            }
        }
        if (step + 1 == a.T) break;
        // ---- grid barrier
        __syncthreads();
        if (threadIdx.x == 0 && !dead) {
            __threadfence();
            atomicAdd(barrier, 1u);
            const unsigned int target = (unsigned int)(step + 1) * nblocks;
            unsigned int spins = 0;
            while (*reinterpret_cast<volatile unsigned int*>(barrier) < target) {
                if (++spins > (1u << 26)) { atomicExch(error_flag, 1); dead = true; break; }
            }
            __threadfence();
        }
        __syncthreads();
    }
}

// x_nchw [B][Cx][512][1024] in [0,1] -> normalised halo-3 NHWC [B][512][1030][3] (stem weight-gradient operand)
__global__ void stem_input_kernel(const float* __restrict__ x, int Cx, float* __restrict__ out, int B) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)B * 512 * 1030 * 3;
    if (i >= total) return;
    const int c = (int)(i % 3);
    size_t t = i / 3;
    const int wp = (int)(t % 1030); t /= 1030;
    const int h = (int)(t % 512);
    const int b = (int)(t / 512);
    int w = wp - 3;
    if (w < 0) w += 1024; else if (w >= 1024) w -= 1024;
    const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
    out[i] = (__ldg(x + (((size_t)b * Cx + c) * 512 + h) * 1024 + w) - mean[c]) / stdv[c];
}

// OIHW of the transposed convolution: out[ci][co][dy][dx] = w[co][ci][kh-1-dy][kw-1-dx]
__global__ void flip_oihw_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int Cin, int kh, int kw) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)Cout * Cin * kh * kw;
    if (i >= total) return;
    const int dx = (int)(i % kw);
    size_t t = i / kw;
    const int dy = (int)(t % kh); t /= kh;
    const int co = (int)(t % Cout);
    const int ci = (int)(t / Cout);
    out[i] = w[(((size_t)co * Cin + ci) * kh + (kh - 1 - dy)) * kw + (kw - 1 - dx)];
}

// Gradients are orders of magnitude smaller than activations, and the fp16 hi/lo planes (conv_tc.cuh: value * 2^-4) only
// carry ~22 bits for values well above 2^-14: a gradient tensor is therefore multiplied by a power of two that brings its
// largest magnitude to [2^11, 2^12) before it is split, and the convolution result is divided by it in the epilogue
// constants (exact: powers of two); pow2_factor lives in conv_tc.cuh (the tensor-core weight-gradient kernel divides it out too).
// 16-byte loads, grid-stride; the tail (n % 4) goes to the first threads
__global__ void absmax_f32_kernel(const float* __restrict__ x, size_t n, float* __restrict__ out) {
    float m = 0.f;
    const size_t n4 = n / 4, stride = (size_t)gridDim.x * blockDim.x, t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (size_t i = t; i < n4; i += stride) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
        m = fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
    }
    if (t < n - n4 * 4) m = fmaxf(m, fabsf(x[n4 * 4 + t]));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));      // m >= 0: int order = float order
}

__global__ void split_pow2_scalar_kernel(const float* __restrict__ in, unsigned short* __restrict__ out, size_t n,
                                         const float* __restrict__ absmax) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    split_scaled(in[i] * pow2_factor(*absmax), out[i], out[n + i]);
}

// n % 8 == 0 (both planes 16-byte aligned): 8 elements per thread, two 16-byte loads, one 16-byte store per plane
__global__ void split_pow2_kernel(const float* __restrict__ in, unsigned short* __restrict__ out, size_t n,
                                  const float* __restrict__ absmax) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n8 = n / 8;
    const float s = pow2_factor(*absmax);
    if (i < n8) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(in) + 2 * i), b = __ldg(reinterpret_cast<const float4*>(in) + 2 * i + 1);
        const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        unsigned short h[8], l[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) split_scaled(v[j] * s, h[j], l[j]);
        *reinterpret_cast<uint4*>(out + 8 * i) = make_uint4((unsigned)h[0] | ((unsigned)h[1] << 16), (unsigned)h[2] | ((unsigned)h[3] << 16),
                                                            (unsigned)h[4] | ((unsigned)h[5] << 16), (unsigned)h[6] | ((unsigned)h[7] << 16));
        *reinterpret_cast<uint4*>(out + n + 8 * i) = make_uint4((unsigned)l[0] | ((unsigned)l[1] << 16), (unsigned)l[2] | ((unsigned)l[3] << 16),
                                                                (unsigned)l[4] | ((unsigned)l[5] << 16), (unsigned)l[6] | ((unsigned)l[7] << 16));
    }
}

__global__ void aux_div_pow2_kernel(float* __restrict__ aux, int C, const float* __restrict__ absmax) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < C) aux[i] /= pow2_factor(*absmax);
}

__global__ void add_kernel(float* __restrict__ dst, const float* __restrict__ src, size_t n4) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 a = reinterpret_cast<float4*>(dst)[i];
    const float4 b = reinterpret_cast<const float4*>(src)[i];
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    reinterpret_cast<float4*>(dst)[i] = a;
}

__global__ void fill_kernel(float* __restrict__ p, size_t n, float v) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;      // out[c][r] = in[r][c]
    if (i >= (size_t)rows * cols) return;
    const int r = (int)(i % rows);
    const int c = (int)(i / rows);
    out[i] = in[(size_t)r * cols + c];
}

inline unsigned blocks_for(size_t n, int per = 256) { return (unsigned)((n + per - 1) / per); }

}  // namespace

// ================================================================================================ host wrappers
int fill_f32(float* p, size_t n, float v, cudaStream_t st) {
    if (n == 0) return 0;
    fill_kernel<<<blocks_for(n), 256, 0, st>>>(p, n, v);
    HN_LAUNCH_OK();
    return 0;
}

int flip_oihw(const float* w_oihw, float* out, int Cout, int Cin, int kh, int kw, cudaStream_t st) {
    flip_oihw_kernel<<<blocks_for((size_t)Cout * Cin * kh * kw), 256, 0, st>>>(w_oihw, out, Cout, Cin, kh, kw);
    HN_LAUNCH_OK();
    return 0;
}

int add_inplace(float* dst, const float* src, size_t n, cudaStream_t st) {
    HN_CHECK(n % 4 == 0, "add_inplace: element count must be a multiple of 4");
    if (n == 0) return 0;
    add_kernel<<<blocks_for(n / 4), 256, 0, st>>>(dst, src, n / 4);
    HN_LAUNCH_OK();
    return 0;
}

int split_planes_pow2(const float* in, unsigned short* out, size_t n, float* absmax_scratch, cudaStream_t st) {
    HN_CUDA_OK(cudaMemsetAsync(absmax_scratch, 0, sizeof(float), st));
    if (n == 0) return 0;
    size_t blocks = (n / 4 + 256 * 4 - 1) / (256 * 4);                                  // >= 4 float4 per thread
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    if (blocks < 1) blocks = 1;
    HN_CHECK((reinterpret_cast<uintptr_t>(in) & 15) == 0, "split_planes_pow2: input must be 16-byte aligned");
    absmax_f32_kernel<<<(unsigned)blocks, 256, 0, st>>>(in, n, absmax_scratch);
    HN_LAUNCH_OK();
    if (n % 8 == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0)
        split_pow2_kernel<<<blocks_for(n / 8), 256, 0, st>>>(in, out, n, absmax_scratch);
    else
        split_pow2_scalar_kernel<<<blocks_for(n), 256, 0, st>>>(in, out, n, absmax_scratch);
    HN_LAUNCH_OK();
    return 0;
}

int tc_aux_div_pow2(float* tc_aux, int C, const float* absmax_scratch, cudaStream_t st) {
    aux_div_pow2_kernel<<<(C + 255) / 256, 256, 0, st>>>(tc_aux, C, absmax_scratch);
    HN_LAUNCH_OK();
    return 0;
}

// zero-dilated copy of dz for the data gradient of a strided conv (see conv_dgrad_f32); out: geometry of din with C = Cout
int dilate_for_dgrad(const Act& dz, const Act& out, int sh, int sw, cudaStream_t st) {
    HN_CHECK(out.halo == 1 && out.C == dz.C && out.C % 4 == 0, "dilate_for_dgrad: bad tensors");
    dilate_kernel<<<blocks_for(out.numel() / 4), 256, 0, st>>>(dz.p, out.p, dz.B, dz.H, dz.W, dz.halo, out.H, out.W, out.C, sh, sw);
    HN_LAUNCH_OK();
    return 0;
}

int transpose_f32(const float* in, float* out, int rows, int cols, cudaStream_t st) {
    transpose_kernel<<<blocks_for((size_t)rows * cols), 256, 0, st>>>(in, out, rows, cols);
    HN_LAUNCH_OK();
    return 0;
}

int conv_wgrad_f32(const ConvDesc& d, const Act& in, const Act& dz, float* dw_ohwi, cudaStream_t st) {
    HN_CHECK(in.C == d.Cin && dz.C == d.Cout && in.B == dz.B, "conv_wgrad: channel / batch mismatch");
    HN_CHECK(d.pw <= in.halo && d.Cout % 4 == 0, "conv_wgrad: circular pad wider than the input halo, or Cout % 4");
    const int Ho = (in.H + 2 * d.ph - d.kh) / d.sh + 1;
    const int Wo = (in.W + 2 * d.pw - d.kw) / d.sw + 1;
    HN_CHECK(Ho == dz.H && Wo == dz.W, "conv_wgrad: output geometry mismatch");
    WgradArgs a;
    a.in = in.p; a.dz = dz.p; a.dw = dw_ohwi;
    a.B = in.B; a.H = in.H; a.Wp = in.Wp(); a.Cin = d.Cin;
    a.Ho = Ho; a.Wo = Wo; a.Wop = dz.Wp(); a.Cout = d.Cout; a.out_halo = dz.halo;
    a.kh = d.kh; a.kw = d.kw; a.sh = d.sh; a.sw = d.sw; a.ph = d.ph; a.woff = in.halo - d.pw;
    const long long M = (long long)in.B * Ho * Wo;
    HN_CHECK(M < (1ll << 31), "conv_wgrad: M overflows int");
    a.M = (int)M; a.K = d.kh * d.kw * d.Cin;
    HN_CUDA_OK(cudaMemsetAsync(dw_ohwi, 0, (size_t)d.Cout * a.K * sizeof(float), st));
    if (a.M == 0) return 0;
    const bool big = d.Cin % 4 == 0 && d.Cout >= 128 && a.K >= 128 && d.Cout % 4 == 0;
    const int tile = big ? 128 : 64;
    const int gx = (a.K + tile - 1) / tile, gy = (d.Cout + tile - 1) / tile;
    // pixel slices: the CTAs of a launch all do the same amount of work, so pick the slice count whose CTA total fills
    // whole waves of the resident slots best (ncu: 320 CTAs on 296 slots left the SMs idle a third of the time)
    const long long tiles = (long long)gx * gy, slots = (long long)num_sms() * (big ? 2 : 4);
    long long max_slices = (M + 255) / 256;                        // at least 256 pixels per slice
    if (max_slices > 64) max_slices = 64;
    long long slices = 1;
    double best = 0.0;
    for (long long s = 1; s <= max_slices; ++s) {
        const long long total = tiles * s, waves = (total + slots - 1) / slots;
        const double fill = (double)total / (double)(waves * slots);
        if (fill > best + 0.02) { best = fill; slices = s; }       // more slices only for a real gain (more atomics)
    }
    a.m_per_slice = (int)(((M + slices - 1) / slices + 15) / 16 * 16);
    slices = (M + a.m_per_slice - 1) / a.m_per_slice;
    dim3 grid((unsigned)gx, (unsigned)gy, (unsigned)slices);
    if (big) conv_wgrad128_kernel<<<grid, 256, 0, st>>>(a);
    else if (d.Cin % 4 == 0) conv_wgrad_kernel<true><<<grid, 256, 0, st>>>(a);
    else conv_wgrad_kernel<false><<<grid, 256, 0, st>>>(a);
    HN_LAUNCH_OK();
    return 0;
}

int ohwi_to_oihw(const float* in, float* out, int Cout, int Cin, int kh, int kw, cudaStream_t st) {
    const size_t n = (size_t)Cout * Cin * kh * kw;
    ohwi_to_oihw_kernel<<<blocks_for(n), 256, 0, st>>>(in, out, Cout, Cin, kh, kw);
    HN_LAUNCH_OK();
    return 0;
}

int pack_dgrad_weight(const float* w_oihw, float* out, int Cout, int Cin, int kh, int kw, cudaStream_t st) {
    const size_t n = (size_t)Cout * Cin * kh * kw;
    pack_dgrad_weight_kernel<<<blocks_for(n), 256, 0, st>>>(w_oihw, out, Cout, Cin, kh, kw);
    HN_LAUNCH_OK();
    return 0;
}

int conv_dgrad_f32(const ConvDesc& d, const float* wd_packed, const Act& dz, const Act& din, bool accumulate,
                   float* dilate_scratch, const float* ones, const float* zeros, cudaStream_t st) {
    HN_CHECK(dz.C == d.Cout && din.C == d.Cin && dz.B == din.B, "conv_dgrad: channel / batch mismatch");
    HN_CHECK(dz.halo == 1 && din.halo == 1, "conv_dgrad: tensors need a halo of 1");
    HN_CHECK(din.H == dz.H * d.sh && din.W == dz.W * d.sw, "conv_dgrad: input size must be stride x output size");
    HN_CHECK(d.Cout % 16 == 0 && d.Cin % 4 == 0, "conv_dgrad: Cout % 16, Cin % 4");
    Act src = dz;
    if (d.sh != 1 || d.sw != 1) {
        src = din; src.C = d.Cout; src.p = dilate_scratch;
        const size_t n4 = src.numel() / 4;
        dilate_kernel<<<blocks_for(n4), 256, 0, st>>>(dz.p, src.p, dz.B, dz.H, dz.W, dz.halo, din.H, din.W, d.Cout, d.sh,
                                                      d.sw);
        HN_LAUNCH_OK();
    }
    ConvDesc t;
    t.Cin = d.Cout; t.Cout = d.Cin; t.kh = d.kh; t.kw = d.kw; t.sh = 1; t.sw = 1;
    t.ph = d.kh - 1 - d.ph; t.pw = d.kw - 1 - d.pw; t.relu = 0;
    t.w = wd_packed; t.scale = ones; t.shift = zeros;
    return conv_f32(t, src, din, accumulate ? din.p : nullptr, st);
}

int bn_finalize_full(const double* sums, long long count, const float* gamma, const float* beta, const float* bias,
                     float* running_mean, float* running_var, double factor, bool train, float* bn, int C, cudaStream_t st) {
    bn_finalize_full_kernel<<<(C + 255) / 256, 256, 0, st>>>(sums, (double)count, gamma, beta, bias, running_mean,
                                                             running_var, factor, train ? 1 : 0, bn, C);
    HN_LAUNCH_OK();
    return 0;
}

int bn_apply_fwd(const Act& z, const float* bn, const float* res, bool relu, const Act& y, unsigned short* y_planes,
                 cudaStream_t st) {
    HN_CHECK(z.halo == 1 && y.halo == 1 && z.C % 4 == 0 && z.numel() == y.numel(), "bn_apply_fwd: bad tensors");
    const size_t n = (size_t)z.B * z.H * z.W * (z.C / 4);
    bn_apply_fwd_kernel<<<blocks_for(n), 256, 0, st>>>(z.p, bn, res, y.p, y_planes, z.B, z.H, z.W, z.C, relu ? 1 : 0);
    HN_LAUNCH_OK();
    return 0;
}

int bn_bwd(const Act& dy, const Act& y, const Act& z, const float* bn, bool train, bool relu, double* sums, const Act& dz,
           float* dres, float* dgamma, float* dbeta, float* dbias, cudaStream_t st) {
    HN_CHECK(dy.halo == 1 && z.halo == 1 && dz.halo == 1 && z.C % 4 == 0, "bn_bwd: bad tensors");
    const int C = z.C, C4 = C / 4;
    HN_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * (size_t)C * sizeof(double), st));
    int CL4 = 1;
    while (CL4 * 2 <= C4 && CL4 * 2 <= 64) CL4 *= 2;
    const int cblocks = (C4 + CL4 - 1) / CL4;
    const long long rows = (long long)z.B * z.H;
    const size_t npix = (size_t)rows * z.W;
    HN_CHECK(rows < (1ll << 31) && npix * C4 < (1ull << 32), "bn_bwd: tensor too large for 32-bit indexing");
    long long ysplit = (num_sms() * 8 + cblocks - 1) / cblocks;
    if (ysplit > rows) ysplit = rows;
    if (ysplit > 65535) ysplit = 65535;
    bn_bwd_reduce_kernel<<<dim3((unsigned)cblocks, (unsigned)ysplit), 256, 0, st>>>(dy.p, y.p, z.p, bn, (int)rows, z.W, C,
                                                                                     relu ? 1 : 0, CL4, sums);
    HN_LAUNCH_OK();
    float* mf = reinterpret_cast<float*>(sums + 2 * (size_t)C);            // 2*C floats behind the 2*C sums
    bn_bwd_means_kernel<<<(C + 255) / 256, 256, 0, st>>>(sums, (double)npix, bn, train ? 1 : 0, mf, dgamma, dbeta, dbias, C);
    HN_LAUNCH_OK();
    const size_t n = npix * C4;
    bn_bwd_apply_kernel<<<blocks_for(n), 256, 0, st>>>(dy.p, y.p, z.p, bn, mf, train ? 1 : 0, relu ? 1 : 0, dz.p, dres,
                                                       (unsigned)n, z.W, C);
    HN_LAUNCH_OK();
    return 0;
}

int maxpool_bwd(const Act& x, const Act& dp, float* dx, cudaStream_t st) {
    const size_t n = (size_t)dp.B * dp.H * dp.W * dp.C;
    maxpool_bwd_kernel<<<blocks_for(n), 256, 0, st>>>(x.p, dp.p, dx, x.B, x.H, x.W, x.C, dp.H, dp.W);
    HN_LAUNCH_OK();
    return 0;
}

int ghc_to_sequence_bwd(const float* dseq, const Act dghc[4], cudaStream_t st) {
    GhcDst s;
    int off = 0;
    for (int i = 0; i < 4; ++i) {
        s.p[i] = dghc[i].p; s.H[i] = dghc[i].H; s.W[i] = dghc[i].W; s.C[i] = dghc[i].C; s.chan_off[i] = off;
        off += dghc[i].C * dghc[i].H;
    }
    HN_CHECK((off == 1024 || off == 256), "ghc_to_sequence_bwd: the 4 scales must flatten to 1024 or 256 channels");
    s.lg = off == 1024 ? 10 : 8;
    const size_t total = (size_t)256 * dghc[0].B * off;
    ghc_to_sequence_bwd_kernel<<<blocks_for(total), 256, 0, st>>>(dseq, s, dghc[0].B);
    HN_LAUNCH_OK();
    return 0;
}

template <int K>
static int head_bwd_k(const float* dbon, const float* dcor, const float* rnn, const float* w, float* drnn, float* dw, float* db,
                      int T, int B, cudaStream_t st) {
    head_bwd_input_kernel<K><<<blocks_for((size_t)T * B * K), 256, 0, st>>>(dbon, dcor, w, drnn, T, B);
    HN_LAUNCH_OK();
    HN_CUDA_OK(cudaMemsetAsync(dw, 0, 12 * K * sizeof(float), st));
    HN_CUDA_OK(cudaMemsetAsync(db, 0, 12 * sizeof(float), st));
    head_bwd_weight_kernel<K><<<dim3(K / 256, 12, 16), 256, 0, st>>>(dbon, dcor, rnn, dw, db, T, B);
    HN_LAUNCH_OK();
    return 0;
}

int head_bwd(const float* dbon, const float* dcor, const float* rnn, const float* w, float* drnn, float* dw, float* db, int T,
             int B, int K, cudaStream_t st) {
    if (K == 1024) return head_bwd_k<1024>(dbon, dcor, rnn, w, drnn, dw, db, T, B, st);
    if (K == 512) return head_bwd_k<512>(dbon, dcor, rnn, w, drnn, dw, db, T, B, st);
    return fail("head_bwd: K must be 1024 or 512");
}

int relu_bwd_inplace(float* dx, const float* y, size_t n, cudaStream_t st) {
    if (n == 0) return 0;
    relu_bwd_inplace_kernel<<<blocks_for(n), 256, 0, st>>>(dx, y, n);
    HN_LAUNCH_OK();
    return 0;
}

int col_sum(const float* x, size_t rows, int cols, float* out, cudaStream_t st) {
    HN_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)cols * sizeof(float), st));
    if (rows == 0) return 0;
    const unsigned gy = (unsigned)(rows < 64 ? rows : 64);
    col_sum_kernel<<<dim3((cols + 255) / 256, gy), 256, 0, st>>>(x, rows, cols, out);
    HN_LAUNCH_OK();
    return 0;
}

int lstm_gather(const float* hout, const float* xp, float* hprev, float* xpd, int T, int B, cudaStream_t st) {
    lstm_gather_kernel<<<blocks_for((size_t)2 * T * B * 2048), 256, 0, st>>>(hout, xp, hprev, xpd, T, B);
    HN_LAUNCH_OK();
    return 0;
}

int lstm_cell_scan(float* gates, float* cell, int T, int B, cudaStream_t st) {
    lstm_cell_scan_kernel<<<(2 * B * 512 + 127) / 128, 128, 0, st>>>(gates, cell, T, B);
    HN_LAUNCH_OK();
    return 0;
}

// the cooperative kernel for batch B: staged for B <= 16 (dynamic shared memory = one step's dG of one direction)
static void* lstm_bwd_persistent_for(int B, size_t* smem) {
    const bool staged = B <= 16;
    *smem = staged ? (size_t)B * 2048 * sizeof(float) : 0;
    return staged ? reinterpret_cast<void*>(lstm_bwd_persistent_kernel<true>)
                  : reinterpret_cast<void*>(lstm_bwd_persistent_kernel<false>);
}

int lstm_bwd_persistent_fits(int B, bool* fits) {
    size_t smem = 0;
    void* kernel = lstm_bwd_persistent_for(B, &smem);
    int dev = 0, coop = 0, sms = 0, per_sm = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    HN_CUDA_OK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    HN_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (smem) HN_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    HN_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, smem));
    *fits = coop && per_sm * sms >= 128;
    return 0;
}

int lstm_bwd_steps(const float* dout, const float* gates, const float* cell, const float* whh_t_f, const float* whh_t_b,
                   float* dgates, float* dc, int T, int B, unsigned int* barrier, int* error_flag, cudaStream_t st) {
    LstmBwdArgs a;
    a.dout = dout; a.gates = gates; a.cell = cell; a.whh_t[0] = whh_t_f; a.whh_t[1] = whh_t_b; a.dgates = dgates; a.dc = dc;
    a.T = T; a.B = B; a.step = 0;
    bool fits = false;
    if (barrier && error_flag && lstm_bwd_persistent_fits(B, &fits)) return -1;
    if (fits) {
        // one cooperative launch for the whole sequence (128 co-resident CTAs, grid barrier between the steps)
        size_t smem = 0;
        void* kernel = lstm_bwd_persistent_for(B, &smem);
        HN_CUDA_OK(cudaMemsetAsync(barrier, 0, sizeof(unsigned int), st));
        void* args[] = {&a, &barrier, &error_flag};
        HN_CUDA_OK(cudaLaunchCooperativeKernel(kernel, dim3(64, 2), dim3(256), args, smem, st));
        HN_LAUNCH_OK();
        return 0;
    }
    for (int s = 0; s < T; ++s) {
        a.step = s;
        lstm_bwd_step_kernel<<<dim3(64, 2), 256, 0, st>>>(a);
        HN_LAUNCH_OK();
    }
    return 0;
}

int stem_input_nhwc(const float* x, int in_channels, float* out, int B, cudaStream_t st) {
    stem_input_kernel<<<blocks_for((size_t)B * 512 * 1030 * 3), 256, 0, st>>>(x, in_channels, out, B);
    HN_LAUNCH_OK();
    return 0;
}

}  // namespace hn
