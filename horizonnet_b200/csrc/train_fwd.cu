// Train-mode pieces of HorizonNet.forward (reference train.py:52 calls net(x) under net.train()) that the training step
// (train_step.cu) runs around its convolutions:
//   * batch statistics for BatchNorm2d (torch.nn.BatchNorm2d training branch; reference model.py:130 and torchvision
//     Bottleneck bn1..bn3 / downsample.1): per-channel sums of the raw convolution output and of its square, from which
//     bn_finalize_full (bwd_kernels.cu) takes the batch mean, the biased variance and the running-statistics update;
//   * dropout (nn.LSTM(dropout=0.5) between the two recurrent layers, model.py:226, and nn.Dropout(0.5) before the
//     linear head, model.py:228 / :265): counter-based Philox4x32-10 masks, so a mask is a pure function of
//     (seed, which, element index) and the oracle can be handed exactly the mask the device applied.
#include "hn_common.cuh"

namespace hn {
namespace {

constexpr int ST_THREADS = 256;

// sums[c] += sum z, sums[C + c] += sum z^2 over the interior pixels of a fp32 halo-NHWC tensor.
// Block = CL4 channel-quad lanes x (256 / CL4) pixel lanes: a thread owns 4 consecutive channels (one 16-byte load per
// pixel) and walks its rows with 32-bit index arithmetic (round 2: the first version spent its time in 64-bit
// divisions of a flat pixel index and scalar loads: 5.3 ms per batch-8 training step for 3.4 GB of input); the sums
// stay fp64 per element, so the statistics are unchanged.
__global__ void __launch_bounds__(ST_THREADS)
bn_stats_kernel(const float* __restrict__ z, int rows, int W, int C, int halo, int CL4, double* __restrict__ sums) {
    __shared__ double sh[ST_THREADS][8];
    const int cl = threadIdx.x % CL4, pl = threadIdx.x / CL4, PL = ST_THREADS / CL4;
    const int c4 = blockIdx.x * CL4 + cl;
    const bool active = c4 * 4 < C;
    const int Wp = W + 2 * halo;
    double a[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (active) {
        for (int row = blockIdx.y; row < rows; row += gridDim.y) {
            const size_t base = ((size_t)row * Wp + halo) * C + (size_t)c4 * 4;
            for (int w = pl; w < W; w += PL) {
                const size_t i = base + (size_t)w * C;
                const float4 f = *reinterpret_cast<const float4*>(z + i);
                const float v[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    a[j] += (double)v[j];
                    a[4 + j] += (double)v[j] * (double)v[j];
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

// ---- Philox4x32-10 (Salmon et al., SC'11): counter = (index / 4, which, 0, 0), key = seed
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const unsigned int hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
        const unsigned int hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += 0x9E3779B9u;
        key.y += 0xBB67AE85u;
    }
    return ctr;
}

__device__ __forceinline__ float keep_factor(unsigned int r, float p, float inv_keep) {
    // uniform in [0, 1) from the top 24 bits; dropped with probability p (torch: mask ~ Bernoulli(1 - p), then / (1 - p))
    return ((float)(r >> 8) * (1.f / 16777216.f)) >= p ? inv_keep : 0.f;
}

template <bool APPLY>
__global__ void dropout_kernel(float* __restrict__ x, size_t n, float p, float inv_keep, unsigned long long seed,
                               unsigned int which) {
    const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;       // group of 4 consecutive elements
    if (g * 4 >= n) return;
    const uint4 r = philox4x32_10(make_uint4((unsigned int)g, (unsigned int)(g >> 32), which, 0u),
                                  make_uint2((unsigned int)seed, (unsigned int)(seed >> 32)));
    const float f[4] = {keep_factor(r.x, p, inv_keep), keep_factor(r.y, p, inv_keep), keep_factor(r.z, p, inv_keep),
                        keep_factor(r.w, p, inv_keep)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const size_t i = g * 4 + j;
        if (i < n) x[i] = APPLY ? x[i] * f[j] : f[j];
    }
}

__global__ void multiply_kernel(float* __restrict__ x, const float* __restrict__ m, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] *= m[i];
}

}  // namespace

int multiply_inplace(float* x, const float* mask, size_t n, cudaStream_t st) {
    if (n == 0) return 0;
    multiply_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, mask, n);
    HN_LAUNCH_OK();
    return 0;
}

int bn_batch_stats(const Act& z, double* sums, cudaStream_t st) {
    HN_CHECK(z.C >= 4 && z.C <= 4096 && z.C % 4 == 0 && z.B >= 1, "bn_batch_stats: bad tensor (C must be a multiple of 4)");
    HN_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * (size_t)z.C * sizeof(double), st));
    const int C4 = z.C / 4;
    int CL4 = 1;
    while (CL4 * 2 <= C4 && CL4 * 2 <= 64) CL4 *= 2;
    const int cblocks = (C4 + CL4 - 1) / CL4;
    const long long rows = (long long)z.B * z.H;
    HN_CHECK(rows < (1ll << 31), "bn_batch_stats: too many rows");
    long long ysplit = (num_sms() * 8 + cblocks - 1) / cblocks;                  // ~8 resident blocks per SM
    if (ysplit > rows) ysplit = rows;
    if (ysplit > 65535) ysplit = 65535;
    dim3 grid((unsigned)cblocks, (unsigned)ysplit);
    bn_stats_kernel<<<grid, ST_THREADS, 0, st>>>(z.p, (int)rows, z.W, z.C, z.halo, CL4, sums);
    HN_LAUNCH_OK();
    return 0;
}

int dropout_inplace(float* x, size_t n, double p, unsigned long long seed, int which, bool mask_only, cudaStream_t st) {
    HN_CHECK(p >= 0.0 && p < 1.0, "dropout: p must be in [0, 1)");
    if (n == 0) return 0;
    const float inv_keep = (float)(1.0 / (1.0 - p));
    const unsigned blocks = (unsigned)(((n + 3) / 4 + 255) / 256);
    if (mask_only) dropout_kernel<false><<<blocks, 256, 0, st>>>(x, n, (float)p, inv_keep, seed, (unsigned)which);
    else dropout_kernel<true><<<blocks, 256, 0, st>>>(x, n, (float)p, inv_keep, seed, (unsigned)which);
    HN_LAUNCH_OK();
    return 0;
}

}  // namespace hn
