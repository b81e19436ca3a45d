// Shared declarations for libhorizonnet_b200 (sm_90a / H100 only).
//
// Activation layout everywhere on the device: "halo-NHWC"
//     act[b][h][wp][c],  wp in [0, W + 2*halo),  interior column w lives at wp = w + halo.
// The halo columns hold the circular left/right wrap of the interior (reference model.py:27-29
// lr_pad materialises a W+2p copy before every wrapped conv; here every producer kernel writes the
// two wrap columns once, so no consumer ever needs modular addressing and TMA boxes never wrap).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <string>

namespace hn {

// SM count of the current device (132 on an H100 SXM, 114 on an H100 PCIe): grid-size heuristics of the CUDA-core kernels
inline int num_sms() {
    static int cached[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        cached[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
    }
    return cached[dev];
}

void set_error(const std::string& msg);
int  fail(const std::string& msg);                 // records msg, returns -1
void count_launch(int n = 1);                      // kernels launched by this library (bench "gpu_launches")

#define HN_CUDA_OK(expr)                                                                          \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess)                                                                    \
            return ::hn::fail(std::string(#expr) + ": " + cudaGetErrorString(_e) + " at " +       \
                              __FILE__ + ":" + std::to_string(__LINE__));                         \
    } while (0)

#define HN_CHECK(cond, msg)                                                                       \
    do {                                                                                          \
        if (!(cond)) return ::hn::fail(std::string(msg) + " [" #cond "] at " + __FILE__ + ":" +   \
                                       std::to_string(__LINE__));                                 \
    } while (0)

#define HN_LAUNCH_OK()                                                                            \
    do {                                                                                          \
        ::hn::count_launch();                                                                     \
        HN_CUDA_OK(cudaGetLastError());                                                           \
    } while (0)

// A device activation tensor in halo-NHWC layout (fp32).
struct Act {
    float* p = nullptr;
    int B = 0, H = 0, W = 0, C = 0;
    int halo = 0;
    __host__ __device__ int Wp() const { return W + 2 * halo; }
    __host__ __device__ size_t numel() const { return (size_t)B * H * Wp() * C; }
};

// One convolution of the graph (all convs of the path: reference model.py:73,129 + torchvision
// Bottleneck).  Weights are packed [K = kh*kw*Cin][Cout] with k = (dy*kw + dx)*Cin + c; the
// epilogue is y = acc*scale[n] + shift[n] (+ residual) (ReLU), i.e. eval-mode BN (and the GHC conv
// bias) folded into scale/shift.
struct ConvDesc {
    int Cin = 0, Cout = 0;
    int kh = 1, kw = 1;
    int sh = 1, sw = 1;
    int ph = 0;           // zero padding along H (reference keeps it: model.py:48)
    int pw = 0;           // circular padding along W, must be <= input halo
    int relu = 0;
    const float* w = nullptr;       // [K][Cout]
    const float* scale = nullptr;   // [Cout]
    const float* shift = nullptr;   // [Cout]
};

int conv_f32(const ConvDesc& d, const Act& in, const Act& out, const float* residual, cudaStream_t st);
// The tile plan conv_f32 launches with on `sms` SMs (host only): plan = BM, BN, grid_m, grid_n; -1 for a shape it rejects
int conv_f32_plan(const ConvDesc& d, const Act& in, const Act& out, int sms, int plan[4]);
int stem_f32(const float* x_nchw, int B, int in_channels, const float* w_packed, const float* scale,
             const float* shift, const Act& out, cudaStream_t st, bool relu = true);
int maxpool3x3s2(const Act& in, const Act& out, cudaStream_t st, bool out_split = false);

// train-mode forward pieces (train_fwd.cu): batch statistics of a fp32 tensor for BN, and Philox dropout
int bn_batch_stats(const Act& z, double* sums /* [2*C] */, cudaStream_t st);
int dropout_inplace(float* x, size_t n, double p, unsigned long long seed, int which, bool mask_only, cudaStream_t st);
int multiply_inplace(float* x, const float* mask, size_t n, cudaStream_t st);

}  // namespace hn
