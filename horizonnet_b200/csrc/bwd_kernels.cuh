// Backward-pass building blocks (bwd_kernels.cu), fp32 halo-NHWC.  See the .cu for what each one computes.
#pragma once
#include "hn_common.cuh"

namespace hn {

int fill_f32(float* p, size_t n, float v, cudaStream_t st);
int transpose_f32(const float* in, float* out, int rows, int cols, cudaStream_t st);           // out[c][r] = in[r][c]
int flip_oihw(const float* w_oihw, float* out, int Cout, int Cin, int kh, int kw, cudaStream_t st);   // OIHW of the transposed conv
int add_inplace(float* dst, const float* src, size_t n, cudaStream_t st);
// fp32 gradient tensor -> fp16 hi/lo planes of (x * 2^k), k from the tensor's absmax (left in absmax_scratch[0]);
// tc_aux_div_pow2 folds 2^-k into the first C epilogue constants (accumulator -> true units) of the conv that consumes them
int split_planes_pow2(const float* in, unsigned short* out, size_t n, float* absmax_scratch, cudaStream_t st);
int tc_aux_div_pow2(float* tc_aux, int C, const float* absmax_scratch, cudaStream_t st);
int dilate_for_dgrad(const Act& dz, const Act& out, int sh, int sw, cudaStream_t st);

// dW[Cout][kh][kw][Cin] (zeroed here, then accumulated); in = the conv's forward input, dz = d(raw conv output)
int conv_wgrad_f32(const ConvDesc& d, const Act& in, const Act& dz, float* dw_ohwi, cudaStream_t st);
// The same product on tensor-core (wgrad_tc.cu) from the split planes of the input and of dz (split_planes_pow2; dz_absmax =
// the float it left behind): Cin, Cout multiples of 64, halo 0 or 1, strides 1 or 2.  HN_WGRAD_TC=0/1 overrides the default.
#ifndef HN_WGRAD_TC_DEFAULT
#define HN_WGRAD_TC_DEFAULT 1
#endif
bool wgrad_tc_on();
bool conv_wgrad_tc_supported(const ConvDesc& d, const Act& in, const Act& dz);
int conv_wgrad_tc_plan(const ConvDesc& d, const Act& in, const Act& dz, int sms, int plan[10]);      // host-only (tests)
int conv_wgrad_tc(const ConvDesc& d, const Act& in, const unsigned short* in_planes, const Act& dz,
                  const unsigned short* dz_planes, const float* dz_absmax, float* dw_ohwi, cudaStream_t st);
int ohwi_to_oihw(const float* in, float* out, int Cout, int Cin, int kh, int kw, cudaStream_t st);
// flipped / transposed weights in conv_f32's [K][N] packing, for conv_dgrad_f32
int pack_dgrad_weight(const float* w_oihw, float* out, int Cout, int Cin, int kh, int kw, cudaStream_t st);
// din (+)= conv_transpose(dz, W).  dz: halo 1 with circular halo columns; dilate_scratch: din.numel()/Cin*Cout floats
// (strided convs only); ones / zeros: >= Cin floats of 1 / 0.
int conv_dgrad_f32(const ConvDesc& d, const float* wd_packed, const Act& dz, const Act& din, bool accumulate,
                   float* dilate_scratch, const float* ones, const float* zeros, cudaStream_t st);

// bn[4*C]: scale, shift, mean of z, invstd.  train: from the batch sums (bn_batch_stats) + running-stat update;
// frozen: from the running statistics.
int bn_finalize_full(const double* sums, long long count, const float* gamma, const float* beta, const float* bias,
                     float* running_mean, float* running_var, double factor, bool train, float* bn, int C, cudaStream_t st);
// y_planes (nullable): also write y as fp16 hi/lo planes, the tensor-core conv kernel's operand format
int bn_apply_fwd(const Act& z, const float* bn, const float* res, bool relu, const Act& y, unsigned short* y_planes,
                 cudaStream_t st);
// dz (with halo columns), dres += relu-masked dy, parameter gradients; sums: 3*C doubles of scratch
int bn_bwd(const Act& dy, const Act& y, const Act& z, const float* bn, bool train, bool relu, double* sums, const Act& dz,
           float* dres, float* dgamma, float* dbeta, float* dbias, cudaStream_t st);

int maxpool_bwd(const Act& x, const Act& dp, float* dx, cudaStream_t st);                      // dx accumulated (atomics)
int ghc_to_sequence_bwd(const float* dseq, const Act dghc[4], cudaStream_t st);                // accumulated (atomics)
// K = 1024 (bi-LSTM head) or 512 (last layer of the MLP head): rnn / drnn [T][B][K], w / dw [12][K]
int head_bwd(const float* dbon, const float* dcor, const float* rnn, const float* w, float* drnn, float* dw, float* db, int T,
             int B, int K, cudaStream_t st);
int relu_bwd_inplace(float* dx, const float* y, size_t n, cudaStream_t st);           // dx *= (y > 0)
int col_sum(const float* x, size_t rows, int cols, float* out, cudaStream_t st);

int lstm_gather(const float* hout, const float* xp, float* hprev, float* xpd, int T, int B, cudaStream_t st);
int lstm_cell_scan(float* gates, float* cell, int T, int B, cudaStream_t st);
// whh_t_*: W_hh transposed, [512][2048] (the same copies the gate GEMM uses)
// barrier (1 uint) / error_flag (1 int): device scratch of the single cooperative launch (grid barrier between the steps;
// a barrier time-out sets *error_flag); nullptr or HN_LSTM_BWD_PERSISTENT=0: one launch per time step
int lstm_bwd_steps(const float* dout, const float* gates, const float* cell, const float* whh_t_f, const float* whh_t_b,
                   float* dgates, float* dc, int T, int B, unsigned int* barrier, int* error_flag, cudaStream_t st);
int stem_input_nhwc(const float* x, int in_channels, float* out, int B, cudaStream_t st);

}  // namespace hn
