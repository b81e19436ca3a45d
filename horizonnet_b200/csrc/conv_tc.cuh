// Split-precision tensor-core (wgmma) convolution entry points (conv_tc.cu) and the plane format helpers.
//
// Plane format ("split planes"): an fp32 tensor v is carried as two fp16 planes of the SCALED value
// s = v * 2^-4:        hi = fp16(s)       (11 significant bits, saturated at +-65504)
//                      lo = fp16(s - hi)  (the next 11 bits)
// hi plane first, lo plane at +numel 16-bit elements; 4 bytes per element in total, like fp32.
// The power-of-two scale is exact; it puts the fp16 range at |v| < 1.05e6 (random-init activations of
// this net peak at 6.3e3, trained ones far lower) and keeps lo normal for |v| > 2; below that lo is
// an fp16 subnormal, i.e. an absolute resolution of 2^-24 * 16 = 9.5e-7 (measured end-to-end effect
// of the whole scheme: 2e-6..1e-5 max-abs, DESIGN.md).  The fp16 x fp16 MMAs take both operands in one format, and a bf16+bf16 split misses the
// 1e-4 contract, hence fp16+fp16.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "hn_common.cuh"

namespace hn {

constexpr float ACT_SCALE = 0.0625f;        // 2^-4
constexpr float ACT_UNSCALE = 16.f;

__device__ __forceinline__ void split_scaled(float v, unsigned short& hi, unsigned short& lo) {
    const float s = fminf(fmaxf(v * ACT_SCALE, -65504.f), 65504.f);
    const __half h = __float2half_rn(s);
    hi = __half_as_ushort(h);
    lo = __half_as_ushort(__float2half_rn(s - __half2float(h)));
}
__device__ __forceinline__ float merge_scaled(unsigned short hi, unsigned short lo) {
    return (__half2float(__ushort_as_half(hi)) + __half2float(__ushort_as_half(lo))) * ACT_UNSCALE;
}

// ---- scaled-domain fast path (conv_tc epilogue): values are already multiplied by ACT_SCALE
__device__ __forceinline__ uint32_t pack_half2_sat(float e0, float e1) {      // e0 -> low half, e1 -> high half
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(e1), "f"(e0));
    return r;
}
__device__ __forceinline__ float2 unpack_half2(uint32_t v) {
    return __half22float2(*reinterpret_cast<const __half2*>(&v));
}
__device__ __forceinline__ void split2_scaled(float s0, float s1, uint32_t& hi2, uint32_t& lo2) {
    hi2 = pack_half2_sat(s0, s1);
    const float2 b = unpack_half2(hi2);
    lo2 = pack_half2_sat(s0 - b.x, s1 - b.y);
}

// Gradient tensors are split after a multiplication by this power of two (largest magnitude -> [2^11, 2^12)), see
// split_planes_pow2 in bwd_kernels.cuh; consumers divide it out again (exact).
__device__ __forceinline__ float pow2_factor(float absmax) {
    if (!(absmax > 0.f) || isinf(absmax)) return 1.f;
    int e;
    frexpf(absmax, &e);                      // absmax = m * 2^e, m in [0.5, 1)
    e = 12 - e;
    e = e < -100 ? -100 : (e > 100 ? 100 : e);
    return ldexpf(1.f, e);
}

bool conv_tc_supported(const ConvDesc& d, const Act& in, const Act& out);
// Launch plan of conv_tc_planes for one shape (host only): which kernel, tile shape, operand boxes and grid.
struct TcPlan {
    int gemm_kernel;          // 1: gemm_tc_kernel (asynchronous epilogue), 0: conv_tc_kernel
    int BN;                   // output channels per tile (128, 64 or 32)
    int mode;                 // 0: GEMM rows over all halo-NHWC pixels, 1: conv rows
    int M;                    // mode 0: pixel rows, mode 1: B * Ho output rows
    int tw, rows_per_tile, wsegs;          // mode 1: tile columns, output rows per tile, tiles per output row
    int box_rows, box_imgs;                // mode 1: the one TMA box of a tile's rows: rows of one image x images
    int dxr, parity;                       // 3x3 dx reuse of one 130-pixel input row; stride 2 along W (parity view)
    int num_kc, seg;                       // K chunks of 64; chunks per tensor-core accumulation segment (SEG)
    int pf;                                // gemm_tc_kernel: L2 prefetch distance in tile rounds, 0 = off
    int n_tiles, num_tiles, grid;          // tiles along Cout, all tiles, CTAs (persistent, min(num_tiles, sms))
};
// A function of the shapes and sms alone; -1 (with hn_last_error set) for a shape conv_tc_supported rejects or a residual
// with fp32 output.  conv_tc_planes launches exactly this plan.
int conv_tc_plan(const ConvDesc& d, const Act& in, const Act& out, bool out_f32, bool has_residual, int sms, TcPlan* p);
// fp32 halo-NHWC in/out convenience wrapper (unit tests): splits, runs the plane kernel, merges the output planes, or with
// out_f32 lets the kernel write fp32 directly (the epilogue of the LSTM projections and of the data gradient; no residual).
int conv_tc(const ConvDesc& d, const Act& in, const Act& out, const float* residual, bool out_f32, cudaStream_t st);
// The real thing: operands and result are split planes.  wq: [2][Cout][K] weight planes
// (fp16 hi, fp16 lo of w * 2^t); tc_aux = 3*Cout floats written by pack_weight_tc:
//   [0,C)  accumulator -> true units   (BN scale * 2^(4-t)),  used with d.shift for fp32 outputs
//   [C,2C) accumulator -> plane units  (the above * 2^-4),    [2C,3C) shift in plane units
int conv_tc_planes(const ConvDesc& d, const unsigned short* wq, const float* tc_aux, const Act& in,
                   const unsigned short* in_planes, const Act& out, unsigned short* out_planes, float* out_f32,
                   const unsigned short* res_planes, cudaStream_t st);
// Eval-mode conv3 of a bottleneck's block 0 with its downsample folded in: out = relu([t2 | x↓] . wq + shift), one GEMM
// with K = t2.C + x.C and no residual.  x↓ = x at every stride-th pixel (the 1x1 downsample), t2 has the output geometry.
// wq: [2][Cout][K] planes of [s3 W3 ; sd Wd] (both BN scales folded into the weights), tc_aux from pack_weight_tc with
// scale 1 and shift f3 + fd.  Plan: conv rows (mode 1) of conv_tc_kernel, the first t2.C / 64 K chunks from t2.
int conv_tc_fold_plan(const Act& t2, const Act& x, int stride, const Act& out, int sms, TcPlan* p);
int conv_tc_fold_planes(const unsigned short* wq, const float* tc_aux, const Act& t2, const unsigned short* t2_planes,
                        const Act& x, const unsigned short* x_planes, int stride, const Act& out, unsigned short* out_planes,
                        cudaStream_t st);
// fp32 halo-NHWC convenience wrapper (unit tests): w = the folded fp32 weights [Cout][K], shift [Cout]
int conv_tc_fold(const float* w, const float* shift, const Act& t2, const Act& x, int stride, const Act& out,
                 cudaStream_t st);
// conv2 (3x3 s1, 64 -> 64) + BN + ReLU fused with conv3 (1x1, 64 -> C3) + BN + identity + ReLU of a layer1 bottleneck
// (conv_tc.cu: bott_tc_kernel).  With the downsample folded in (res_planes null, x_planes the block input in `in`'s
// geometry, wq3 / aux3 the folded pack of conv_tc_fold_planes) conv3 has no residual.
bool bott_tc_supported(const ConvDesc& d2, const ConvDesc& d3, const Act& in, const Act& out);
int bott_tc_planes(const ConvDesc& d2, const unsigned short* wq2, const float* aux2, const ConvDesc& d3,
                   const unsigned short* wq3, const float* aux3, const Act& in, const unsigned short* in_planes, const Act& out,
                   unsigned short* out_planes, const unsigned short* res_planes, const unsigned short* x_planes,
                   cudaStream_t st);
// fp32 convenience wrapper of bott_tc_planes (unit tests): w2 OIHW [64][64][3][3] with BN scale2 / shift2; in / out fp32
// halo-NHWC.  Exactly one of res (the block's identity, out's geometry; w3 the conv3 weights [C3][64] with scale3 /
// shift3) and x (the block input, in's geometry; w3 the folded weights [C3][128] with shift3, scale3 null).
int bott_tc_f32(const float* w2, const float* scale2, const float* shift2, const float* w3, const float* scale3,
                const float* shift3, const Act& in, const float* res, const float* x, const Act& out, cudaStream_t st);
// 7x7 stride-2 stem on wgmma (conv_tc.cu: stem_tc_kernel): NCHW fp32 input -> fp32 halo-NHWC [B][256][514][64]
// (interior columns only).  wq [2][64][224] / tc_aux [3*64+1] come from stem_tc_pack_weights (pad_scratch: 64*224 floats);
// scratch: stem_tc_scratch_bytes(B) bytes of packed input planes.
size_t stem_tc_scratch_bytes(int B);
int stem_tc_pack_weights(const float* w_oihw, float* pad_scratch, unsigned short* wq, const float* scale,
                         const float* shift, float* tc_aux, cudaStream_t st);
int stem_tc(const float* x_nchw, int B, int in_channels, const unsigned short* wq, const float* tc_aux,
            const float* shift, unsigned short* scratch, const Act& out, cudaStream_t st, bool relu = true);
int split_planes(const float* in, unsigned short* out, size_t n, cudaStream_t st);
int merge_planes(const unsigned short* in, float* out, size_t n, cudaStream_t st);
// OIHW fp32 weights -> wq planes + tc_aux[3*Cout] (scale/shift may be null = ones/zeros); scratch: 1 float.
int pack_weight_tc(const float* w_oihw, unsigned short* wq, const float* scale, const float* shift, float* tc_aux,
                   float* scratch, int Cout, int Cin, int kh, int kw, cudaStream_t st);
// New epilogue constants for already packed weights (train mode: batch-statistics scale/shift); absmax = the scratch
// float pack_weight_tc left behind (weight plane scale).
int tc_aux_update(const float* scale, const float* shift, const float* absmax, float* tc_aux, int Cout, cudaStream_t st);

}  // namespace hn
