// Narrow height-reduction convolution: 3x3, stride (2, 1), zero padding along H, circular along W (the input halo), for
// channel counts below what conv_tc_kernel takes (Cin < 64 or Cout < 32).  resnet18 has four of them -- ghc0.1 32 -> 32,
// ghc0.2 32 -> 16, ghc0.3 16 -> 8 and ghc1.3 32 -> 16 -- about 0.2 GFLOP per panorama in all, too little for tensor cores.
//
// It sits on the tensor-core path of the forward, so activations arrive and leave as split fp16 hi/lo planes
// (conv_tc.cuh): the kernel merges its input rows to fp32 in shared memory, accumulates in fp32 from the fp32 packed
// weights [K = (dy*3 + dx)*Cin + c][Cout], applies scale/shift (BN with the conv bias folded in) and ReLU, and re-splits
// into planes, interior and circular halo columns -- no separate split or merge pass.
//
// CTA = one output row segment of up to 128 columns x all Cout; thread = one output column.  Shared memory: the weights
// (read as broadcasts) and the three input rows [3][130][Cin + 1] (the +1 keeps the per-thread pixel reads conflict-free).
#include "model.cuh"

namespace hn {
namespace {

constexpr int NW = 128;       // output columns per CTA (= threads)

template <int CIN, int COUT>
struct NarrowSmem {
    static constexpr int W_FLOATS = 9 * CIN * COUT;
    static constexpr int ROW = NW + 2;
    static constexpr int PIX = CIN + 1;
    static constexpr int IN_FLOATS = 3 * ROW * PIX;
    static constexpr size_t BYTES = (size_t)(W_FLOATS + IN_FLOATS) * sizeof(float);
};

struct NarrowArgs {
    const unsigned short* in; size_t in_plane;     // hi plane, lo plane at + in_plane
    unsigned short* out; size_t out_plane;
    const float* w; const float* scale; const float* shift;
    int H, Wp, Ho, Wo, Wop, relu;
};

template <int CIN, int COUT>
__global__ void __launch_bounds__(NW) conv_narrow_kernel(const NarrowArgs a) {
    using S = NarrowSmem<CIN, COUT>;
    extern __shared__ __align__(16) float sm[];
    float* ws = sm;
    float* xs = sm + S::W_FLOATS;
    const int seg = blockIdx.x, ho = blockIdx.y, b = blockIdx.z;
    const int wo0 = seg * NW;
    for (int i = threadIdx.x; i < S::W_FLOATS / 4; i += NW)
        reinterpret_cast<float4*>(ws)[i] = __ldg(reinterpret_cast<const float4*>(a.w) + i);
    // input rows 2 ho - 1 .. 2 ho + 1 (zero outside the image), halo columns wo0 .. wo0 + NW + 1 of the halo-1 row
    for (int i = threadIdx.x; i < 3 * S::ROW * CIN; i += NW) {
        const int c = i % CIN, r = i / CIN;
        const int col = r % S::ROW, dy = r / S::ROW;
        const int hin = 2 * ho + dy - 1, wp = wo0 + col;
        float v = 0.f;
        if (hin >= 0 && hin < a.H && wp < a.Wp) {
            const size_t o = (((size_t)b * a.H + hin) * a.Wp + wp) * CIN + c;
            v = merge_scaled(a.in[o], a.in[a.in_plane + o]);
        }
        xs[(dy * S::ROW + col) * S::PIX + c] = v;
    }
    __syncthreads();
    const int wo = wo0 + threadIdx.x;
    if (wo >= a.Wo) return;
    float acc[COUT];
#pragma unroll
    for (int n = 0; n < COUT; ++n) acc[n] = 0.f;
    for (int tap = 0; tap < 9; ++tap) {
        const int dy = tap / 3, dx = tap - dy * 3;
        const float* x = xs + (dy * S::ROW + threadIdx.x + dx) * S::PIX;
        const float* w = ws + tap * CIN * COUT;
#pragma unroll 4
        for (int c = 0; c < CIN; ++c) {
            const float v = x[c];
            const float4* wr = reinterpret_cast<const float4*>(w + c * COUT);
#pragma unroll
            for (int q = 0; q < COUT / 4; ++q) {
                const float4 wv = wr[q];
                acc[4 * q + 0] = fmaf(v, wv.x, acc[4 * q + 0]);
                acc[4 * q + 1] = fmaf(v, wv.y, acc[4 * q + 1]);
                acc[4 * q + 2] = fmaf(v, wv.z, acc[4 * q + 2]);
                acc[4 * q + 3] = fmaf(v, wv.w, acc[4 * q + 3]);
            }
        }
    }
    // epilogue: scale/shift (+ReLU), split into planes; interior column plus its circular halo copy
    const size_t row = ((size_t)b * a.Ho + ho) * a.Wop;
    size_t dst[2] = {(row + wo + 1) * COUT, 0};
    int ndst = 1;
    if (wo == 0) dst[ndst++] = (row + a.Wo + 1) * COUT;
    else if (wo == a.Wo - 1) dst[ndst++] = row * COUT;
#pragma unroll
    for (int g = 0; g < COUT / 8; ++g) {
        __align__(16) unsigned short hi[8];
        __align__(16) unsigned short lo[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = 8 * g + j;
            float v = fmaf(acc[n], __ldg(a.scale + n), __ldg(a.shift + n));
            if (a.relu) v = fmaxf(v, 0.f);
            split_scaled(v, hi[j], lo[j]);
        }
        for (int k = 0; k < ndst; ++k) {
            *reinterpret_cast<uint4*>(a.out + dst[k] + 8 * g) = *reinterpret_cast<const uint4*>(hi);
            *reinterpret_cast<uint4*>(a.out + a.out_plane + dst[k] + 8 * g) = *reinterpret_cast<const uint4*>(lo);
        }
    }
}

template <int CIN, int COUT>
int launch_narrow(const NarrowArgs& a, int B, cudaStream_t st) {
    constexpr size_t smem = NarrowSmem<CIN, COUT>::BYTES;
    HN_CUDA_OK(cudaFuncSetAttribute(conv_narrow_kernel<CIN, COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((a.Wo + NW - 1) / NW, a.Ho, B);
    conv_narrow_kernel<CIN, COUT><<<grid, NW, smem, st>>>(a);
    HN_LAUNCH_OK();
    return 0;
}

// the channel pairs of the four resnet18 convs
bool narrow_channels(int cin, int cout) {
    return (cin == 32 && (cout == 32 || cout == 16)) || (cin == 16 && cout == 8);
}

}  // namespace

bool conv_narrow_supported(const ConvDesc& d, const Act& in, const Act& out) {
    return narrow_channels(d.Cin, d.Cout) && in.C == d.Cin && out.C == d.Cout && d.kh == 3 && d.kw == 3 && d.sh == 2 &&
           d.sw == 1 && d.ph == 1 && d.pw == 1 && in.halo == 1 && out.halo == 1 && out.B == in.B &&
           out.H == (in.H - 1) / 2 + 1 && out.W == in.W;
}

int conv_narrow_planes(const ConvDesc& d, const Act& in, const unsigned short* in_planes, const Act& out,
                       unsigned short* out_planes, cudaStream_t st) {
    HN_CHECK(conv_narrow_supported(d, in, out), "conv_narrow: unsupported shape");
    HN_CHECK(d.w && d.scale && d.shift, "conv_narrow: weights and epilogue constants must be set");
    if (in.B == 0 || out.H == 0) return 0;
    NarrowArgs a;
    a.in = in_planes; a.in_plane = in.numel();
    a.out = out_planes; a.out_plane = out.numel();
    a.w = d.w; a.scale = d.scale; a.shift = d.shift;
    a.H = in.H; a.Wp = in.Wp(); a.Ho = out.H; a.Wo = out.W; a.Wop = out.Wp(); a.relu = d.relu;
    const int key = d.Cin * 100 + d.Cout;
    switch (key) {
        case 3232: return launch_narrow<32, 32>(a, in.B, st);
        case 3216: return launch_narrow<32, 16>(a, in.B, st);
        default: return launch_narrow<16, 8>(a, in.B, st);
    }
}

}  // namespace hn
