// Height-reduction tail and linear head.
//
// ghc_to_sequence: reference model.py:152-155 (circular pad by 1, bilinear W-upsample to 256+2f
//   columns, crop f) + model.py:175-178 (reshape (C,H)->C*H, concat 4 scales) + model.py:263
//   (permute to [T=256, B, c_last], c_last = 1024 resnet50 / 256 resnet18) in one pass.  Because (W+2)*f == 256+2f the interpolate scale is
//   exactly 1/f, so out[col] = (1-l)*x[i0] + l*x[i0+1] with s = (col+0.5)/f + 0.5 in halo
//   coordinates, i0 = floor(s), l = s - i0 (all exactly representable in fp32; f=1 is the identity).
// head_kernel<K>: model.py:266-269, Linear(K -> 12) + the [T,B,3,4] -> [B,3,T*4] scatter;
//   channel 0 = cor, 1..2 = bon (model.py:278-279).  K = 1024: the bi-LSTM head; K = 512: the last layer of the
//   per-column MLP head of use_rnn=False (model.py:238-243, :270-275), whose rows are the same t*B + b.
#include "hn_common.cuh"
#include "conv_tc.cuh"

namespace hn {

namespace {

struct GhcSrc {
    const float* p[4];
    int H[4], W[4], C[4], chan_off[4];
    int lg;                   // log2 of the sequence width (1024 or 256)
};

template <bool SPLIT>
__global__ void __launch_bounds__(256) ghc_to_sequence_kernel(const GhcSrc s, float* __restrict__ seq, int B) {
    // seq[t][b][ch], ch = chan_off[s] + c*H + h ; one thread per (t, b, ch), ch fastest
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
    const float pos = ((float)t + 0.5f) / (float)f + 0.5f;      // halo (padded) coordinate
    const int i0 = (int)floorf(pos);
    const float l1 = pos - (float)i0;
    const float l0 = 1.f - l1;
    const size_t o0 = (((size_t)b * H + h) * (W + 2) + i0) * C + c;
    const size_t o1 = (((size_t)b * H + h) * (W + 2) + min(i0 + 1, W + 1)) * C + c;
    if (!SPLIT) {
        seq[i] = l0 * __ldg(s.p[sc] + o0) + l1 * __ldg(s.p[sc] + o1);
    } else {
        // inputs and output are hi/lo plane pairs (conv_tc.cuh)
        const unsigned short* pb = reinterpret_cast<const unsigned short*>(s.p[sc]);
        const size_t plane = (size_t)B * H * (W + 2) * C;
        const float v0 = merge_scaled(pb[o0], pb[plane + o0]);
        const float v1 = merge_scaled(pb[o1], pb[plane + o1]);
        const float v = l0 * v0 + l1 * v1;
        unsigned short* ob = reinterpret_cast<unsigned short*>(seq);
        split_scaled(v, ob[i], ob[total + i]);
    }
}

template <int K>
__global__ void __launch_bounds__(256) head_kernel(const float* __restrict__ rnn,   // [T][B][K]
                                                   const float* __restrict__ w,     // [12][K]
                                                   const float* __restrict__ bias,  // [12]
                                                   float* __restrict__ bon,         // [B][2][1024]
                                                   float* __restrict__ cor,         // [B][1][1024]
                                                   int T, int B) {
    static_assert(K % 128 == 0, "one float4 per lane per 128 inputs");
    __shared__ __align__(16) float ws[12 * K];
    for (int i = threadIdx.x; i < 12 * K / 4; i += 256)
        reinterpret_cast<float4*>(ws)[i] = __ldg(reinterpret_cast<const float4*>(w) + i);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + warp;           // row = t*B + b
    if (row >= T * B) return;
    const int t = row / B, b = row - t * B;
    const float4* x = reinterpret_cast<const float4*>(rnn + (size_t)row * K);
    float acc[12];
#pragma unroll
    for (int o = 0; o < 12; ++o) acc[o] = 0.f;
#pragma unroll
    for (int q = 0; q < K / 128; ++q) {
        const float4 xv = x[q * 32 + lane];
#pragma unroll
        for (int o = 0; o < 12; ++o) {
            const float4 wv = reinterpret_cast<const float4*>(ws + o * K)[q * 32 + lane];
            acc[o] = fmaf(xv.x, wv.x, acc[o]);
            acc[o] = fmaf(xv.y, wv.y, acc[o]);
            acc[o] = fmaf(xv.z, wv.z, acc[o]);
            acc[o] = fmaf(xv.w, wv.w, acc[o]);
        }
    }
#pragma unroll
    for (int o = 0; o < 12; ++o)
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], off);
    if (lane == 0) {
#pragma unroll
        for (int o = 0; o < 12; ++o) {
            const int s = o >> 2, k = o & 3;                // output column = t*4 + k (model.py:267-269)
            const float v = acc[o] + __ldg(bias + o);
            if (s == 0) cor[(size_t)b * 1024 + t * 4 + k] = v;
            else bon[((size_t)b * 2 + (s - 1)) * 1024 + t * 4 + k] = v;
        }
    }
}

}  // namespace

int ghc_to_sequence(const Act ghc[4], float* seq, cudaStream_t st, bool split) {
    GhcSrc s;
    int off = 0;
    for (int i = 0; i < 4; ++i) {
        HN_CHECK(ghc[i].halo == 1 && 256 % ghc[i].W == 0 && ghc[i].B == ghc[0].B, "ghc_to_sequence: bad input");
        s.p[i] = ghc[i].p; s.H[i] = ghc[i].H; s.W[i] = ghc[i].W; s.C[i] = ghc[i].C; s.chan_off[i] = off;
        off += ghc[i].C * ghc[i].H;
    }
    HN_CHECK((off == 1024 || off == 256),
             "ghc_to_sequence: the 4 scales must flatten to 1024 (resnet50) or 256 (resnet18) channels (model.py:218)");
    s.lg = off == 1024 ? 10 : 8;
    const size_t total = (size_t)256 * ghc[0].B * off;
    if (split)
        ghc_to_sequence_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(s, seq, ghc[0].B);
    else
        ghc_to_sequence_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(s, seq, ghc[0].B);
    HN_LAUNCH_OK();
    return 0;
}

int linear_head(const float* rnn, const float* w, const float* bias, float* bon, float* cor, int T, int B, int K,
                cudaStream_t st) {
    if (K == 1024) head_kernel<1024><<<(T * B + 7) / 8, 256, 0, st>>>(rnn, w, bias, bon, cor, T, B);
    else if (K == 512) head_kernel<512><<<(T * B + 7) / 8, 256, 0, st>>>(rnn, w, bias, bon, cor, T, B);
    else return fail("linear_head: K must be 1024 or 512");
    HN_LAUNCH_OK();
    return 0;
}

}  // namespace hn
