// fp32 CUDA-core convolution kernels over halo-NHWC activations.
//
// conv_igemm_f32: implicit GEMM  D[M = B*Ho*Wo][N = Cout] = A[M][K = kh*kw*Cin] * Wp[K][N]
//   for every conv of the path except the stem (reference model.py:78-81 Bottleneck convs,
//   model.py:129 ConvCompressH convs, and the LSTM input projections treated as 1x1 convs).
//   Epilogue fuses eval-mode BN / conv bias (scale, shift), the residual add and ReLU, and writes the
//   circular halo columns of the output.  This is the exact-fp32 path: it is the on-device
//   reference the split-fp16 tensor-core kernels (conv_tc.cu) are validated against, and the fallback
//   geometry for shapes the tensor-core kernel does not cover.
// stem_f32: 7x7 stride-2 conv on the NCHW fp32 input with the input normalisation
//   (model.py:248-252), BN and ReLU fused (model.py:73-75).
// maxpool3x3s2: model.py:76 (padding is -inf on both axes -- NOT circular, see SURVEY 2b).
#include "hn_common.cuh"
#include "conv_tc.cuh"

namespace hn {

namespace {

struct ConvArgs {
    const float* in;
    float* out;
    const float* res;
    const float* w;
    const float* scale;
    const float* shift;
    int B, H, Wp, Cin;          // input geometry (Wp = padded pitch)
    int Ho, Wo, Wop, Cout, out_halo;
    int kh, kw, sh, sw, ph, woff;
    int relu, M, K;
};

constexpr int BK = 16;

template <int BM, int BN>
__global__ void __launch_bounds__(256) conv_igemm_f32(const ConvArgs a) {
    constexpr int RC = BM / 64;     // row chunks of 4 per thread (stride 64)
    constexpr int CC = BN / 64;     // col chunks of 4 per thread (stride 64)
    constexpr int APAD = 4;
    __shared__ __align__(16) float As[2][BK][BM + APAD];
    __shared__ __align__(16) float Bs[2][BK][BN];

    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;

    // ---- A loader state: RC rows per thread, one float4 (4 consecutive channels) each
    const int a_kq = tid & 3;
    size_t a_base[RC];
    int a_h[RC];
#pragma unroll
    for (int l = 0; l < RC; ++l) {
        int m = m0 + (tid >> 2) + 64 * l;
        if (m < a.M) {
            int wo = m % a.Wo;
            int t = m / a.Wo;
            int ho = t % a.Ho;
            int b = t / a.Ho;
            a_base[l] = ((size_t)b * a.H * a.Wp + (size_t)(wo * a.sw + a.woff)) * a.Cin + a_kq * 4;
            a_h[l] = ho * a.sh - a.ph;
        } else {
            a_base[l] = 0;
            a_h[l] = -(1 << 28);
        }
    }
    // ---- B loader state
    constexpr int BQ = BN / 4;
    float4 ra[RC], rb[CC];

    auto load_tiles = [&](int kt) {
        const int k0 = kt * BK;
        const int tap = k0 / a.Cin;
        const int c0 = k0 - tap * a.Cin;
        const int dy = tap / a.kw;
        const int dx = tap - dy * a.kw;
#pragma unroll
        for (int l = 0; l < RC; ++l) {
            int hin = a_h[l] + dy;
            if (hin >= 0 && hin < a.H) {
                const float* p = a.in + a_base[l] + ((size_t)hin * a.Wp + dx) * a.Cin + c0;
                ra[l] = __ldg(reinterpret_cast<const float4*>(p));
            } else {
                ra[l] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
#pragma unroll
        for (int l = 0; l < CC; ++l) {
            int idx = tid + 256 * l;
            int kr = idx / BQ, cq = idx - kr * BQ;
            int n = n0 + cq * 4;
            if (n < a.Cout)
                rb[l] = __ldg(reinterpret_cast<const float4*>(a.w + (size_t)(k0 + kr) * a.Cout + n));
            else
                rb[l] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto store_tiles = [&](int buf) {
#pragma unroll
        for (int l = 0; l < RC; ++l) {
            int r = (tid >> 2) + 64 * l;
            As[buf][a_kq * 4 + 0][r] = ra[l].x;
            As[buf][a_kq * 4 + 1][r] = ra[l].y;
            As[buf][a_kq * 4 + 2][r] = ra[l].z;
            As[buf][a_kq * 4 + 3][r] = ra[l].w;
        }
#pragma unroll
        for (int l = 0; l < CC; ++l) {
            int idx = tid + 256 * l;
            int kr = idx / BQ, cq = idx - kr * BQ;
            *reinterpret_cast<float4*>(&Bs[buf][kr][cq * 4]) = rb[l];
        }
    };

    float acc[RC * 4][CC * 4];
#pragma unroll
    for (int i = 0; i < RC * 4; ++i)
#pragma unroll
        for (int j = 0; j < CC * 4; ++j) acc[i][j] = 0.f;

    const int KT = a.K / BK;
    load_tiles(0);
    store_tiles(0);
    __syncthreads();
    for (int kt = 0; kt < KT; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < KT) load_tiles(kt + 1);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float av[RC * 4], bv[CC * 4];
#pragma unroll
            for (int rc = 0; rc < RC; ++rc) {
                float4 v = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4 + 64 * rc]);
                av[rc * 4 + 0] = v.x; av[rc * 4 + 1] = v.y; av[rc * 4 + 2] = v.z; av[rc * 4 + 3] = v.w;
            }
#pragma unroll
            for (int cc = 0; cc < CC; ++cc) {
                float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4 + 64 * cc]);
                bv[cc * 4 + 0] = v.x; bv[cc * 4 + 1] = v.y; bv[cc * 4 + 2] = v.z; bv[cc * 4 + 3] = v.w;
            }
#pragma unroll
            for (int i = 0; i < RC * 4; ++i)
#pragma unroll
                for (int j = 0; j < CC * 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (kt + 1 < KT) store_tiles(buf ^ 1);
        __syncthreads();
    }

    // ---- epilogue: scale/shift (+residual) (+ReLU), interior store + circular halo columns
#pragma unroll
    for (int cc = 0; cc < CC; ++cc) {
        const int n = n0 + tx * 4 + 64 * cc;
        if (n >= a.Cout) continue;
        const float4 sc = __ldg(reinterpret_cast<const float4*>(a.scale + n));
        const float4 sf = __ldg(reinterpret_cast<const float4*>(a.shift + n));
#pragma unroll
        for (int i = 0; i < RC * 4; ++i) {
            const int m = m0 + ty * 4 + (i & 3) + 64 * (i >> 2);
            if (m >= a.M) continue;
            const int wo = m % a.Wo;
            const int t = m / a.Wo;     // = b*Ho + ho
            const size_t row = (size_t)t * a.Wop;
            const size_t o = (row + wo + a.out_halo) * a.Cout + n;
            float4 v;
            v.x = fmaf(acc[i][cc * 4 + 0], sc.x, sf.x);
            v.y = fmaf(acc[i][cc * 4 + 1], sc.y, sf.y);
            v.z = fmaf(acc[i][cc * 4 + 2], sc.z, sf.z);
            v.w = fmaf(acc[i][cc * 4 + 3], sc.w, sf.w);
            if (a.res) {
                const float4 r = __ldg(reinterpret_cast<const float4*>(a.res + o));
                v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
            }
            if (a.relu) {
                v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
            }
            *reinterpret_cast<float4*>(a.out + o) = v;
            if (a.out_halo) {
                if (wo == 0)
                    *reinterpret_cast<float4*>(a.out + (row + a.Wo + 1) * a.Cout + n) = v;
                if (wo == a.Wo - 1)
                    *reinterpret_cast<float4*>(a.out + row * a.Cout + n) = v;
            }
        }
    }
}

// Checks one convolution against what conv_igemm_f32 takes and fills its geometry (no pointers, no GPU work).
int conv_f32_args(const ConvDesc& d, const Act& in, const Act& out, ConvArgs* a) {
    HN_CHECK(in.C == d.Cin && out.C == d.Cout, "conv_f32: channel mismatch");
    HN_CHECK(d.Cin % BK == 0 && d.Cout % 4 == 0, "conv_f32: Cin must be a multiple of 16, Cout of 4");
    HN_CHECK(d.pw <= in.halo, "conv_f32: circular pad wider than the input halo");
    HN_CHECK(out.halo == 0 || out.halo == 1, "conv_f32: output halo must be 0 or 1");
    const int Ho = (in.H + 2 * d.ph - d.kh) / d.sh + 1;
    const int Wo = (in.W + 2 * d.pw - d.kw) / d.sw + 1;
    HN_CHECK(Ho == out.H && Wo == out.W && in.B == out.B, "conv_f32: output geometry mismatch");
    a->B = in.B; a->H = in.H; a->Wp = in.Wp(); a->Cin = d.Cin;
    a->Ho = Ho; a->Wo = Wo; a->Wop = out.Wp(); a->Cout = d.Cout; a->out_halo = out.halo;
    a->kh = d.kh; a->kw = d.kw; a->sh = d.sh; a->sw = d.sw; a->ph = d.ph; a->woff = in.halo - d.pw;
    a->relu = d.relu;
    const long long M = (long long)in.B * Ho * Wo;
    HN_CHECK(M < (1ll << 31), "conv_f32: M overflows int");
    a->M = (int)M; a->K = d.kh * d.kw * d.Cin;
    return 0;
}

// Tile choice: big tiles when they still fill the SMs, else 64x64.  plan = BM, BN, grid_m, grid_n.
void conv_f32_tiles(long long M, int Cout, int sms, int plan[4]) {
    const long long big = ((M + 127) / 128) * ((Cout + 127) / 128);
    int bm = 64, bn = 64;
    if (Cout >= 128 && big >= sms) bm = bn = 128;
    else if (Cout <= 64 && (M + 127) / 128 >= sms) bm = 128;
    plan[0] = bm; plan[1] = bn; plan[2] = (int)((M + bm - 1) / bm); plan[3] = (Cout + bn - 1) / bn;
}

}  // namespace

int conv_f32_plan(const ConvDesc& d, const Act& in, const Act& out, int sms, int plan[4]) {
    HN_CHECK(sms >= 1, "conv_f32_plan: sms must be positive");
    ConvArgs a;
    if (conv_f32_args(d, in, out, &a)) return -1;
    conv_f32_tiles(a.M, d.Cout, sms, plan);
    return 0;
}

int conv_f32(const ConvDesc& d, const Act& in, const Act& out, const float* residual, cudaStream_t st) {
    ConvArgs a;
    if (conv_f32_args(d, in, out, &a)) return -1;
    a.in = in.p; a.out = out.p; a.res = residual; a.w = d.w; a.scale = d.scale; a.shift = d.shift;
    if (a.M == 0) return 0;
    int p[4];
    conv_f32_tiles(a.M, d.Cout, num_sms(), p);
    const dim3 g((unsigned)p[2], (unsigned)p[3]);
    if (p[0] == 128 && p[1] == 128) conv_igemm_f32<128, 128><<<g, 256, 0, st>>>(a);
    else if (p[0] == 128) conv_igemm_f32<128, 64><<<g, 256, 0, st>>>(a);
    else conv_igemm_f32<64, 64><<<g, 256, 0, st>>>(a);
    HN_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Stem: x[B][Cx][512][1024] NCHW fp32 -> normalise -> 7x7 s2 conv (circular W pad 3, zero H pad 3)
//       -> BN -> ReLU -> halo-NHWC [B][256][512+2][64].
// One CTA = 4 output rows x 64 output cols (256 threads, one output pixel each, all 64 channels).
namespace {

constexpr int ST_TW = 64, ST_TH = 4;
constexpr int ST_PW = ST_TW * 2 + 5;   // 133 input cols
constexpr int ST_PH = ST_TH * 2 + 5;   // 13 input rows
constexpr int ST_PP = 136;             // patch row pitch: multiple of 4 floats so rows can be read as float4

// thread = 4 consecutive output pixels x 16 output channels.  Per (dy, c) the 13 input values the 4 pixels
// need for all 7 dx taps are read once (4 x LDS.128) and the 7 x 4 weight vectors once each, i.e. 32 shared
// loads per 448 FMAs: the kernel runs at the fp32 FMA rate instead of the shared-memory rate.
__global__ void __launch_bounds__(256) stem_kernel(const float* __restrict__ x, int Cx,
                                                   const float* __restrict__ w,      // [147][64], k=(dy*7+dx)*3+c
                                                   const float* __restrict__ scale,
                                                   const float* __restrict__ shift,
                                                   float* __restrict__ out, int Hin, int Win, float flo) {
    extern __shared__ __align__(16) float smem[];
    float* ws = smem;                              // 147*64
    float* patch = smem + 147 * 64;                // [3][ST_PH][ST_PP]
    const int Ho = Hin / 2, Wo = Win / 2;
    const int b = blockIdx.z;
    const int ho0 = blockIdx.y * ST_TH, wo0 = blockIdx.x * ST_TW;
    const int tid = threadIdx.x;
    for (int i = tid; i < 147 * 64 / 4; i += 256)
        reinterpret_cast<float4*>(ws)[i] = __ldg(reinterpret_cast<const float4*>(w) + i);
    const float mean[3] = {0.485f, 0.456f, 0.406f};       // reference model.py:186
    const float stdv[3] = {0.229f, 0.224f, 0.225f};       // reference model.py:187
    const int hi0 = ho0 * 2 - 3, wi0 = wo0 * 2 - 3;
    for (int i = tid; i < 3 * ST_PH * ST_PP; i += 256) {
        int c = i / (ST_PH * ST_PP);
        int r = i - c * (ST_PH * ST_PP);
        int py = r / ST_PP, px = r - py * ST_PP;
        int hi = hi0 + py;
        int wi = wi0 + px;
        wi = wi < 0 ? wi + Win : (wi >= Win ? wi - Win : wi);       // circular W (model.py:27-29)
        float v = 0.f;                                               // zero H pad of the *normalised* input
        if (px < ST_PW && hi >= 0 && hi < Hin)
            v = (__ldg(x + (((size_t)b * Cx + c) * Hin + hi) * Win + wi) - mean[c]) / stdv[c];
        patch[i] = v;
    }
    __syncthreads();
    const int cg = tid & 3;                        // channel group: channels cg*16 .. +15
    const int pg = tid >> 2;                       // pixel group: 4 consecutive pixels of one row
    const int ly = pg >> 4, lx0 = (pg & 15) * 4;
    float acc[4][16];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int n = 0; n < 16; ++n) acc[p][n] = 0.f;
    for (int dy = 0; dy < 7; ++dy) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float in[16];                          // input columns 2*lx0 .. 2*lx0+15 (13 are used)
            const float4* ip = reinterpret_cast<const float4*>(patch + (c * ST_PH + ly * 2 + dy) * ST_PP + lx0 * 2);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 v = ip[q];
                in[q * 4 + 0] = v.x; in[q * 4 + 1] = v.y; in[q * 4 + 2] = v.z; in[q * 4 + 3] = v.w;
            }
#pragma unroll
            for (int dx = 0; dx < 7; ++dx) {
                const float4* wr = reinterpret_cast<const float4*>(ws + ((dy * 7 + dx) * 3 + c) * 64 + cg * 16);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 wv = wr[q];
#pragma unroll
                    for (int p = 0; p < 4; ++p) {
                        const float v = in[2 * p + dx];
                        acc[p][q * 4 + 0] = fmaf(v, wv.x, acc[p][q * 4 + 0]);
                        acc[p][q * 4 + 1] = fmaf(v, wv.y, acc[p][q * 4 + 1]);
                        acc[p][q * 4 + 2] = fmaf(v, wv.z, acc[p][q * 4 + 2]);
                        acc[p][q * 4 + 3] = fmaf(v, wv.w, acc[p][q * 4 + 3]);
                    }
                }
            }
        }
    }
    const int ho = ho0 + ly;
    if (ho >= Ho) return;
    const int Wop = Wo + 2;
    float4 sc[4], sf[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        sc[q] = __ldg(reinterpret_cast<const float4*>(scale + cg * 16) + q);
        sf[q] = __ldg(reinterpret_cast<const float4*>(shift + cg * 16) + q);
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        const int wo = wo0 + lx0 + p;
        if (wo >= Wo) continue;
        const size_t row = ((size_t)b * Ho + ho) * Wop;
        float* o = out + (row + wo + 1) * 64 + cg * 16;
        float* oh = (wo == 0) ? out + (row + Wo + 1) * 64 + cg * 16 : ((wo == Wo - 1) ? out + row * 64 + cg * 16 : nullptr);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float4 v;
            v.x = fmaxf(fmaf(acc[p][q * 4 + 0], sc[q].x, sf[q].x), flo);
            v.y = fmaxf(fmaf(acc[p][q * 4 + 1], sc[q].y, sf[q].y), flo);
            v.z = fmaxf(fmaf(acc[p][q * 4 + 2], sc[q].z, sf[q].z), flo);
            v.w = fmaxf(fmaf(acc[p][q * 4 + 3], sc[q].w, sf[q].w), flo);
            reinterpret_cast<float4*>(o)[q] = v;
            if (oh) reinterpret_cast<float4*>(oh)[q] = v;
        }
    }
}

__device__ __forceinline__ uint2 split4(const float4 m, bool lo) {
    const float f[4] = {m.x, m.y, m.z, m.w};
    unsigned short u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        unsigned short h, l;
        split_scaled(f[j], h, l);
        u[j] = lo ? l : h;
    }
    return make_uint2((unsigned)u[0] | ((unsigned)u[1] << 16), (unsigned)u[2] | ((unsigned)u[3] << 16));
}

template <bool SPLIT>
__global__ void __launch_bounds__(256) maxpool_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                      int B, int H, int W, int C, int Ho, int Wo) {
    // one thread = one output pixel x 4 channels; input/output halo = 1
    const int C4 = C / 4;
    const size_t total = (size_t)B * Ho * Wo * C4;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c4 = (int)(i % C4);
    size_t t = i / C4;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    const int Wp = W + 2, Wop = Wo + 2;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
        const int hi = ho * 2 + dy - 1;
        if (hi < 0 || hi >= H) continue;
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
            const int wi = wo * 2 + dx - 1;
            if (wi < 0 || wi >= W) continue;               // -inf padding, not circular (model.py:76)
            const float4 v = __ldg(reinterpret_cast<const float4*>(
                in + (((size_t)b * H + hi) * Wp + wi + 1) * C) + c4);
            m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
        }
    }
    const size_t row = ((size_t)b * Ho + ho) * Wop;
    if (!SPLIT) {
        reinterpret_cast<float4*>(out + (row + wo + 1) * C)[c4] = m;
        if (wo == 0) reinterpret_cast<float4*>(out + (row + Wo + 1) * C)[c4] = m;
        if (wo == Wo - 1) reinterpret_cast<float4*>(out + row * C)[c4] = m;
    } else {
        // hi/lo planes for the tensor-core convs (plane = B*Ho*Wop*C elements)
        unsigned short* ob = reinterpret_cast<unsigned short*>(out);
        const size_t plane = (size_t)B * Ho * Wop * C;
        const uint2 hi = split4(m, false), lo = split4(m, true);
        auto put = [&](size_t pix) {
            reinterpret_cast<uint2*>(ob + pix * C)[c4] = hi;
            reinterpret_cast<uint2*>(ob + plane + pix * C)[c4] = lo;
        };
        put(row + wo + 1);
        if (wo == 0) put(row + Wo + 1);
        if (wo == Wo - 1) put(row);
    }
}

}  // namespace

int stem_f32(const float* x_nchw, int B, int in_channels, const float* w_packed, const float* scale,
             const float* shift, const Act& out, cudaStream_t st, bool relu) {
    HN_CHECK(in_channels >= 3, "stem: input needs >= 3 channels (reference model.py:252 uses x[:, :3])");
    HN_CHECK(out.B == B && out.H == 256 && out.W == 512 && out.C == 64 && out.halo == 1, "stem: bad output tensor");
    const size_t smem = (147 * 64 + 3 * ST_PH * ST_PP) * sizeof(float);
    HN_CUDA_OK(cudaFuncSetAttribute(stem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 g(512 / ST_TW, 256 / ST_TH, B);
    // relu = false (train-mode statistics pass): floor at -inf, i.e. the raw conv * scale + shift
    stem_kernel<<<g, 256, smem, st>>>(x_nchw, in_channels, w_packed, scale, shift, out.p, 512, 1024, relu ? 0.f : -INFINITY);
    HN_LAUNCH_OK();
    return 0;
}

int maxpool3x3s2(const Act& in, const Act& out, cudaStream_t st, bool out_split) {
    HN_CHECK(in.halo == 1 && out.halo == 1 && in.C == out.C && in.C % 4 == 0, "maxpool: bad tensors");
    HN_CHECK(out.H == (in.H + 2 - 3) / 2 + 1 && out.W == (in.W + 2 - 3) / 2 + 1 && in.B == out.B, "maxpool: geometry");
    const size_t total = (size_t)out.B * out.H * out.W * (out.C / 4);
    if (out_split)
        maxpool_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in.p, out.p, in.B, in.H, in.W, in.C, out.H, out.W);
    else
        maxpool_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in.p, out.p, in.B, in.H, in.W, in.C, out.H, out.W);
    HN_LAUNCH_OK();
    return 0;
}

}  // namespace hn
