// hn_model: weight registry (reference checkpoint layout, misc/utils.py:49-65), BN folding and
// weight packing, activation workspace, and the forward schedule of HorizonNet('resnet50' or 'resnet18', rnn)
// (reference model.py:254-281), plus the C ABI (include/horizonnet_b200.h).
#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include <atomic>

#include "model.cuh"
#include "bwd_kernels.cuh"
#include "../../include/horizonnet_b200.h"

#ifndef HN_BUILD_DIGEST
#define HN_BUILD_DIGEST "unknown"
#endif

namespace hn {

// ---- error / launch accounting -----------------------------------------------------------------
static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};
void set_error(const std::string& m) { g_err = m; }
int fail(const std::string& m) { g_err = m; return -1; }
void count_launch(int n) { g_launches += n; }

namespace {
// ---- packing kernels ---------------------------------------------------------------------------
// OIHW [Cout][Cin][kh][kw] -> [K = (dy*kw+dx)*Cin + c][Cout]
__global__ void pack_oihw_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int Cin, int kh,
                                 int kw) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)Cout * Cin * kh * kw;
    if (i >= total) return;
    const int n = (int)(i % Cout);
    const size_t k = i / Cout;
    const int c = (int)(k % Cin);
    const int tap = (int)(k / Cin);
    const int dy = tap / kw, dx = tap % kw;
    out[i] = w[(((size_t)n * Cin + c) * kh + dy) * kw + dx];
}

// eval-mode BN (+ optional conv bias) -> scale/shift:  y = conv*scale + shift
__global__ void fold_bn_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                               const float* __restrict__ mean, const float* __restrict__ var,
                               const float* __restrict__ bias, float* __restrict__ scale,
                               float* __restrict__ shift, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C) return;
    const double s = (double)gamma[i] / sqrt((double)var[i] + 1e-5);      // BatchNorm2d eps (model.py:130)
    const double b = bias ? (double)bias[i] : 0.0;
    scale[i] = (float)s;
    shift[i] = (float)((double)beta[i] + (b - (double)mean[i]) * s);
}

// block 0: [s3 W3 | sd Wd] per output channel n (1x1 OIHW weights [Cout][Cmid], [Cout][Cin]) and f3 + fd.  Both scales go
// into the weights (not their ratio: a BN scale can be near 0)
__global__ void fold_downsample_kernel(const float* __restrict__ w3, const float* __restrict__ s3, const float* __restrict__ f3,
                                       const float* __restrict__ wd, const float* __restrict__ sd,
                                       const float* __restrict__ fd, float* __restrict__ w, float* __restrict__ shift,
                                       int Cout, int Cmid, int Cin) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int K = Cmid + Cin;
    if (i >= (size_t)Cout * K) return;
    const int n = (int)(i / K), k = (int)(i - (size_t)n * K);
    w[i] = k < Cmid ? s3[n] * w3[(size_t)n * Cmid + k] : sd[n] * wd[(size_t)n * Cin + (k - Cmid)];
    if (k == 0) shift[n] = f3[n] + fd[n];
}

__global__ void lstm_bias_kernel(const float* __restrict__ bih_f, const float* __restrict__ bhh_f,
                                 const float* __restrict__ bih_b, const float* __restrict__ bhh_b,
                                 float* __restrict__ scale, float* __restrict__ shift) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 4096) return;
    scale[i] = 1.f;
    shift[i] = i < 2048 ? bih_f[i] + bhh_f[i] : bih_b[i - 2048] + bhh_b[i - 2048];
}

// halo-NHWC interior -> NCHW (test hook)
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W,
                                    int C, int halo) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)B * C * H * W;
    if (i >= total) return;
    const int w = (int)(i % W);
    size_t t = i / W;
    const int h = (int)(t % H); t /= H;
    const int c = (int)(t % C);
    const int b = (int)(t / C);
    out[i] = in[(((size_t)b * H + h) * (W + 2 * halo) + w + halo) * C + c];
}

// MLP head layer 1 epilogue: y = acc * 1 + linear.0.bias
__global__ void bias_constants_kernel(const float* __restrict__ bias, float* __restrict__ scale, float* __restrict__ shift,
                                      int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C) return;
    scale[i] = 1.f;
    shift[i] = bias[i];
}

// rows [T][B][C] -> [B][T][C] (test hook: the MLP hidden layer in the reference's [B, W, C] layout)
__global__ void rows_to_batch_major_kernel(const float* __restrict__ in, float* __restrict__ out, int T, int B, int C) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)T * B * C;
    if (i >= total) return;
    const int c = (int)(i % C);
    const int t = (int)((i / C) % T);
    const int b = (int)(i / C / T);
    out[i] = in[((size_t)t * B + b) * C + c];
}

// seq [T][B][C] -> feature [B][C][T]
__global__ void seq_to_feature_kernel(const float* __restrict__ seq, float* __restrict__ out, int T, int B, int C) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)T * B * C;
    if (i >= total) return;
    const int t = (int)(i % T);
    const int ch = (int)((i / T) % C);
    const int b = (int)(i / T / C);
    out[i] = seq[((size_t)t * B + b) * C + ch];
}

}  // namespace
}  // namespace hn

using namespace hn;


namespace {

ConvLayer make_conv(hn_model* m, const std::string& wkey, const std::string& bn, const std::string& biaskey, int cin,
                    int cout, int k, int sh, int sw, int relu) {
    ConvLayer c;
    c.d.Cin = cin; c.d.Cout = cout; c.d.kh = k; c.d.kw = k; c.d.sh = sh; c.d.sw = sw;
    c.d.ph = k / 2; c.d.pw = k / 2; c.d.relu = relu;
    c.wkey = wkey; c.bnprefix = bn; c.biaskey = biaskey;
    m->add_slot(wkey, (long long)cout * cin * k * k);
    if (!biaskey.empty()) m->add_slot(biaskey, cout);
    m->add_bn(bn, cout);
    c.bn_index = (int)m->bn_names.size();
    m->bn_names.push_back(bn);
    return c;
}

// The encoders the library builds (torchvision resnet.py): block kind, blocks per layer, channel expansion
struct Arch {
    const char* name;
    hn_model::Kind kind;
    int nblk[4];
    int expansion;
};
const Arch ARCHS[] = {{"resnet50", hn_model::BOTTLENECK, {3, 4, 6, 3}, 4}, {"resnet18", hn_model::BASIC, {2, 2, 2, 2}, 1}};

int block_out_channels(const hn_model::Block& b) { return b.kind == hn_model::BASIC ? b.c2.d.Cout : b.c3.d.Cout; }

// Builds the key list in the reference's own order (tests/golden/state_dict_keys*.json) and the graph.
void build_graph(hn_model* m, const Arch& arch) {
    const std::string enc = "feature_extractor.encoder.";
    m->stem = make_conv(m, enc + "conv1.1.weight", enc + "bn1", "", 3, 64, 7, 2, 2, 1);
    const int planes[4] = {64, 128, 256, 512};
    int inpl = 64;
    for (int l = 0; l < 4; ++l) {
        const int cout = planes[l] * arch.expansion;
        for (int b = 0; b < arch.nblk[l]; ++b) {
            const std::string p = enc + "layer" + std::to_string(l + 1) + "." + std::to_string(b) + ".";
            const int stride = (b == 0 && l > 0) ? 2 : 1;
            hn_model::Block blk;
            blk.kind = arch.kind;
            if (arch.kind == hn_model::BOTTLENECK) {
                blk.c1 = make_conv(m, p + "conv1.weight", p + "bn1", "", inpl, planes[l], 1, 1, 1, 1);
                blk.c2 = make_conv(m, p + "conv2.1.weight", p + "bn2", "", planes[l], planes[l], 3, stride, stride, 1);
                blk.c3 = make_conv(m, p + "conv3.weight", p + "bn3", "", planes[l], cout, 1, 1, 1, 1);
            } else {       // BasicBlock: conv1 3x3 carries the stride, conv2 3x3 + identity
                blk.c1 = make_conv(m, p + "conv1.1.weight", p + "bn1", "", inpl, planes[l], 3, stride, stride, 1);
                blk.c2 = make_conv(m, p + "conv2.1.weight", p + "bn2", "", planes[l], cout, 3, 1, 1, 1);
            }
            blk.has_ds = (b == 0) && (stride != 1 || inpl != cout);
            if (blk.has_ds)
                blk.ds = make_conv(m, p + "downsample.0.weight", p + "downsample.1", "", inpl, cout, 1, stride, stride, 0);
            inpl = cout;
            m->blocks[l].push_back(blk);
        }
    }
    for (int s = 0; s < 4; ++s) {
        const int c = planes[s] * arch.expansion;
        const int ch[5] = {c, c / 2, c / 2, c / 4, c / 8};
        for (int j = 0; j < 4; ++j) {
            const std::string p =
                "reduce_height_module.ghc_lst." + std::to_string(s) + ".layer." + std::to_string(j) + ".layers.";
            m->ghc[s][j] = make_conv(m, p + "0.1.weight", p + "1", p + "0.1.bias", ch[j], ch[j + 1], 3, 2, 1, 1);
        }
    }
    m->c_last = 0;                                   // model.py:175-178: C/8 channels at H = 8, 4, 2, 1 per scale
    for (int s = 0; s < 4; ++s) m->c_last += m->ghc[s][3].d.Cout * (8 >> s);
    const int K0 = m->c_last;
    if (!m->use_rnn) {
        // model.py:234-243: Linear(c_last, 512), ReLU, Dropout, Linear(512, 12)
        m->add_slot("linear.0.weight", 512ll * K0);
        m->add_slot("linear.0.bias", 512);
        m->add_slot("linear.3.weight", 12 * 512);
        m->add_slot("linear.3.bias", 12);
        ConvLayer& c = m->mlp1;
        c.d.Cin = K0; c.d.Cout = 512; c.d.kh = c.d.kw = 1; c.d.sh = c.d.sw = 1; c.d.ph = c.d.pw = 0; c.d.relu = 1;
        c.wkey = "linear.0.weight"; c.biaskey = "linear.0.bias";
        return;
    }
    for (int layer = 0; layer < 2; ++layer)
        for (int dir = 0; dir < 2; ++dir) {
            const std::string sfx = "_l" + std::to_string(layer) + (dir ? "_reverse" : "");
            m->add_slot("bi_rnn.weight_ih" + sfx, 2048ll * (layer == 0 ? K0 : 1024));
            m->add_slot("bi_rnn.weight_hh" + sfx, 2048ll * 512);
            m->add_slot("bi_rnn.bias_ih" + sfx, 2048);
            m->add_slot("bi_rnn.bias_hh" + sfx, 2048);
        }
    m->add_slot("linear.weight", 12 * 1024);
    m->add_slot("linear.bias", 12);
    for (int layer = 0; layer < 2; ++layer) {
        ConvLayer& c = m->xproj[layer];
        c.d.Cin = layer == 0 ? K0 : 1024; c.d.Cout = 4096; c.d.kh = c.d.kw = 1; c.d.sh = c.d.sw = 1; c.d.ph = c.d.pw = 0;
        c.d.relu = 0;
    }
}

int pack_conv(hn_model* m, ConvLayer& c, cudaStream_t st) {
    const size_t nw = (size_t)c.d.Cout * c.d.Cin * c.d.kh * c.d.kw;
    if (!c.w) {
        if (m->alloc_t(&c.w, nw)) return -1;
        if (m->alloc_t(&c.scale, c.d.Cout)) return -1;
        if (m->alloc_t(&c.shift, c.d.Cout)) return -1;
        if (c.d.Cin % 64 == 0 && (m->alloc_t(&c.wq, 2 * nw) || m->alloc_t(&c.tc_scale, 3 * c.d.Cout + 1))) return -1;
    }
    pack_oihw_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, st>>>(m->T(c.wkey), c.w, c.d.Cout, c.d.Cin, c.d.kh, c.d.kw);
    HN_LAUNCH_OK();
    fold_bn_kernel<<<(c.d.Cout + 255) / 256, 256, 0, st>>>(
        m->T(c.bnprefix + ".weight"), m->T(c.bnprefix + ".bias"), m->T(c.bnprefix + ".running_mean"),
        m->T(c.bnprefix + ".running_var"), c.biaskey.empty() ? nullptr : m->T(c.biaskey), c.scale, c.shift, c.d.Cout);
    HN_LAUNCH_OK();
    if (c.wq && pack_weight_tc(m->T(c.wkey), c.wq, c.scale, c.shift, c.tc_scale, c.tc_scale + 3 * c.d.Cout, c.d.Cout,
                               c.d.Cin, c.d.kh, c.d.kw, st))
        return -1;
    c.d.w = c.w; c.d.scale = c.scale; c.d.shift = c.shift;
    return 0;
}

// Folded conv3 + downsample pack of a block 0 (hn_model::Block::fold) from the eval-mode BN constants of both; built by
// the first eval forward that uses it after hn_model_finalize or refold_bn (hn_model::fold_stale)
int alloc_fold(hn_model* m, hn_model::Block& b) {
    ConvLayer& f = b.fold;
    const int Cout = b.c3.d.Cout;
    const size_t nw = (size_t)Cout * (b.c3.d.Cin + b.ds.d.Cin);
    if (f.w) return 0;
    return (m->alloc_t(&f.w, nw) || m->alloc_t(&f.shift, Cout) || m->alloc_t(&f.wq, 2 * nw) ||
            m->alloc_t(&f.tc_scale, 3 * Cout + 1)) ? -1 : 0;
}

int pack_fold(hn_model* m, hn_model::Block& b, cudaStream_t st) {
    ConvLayer& f = b.fold;
    const int Cout = b.c3.d.Cout, Cmid = b.c3.d.Cin, Cin = b.ds.d.Cin, K = Cmid + Cin;
    const size_t nw = (size_t)Cout * K;
    fold_downsample_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, st>>>(m->T(b.c3.wkey), b.c3.scale, b.c3.shift,
                                                                         m->T(b.ds.wkey), b.ds.scale, b.ds.shift, f.w,
                                                                         f.shift, Cout, Cmid, Cin);
    HN_LAUNCH_OK();
    return pack_weight_tc(f.w, f.wq, nullptr, f.shift, f.tc_scale, f.tc_scale + 3 * Cout, Cout, K, 1, 1, st);
}


int run_conv(hn_model* m, const ConvLayer& c, const Act& in, const Act& out, const float* res, cudaStream_t st,
             int cls, bool out_f32 = false) {
    const double flops = 2.0 * (double)out.B * out.H * out.W * c.d.Cout * c.d.kh * c.d.kw * c.d.Cin;
    Scope sc(m, cls, flops, st);
    if (!m->use_tc) return conv_f32(c.d, in, out, res, st);
    // tensor-core path: every activation buffer holds fp16 hi/lo planes (same bytes as fp32)
    if (!c.wq || !conv_tc_supported(c.d, in, out)) {
        // resnet18's narrow height-reduction convs (Cin 16 / 32): fp32 CUDA-core kernel on the same planes (conv_narrow.cu)
        if (!res && !out_f32 && conv_narrow_supported(c.d, in, out))
            return conv_narrow_planes(c.d, in, reinterpret_cast<const unsigned short*>(in.p), out,
                                      reinterpret_cast<unsigned short*>(out.p), st);
        return fail("hn_model_forward: a convolution of the graph is not covered by the tensor-core kernel");
    }
    return conv_tc_planes(c.d, c.wq, c.tc_scale, in, reinterpret_cast<const unsigned short*>(in.p), out,
                          out_f32 ? nullptr : reinterpret_cast<unsigned short*>(out.p), out_f32 ? out.p : nullptr,
                          reinterpret_cast<const unsigned short*>(res), st);
}

// Eval-mode epilogue constants again from the (moved) running statistics; the packed weights are untouched.
int refold_bn(hn_model* m, cudaStream_t st) {
    std::vector<ConvLayer*> all{&m->stem};
    for (int l = 0; l < 4; ++l)
        for (auto& b : m->blocks[l]) {
            all.push_back(&b.c1); all.push_back(&b.c2);
            if (b.kind == hn_model::BOTTLENECK) all.push_back(&b.c3);
            if (b.has_ds) all.push_back(&b.ds);
        }
    for (int s = 0; s < 4; ++s)
        for (int j = 0; j < 4; ++j) all.push_back(&m->ghc[s][j]);
    for (ConvLayer* c : all) {
        const int C = c->d.Cout;
        fold_bn_kernel<<<(C + 255) / 256, 256, 0, st>>>(
            m->T(c->bnprefix + ".weight"), m->T(c->bnprefix + ".bias"), m->T(c->bnprefix + ".running_mean"),
            m->T(c->bnprefix + ".running_var"), c->biaskey.empty() ? nullptr : m->T(c->biaskey), c->scale, c->shift, C);
        HN_LAUNCH_OK();
        if (c->tc_scale && tc_aux_update(c->scale, c->shift, c->tc_scale + 3 * C, c->tc_scale, C, st)) return -1;
    }
    m->fold_stale = true;                            // the folded packs carry the BN scales in their weights
    if (tc_aux_update(m->stem.scale, m->stem.shift, m->stem_aux + 3 * 64, m->stem_aux, 64, st)) return -1;
    m->bn_stale = false;
    return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
extern "C" {

const char* hn_last_error(void) { return g_err.c_str(); }
int hn_abi_version(void) { return 11; }
const char* hn_build_digest(void) { return HN_BUILD_DIGEST; }
long long hn_kernel_launches(void) { return g_launches.load(); }

int hn_model_create(int device, int max_batch, hn_model** out) { return hn_model_create_arch(device, max_batch, "resnet50", 1, out); }

int hn_model_create_head(int device, int max_batch, int use_rnn, hn_model** out) {
    return hn_model_create_arch(device, max_batch, "resnet50", use_rnn, out);
}

int hn_model_create_arch(int device, int max_batch, const char* backbone, int use_rnn, hn_model** out) {
    HN_CHECK(out != nullptr && backbone != nullptr, "hn_model_create: NULL argument");
    HN_CHECK(max_batch >= 1 && max_batch <= 1024, "hn_model_create: max_batch must be in 1..1024");
    HN_CHECK(use_rnn == 0 || use_rnn == 1, "hn_model_create_head: use_rnn must be 0 or 1");
    const Arch* arch = nullptr;
    for (const Arch& a : ARCHS)
        if (std::strcmp(a.name, backbone) == 0) arch = &a;
    if (!arch) return fail(std::string("hn_model_create_arch: unsupported backbone '") + backbone + "' (resnet50, resnet18)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail("hn_model_create: no CUDA device -- libhorizonnet_b200 has no CPU path");
    HN_CHECK(device >= 0 && device < ndev, "hn_model_create: bad device index");
    HN_ON_DEVICE(device);
    cudaDeviceProp prop;
    HN_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    HN_CHECK(prop.major == 9 && prop.minor == 0, "hn_model_create: this library is built for sm_90a (H100) only");
    std::unique_ptr<hn_model> m(new hn_model());
    m->device = device;
    m->max_batch = max_batch;
    m->use_rnn = use_rnn;
    build_graph(m.get(), *arch);
    for (auto& s : m->slots)
        if (!s.ignored && m->alloc_t(&s.dev, (size_t)s.numel)) return -1;
    const size_t B = (size_t)max_batch;
    const size_t CL = (size_t)m->c_last;
    // encoder workspace from the graph, per image: X block outputs, F stage outputs, T1 / T2 the intermediates of a
    // block, IDN its downsample, G / GO the height reduction (halo-NHWC: H x (W + 2) x C)
    size_t x_img = 0, t1_img = 0, t2_img = 0, idn_img = 0, f_img[4] = {0, 0, 0, 0}, g_img = 0, go_img[4] = {0, 0, 0, 0};
    {
        auto px = [](int h, int w, int c) { return (size_t)h * (w + 2) * c; };
        int H = 128, W = 256;                              // after the stem and the max-pool
        for (int l = 0; l < 4; ++l) {
            const int nb = (int)m->blocks[l].size();
            for (int b = 0; b < nb; ++b) {
                const hn_model::Block& blk = m->blocks[l][b];
                const bool basic = blk.kind == hn_model::BASIC;
                const int s = basic ? blk.c1.d.sh : blk.c2.d.sh, Ho = H / s, Wo = W / s;
                t1_img = std::max(t1_img, basic ? px(Ho, Wo, blk.c1.d.Cout) : px(H, W, blk.c1.d.Cout));
                if (!basic) t2_img = std::max(t2_img, px(Ho, Wo, blk.c2.d.Cout));
                if (blk.has_ds) idn_img = std::max(idn_img, px(Ho, Wo, blk.ds.d.Cout));
                const size_t y = px(Ho, Wo, block_out_channels(blk));
                if (b == nb - 1) f_img[l] = y; else x_img = std::max(x_img, y);
                H = Ho; W = Wo;
            }
            int h = H;
            for (int j = 0; j < 4; ++j) {
                h /= 2;
                const size_t o = px(h, W, m->ghc[l][j].d.Cout);
                if (j == 3) go_img[l] = o; else g_img = std::max(g_img, o);
            }
        }
    }
    // X[0] is also the stem's packed-input scratch (stem_tc) and the plane-merge scratch of hn_model_stage("layerN")
    const size_t x0 = std::max({x_img * B, (stem_tc_scratch_bytes((int)B) + 3) / 4, f_img[0] * B, f_img[1] * B,
                                f_img[2] * B, f_img[3] * B});
    m->x0_cap = x0;
    if (!use_rnn) {
        // MLP head: no projections / recurrence buffers.  XP stays as scratch: stem weight packing at finalize and the
        // plane merge of the "feature" test stage.
        struct { float** p; size_t n; } head_bufs[] = {
            {&m->XP, std::max((size_t)256 * B * CL, (size_t)4096 * 1024)},
            {&m->HID, 256 * B * 512},
        };
        for (auto& b : head_bufs)
            if (m->alloc_t(b.p, b.n)) return -1;
    }
    struct { float** p; size_t n; } bufs[] = {
        {&m->S0, B * 256 * 514 * 64},   {&m->S1, B * 128 * 258 * 64},  {&m->X[0], x0},
        {&m->X[1], B * x_img},          {&m->IDN, B * idn_img},        {&m->T1, B * t1_img},
        {&m->T2, B * t2_img},           {&m->F[0], B * f_img[0]},      {&m->F[1], B * f_img[1]},
        {&m->F[2], B * f_img[2]},       {&m->F[3], B * f_img[3]},      {&m->G[0], B * g_img},
        {&m->G[1], B * g_img},          {&m->GO[0], B * go_img[0]},    {&m->GO[1], B * go_img[1]},
        {&m->GO[2], B * go_img[2]},     {&m->GO[3], B * go_img[3]},    {&m->SEQ, 256 * B * CL},
        {&m->x_in, B * 3 * 512 * 1024}, {&m->bon_out, B * 2 * 1024},    {&m->cor_out, B * 1024},
        {&m->x_slot[1], B * 3 * 512 * 1024},
        {&m->bon_slot[1], B * 2 * 1024},  {&m->cor_slot[1], B * 1024},
        {&m->head_w, 12 * 1024},        {&m->head_b, 12},
    };
    for (auto& b : bufs)
        if (m->alloc_t(b.p, b.n)) return -1;
    if (use_rnn) {
        struct { float** p; size_t n; } rnn_bufs[] = {
            {&m->XP, (256 * B * 4096 > (size_t)4096 * 1024) ? 256 * B * 4096 : (size_t)4096 * 1024},       {&m->R1, 256 * B * 1024},       {&m->R2, 256 * B * 1024},       {&m->R1S, 256 * B * 1024},
        };
        for (auto& b : rnn_bufs)
            if (m->alloc_t(b.p, b.n)) return -1;
    }
    if (m->alloc_t(&m->error_flag, 1)) return -1;
    if (m->alloc_t(&m->tta_ints, 128)) return -1;
    HN_CUDA_OK(cudaMemset(m->error_flag, 0, sizeof(int)));
    m->x_slot[0] = m->x_in;
    m->bon_slot[0] = m->bon_out; m->cor_slot[0] = m->cor_out;
    HN_CUDA_OK(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
    HN_CUDA_OK(cudaStreamCreateWithFlags(&m->compute_stream, cudaStreamNonBlocking));
    {
        int prio_lo = 0, prio_hi = 0;
        HN_CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
        HN_CUDA_OK(cudaStreamCreateWithPriority(&m->enc_stream, cudaStreamNonBlocking, prio_lo));
        // the recurrence's 16-CTA clusters must get their SMs as soon as a convolution kernel retires
        HN_CUDA_OK(cudaStreamCreateWithPriority(&m->rnn_stream, cudaStreamNonBlocking, prio_hi));
    }
    for (int i = 0; i < 2; ++i) {
        HN_CUDA_OK(cudaEventCreateWithFlags(&m->slot_ready[i], cudaEventDisableTiming));
        HN_CUDA_OK(cudaEventCreateWithFlags(&m->slot_done[i], cudaEventDisableTiming));
        HN_CUDA_OK(cudaEventCreateWithFlags(&m->async_done[i], cudaEventDisableTiming));
    }
    for (cudaEvent_t* e : {&m->ev_in, &m->ev_xfree, &m->ev_seq, &m->ev_rnn_last, &m->ev_plain_done})
        HN_CUDA_OK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    *out = m.release();
    return 0;
}

int hn_model_num_tensors(const hn_model* m) { return m ? (int)m->slots.size() : 0; }

int hn_model_tensor_info(const hn_model* m, int i, const char** key, long long* numel) {
    HN_CHECK(m && i >= 0 && i < (int)m->slots.size(), "hn_model_tensor_info: bad index");
    if (key) *key = m->slots[i].key.c_str();
    if (numel) *numel = m->slots[i].numel;
    return 0;
}

int hn_model_set_tensor(hn_model* m, const char* key, const float* data, long long numel, int on_device) {
    HN_CHECK(m && key, "hn_model_set_tensor: NULL argument");
    auto it = m->index.find(key);
    if (it == m->index.end()) return fail(std::string("hn_model_set_tensor: unexpected key '") + key + "'");
    TensorSlot& s = m->slots[it->second];
    if (s.ignored) { s.set = true; return 0; }
    HN_CHECK(data != nullptr, "hn_model_set_tensor: data is NULL");
    if (numel != s.numel)
        return fail(std::string("hn_model_set_tensor: size mismatch for '") + key + "': got " + std::to_string(numel) +
                    ", expected " + std::to_string(s.numel));
    HN_ON_DEVICE(m->device);
    if (m->rnn_inflight) {        // forwards may still be running on the internal (non-blocking) streams: do not race them
        HN_CUDA_OK(cudaStreamSynchronize(m->enc_stream));
        HN_CUDA_OK(cudaStreamSynchronize(m->rnn_stream));
        m->rnn_inflight = false;
    }
    HN_CUDA_OK(cudaMemcpy(s.dev, data, (size_t)numel * sizeof(float),
                          on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    s.set = true;
    m->finalized = false;
    return 0;
}

int hn_model_set_option(hn_model* m, const char* name, int value) {
    HN_CHECK(m && name, "hn_model_set_option: NULL argument");
    if (std::strcmp(name, "tensor_cores") == 0) { m->use_tc = value; return 0; }
    if (std::strcmp(name, "profile") == 0) { m->profile = value; return 0; }
    if (std::strcmp(name, "fold_downsample") == 0) { m->fold_on = value; return 0; }
    return fail(std::string("hn_model_set_option: unknown option '") + name + "'");
}

int hn_model_finalize(hn_model* m) {
    HN_CHECK(m, "hn_model_finalize: NULL model");
    for (auto& s : m->slots)
        if (!s.set && !s.ignored) return fail("hn_model_finalize: missing key '" + s.key + "' (strict load, utils.py:64)");
    HN_ON_DEVICE(m->device);
    cudaStream_t st = 0;
    if (pack_conv(m, m->stem, st)) return -1;
    if (!m->stem_wq && (m->alloc_t(&m->stem_wq, (size_t)2 * 64 * 224) || m->alloc_t(&m->stem_aux, 3 * 64 + 1))) return -1;
    if (stem_tc_pack_weights(m->T(m->stem.wkey), m->XP, m->stem_wq, m->stem.scale, m->stem.shift, m->stem_aux, st)) return -1;
    for (int l = 0; l < 4; ++l)
        for (auto& b : m->blocks[l]) {
            if (pack_conv(m, b.c1, st) || pack_conv(m, b.c2, st)) return -1;
            if (b.kind == hn_model::BOTTLENECK && pack_conv(m, b.c3, st)) return -1;
            if (b.has_ds && pack_conv(m, b.ds, st)) return -1;
            if (b.has_ds && b.kind == hn_model::BOTTLENECK && alloc_fold(m, b)) return -1;
        }
    m->fold_stale = true;
    for (int s = 0; s < 4; ++s)
        for (int j = 0; j < 4; ++j)
            if (pack_conv(m, m->ghc[s][j], st)) return -1;
    if (!m->use_rnn) {
        // MLP layer 1: OIHW [512][K] -> [K][N=512] (K = c_last), epilogue 1 * acc + linear.0.bias, ReLU in the kernel
        ConvLayer& c = m->mlp1;
        const int K = m->c_last;
        if (!c.w) {
            if (m->alloc_t(&c.w, (size_t)512 * K) || m->alloc_t(&c.scale, 512) || m->alloc_t(&c.shift, 512)) return -1;
            if (m->alloc_t(&c.wq, (size_t)2 * 512 * K) || m->alloc_t(&c.tc_scale, 3 * 512 + 1)) return -1;
        }
        pack_oihw_kernel<<<(512 * K + 255) / 256, 256, 0, st>>>(m->T(c.wkey), c.w, 512, K, 1, 1);
        HN_LAUNCH_OK();
        bias_constants_kernel<<<2, 256, 0, st>>>(m->T(c.biaskey), c.scale, c.shift, 512);
        HN_LAUNCH_OK();
        if (pack_weight_tc(m->T(c.wkey), c.wq, c.scale, c.shift, c.tc_scale, c.tc_scale + 3 * 512, 512, K, 1, 1, st)) return -1;
        c.d.w = c.w; c.d.scale = c.scale; c.d.shift = c.shift;
        HN_CUDA_OK(cudaMemcpyAsync(m->head_w, m->T("linear.3.weight"), 12 * 512 * sizeof(float), cudaMemcpyDeviceToDevice, st));
        HN_CUDA_OK(cudaMemcpyAsync(m->head_b, m->T("linear.3.bias"), 12 * sizeof(float), cudaMemcpyDeviceToDevice, st));
        HN_CUDA_OK(cudaStreamSynchronize(st));
        m->bn_stale = false;
        m->finalized = true;
        return 0;
    }
    for (int layer = 0; layer < 2; ++layer) {
        ConvLayer& c = m->xproj[layer];
        const int K = c.d.Cin;                       // c_last for layer 0, 1024 for layer 1
        if (!c.w) {
            if (m->alloc_t(&c.w, (size_t)4096 * K) || m->alloc_t(&c.scale, 4096) || m->alloc_t(&c.shift, 4096)) return -1;
            if (m->alloc_t(&c.wq, (size_t)2 * 4096 * K) || m->alloc_t(&c.tc_scale, 3 * 4096 + 1)) return -1;
        }
        const std::string l = "_l" + std::to_string(layer);
        // [4096][K] (fwd rows then reverse rows) -> [K][N=4096]
        for (int dir = 0; dir < 2; ++dir) {
            const float* w = m->T("bi_rnn.weight_ih" + l + (dir ? "_reverse" : ""));
            HN_CUDA_OK(cudaMemcpyAsync(m->XP + (size_t)dir * 2048 * K, w, (size_t)2048 * K * sizeof(float),
                                       cudaMemcpyDeviceToDevice, st));
            m->whh[layer][dir] = m->T("bi_rnn.weight_hh" + l + (dir ? "_reverse" : ""));
        }
        pack_oihw_kernel<<<(4096 * K + 255) / 256, 256, 0, st>>>(m->XP, c.w, 4096, K, 1, 1);
        HN_LAUNCH_OK();

        lstm_bias_kernel<<<16, 256, 0, st>>>(m->T("bi_rnn.bias_ih" + l), m->T("bi_rnn.bias_hh" + l),
                                             m->T("bi_rnn.bias_ih" + l + "_reverse"),
                                             m->T("bi_rnn.bias_hh" + l + "_reverse"), c.scale, c.shift);
        HN_LAUNCH_OK();
        if (pack_weight_tc(m->XP, c.wq, c.scale, c.shift, c.tc_scale, c.tc_scale + 3 * 4096, 4096, K, 1, 1, st)) return -1;
        c.d.w = c.w; c.d.scale = c.scale; c.d.shift = c.shift;
    }
    HN_CUDA_OK(cudaMemcpyAsync(m->head_w, m->T("linear.weight"), 12 * 1024 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    HN_CUDA_OK(cudaMemcpyAsync(m->head_b, m->T("linear.bias"), 12 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    HN_CUDA_OK(cudaStreamSynchronize(st));
    m->bn_stale = false;
    m->finalized = true;
    return 0;
}

// ---- the three parts of HorizonNet.forward (model.py:254-281); static helpers (no extern "C" linkage needed)
// (1) normalise + stem + max-pool + layer1..4 + the 16 height-reduction convs: leaves gout[] in GO[0..3]
static int forward_encoder(hn_model* m, const float* x, int B, int in_channels, Act gout[4], cudaStream_t st,
                           cudaEvent_t x_consumed) {
    if (m->bn_stale && refold_bn(m, st)) return -1;
    if (m->use_tc && m->fold_on && m->fold_stale) {
        for (int l = 0; l < 4; ++l)
            for (auto& b : m->blocks[l])
                if (b.has_ds && b.kind == hn_model::BOTTLENECK && pack_fold(m, b, st)) return -1;
        m->fold_stale = false;
    }
    // model.py:248-252 + :73-76: normalise, stem conv/BN/ReLU, max-pool
    Act s0 = mk(m->S0, B, 256, 512, 64);
    {
        Scope sc(m, CLS_STEM, 2.0 * B * 256 * 512 * 64 * 147, st);
        if (m->use_tc) {
            // packed input planes live in X[0] (free until layer1): B * 8.6 MB of its B * 33.8 MB
            if (stem_tc(x, B, in_channels, m->stem_wq, m->stem_aux, m->stem.shift, reinterpret_cast<unsigned short*>(m->X[0]),
                        s0, st))
                return -1;
        } else if (stem_f32(x, B, in_channels, m->stem.w, m->stem.scale, m->stem.shift, s0, st)) return -1;
    }
    if (x_consumed) HN_CUDA_OK(cudaEventRecord(x_consumed, st));       // the input batch is not read after the stem
    Act cur = mk(m->S1, B, 128, 256, 64);
    {
        Scope sc(m, CLS_POOL, 0.0, st);
        if (maxpool3x3s2(s0, cur, st, m->use_tc != 0)) return -1;
    }

    // model.py:78-81: layer1..layer4 (torchvision Bottleneck v1.5, or BasicBlock)
    Act feats[4];
    for (int l = 0; l < 4; ++l) {
        const int nb = (int)m->blocks[l].size();
        for (int b = 0; b < nb; ++b) {
            const hn_model::Block& blk = m->blocks[l][b];
            if (blk.kind == hn_model::BASIC) {
                // conv1 3x3 (stride) + BN + ReLU; the downsample (block 0 of layers 2-4) as its own launch; conv2 3x3 + BN +
                // identity + ReLU.  No fold / fused kernel for this block kind: option fold_downsample changes nothing here
                const int s = blk.c1.d.sh;
                Act t1 = mk(m->T1, B, cur.H / s, cur.W / s, blk.c1.d.Cout);
                Act y = mk(b == nb - 1 ? m->F[l] : m->X[b & 1], B, t1.H, t1.W, blk.c2.d.Cout);
                if (run_conv(m, blk.c1, cur, t1, nullptr, st, CLS_ENC_CONV)) return -1;
                const float* idn = cur.p;
                if (blk.has_ds) {
                    Act d = mk(m->IDN, B, t1.H, t1.W, blk.ds.d.Cout);
                    if (run_conv(m, blk.ds, cur, d, nullptr, st, CLS_ENC_CONV)) return -1;
                    idn = d.p;
                }
                if (run_conv(m, blk.c2, t1, y, idn, st, CLS_ENC_CONV)) return -1;
                cur = y;
                continue;
            }
            const int s = blk.c2.d.sh;
            const int Ho = cur.H / s, Wo = cur.W / s;
            Act t1 = mk(m->T1, B, cur.H, cur.W, blk.c1.d.Cout);
            Act t2 = mk(m->T2, B, Ho, Wo, blk.c2.d.Cout);
            Act y = mk(b == nb - 1 ? m->F[l] : m->X[b & 1], B, Ho, Wo, blk.c3.d.Cout);
            if (run_conv(m, blk.c1, cur, t1, nullptr, st, CLS_ENC_CONV)) return -1;
            // on the tensor cores: the downsample runs inside conv3, one GEMM over [t2 | x] (no identity tensor)
            const bool fold = blk.has_ds && m->use_tc && m->fold_on;
            const float* idn = cur.p;
            if (blk.has_ds && !fold) {
                Act d = mk(m->IDN, B, Ho, Wo, blk.ds.d.Cout);
                if (run_conv(m, blk.ds, cur, d, nullptr, st, CLS_ENC_CONV)) return -1;
                idn = d.p;
            }
            const double conv3_k = blk.c3.d.Cin + (fold ? (double)blk.ds.d.Cin : 0.0);
            if (m->use_tc && blk.c2.wq && blk.c3.wq && bott_tc_supported(blk.c2.d, blk.c3.d, t1, y) &&
                (!fold || (cur.C == 64 && cur.H == t1.H && cur.W == t1.W))) {
                // layer1: conv2 + conv3 in one kernel, the 64-channel intermediate stays in shared memory (conv_tc.cu)
                const double flops = 2.0 * (double)B * Ho * Wo * (64.0 * 9 * 64 + (double)blk.c3.d.Cout * conv3_k);
                Scope sc(m, CLS_ENC_CONV, flops, st);
                const ConvLayer& c3 = fold ? blk.fold : blk.c3;
                const unsigned short* idn_planes = reinterpret_cast<const unsigned short*>(idn);
                if (bott_tc_planes(blk.c2.d, blk.c2.wq, blk.c2.tc_scale, blk.c3.d, c3.wq, c3.tc_scale, t1,
                                   reinterpret_cast<const unsigned short*>(t1.p), y, reinterpret_cast<unsigned short*>(y.p),
                                   fold ? nullptr : idn_planes, fold ? idn_planes : nullptr, st))
                    return -1;
            } else {
                if (run_conv(m, blk.c2, t1, t2, nullptr, st, CLS_ENC_CONV)) return -1;
                if (fold) {
                    Scope sc(m, CLS_ENC_CONV, 2.0 * (double)B * Ho * Wo * blk.c3.d.Cout * conv3_k, st);
                    if (conv_tc_fold_planes(blk.fold.wq, blk.fold.tc_scale, t2, reinterpret_cast<const unsigned short*>(t2.p),
                                            cur, reinterpret_cast<const unsigned short*>(cur.p), s, y,
                                            reinterpret_cast<unsigned short*>(y.p), st))
                        return -1;
                } else if (run_conv(m, blk.c3, t2, y, idn, st, CLS_ENC_CONV)) return -1;   // + identity, ReLU
            }
            cur = y;
        }
        feats[l] = cur;
    }

    // model.py:148-151: 4 x (3x3 stride (2,1) conv + bias + BN + ReLU) per scale
    for (int s = 0; s < 4; ++s) {
        Act g = feats[s];
        for (int j = 0; j < 4; ++j) {
            const ConvLayer& c = m->ghc[s][j];
            Act o = mk(j == 3 ? m->GO[s] : m->G[j & 1], B, g.H / 2, g.W, c.d.Cout);
            if (run_conv(m, c, g, o, nullptr, st, CLS_GHC_CONV)) return -1;
            g = o;
        }
        gout[s] = g;
    }
    return 0;
}

// (2) model.py:152-155 + :175-178 + :263: upsample + flatten + concat + permute -> SEQ [T=256][B][c_last]
static int forward_sequence(hn_model* m, const Act gout[4], cudaStream_t st) {
    Scope sc(m, CLS_TAIL, 0.0, st);
    return ghc_to_sequence(gout, m->SEQ, st, m->use_tc != 0);
}

// (3') model.py:270-279 (use_rnn=False): per-column MLP over the rows of SEQ.  Layer 1 (c_last -> 512, bias, ReLU) is the
// same GEMM-row convolution as the LSTM projections; layer 2 + the scatter (eval: the dropout between them = identity).
static int forward_mlp(hn_model* m, int B, float* bon, float* cor, cudaStream_t st) {
    const Act a = mk(m->SEQ, 1, 1, 256 * B, m->c_last, 0);
    const Act h = mk(m->HID, 1, 1, 256 * B, 512, 0);
    if (run_conv(m, m->mlp1, a, h, nullptr, st, CLS_HEAD, true)) return -1;
    Scope sc(m, CLS_HEAD, 2.0 * 256 * B * 12 * 512, st);
    return linear_head(m->HID, m->head_w, m->head_b, bon, cor, 256, B, 512, st);
}

// (3) model.py:264-281: 2-layer bidirectional LSTM (eval: dropout = identity), linear head, reshape, split
static int forward_rnn(hn_model* m, int B, float* bon, float* cor, cudaStream_t st) {
    if (!m->use_rnn) return forward_mlp(m, B, bon, cor, st);
    const float* lin = m->SEQ;
    float* louts[2] = {m->R1, m->R2};
    for (int layer = 0; layer < 2; ++layer) {
        Act a = mk(const_cast<float*>(lin), 1, 1, 256 * B, m->xproj[layer].d.Cin, 0);
        Act xp = mk(m->XP, 1, 1, 256 * B, 4096, 0);
        if (m->use_tc && layer == 1) {
            // layer-2 projection operand: the fp32 recurrence output as fp16 hi/lo planes
            Scope sc(m, CLS_TAIL, 0.0, st);
            if (split_planes(m->R1, reinterpret_cast<unsigned short*>(m->R1S), (size_t)256 * B * 1024, st)) return -1;
            a.p = m->R1S;
        }
        if (run_conv(m, m->xproj[layer], a, xp, nullptr, st, CLS_XPROJ, true)) return -1;
        {
            Scope sc(m, CLS_LSTM, 2.0 * 256 * B * 2 * 2048 * 512, st);
            if (lstm_layer(m->XP, m->whh[layer][0], m->whh[layer][1], louts[layer], 256, B, st)) return -1;
        }
        lin = louts[layer];
    }
    {
        Scope sc(m, CLS_HEAD, 2.0 * 256 * B * 12 * 1024, st);
        if (linear_head(m->R2, m->head_w, m->head_b, bon, cor, 256, B, 1024, st)) return -1;
    }
    return 0;
}

static int forward_args_ok(hn_model* m, const void* x, int B, const void* bon, const void* cor, const char* who) {
    if (!(m && x && bon && cor)) return fail(std::string(who) + ": NULL argument");
    if (!m->finalized) return fail(std::string(who) + ": call hn_model_finalize after setting all tensors");
    if (!(B >= 1 && B <= m->max_batch)) return fail(std::string(who) + ": batch exceeds max_batch given at create");
    return 0;
}

// Two-stream enqueue of one forward: encoder + height reduction on enc_stream (the caller has already made
// enc_stream wait for the input), sequence assembly once the previous batch's recurrence no longer reads SEQ,
// then projections + recurrence + head on rnn_stream.  `done` (optional) is recorded when bon/cor are complete.
static int enqueue_two_stream(hn_model* m, const float* x, int B, int in_channels, float* bon, float* cor,
                              cudaEvent_t done) {
    if (m->plain_recorded) {      // a plain hn_model_forward on a caller stream may still use the workspace
        HN_CUDA_OK(cudaStreamWaitEvent(m->enc_stream, m->ev_plain_done, 0));
        HN_CUDA_OK(cudaStreamWaitEvent(m->rnn_stream, m->ev_plain_done, 0));
        m->plain_recorded = false;
    }
    Act gout[4];
    if (forward_encoder(m, x, B, in_channels, gout, m->enc_stream, m->ev_xfree)) return -1;
    if (m->rnn_inflight) HN_CUDA_OK(cudaStreamWaitEvent(m->enc_stream, m->ev_rnn_last, 0));
    if (forward_sequence(m, gout, m->enc_stream)) return -1;
    HN_CUDA_OK(cudaEventRecord(m->ev_seq, m->enc_stream));
    HN_CUDA_OK(cudaStreamWaitEvent(m->rnn_stream, m->ev_seq, 0));
    if (forward_rnn(m, B, bon, cor, m->rnn_stream)) return -1;
    HN_CUDA_OK(cudaEventRecord(m->ev_rnn_last, m->rnn_stream));
    if (done) HN_CUDA_OK(cudaEventRecord(done, m->rnn_stream));
    m->rnn_inflight = true;
    m->last_batch = B;
    return 0;
}

int hn_model_forward(hn_model* m, const float* x, int B, int in_channels, float* bon, float* cor, void* stream) {
    if (forward_args_ok(m, x, B, bon, cor, "hn_model_forward")) return -1;
    HN_ON_DEVICE(m->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (m->rnn_inflight) {        // join batches still in flight on the internal streams (they share the workspace)
        HN_CUDA_OK(cudaStreamWaitEvent(st, m->ev_rnn_last, 0));
        m->rnn_inflight = false;
    }
    m->last_batch = B;
    Act gout[4];
    if (forward_encoder(m, x, B, in_channels, gout, st, nullptr)) return -1;
    if (forward_sequence(m, gout, st)) return -1;
    if (forward_rnn(m, B, bon, cor, st)) return -1;
    HN_CUDA_OK(cudaEventRecord(m->ev_plain_done, st));
    m->plain_recorded = true;
    return 0;
}

int hn_model_num_bn(const hn_model* m) { return m ? (int)m->bn_names.size() : 0; }

const char* hn_model_bn_name(const hn_model* m, int i) {
    return (m && i >= 0 && i < (int)m->bn_names.size()) ? m->bn_names[i].c_str() : nullptr;
}

int hn_model_get_tensor(hn_model* m, const char* key, float* out, long long numel, int on_device, void* stream) {
    HN_CHECK(m && key && out, "hn_model_get_tensor: NULL argument");
    auto it = m->index.find(key);
    if (it == m->index.end()) return fail(std::string("hn_model_get_tensor: unknown key '") + key + "'");
    const TensorSlot& s = m->slots[it->second];
    HN_CHECK(!s.ignored && s.set && s.dev, "hn_model_get_tensor: tensor was never set");
    HN_CHECK(numel == s.numel, "hn_model_get_tensor: element count differs from the tensor's");
    HN_ON_DEVICE(m->device);
    cudaStream_t st = (cudaStream_t)stream;
    HN_CUDA_OK(cudaMemcpyAsync(out, s.dev, (size_t)numel * sizeof(float),
                               on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
    if (!on_device) HN_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

int hn_dropout_mask(unsigned long long seed, int which, double p, float* out, long long n, void* stream) {
    HN_CHECK(out && n >= 0, "hn_dropout_mask: bad argument");
    return dropout_inplace(out, (size_t)n, p, seed, which, true, (cudaStream_t)stream);
}

int hn_model_forward_async(hn_model* m, const float* x, int B, int in_channels, float* bon, float* cor, void* stream) {
    if (forward_args_ok(m, x, B, bon, cor, "hn_model_forward_async")) return -1;
    HN_ON_DEVICE(m->device);
    cudaStream_t st = (cudaStream_t)stream;
    HN_CUDA_OK(cudaEventRecord(m->ev_in, st));                          // x (and everything before it on st) is ready
    HN_CUDA_OK(cudaStreamWaitEvent(m->enc_stream, m->ev_in, 0));
    const int slot = (int)(m->async_count & 1);
    const bool had_prev = m->async_count > 0;
    if (enqueue_two_stream(m, x, B, in_channels, bon, cor, m->async_done[slot])) return -1;
    HN_CUDA_OK(cudaStreamWaitEvent(st, m->ev_xfree, 0));                // x may be overwritten by later work on st
    if (had_prev) HN_CUDA_OK(cudaStreamWaitEvent(st, m->async_done[slot ^ 1], 0));   // outputs of the PREVIOUS call
    ++m->async_count;
    return 0;
}

int hn_model_flush(hn_model* m, void* stream) {
    HN_CHECK(m, "hn_model_flush: NULL model");
    HN_ON_DEVICE(m->device);
    if (m->rnn_inflight) HN_CUDA_OK(cudaStreamWaitEvent((cudaStream_t)stream, m->ev_rnn_last, 0));
    return 0;
}

int hn_model_profile_read(hn_model* m, double* ms, double* flops, long long* launches, int reset) {
    HN_CHECK(m, "hn_model_profile_read: NULL model");
    HN_ON_DEVICE(m->device);
    for (auto& sp : m->spans) {
        HN_CUDA_OK(cudaEventSynchronize(sp.b));
        float t = 0.f;
        HN_CUDA_OK(cudaEventElapsedTime(&t, sp.a, sp.b));
        m->prof_ms[sp.cls] += t; m->prof_flops[sp.cls] += sp.flops; m->prof_launches[sp.cls] += 1;
        m->free_events.push_back(sp.a); m->free_events.push_back(sp.b);
    }
    m->spans.clear();
    for (int i = 0; i < HN_NUM_CLASSES; ++i) {
        if (ms) ms[i] = m->prof_ms[i];
        if (flops) flops[i] = m->prof_flops[i];
        if (launches) launches[i] = m->prof_launches[i];
        if (reset) { m->prof_ms[i] = 0; m->prof_flops[i] = 0; m->prof_launches[i] = 0; }
    }
    return 0;
}

int hn_model_check(hn_model* m) {
    // surfaces device-side failures (grid-barrier time-out of the cooperative BPTT kernel) after a synchronisation point
    HN_CHECK(m, "hn_model_check: NULL model");
    HN_ON_DEVICE(m->device);
    int flag = 0;
    HN_CUDA_OK(cudaMemcpy(&flag, m->error_flag, sizeof(int), cudaMemcpyDeviceToHost));
    if (flag) {
        cudaMemset(m->error_flag, 0, sizeof(int));
        return fail("hn_model: the persistent LSTM kernel timed out waiting for a peer CTA");
    }
    return 0;
}

int hn_model_forward_host(hn_model* m, const float* x, int B, int in_channels, float* bon, float* cor) {
    HN_CHECK(m && x && bon && cor, "hn_model_forward_host: NULL argument");
    HN_CHECK(B >= 1 && B <= m->max_batch, "hn_model_forward_host: batch exceeds max_batch");
    HN_CHECK(in_channels >= 3, "hn_model_forward_host: need >= 3 channels");
    HN_CHECK(m->submit_count == m->collect_count, "hn_model_forward_host: collect the submitted batches first");
    HN_ON_DEVICE(m->device);
    cudaStream_t st = 0;
    // only the first 3 channels are used (model.py:252): copy them image by image
    for (int b = 0; b < B; ++b)
        HN_CUDA_OK(cudaMemcpyAsync(m->x_in + (size_t)b * 3 * 512 * 1024, x + (size_t)b * in_channels * 512 * 1024,
                                   (size_t)3 * 512 * 1024 * sizeof(float), cudaMemcpyHostToDevice, st));
    if (hn_model_forward(m, m->x_in, B, 3, m->bon_out, m->cor_out, st)) return -1;
    HN_CUDA_OK(cudaMemcpyAsync(bon, m->bon_out, (size_t)B * 2 * 1024 * sizeof(float), cudaMemcpyDeviceToHost, st));
    HN_CUDA_OK(cudaMemcpyAsync(cor, m->cor_out, (size_t)B * 1024 * sizeof(float), cudaMemcpyDeviceToHost, st));
    HN_CUDA_OK(cudaStreamSynchronize(st));
    return hn_model_check(m);
}

int hn_model_submit_host(hn_model* m, const float* x, int B, int in_channels) {
    HN_CHECK(m && x, "hn_model_submit_host: NULL argument");
    HN_CHECK(m->finalized, "hn_model_submit_host: call hn_model_finalize after setting all tensors");
    HN_CHECK(B >= 1 && B <= m->max_batch, "hn_model_submit_host: batch exceeds max_batch");
    HN_CHECK(in_channels >= 3, "hn_model_submit_host: need >= 3 channels");
    HN_CHECK(m->submit_count - m->collect_count < 2, "hn_model_submit_host: both input slots are in flight (collect first)");
    HN_ON_DEVICE(m->device);
    const int slot = m->submit_count & 1;
    // the slot's previous batch was collected (fully synchronised), so its input buffer is free
    for (int b = 0; b < B; ++b)
        HN_CUDA_OK(cudaMemcpyAsync(m->x_slot[slot] + (size_t)b * 3 * 512 * 1024, x + (size_t)b * in_channels * 512 * 1024,
                                   (size_t)3 * 512 * 1024 * sizeof(float), cudaMemcpyHostToDevice, m->copy_stream));
    HN_CUDA_OK(cudaEventRecord(m->slot_ready[slot], m->copy_stream));
    // the forward is enqueued right away: the encoder of this batch overlaps the recurrence of the previous one
    HN_CUDA_OK(cudaStreamWaitEvent(m->enc_stream, m->slot_ready[slot], 0));
    if (enqueue_two_stream(m, m->x_slot[slot], B, 3, m->bon_slot[slot], m->cor_slot[slot], m->slot_done[slot])) return -1;
    m->slot_batch[slot] = B;
    ++m->submit_count;
    return 0;
}

int hn_model_collect_host(hn_model* m, float* bon, float* cor) {
    HN_CHECK(m && bon && cor, "hn_model_collect_host: NULL argument");
    HN_CHECK(m->collect_count < m->submit_count, "hn_model_collect_host: nothing submitted");
    HN_ON_DEVICE(m->device);
    const int slot = m->collect_count & 1;
    const int B = m->slot_batch[slot];
    cudaStream_t st = m->compute_stream;
    HN_CUDA_OK(cudaStreamWaitEvent(st, m->slot_done[slot], 0));
    HN_CUDA_OK(cudaMemcpyAsync(bon, m->bon_slot[slot], (size_t)B * 2 * 1024 * sizeof(float), cudaMemcpyDeviceToHost, st));
    HN_CUDA_OK(cudaMemcpyAsync(cor, m->cor_slot[slot], (size_t)B * 1024 * sizeof(float), cudaMemcpyDeviceToHost, st));
    // a device-side LSTM timeout of this batch is surfaced here (the flag is written before the outputs complete)
    int flag = 0;
    HN_CUDA_OK(cudaMemcpyAsync(&flag, m->error_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    HN_CUDA_OK(cudaStreamSynchronize(st));
    ++m->collect_count;
    if (flag) {
        cudaMemsetAsync(m->error_flag, 0, sizeof(int), st);
        cudaStreamSynchronize(st);
        return fail("hn_model: the persistent LSTM kernel timed out waiting for a peer CTA");
    }
    return 0;
}

// The views of P panoramas (view-major, as reference augment concatenates them), one forward, the per-panorama merge
static int infer_views(hn_model* m, const float* x, int P, int flip, const int* shifts, int n_rotate, float* y_bon_pix,
                       float* y_cor, cudaStream_t st, const char* who) {
    const std::string w(who);
    HN_CHECK(n_rotate >= 0 && n_rotate <= 32 && (n_rotate == 0 || shifts), w + ": bad rotate list");
    const int V = 1 + (flip ? 1 : 0) + n_rotate;
    HN_CHECK(P >= 1, w + ": no panoramas");
    HN_CHECK(V <= 64 && (long long)V * P <= m->max_batch, w + ": panoramas x views exceed max_batch");
    HN_CHECK(m->submit_count == m->collect_count, w + ": collect the submitted batches first");
    int host[128];
    int v = 0;
    host[v] = 0; host[64 + v] = 0; ++v;                         // aug_type '' (inference.py:34)
    if (flip) { host[v] = 1; host[64 + v] = 0; ++v; }           // 'flip' (:36-38)
    for (int i = 0; i < n_rotate; ++i, ++v) { host[v] = 2; host[64 + v] = shifts[i]; }   // 'rotate shift' (:39-42)
    HN_CUDA_OK(cudaMemcpyAsync(m->tta_ints, host, sizeof(host), cudaMemcpyHostToDevice, st));
    HN_CUDA_OK(cudaStreamSynchronize(st));                      // host[] is a stack array
    if (tta_views(x, m->x_slot[1], V, P, m->tta_ints, m->tta_ints + 64, st)) return -1;
    if (hn_model_forward(m, m->x_slot[1], V * P, 3, m->bon_out, m->cor_out, st)) return -1;
    return tta_merge(m->bon_out, m->cor_out, V, P, m->tta_ints, m->tta_ints + 64, y_bon_pix, y_cor, st);
}

int hn_model_infer_tta(hn_model* m, const float* x, int in_channels, int flip, const int* shifts, int n_rotate,
                       float* y_bon_pix, float* y_cor, void* stream) {
    HN_CHECK(m && x && y_bon_pix && y_cor, "hn_model_infer_tta: NULL argument");
    HN_CHECK(in_channels == 3, "hn_model_infer_tta: expects a 3-channel panorama (inference.py:196-200)");
    HN_ON_DEVICE(m->device);
    return infer_views(m, x, 1, flip, shifts, n_rotate, y_bon_pix, y_cor, (cudaStream_t)stream, "hn_model_infer_tta");
}

int hn_model_infer_layout(hn_model* m, const float* x, int B, int in_channels, int flip, const int* shifts, int n_rotate,
                          int r_px, float min_v, int force_cuboid, int force_raw, int max_rows, float* y_bon_pix,
                          float* y_cor, float* cor_id, int* n_rows, float* z0, float* z1, int* status, void* stream) {
    HN_CHECK(m && x && y_bon_pix && y_cor && cor_id && n_rows && z0 && z1 && status, "hn_model_infer_layout: NULL argument");
    HN_CHECK(in_channels == 3, "hn_model_infer_layout: expects 3-channel panoramas (inference.py:196-200)");
    HN_CHECK(r_px >= 1 && r_px <= 1024 && max_rows >= 0, "hn_model_infer_layout: bad r_px or max_rows");
    HN_ON_DEVICE(m->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (infer_views(m, x, B, flip, shifts, n_rotate, y_bon_pix, y_cor, st, "hn_model_infer_layout")) return -1;
    return layout_postproc(y_bon_pix, y_cor, B, r_px, min_v, force_cuboid, force_raw, max_rows, cor_id, n_rows, z0, z1,
                           status, nullptr, nullptr, st);
}

int hn_layout_postproc(const float* y_bon_pix, const float* y_cor, int B, int r_px, float min_v, int force_cuboid,
                       int force_raw, int max_rows, float* cor_id, int* n_rows, float* z0, float* z1, int* status,
                       int* peaks, int* n_peaks, void* stream) {
    HN_CHECK(y_bon_pix && y_cor && cor_id && n_rows && z0 && z1 && status, "hn_layout_postproc: NULL argument");
    HN_CHECK(B >= 1 && B <= 65535, "hn_layout_postproc: bad panorama count");
    HN_CHECK(r_px >= 1 && r_px <= 1024 && max_rows >= 0, "hn_layout_postproc: bad r_px or max_rows");
    return layout_postproc(y_bon_pix, y_cor, B, r_px, min_v, force_cuboid, force_raw, max_rows, cor_id, n_rows, z0, z1,
                           status, peaks, n_peaks, (cudaStream_t)stream);
}

int hn_model_validate(hn_model* m, const float* x, int B, int in_channels, const float* gt, const int* gt_rows,
                      int max_rows, double* iou2d, double* iou3d, double* rmse, double* delta_1, int* status,
                      void* stream) {
    HN_CHECK(m && x && gt && gt_rows && iou2d && iou3d && rmse && delta_1 && status, "hn_model_validate: NULL argument");
    HN_CHECK(in_channels == 3, "hn_model_validate: expects 3-channel panoramas (inference.py:196-200)");
    HN_CHECK(B >= 1 && B <= 65535 && max_rows >= 0 && max_rows <= 2048, "hn_model_validate: bad B or max_rows");
    HN_ON_DEVICE(m->device);
    cudaStream_t st = (cudaStream_t)stream;
    // inference(net, x, force_raw=True) without augmentation (train.py:306), its outputs kept on the device
    constexpr int R = 2048;
    const size_t nf = (size_t)B * (2 * 1024 + 1024 + R * 2 + 2);
    float* buf = nullptr;
    int* ibuf = nullptr;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&buf), nf * sizeof(float), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ibuf), (size_t)B * 2 * sizeof(int), st));
    float* y_bon = buf;
    float* y_cor = y_bon + (size_t)B * 2 * 1024;
    float* cor_id = y_cor + (size_t)B * 1024;
    float* z0 = cor_id + (size_t)B * R * 2;
    float* z1 = z0 + B;
    int rc = infer_views(m, x, B, 0, nullptr, 0, y_bon, y_cor, st, "hn_model_validate");
    if (!rc) rc = layout_postproc(y_bon, y_cor, B, 26, 0.05f, 0, 1, R, cor_id, ibuf, z0, z1, ibuf + B, nullptr, nullptr, st);
    // a failed inference is scored as train.py:309-313's fallback box (layout statuses 2..5)
    if (!rc) rc = layout_eval_general(cor_id, ibuf, ibuf + B, R, gt, gt_rows, max_rows, B, iou2d, iou3d, rmse, delta_1,
                                      status, nullptr, st);
    cudaFreeAsync(buf, st);
    cudaFreeAsync(ibuf, st);
    return rc;
}

int hn_layout_eval_general(const float* dt, const int* dt_rows, const int* dt_status, const float* gt, const int* gt_rows,
                           int B, int max_rows, double* iou2d, double* iou3d, double* rmse, double* delta_1, int* status,
                           float* depth_out, void* stream) {
    HN_CHECK(dt && dt_rows && gt && gt_rows && iou2d && iou3d && rmse && delta_1 && status,
             "hn_layout_eval_general: NULL argument");
    HN_CHECK(B >= 1 && B <= 65535, "hn_layout_eval_general: bad pair count");
    HN_CHECK(max_rows >= 0 && max_rows <= 2048, "hn_layout_eval_general: max_rows must be in 0..2048");
    return layout_eval_general(dt, dt_rows, dt_status, max_rows, gt, gt_rows, max_rows, B, iou2d, iou3d, rmse, delta_1,
                               status, depth_out, (cudaStream_t)stream);
}

int hn_layout_eval_cuboid(const float* dt, const int* dt_rows, const int* dt_status, const double* z0, const double* z1,
                          const float* gt, const int* gt_rows, int B, int max_rows, double* ce, double* pe, double* iou3d,
                          int* status, void* stream) {
    HN_CHECK(dt && dt_rows && z0 && z1 && gt && gt_rows && ce && pe && iou3d && status,
             "hn_layout_eval_cuboid: NULL argument");
    HN_CHECK(B >= 1 && B <= 65535, "hn_layout_eval_cuboid: bad pair count");
    HN_CHECK(max_rows >= 8 && max_rows <= 2048, "hn_layout_eval_cuboid: max_rows must be in 8..2048");
    return layout_eval_cuboid(dt, dt_rows, dt_status, max_rows, z0, z1, nullptr, nullptr, gt, gt_rows, max_rows, B, ce, pe,
                              iou3d, status, (cudaStream_t)stream);
}

int hn_train_targets(const float* cor0, const float* cor, const int* rows, const int* flip, const int* dx, int N, int max_rows,
                     double p_base, float* y_bon, float* y_cor, float* cor_out, int* occlusion, int* status, void* stream) {
    HN_CHECK(cor0 && cor && rows && flip && dx && y_bon && y_cor && status, "hn_train_targets: NULL argument");
    HN_CHECK(N >= 1 && N <= 65535, "hn_train_targets: bad sample count");
    HN_CHECK(max_rows >= 1 && max_rows <= 2048, "hn_train_targets: max_rows must be in 1..2048");
    HN_CHECK(p_base > 0 && p_base < 1, "hn_train_targets: p_base must be in (0, 1)");
    return train_targets(cor0, cor, rows, flip, dx, N, max_rows, p_base, y_bon, y_cor, cor_out, occlusion, status,
                         (cudaStream_t)stream);
}

int hn_model_eval_cuboid(hn_model* m, const float* x, int B, int in_channels, int flip, const int* shifts, int n_rotate,
                         int r_px, float min_v, const float* gt, const int* gt_rows, int max_rows, double* ce, double* pe,
                         double* iou3d, int* status, void* stream) {
    HN_CHECK(m && x && gt && gt_rows && ce && pe && iou3d && status, "hn_model_eval_cuboid: NULL argument");
    HN_CHECK(in_channels == 3, "hn_model_eval_cuboid: expects 3-channel panoramas (inference.py:196-200)");
    HN_CHECK(B >= 1 && B <= 65535 && max_rows >= 8 && max_rows <= 2048, "hn_model_eval_cuboid: bad B or max_rows");
    HN_CHECK(r_px >= 1 && r_px <= 1024, "hn_model_eval_cuboid: bad r_px");
    HN_ON_DEVICE(m->device);
    cudaStream_t st = (cudaStream_t)stream;
    // inference(net, x, flip, rotate, force_cuboid=True) (eval_cuboid's protocol), its outputs kept on the device
    constexpr int R = 8;
    const size_t nf = (size_t)B * (2 * 1024 + 1024 + R * 2 + 2);
    float* buf = nullptr;
    int* ibuf = nullptr;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&buf), nf * sizeof(float), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ibuf), (size_t)B * 2 * sizeof(int), st));
    float* y_bon = buf;
    float* y_cor = y_bon + (size_t)B * 2 * 1024;
    float* cor_id = y_cor + (size_t)B * 1024;
    float* z0 = cor_id + (size_t)B * R * 2;
    float* z1 = z0 + B;
    int rc = infer_views(m, x, B, flip, shifts, n_rotate, y_bon, y_cor, st, "hn_model_eval_cuboid");
    if (!rc) rc = layout_postproc(y_bon, y_cor, B, r_px, min_v, 1, 0, R, cor_id, ibuf, z0, z1, ibuf + B, nullptr, nullptr, st);
    // a failed inference has no cuboid to score (status HN_CUBOID_DT_FAILED)
    if (!rc) rc = layout_eval_cuboid(cor_id, ibuf, ibuf + B, R, nullptr, nullptr, z0, z1, gt, gt_rows, max_rows, B, ce, pe,
                                     iou3d, status, st);
    cudaFreeAsync(buf, st);
    cudaFreeAsync(ibuf, st);
    return rc;
}

int hn_model_stage(hn_model* m, const char* stage, float* out, long long capacity, int dims[4], void* stream) {
    HN_CHECK(m && stage && out && dims, "hn_model_stage: NULL argument");
    HN_CHECK(m->last_batch > 0, "hn_model_stage: no forward has run yet");
    HN_ON_DEVICE(m->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (m->rnn_inflight) HN_CUDA_OK(cudaStreamWaitEvent(st, m->ev_rnn_last, 0));
    const int B = m->last_batch;
    const std::string s(stage);
    for (int l = 0; l < 4; ++l)
        if (s == "layer" + std::to_string(l + 1)) {
            const int C = block_out_channels(m->blocks[l].back()), H = 128 >> l, W = 256 >> l;
            const size_t total = (size_t)B * C * H * W;
            HN_CHECK((long long)total <= capacity, "hn_model_stage: output buffer too small");
            const float* src = m->F[l];
            if (m->use_tc) {       // F[l] holds fp16 hi/lo planes: merge into X[0] (free after the forward)
                const size_t n = (size_t)B * H * (W + 2) * C;
                float* tmp = m->X[0];
                HN_CHECK(n <= m->x0_cap, "hn_model_stage: scratch buffer too small");
                if (merge_planes(reinterpret_cast<const unsigned short*>(m->F[l]), tmp, n, st)) return -1;
                src = tmp;
            }
            nhwc_to_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(src, out, B, H, W, C, 1);
            HN_LAUNCH_OK();
            dims[0] = B; dims[1] = C; dims[2] = H; dims[3] = W;
            return 0;
        }
    if (s == "stem") {           // conv1 + bn1 + relu (model.py:73-75), before the max-pool; S0 is fp32 on both paths
        const size_t n = (size_t)B * 64 * 256 * 512;
        HN_CHECK((long long)n <= capacity, "hn_model_stage: output buffer too small");
        nhwc_to_nchw_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(m->S0, out, B, 256, 512, 64, 1);
        HN_LAUNCH_OK();
        dims[0] = B; dims[1] = 64; dims[2] = 256; dims[3] = 512;
        return 0;
    }
    const size_t total = (size_t)256 * B * 1024;
    HN_CHECK((long long)total <= capacity, "hn_model_stage: output buffer too small");
    if (s == "feature") {
        const size_t n = (size_t)256 * B * m->c_last;
        const float* seq = m->SEQ;
        if (m->use_tc) {      // SEQ holds fp16 hi/lo planes; XP is dead after the forward and large enough
            if (merge_planes(reinterpret_cast<const unsigned short*>(m->SEQ), m->XP, n, st)) return -1;
            seq = m->XP;
        }
        seq_to_feature_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seq, out, 256, B, m->c_last);
        HN_LAUNCH_OK();
        dims[0] = B; dims[1] = m->c_last; dims[2] = 256; dims[3] = 0;
        return 0;
    }
    if (s == "mlp_hidden") {      // post-ReLU, pre-dropout hidden layer -> [B][256][512] (reference linear[1], model.py:272)
        if (m->use_rnn) return fail("hn_model_stage: 'mlp_hidden' exists only in the MLP-head model (use_rnn = 0)");
        const size_t nh = (size_t)256 * B * 512;
        rows_to_batch_major_kernel<<<(unsigned)((nh + 255) / 256), 256, 0, st>>>(m->HID, out, 256, B, 512);
        HN_LAUNCH_OK();
        dims[0] = B; dims[1] = 256; dims[2] = 512; dims[3] = 0;
        return 0;
    }
    if (s == "rnn_out") {
        if (!m->use_rnn) return fail("hn_model_stage: 'rnn_out' does not exist in the MLP-head model (use_rnn = 0)");
        HN_CUDA_OK(cudaMemcpyAsync(out, m->R2, total * sizeof(float), cudaMemcpyDeviceToDevice, st));
        dims[0] = 256; dims[1] = B; dims[2] = 1024; dims[3] = 0;
        return 0;
    }
    return fail("hn_model_stage: unknown stage '" + s + "'");
}

void hn_model_destroy(hn_model* m) { delete m; }

// ---- pano_stretch ------------------------------------------------------------------------------
static int pano_stretch_any(const void* img, void* out, int f64, int n, int h, int w, int c, const double* kx, const double* ky,
                            int order, void* stream, const char* who) {
    if (!(n >= 0 && h >= 1 && w >= 1)) return fail(std::string(who) + ": bad geometry");
    if (n == 0) return 0;
    if (!(img && out && kx && ky)) return fail(std::string(who) + ": NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(std::string(who) + ": no CUDA device -- libhorizonnet_b200 has no CPU path");
    for (int i = 0; i < n; ++i)
        if (!(kx[i] > 0 && ky[i] > 0)) return fail(std::string(who) + ": kx, ky must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    double* scratch = nullptr;
    const size_t nd = (size_t)2 * n + (size_t)4 * n * w + h;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&scratch), nd * sizeof(double), st));
    HN_CUDA_OK(cudaMemcpyAsync(scratch, kx, n * sizeof(double), cudaMemcpyHostToDevice, st));
    HN_CUDA_OK(cudaMemcpyAsync(scratch + n, ky, n * sizeof(double), cudaMemcpyHostToDevice, st));
    int rc = f64 ? pano_stretch_device_f64(static_cast<const double*>(img), static_cast<double*>(out), n, h, w, c, scratch,
                                           scratch + n, scratch + 2 * (size_t)n, order, st)
                 : pano_stretch_device(static_cast<const float*>(img), static_cast<float*>(out), n, h, w, c, scratch,
                                       scratch + n, scratch + 2 * (size_t)n, order, st);
    cudaFreeAsync(scratch, st);
    return rc;
}

static int pano_stretch_any_host(const void* img, void* out, int f64, int n, int h, int w, int c, const double* kx,
                                 const double* ky, int order, const char* who) {
    if (n == 0) return 0;
    if (!(img && out && kx && ky)) return fail(std::string(who) + ": NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(std::string(who) + ": no CUDA device -- libhorizonnet_b200 has no CPU path");
    const size_t bytes = (size_t)n * h * w * c * (f64 ? sizeof(double) : sizeof(float));
    void *d_in = nullptr, *d_out = nullptr;
    HN_CUDA_OK(cudaMalloc(&d_in, bytes));
    if (cudaMalloc(&d_out, bytes) != cudaSuccess) { cudaFree(d_in); return fail(std::string(who) + ": out of memory"); }
    int rc = 0;
    if (cudaMemcpy(d_in, img, bytes, cudaMemcpyHostToDevice) != cudaSuccess) rc = fail(std::string(who) + ": H2D failed");
    if (!rc) rc = pano_stretch_any(d_in, d_out, f64, n, h, w, c, kx, ky, order, nullptr, who);
    if (!rc && cudaMemcpy(out, d_out, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) rc = fail(std::string(who) + ": D2H failed");
    cudaFree(d_in);
    cudaFree(d_out);
    return rc;
}

int hn_pano_stretch(const float* img, float* out, int n, int h, int w, int c, const double* kx, const double* ky,
                    int order, void* stream) {
    return pano_stretch_any(img, out, 0, n, h, w, c, kx, ky, order, stream, "hn_pano_stretch");
}
int hn_pano_stretch_host(const float* img, float* out, int n, int h, int w, int c, const double* kx,
                         const double* ky, int order) {
    return pano_stretch_any_host(img, out, 0, n, h, w, c, kx, ky, order, "hn_pano_stretch_host");
}
int hn_pano_stretch_f64(const double* img, double* out, int n, int h, int w, int c, const double* kx, const double* ky,
                        int order, void* stream) {
    return pano_stretch_any(img, out, 1, n, h, w, c, kx, ky, order, stream, "hn_pano_stretch_f64");
}
int hn_pano_stretch_host_f64(const double* img, double* out, int n, int h, int w, int c, const double* kx,
                             const double* ky, int order) {
    return pano_stretch_any_host(img, out, 1, n, h, w, c, kx, ky, order, "hn_pano_stretch_host_f64");
}

// ---- training augmentation, image path (reference dataset.py:53, 69-105, 124) ----------------------
int hn_augment(const unsigned char* img, float* out, int n, int h, int w, const double* kx, const double* ky,
               const int* flip, const int* dx, const float* gamma, void* stream) {
    HN_CHECK(n >= 0 && h >= 1 && w >= 1, "hn_augment: bad geometry");
    if (n == 0) return 0;
    HN_CHECK(img && out, "hn_augment: NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail("hn_augment: no CUDA device -- libhorizonnet_b200 has no CPU path");
    std::vector<double> k((size_t)2 * n, 1.0);
    std::vector<int> prm((size_t)4 * n, 0);
    for (int i = 0; i < n; ++i) {
        const bool stretch = kx && ky && kx[i] > 0 && ky[i] > 0;
        if (kx && ky) HN_CHECK((kx[i] > 0) == (ky[i] > 0), "hn_augment: kx and ky must both be positive, or both <= 0 (no stretch)");
        if (stretch) { k[i] = kx[i]; k[(size_t)n + i] = ky[i]; }
        const int d = dx ? dx[i] : 0;
        HN_CHECK(d >= 0 && d < w, "hn_augment: dx must be in [0, W) (dataset.py:95 np.random.randint(W))");
        const float g = gamma ? gamma[i] : 0.f;
        prm[(size_t)4 * i + 0] = (flip && flip[i]) ? 1 : 0;
        prm[(size_t)4 * i + 1] = d;
        std::memcpy(&prm[(size_t)4 * i + 2], &g, sizeof(float));
        prm[(size_t)4 * i + 3] = stretch ? 1 : 0;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double* scratch = nullptr;
    const size_t nd = (size_t)2 * n + (size_t)4 * n * w + h + (size_t)2 * n + 2;     // kx, ky, tables, params (4 ints = 2 doubles)
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&scratch), nd * sizeof(double), st));
    double* tables = scratch + 2 * (size_t)n;
    int* prm_dev = reinterpret_cast<int*>(tables + (size_t)4 * n * w + h);
    int rc = 0;
    if (cudaMemcpyAsync(scratch, k.data(), (size_t)2 * n * sizeof(double), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(prm_dev, prm.data(), (size_t)4 * n * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess)
        rc = fail("hn_augment: parameter upload failed");
    // the host vectors are pageable: the runtime has staged them when cudaMemcpyAsync returns
    if (!rc) rc = augment_device(img, out, n, h, w, scratch, scratch + n, prm_dev, tables, st);
    cudaFreeAsync(scratch, st);
    return rc;
}

// ---- misc.pano_lsd_align.rotatePanorama (reference misc/pano_lsd_align.py:125-171) -------------------
int hn_rotate_panorama(const void* img, int in_is_f64, double* out, int n, int h, int w, int c, const double* rinv,
                       void* stream) {
    if (n == 0) return 0;
    HN_CHECK(img && out && rinv, "hn_rotate_panorama: NULL argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail("hn_rotate_panorama: no CUDA device -- libhorizonnet_b200 has no CPU path");
    return rotate_panorama_device(img, in_is_f64, out, n, h, w, c, rinv, (cudaStream_t)stream);
}

// ---- kernel-level entry points -----------------------------------------------------------------
int hn_conv2d(const float* in, int B, int H, int W, int Cin, int in_halo, const float* w, const float* scale,
              const float* shift, const float* residual, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
              int relu, float* out, int out_halo, int impl, void* stream) {
    HN_CHECK(in && w && scale && shift && out, "hn_conv2d: NULL argument");
    ConvDesc d;
    d.Cin = Cin; d.Cout = Cout; d.kh = kh; d.kw = kw; d.sh = sh; d.sw = sw; d.ph = ph; d.pw = pw; d.relu = relu;
    d.w = w; d.scale = scale; d.shift = shift;
    Act a = mk(const_cast<float*>(in), B, H, W, Cin, in_halo);
    const int Ho = (H + 2 * ph - kh) / sh + 1, Wo = (W + 2 * pw - kw) / sw + 1;
    Act o = mk(out, B, Ho, Wo, Cout, out_halo);
    if (impl == 1 || impl == 2) {
        if (!conv_tc_supported(d, a, o)) return fail("hn_conv2d: shape not supported by the tensor-core kernel");
        if (impl == 2 && residual) return fail("hn_conv2d: the fp32-output tensor-core epilogue takes no residual");
        return conv_tc(d, a, o, residual, impl == 2, (cudaStream_t)stream);
    }
    if (impl == 3) {              // the narrow height-reduction kernel, through split planes of in / out
        if (!conv_narrow_supported(d, a, o) || residual) return fail("hn_conv2d: shape not supported by the narrow kernel");
        cudaStream_t st = (cudaStream_t)stream;
        unsigned short *ip = nullptr, *op = nullptr;
        HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ip), a.numel() * 2 * sizeof(unsigned short), st));
        HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&op), o.numel() * 2 * sizeof(unsigned short), st));
        int rc = split_planes(in, ip, a.numel(), st) || conv_narrow_planes(d, a, ip, o, op, st) ||
                 merge_planes(op, out, o.numel(), st);
        cudaFreeAsync(ip, st); cudaFreeAsync(op, st);
        return rc ? -1 : 0;
    }
    HN_CHECK(impl == 0, "hn_conv2d: impl must be 0, 1, 2 or 3");
    return conv_f32(d, a, o, residual, (cudaStream_t)stream);
}

// Launch plan of the tensor-core convolution for one shape (no GPU work): the one conv_tc_planes launches with.
int hn_conv_tc_plan(int B, int H, int W, int Cin, int in_halo, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
                    int out_halo, int out_f32, int has_residual, int sms, int plan[18]) {
    HN_CHECK(plan, "hn_conv_tc_plan: NULL argument");
    HN_CHECK(B >= 1 && H >= 1 && W >= 1 && kh >= 1 && kw >= 1 && sh >= 1 && sw >= 1 && in_halo >= 0 && out_halo >= 0,
             "hn_conv_tc_plan: bad geometry");
    ConvDesc d;
    d.Cin = Cin; d.Cout = Cout; d.kh = kh; d.kw = kw; d.sh = sh; d.sw = sw; d.ph = ph; d.pw = pw;
    const Act a = mk(nullptr, B, H, W, Cin, in_halo);
    const Act o = mk(nullptr, B, (H + 2 * ph - kh) / sh + 1, (W + 2 * pw - kw) / sw + 1, Cout, out_halo);
    TcPlan p;
    if (conv_tc_plan(d, a, o, out_f32 != 0, has_residual != 0, sms, &p)) return -1;
    const int rowbox = p.mode == 1 && p.rows_per_tile > 1;
    const int v[18] = {p.gemm_kernel, p.BN, p.mode, p.M, p.tw, p.rows_per_tile, p.wsegs, rowbox, p.box_rows, p.box_imgs,
                       p.dxr, p.parity, p.num_kc, p.seg, p.pf, p.n_tiles, p.num_tiles, p.grid};
    memcpy(plan, v, sizeof(v));
    return 0;
}

// Tile plan of the fp32 CUDA-core convolution for one shape (no GPU work): the one conv_f32 launches with.
int hn_conv_f32_plan(int B, int H, int W, int Cin, int in_halo, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
                     int out_halo, int sms, int plan[4]) {
    HN_CHECK(plan, "hn_conv_f32_plan: NULL argument");
    HN_CHECK(B >= 1 && H >= 1 && W >= 1 && kh >= 1 && kw >= 1 && sh >= 1 && sw >= 1 && in_halo >= 0 && out_halo >= 0,
             "hn_conv_f32_plan: bad geometry");
    ConvDesc d;
    d.Cin = Cin; d.Cout = Cout; d.kh = kh; d.kw = kw; d.sh = sh; d.sw = sw; d.ph = ph; d.pw = pw;
    const Act a = mk(nullptr, B, H, W, Cin, in_halo);
    const Act o = mk(nullptr, B, (H + 2 * ph - kh) / sh + 1, (W + 2 * pw - kw) / sw + 1, Cout, out_halo);
    return conv_f32_plan(d, a, o, sms, plan);
}

int hn_conv_tc_fold_plan(int B, int H, int W, int Cin, int Cmid, int Cout, int stride, int sms, int plan[18]) {
    HN_CHECK(plan, "hn_conv_tc_fold_plan: NULL argument");
    HN_CHECK(B >= 1 && H >= 1 && W >= 1 && (stride == 1 || stride == 2) && H % stride == 0 && W % stride == 0,
             "hn_conv_tc_fold_plan: bad geometry");
    const Act x = mk(nullptr, B, H, W, Cin), t2 = mk(nullptr, B, H / stride, W / stride, Cmid);
    const Act o = mk(nullptr, B, H / stride, W / stride, Cout);
    TcPlan p;
    if (conv_tc_fold_plan(t2, x, stride, o, sms, &p)) return -1;
    const int v[18] = {p.gemm_kernel, p.BN, p.mode, p.M, p.tw, p.rows_per_tile, p.wsegs, p.rows_per_tile > 1, p.box_rows,
                       p.box_imgs, p.dxr, p.parity, p.num_kc, p.seg, p.pf, p.n_tiles, p.num_tiles, p.grid};
    memcpy(plan, v, sizeof(v));
    return 0;
}

int hn_conv_tc_fold(const float* t2, const float* x, int B, int H, int W, int Cin, int Cmid, int Cout, int stride,
                    const float* w, const float* shift, float* out, void* stream) {
    HN_CHECK(t2 && x && w && shift && out, "hn_conv_tc_fold: NULL argument");
    HN_CHECK(B >= 1 && H >= 1 && W >= 1 && (stride == 1 || stride == 2) && H % stride == 0 && W % stride == 0,
             "hn_conv_tc_fold: bad geometry");
    const Act xa = mk(const_cast<float*>(x), B, H, W, Cin);
    const Act ta = mk(const_cast<float*>(t2), B, H / stride, W / stride, Cmid);
    const Act oa = mk(out, B, H / stride, W / stride, Cout);
    return conv_tc_fold(w, shift, ta, xa, stride, oa, (cudaStream_t)stream);
}

int hn_bott_tc(const float* in, const float* res, const float* x, int B, int H, int W, const float* w2, const float* scale2,
               const float* shift2, const float* w3, const float* scale3, const float* shift3, int C3, float* out,
               void* stream) {
    HN_CHECK(in && w2 && scale2 && shift2 && w3 && shift3 && out && (!res || scale3), "hn_bott_tc: NULL argument");
    HN_CHECK(B >= 1 && H >= 1 && W >= 1 && C3 >= 64, "hn_bott_tc: bad geometry");
    return bott_tc_f32(w2, scale2, shift2, w3, res ? scale3 : nullptr, shift3, mk(const_cast<float*>(in), B, H, W, 64), res,
                       x, mk(out, B, H, W, C3), (cudaStream_t)stream);
}

int hn_lstm_layer(const float* xproj, const float* whf, const float* whb, float* out, int T, int B, void* stream) {
    HN_CHECK(xproj && whf && whb && out && T >= 1 && B >= 1, "hn_lstm_layer: bad argument");
    return lstm_layer(xproj, whf, whb, out, T, B, (cudaStream_t)stream);
}

// Launch layout of hn_lstm_layer (no GPU work unless max_clusters <= 0 asks the current device): the one lstm_layer takes.
int hn_lstm_plan(int T, int B, int max_clusters, int plan[7]) {
    HN_CHECK(plan, "hn_lstm_plan: NULL argument");
    return lstm_plan(T, B, max_clusters, plan);
}

// The stem as the model runs it: impl 0 = stem_f32 on the weights packed as pack_conv packs them; impl 1 = the weight
// planes and epilogue constants of stem_tc_pack_weights (as finalize makes them) and stem_tc.  relu = 0 with ones / zeros
// is the training step's raw pass: there tc_aux_update(ones, zeros) replaces the constants of weights packed with the BN
// scale, and the planes depend on the weights alone (their power of two), so packing with ones / zeros gives the same
// planes and the same constants.
int hn_stem(const float* x_nchw, int B, int in_channels, const float* w_oihw, const float* scale, const float* shift,
            int relu, int impl, float* out, void* stream) {
    HN_CHECK(x_nchw && w_oihw && scale && shift && out, "hn_stem: NULL argument");
    HN_CHECK(B >= 1 && B <= 2048 && in_channels >= 3, "hn_stem: bad geometry");
    HN_CHECK(impl == 0 || impl == 1, "hn_stem: impl must be 0 or 1");
    cudaStream_t st = (cudaStream_t)stream;
    const Act o = mk(out, B, 256, 512, 64);
    if (impl == 0) {
        float* wp = nullptr;
        HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&wp), 64 * 147 * sizeof(float), st));
        pack_oihw_kernel<<<(64 * 147 + 255) / 256, 256, 0, st>>>(w_oihw, wp, 64, 3, 7, 7);
        count_launch();
        int rc = cudaGetLastError() != cudaSuccess ? fail("hn_stem: weight packing failed") : 0;
        if (!rc) rc = stem_f32(x_nchw, B, in_channels, wp, scale, shift, o, st, relu != 0);
        cudaFreeAsync(wp, st);
        return rc;
    }
    // one scratch block: packed input planes | weight planes [2][64][224] | padded weights [64][224] | tc_aux [3*64+1]
    const size_t n_planes = stem_tc_scratch_bytes(B), n_wq = 2 * 64 * 224 * sizeof(unsigned short);
    const size_t n_pad = 64 * 224 * sizeof(float), n_aux = (3 * 64 + 1) * sizeof(float);
    uint8_t* scratch = nullptr;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&scratch), n_planes + n_wq + n_pad + n_aux, st));
    unsigned short* planes = reinterpret_cast<unsigned short*>(scratch);
    unsigned short* wq = reinterpret_cast<unsigned short*>(scratch + n_planes);
    float* pad = reinterpret_cast<float*>(scratch + n_planes + n_wq);
    float* aux = reinterpret_cast<float*>(scratch + n_planes + n_wq + n_pad);
    int rc = stem_tc_pack_weights(w_oihw, pad, wq, scale, shift, aux, st);
    if (!rc) rc = stem_tc(x_nchw, B, in_channels, wq, aux, shift, planes, o, st, relu != 0);
    cudaFreeAsync(scratch, st);
    return rc;
}

int hn_maxpool(const float* in, int B, int H, int W, int C, int out_planes, float* out, void* stream) {
    HN_CHECK(in && out && B >= 1 && H >= 1 && W >= 1 && C >= 4, "hn_maxpool: bad argument");
    return maxpool3x3s2(mk(const_cast<float*>(in), B, H, W, C), mk(out, B, (H - 1) / 2 + 1, (W - 1) / 2 + 1, C),
                        (cudaStream_t)stream, out_planes != 0);
}

int hn_maxpool_backward(const float* x, const float* dp, int B, int H, int W, int C, float* dx, void* stream) {
    HN_CHECK(x && dp && dx && B >= 1 && H >= 1 && W >= 1 && C >= 1, "hn_maxpool_backward: bad argument");
    return maxpool_bwd(mk(const_cast<float*>(x), B, H, W, C), mk(const_cast<float*>(dp), B, (H - 1) / 2 + 1, (W - 1) / 2 + 1, C),
                       dx, (cudaStream_t)stream);
}

namespace {
// The four height-reduction outputs of an encoder as build_graph makes them: C/8 channels of layer s at H = 8 >> s,
// W = 256 >> s (halo 1)
int ghc_outputs(const char* backbone, int B, float* const p[4], Act a[4]) {
    HN_CHECK(backbone && B >= 1, "feature sequence: bad argument");
    const Arch* arch = nullptr;
    for (const Arch& c : ARCHS)
        if (std::string(backbone) == c.name) arch = &c;
    HN_CHECK(arch, std::string("feature sequence: unknown backbone ") + backbone);
    for (int s = 0; s < 4; ++s) {
        HN_CHECK(p[s], "feature sequence: NULL argument");
        a[s] = mk(p[s], B, 8 >> s, 256 >> s, (64 << s) * arch->expansion / 8);
    }
    return 0;
}
}  // namespace

int hn_feature_sequence(const char* backbone, int B, const float* const ghc[4], int planes, float* seq, void* stream) {
    HN_CHECK(ghc && seq, "hn_feature_sequence: NULL argument");
    Act a[4];
    float* const p[4] = {const_cast<float*>(ghc[0]), const_cast<float*>(ghc[1]), const_cast<float*>(ghc[2]),
                         const_cast<float*>(ghc[3])};
    if (ghc_outputs(backbone, B, p, a)) return -1;
    return ghc_to_sequence(a, seq, (cudaStream_t)stream, planes != 0);
}

int hn_feature_sequence_backward(const char* backbone, int B, const float* dseq, float* const dghc[4], void* stream) {
    HN_CHECK(dseq && dghc, "hn_feature_sequence_backward: NULL argument");
    Act a[4];
    if (ghc_outputs(backbone, B, dghc, a)) return -1;
    return ghc_to_sequence_bwd(dseq, a, (cudaStream_t)stream);
}

int hn_linear_head(const float* rnn, const float* w, const float* b, float* bon, float* cor, int T, int B, int K,
                   void* stream) {
    HN_CHECK(rnn && w && b && bon && cor && T >= 1 && T <= 256 && B >= 1, "hn_linear_head: bad argument");
    return linear_head(rnn, w, b, bon, cor, T, B, K, (cudaStream_t)stream);
}

int hn_linear_head_backward(const float* dbon, const float* dcor, const float* rnn, const float* w, float* drnn, float* dw,
                            float* db, int T, int B, int K, void* stream) {
    HN_CHECK(dbon && dcor && rnn && w && drnn && dw && db && T >= 1 && T <= 256 && B >= 1,
             "hn_linear_head_backward: bad argument");
    return head_bwd(dbon, dcor, rnn, w, drnn, dw, db, T, B, K, (cudaStream_t)stream);
}

int hn_col_sum(const float* x, long long rows, int cols, float* out, void* stream) {
    HN_CHECK(x && out && rows >= 0 && cols >= 1, "hn_col_sum: bad argument");
    return col_sum(x, (size_t)rows, cols, out, (cudaStream_t)stream);
}

int hn_stem_input(const float* x_nchw, int in_channels, int B, float* out, void* stream) {
    HN_CHECK(x_nchw && out && in_channels >= 3 && B >= 1, "hn_stem_input: bad argument");
    return stem_input_nhwc(x_nchw, in_channels, out, B, (cudaStream_t)stream);
}

}  // extern "C"
