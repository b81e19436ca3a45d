// Training step of HorizonNet('resnet50' or 'resnet18', rnn): forward with a tape + backward (SURVEY 8 row f1; reference
// train.py:44-58 feed_forward and :272-281 loss.backward()).  The losses and the optimizer stay in PyTorch (they are
// elementwise on [B,3,1024] outputs and on the parameters): the boundary is an autograd.Function whose forward is
// hn_train_forward and whose backward hands d(bon), d(cor) to hn_train_backward and reads one gradient per
// parameter back with hn_model_get_grad (horizonnet_b200/model.py).
//
// Every convolution output z (pre-BN) and every activation y is kept in fp32 on a tape; one gradient buffer mirrors
// every y.  With the model option tensor_cores (default) the forward convolutions and their data gradients run on the
// tensor-core conv kernel (conv_tc.cu: fp16 hi/lo operand planes, fp32 result; a data gradient is the same kernel on the
// zero-dilated dz with flipped weights); the weight gradients of the convolutions with Cin, Cout multiples of 64 can run
// on the tensor-core weight-gradient kernel (wgrad_tc.cu, HN_WGRAD_TC); the other weight gradients, BatchNorm, LSTM BPTT and
// the rest are fp32 CUDA-core kernels (bwd_kernels.cu).  tensor_cores = 0: conv_f32.cu everywhere.  Not built: loss
// scaling, gradient all-reduce overlapped with the backward.
#include <cstdlib>
#include <cstring>
#include <memory>

#include "model.cuh"
#include "bwd_kernels.cuh"
#include "../../include/horizonnet_b200.h"

namespace hn {
namespace {

constexpr int T_STEPS = 256;

struct Bump {
    float* base = nullptr;
    size_t off = 0;
    float* take(size_t n) {
        float* p = base ? base + off : nullptr;
        off += (n + 63) / 64 * 64;
        return p;
    }
};

struct Unit {
    const ConvLayer* c = nullptr;
    ConvDesc d;            // geometry of c->d
    Act in, z, y;
    const float* res = nullptr;
    float* bn = nullptr;   // [4*C] scale, shift, mean(z), invstd
    bool train = false, relu = false, is_stem = false;
};

struct TrainState {
    int B = 0;
    bool sized = false, have_tape = false;
    size_t ysize = 0, zsize = 0, bnsize = 0;
    float *yarena = nullptr, *garena = nullptr, *zarena = nullptr, *bnarena = nullptr;
    size_t dz_max = 0, dil_max = 0, w_max = 0;
    float *dz_scratch = nullptr, *dil_scratch = nullptr, *wd_scratch = nullptr, *dw_scratch = nullptr;
    // tensor-core variant of the step (hn_model option tensor_cores): fp16 hi/lo planes of every activation (same
    // offsets as yarena), of the current dz / dilated dz, an fp32 landing buffer for data gradients, epilogue constants
    float *parena = nullptr, *pl_scratch = nullptr, *pl2_scratch = nullptr, *dtmp = nullptr, *aux_tmp = nullptr;
    size_t din_max = 0;
    float *ones = nullptr, *zeros = nullptr;
    double* sums = nullptr;
    float* stem_in = nullptr;
    float *seq = nullptr, *xp[2] = {nullptr, nullptr}, *r[2] = {nullptr, nullptr}, *rm[2] = {nullptr, nullptr};
    float *hprev = nullptr, *gates = nullptr, *cell = nullptr, *dgates = nullptr, *dc = nullptr;
    float *da = nullptr, *db = nullptr, *whh_t = nullptr;
    float *mh = nullptr, *mhd = nullptr;          // MLP head: hidden layer [T][B][512] after ReLU, and after dropout
    unsigned int* barrier = nullptr;
    std::vector<Unit> units;
    Act stem_y, pool_y, gout[4];
    TrainCtx ctx{};
    std::vector<float*> grads;           // per TensorSlot
    // phase boundaries of the last backward: start, head, lstm, tail, conv units, end
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    bool timed = false;
    std::vector<cudaEvent_t> uev;        // HN_TRAIN_PROF=1: 4 events per conv unit (start, BN backward, weight gradient, data gradient)
    bool units_timed = false;
    std::vector<void*> owned;            // batch-sized buffers (freed and laid out again when a larger batch arrives)
    template <typename T>
    int alloc_t(T** p, size_t n) {
        HN_CUDA_OK(cudaMalloc(reinterpret_cast<void**>(p), (n ? n : 1) * sizeof(T)));
        owned.push_back(*p);
        return 0;
    }
    void release() {
        for (void* q : owned) cudaFree(q);
        owned.clear();
        sized = false; have_tape = false;
    }
    ~TrainState() {
        release();
        for (auto e : ev) if (e) cudaEventDestroy(e);
        for (auto e : uev) if (e) cudaEventDestroy(e);
    }
};

TrainState* state_of(hn_model* m) {
    if (!m->train_state) m->train_state = std::shared_ptr<void>(new TrainState, [](void* p) { delete static_cast<TrainState*>(p); });
    return static_cast<TrainState*>(m->train_state.get());
}

float* grad_buffer(hn_model* m, TrainState* ts, const std::string& key) {
    const int i = m->index.at(key);
    if (ts->grads.size() != m->slots.size()) ts->grads.assign(m->slots.size(), nullptr);
    if (!ts->grads[i]) {
        float* p = nullptr;
        if (m->alloc_t(&p, (size_t)m->slots[i].numel)) return nullptr;
        ts->grads[i] = p;
    }
    return ts->grads[i];
}

unsigned short* planes_of(const TrainState* ts, const Act& y);

// conv + BatchNorm2d (+ identity, ReLU) with tape.  run = false: only lay the buffers out (sizing pass).
int unit_forward(hn_model* m, TrainState* ts, Bump& Y, Bump& Z, Bump& BN, const ConvLayer& c, const Act& in, const float* res,
                 const TrainCtx& tr, cudaStream_t st, bool run, Act* out) {
    Unit u;
    u.c = &c; u.d = c.d; u.in = in; u.res = res;
    u.train = tr.bn_train[c.bn_index] != 0;
    u.relu = c.d.relu != 0;
    const int Ho = in.H / c.d.sh, Wo = in.W / c.d.sw;
    u.z = mk(nullptr, in.B, Ho, Wo, c.d.Cout);
    u.y = u.z;
    u.z.p = Z.take(u.z.numel());
    u.y.p = Y.take(u.y.numel());
    u.bn = BN.take((size_t)4 * c.d.Cout);
    ts->dz_max = std::max(ts->dz_max, u.z.numel());
    // (the fp32 data gradient pads Cout to a multiple of 16, see walk_backward)
    if (c.d.sh != 1 || c.d.sw != 1) ts->dil_max = std::max(ts->dil_max, (size_t)in.B * in.H * in.Wp() * ((c.d.Cout + 15) / 16 * 16));
    ts->w_max = std::max(ts->w_max, (size_t)c.d.Cout * c.d.Cin * c.d.kh * c.d.kw);
    ts->din_max = std::max(ts->din_max, in.numel());
    if (run) {
        const float* bias = c.biaskey.empty() ? nullptr : m->T(c.biaskey);
        ConvDesc raw = c.d;                       // z = conv + bias, no BN, no ReLU
        raw.relu = 0; raw.scale = ts->ones; raw.shift = bias ? bias : ts->zeros;
        if (m->use_tc && c.wq && conv_tc_supported(raw, in, u.z)) {
            // tensor-core kernel, fp32 output: identity epilogue constants for this layer's weight-plane scale
            if (tc_aux_update(ts->ones, raw.shift, c.tc_scale + 3 * c.d.Cout, ts->aux_tmp, c.d.Cout, st)) return -1;
            if (conv_tc_planes(raw, c.wq, ts->aux_tmp, in, planes_of(ts, in), u.z, nullptr, u.z.p, nullptr, st)) return -1;
        } else if (conv_f32(raw, in, u.z, nullptr, st)) return -1;
        if (u.train && bn_batch_stats(u.z, false, ts->sums, st)) return -1;
        if (bn_finalize_full(ts->sums, (long long)in.B * Ho * Wo, m->T(c.bnprefix + ".weight"), m->T(c.bnprefix + ".bias"),
                             bias, const_cast<float*>(m->T(c.bnprefix + ".running_mean")),
                             const_cast<float*>(m->T(c.bnprefix + ".running_var")), tr.bn_factor[c.bn_index], u.train, u.bn,
                             c.d.Cout, st))
            return -1;
        if (bn_apply_fwd(u.z, u.bn, res, u.relu, u.y, m->use_tc ? planes_of(ts, u.y) : nullptr, st)) return -1;
    }
    ts->units.push_back(u);
    *out = u.y;
    return 0;
}

int walk_forward(hn_model* m, TrainState* ts, const float* x, int B, int in_channels, float* bon, float* cor,
                 const TrainCtx& tr, cudaStream_t st, bool run) {
    Bump Y, Z, BN;
    if (run) { Y.base = ts->yarena; Z.base = ts->zarena; BN.base = ts->bnarena; }
    ts->units.clear();
    // ---- stem (model.py:73-75) + max-pool (:76)
    {
        Unit u;
        u.c = &m->stem; u.d = m->stem.d; u.is_stem = true; u.relu = true;
        u.train = tr.bn_train[m->stem.bn_index] != 0;
        u.in = mk(ts->stem_in, B, 512, 1024, 3, 3);
        u.z = mk(nullptr, B, 256, 512, 64);
        u.y = u.z;
        u.z.p = Z.take(u.z.numel());
        u.y.p = Y.take(u.y.numel());
        u.bn = BN.take(4 * 64);
        ts->dz_max = std::max(ts->dz_max, u.z.numel());
        ts->w_max = std::max(ts->w_max, (size_t)64 * 3 * 49);
        if (run) {
            if (stem_input_nhwc(x, in_channels, ts->stem_in, B, st)) return -1;
            if (m->use_tc && m->stem_tc_on) {
                if (tc_aux_update(ts->ones, ts->zeros, m->stem_aux + 3 * 64, ts->aux_tmp, 64, st)) return -1;
                if (stem_tc(x, B, in_channels, m->stem_wq, ts->aux_tmp, ts->zeros, reinterpret_cast<unsigned short*>(m->X[0]),
                            u.z, st, false))
                    return -1;
            } else if (stem_f32(x, B, in_channels, m->stem.w, ts->ones, ts->zeros, u.z, st, false)) return -1;
            if (u.train && bn_batch_stats(u.z, false, ts->sums, st)) return -1;
            const std::string& p = m->stem.bnprefix;
            if (bn_finalize_full(ts->sums, (long long)B * 256 * 512, m->T(p + ".weight"), m->T(p + ".bias"), nullptr,
                                 const_cast<float*>(m->T(p + ".running_mean")), const_cast<float*>(m->T(p + ".running_var")),
                                 tr.bn_factor[m->stem.bn_index], u.train, u.bn, 64, st))
                return -1;
            if (bn_apply_fwd(u.z, u.bn, nullptr, true, u.y, nullptr, st)) return -1;
        }
        ts->units.push_back(u);
        ts->stem_y = u.y;
    }
    ts->pool_y = mk(Y.take((size_t)B * 128 * 258 * 64), B, 128, 256, 64);
    if (run && maxpool3x3s2(ts->stem_y, ts->pool_y, st, false)) return -1;
    if (run && m->use_tc && split_planes(ts->pool_y.p, planes_of(ts, ts->pool_y), ts->pool_y.numel(), st)) return -1;

    // ---- layer1..4 (model.py:78-81, torchvision Bottleneck v1.5 or BasicBlock)
    Act cur = ts->pool_y, feats[4];
    for (int l = 0; l < 4; ++l) {
        for (size_t b = 0; b < m->blocks[l].size(); ++b) {
            const hn_model::Block& blk = m->blocks[l][b];
            Act t1, t2, y, dsy;
            if (blk.kind == hn_model::BASIC) {       // units conv1, downsample, conv2 (+ identity: its gradient goes to idn)
                if (unit_forward(m, ts, Y, Z, BN, blk.c1, cur, nullptr, tr, st, run, &t1)) return -1;
                const float* idn = cur.p;
                if (blk.has_ds) {
                    if (unit_forward(m, ts, Y, Z, BN, blk.ds, cur, nullptr, tr, st, run, &dsy)) return -1;
                    idn = dsy.p;
                }
                if (unit_forward(m, ts, Y, Z, BN, blk.c2, t1, idn, tr, st, run, &y)) return -1;
                cur = y;
                continue;
            }
            if (unit_forward(m, ts, Y, Z, BN, blk.c1, cur, nullptr, tr, st, run, &t1)) return -1;
            const float* idn = cur.p;
            if (blk.has_ds) {
                if (unit_forward(m, ts, Y, Z, BN, blk.ds, cur, nullptr, tr, st, run, &dsy)) return -1;
                idn = dsy.p;
            }
            if (unit_forward(m, ts, Y, Z, BN, blk.c2, t1, nullptr, tr, st, run, &t2)) return -1;
            if (unit_forward(m, ts, Y, Z, BN, blk.c3, t2, idn, tr, st, run, &y)) return -1;
            cur = y;
        }
        feats[l] = cur;
    }
    // ---- height reduction (model.py:148-151)
    for (int s = 0; s < 4; ++s) {
        Act g = feats[s];
        for (int j = 0; j < 4; ++j)
            if (unit_forward(m, ts, Y, Z, BN, m->ghc[s][j], g, nullptr, tr, st, run, &g)) return -1;
        ts->gout[s] = g;
    }
    ts->ysize = Y.off; ts->zsize = Z.off; ts->bnsize = BN.off;
    if (!run) return 0;

    // ---- model.py:152-155, 175-178, 263: sequence; :264-266 bi-LSTM, dropouts, head
    if (ghc_to_sequence(ts->gout, ts->seq, st, false)) return -1;
    if (!m->use_rnn) {
        // model.py:270-275: MLP per row, layer 1 on the exact fp32 kernel; both hidden layers stay on the tape
        const size_t nh = (size_t)T_STEPS * B * 512;
        const Act a = mk(ts->seq, 1, 1, T_STEPS * B, m->c_last, 0);
        const Act h = mk(ts->mh, 1, 1, T_STEPS * B, 512, 0);
        if (conv_f32(m->mlp1.d, a, h, nullptr, st)) return -1;
        HN_CUDA_OK(cudaMemcpyAsync(ts->mhd, ts->mh, nh * sizeof(float), cudaMemcpyDeviceToDevice, st));
        // hn_model_stage("mlp_hidden") shows the hidden layer of the last forward, this one included
        HN_CUDA_OK(cudaMemcpyAsync(m->HID, ts->mh, nh * sizeof(float), cudaMemcpyDeviceToDevice, st));
        if (tr.head_p > 0.0 && (tr.mask[1] ? multiply_inplace(ts->mhd, tr.mask[1], nh, st)
                                           : dropout_inplace(ts->mhd, nh, tr.head_p, tr.seed, 1, false, st)))
            return -1;
        return linear_head(ts->mhd, m->head_w, m->head_b, bon, cor, T_STEPS, B, 512, st);
    }
    const size_t nseq = (size_t)T_STEPS * B * 1024;
    const float* lin = ts->seq;
    for (int layer = 0; layer < 2; ++layer) {
        Act a = mk(const_cast<float*>(lin), 1, 1, T_STEPS * B, m->xproj[layer].d.Cin, 0);
        Act xp = mk(ts->xp[layer], 1, 1, T_STEPS * B, 4096, 0);
        if (conv_f32(m->xproj[layer].d, a, xp, nullptr, st)) return -1;
        if (lstm_layer(ts->xp[layer], m->whh[layer][0], m->whh[layer][1], ts->r[layer], T_STEPS, B, st)) return -1;
        // the un-dropped outputs stay on the tape (the backward recomputes the gates from them); rm = what the next
        // consumer sees
        HN_CUDA_OK(cudaMemcpyAsync(ts->rm[layer], ts->r[layer], nseq * sizeof(float), cudaMemcpyDeviceToDevice, st));
        const double p = layer == 0 ? tr.rnn_p : tr.head_p;
        if (p > 0.0) {
            if (tr.mask[layer] ? multiply_inplace(ts->rm[layer], tr.mask[layer], nseq, st)
                               : dropout_inplace(ts->rm[layer], nseq, p, tr.seed, layer, false, st))
                return -1;
        }
        lin = ts->rm[layer];
    }
    return linear_head(ts->rm[1], m->head_w, m->head_b, bon, cor, T_STEPS, B, 1024, st);
}

int ensure_buffers(hn_model* m, TrainState* ts, int B, const TrainCtx& tr) {
    if (ts->sized && ts->B >= B) return 0;
    if (ts->sized) {                      // a larger batch than the buffers were laid out for
        HN_CUDA_OK(cudaDeviceSynchronize());
        ts->release();
    }
    ts->dz_max = ts->dil_max = ts->w_max = ts->din_max = 0;
    if (walk_forward(m, ts, nullptr, B, 3, nullptr, nullptr, tr, 0, false)) return -1;     // sizing pass
    if (ts->alloc_t(&ts->yarena, ts->ysize) || ts->alloc_t(&ts->garena, ts->ysize) || ts->alloc_t(&ts->zarena, ts->zsize) ||
        ts->alloc_t(&ts->bnarena, ts->bnsize))
        return -1;
    if (ts->alloc_t(&ts->dz_scratch, ts->dz_max) || ts->alloc_t(&ts->dil_scratch, ts->dil_max) ||
        ts->alloc_t(&ts->wd_scratch, ts->w_max) || ts->alloc_t(&ts->dw_scratch, ts->w_max))
        return -1;
    if (ts->alloc_t(&ts->parena, ts->ysize) || ts->alloc_t(&ts->pl_scratch, std::max(ts->dz_max, ts->dil_max)) ||
        ts->alloc_t(&ts->pl2_scratch, ts->dz_max) || ts->alloc_t(&ts->dtmp, ts->din_max) ||
        ts->alloc_t(&ts->aux_tmp, 3 * 4096 + 3))
        return -1;
    if (ts->alloc_t(&ts->ones, 4096) || ts->alloc_t(&ts->zeros, 4096) || ts->alloc_t(&ts->sums, 2 * 4096)) return -1;
    if (fill_f32(ts->ones, 4096, 1.f, 0) || fill_f32(ts->zeros, 4096, 0.f, 0)) return -1;
    if (ts->alloc_t(&ts->stem_in, (size_t)B * 512 * 1030 * 3)) return -1;
    const size_t rows = (size_t)T_STEPS * B;
    // da / db: gradients of the LSTM outputs (1024 wide) and of the sequence (c_last <= 1024)
    if (ts->alloc_t(&ts->seq, rows * m->c_last) || ts->alloc_t(&ts->da, rows * 1024) || ts->alloc_t(&ts->db, rows * 1024))
        return -1;
    if (!m->use_rnn) {
        if (ts->alloc_t(&ts->mh, rows * 512) || ts->alloc_t(&ts->mhd, rows * 512)) return -1;
        HN_CUDA_OK(cudaStreamSynchronize(0));
        ts->B = B;
        ts->sized = true;
        return 0;
    }
    for (int l = 0; l < 2; ++l)
        if (ts->alloc_t(&ts->xp[l], rows * 4096) || ts->alloc_t(&ts->r[l], rows * 1024) || ts->alloc_t(&ts->rm[l], rows * 1024))
            return -1;
    if (ts->alloc_t(&ts->hprev, 2 * rows * 512) || ts->alloc_t(&ts->gates, 2 * rows * 2048) ||
        ts->alloc_t(&ts->cell, 2 * rows * 512) || ts->alloc_t(&ts->dgates, 2 * rows * 2048) ||
        ts->alloc_t(&ts->dc, (size_t)2 * B * 512) || ts->alloc_t(&ts->whh_t, (size_t)2 * 512 * 2048) ||
        ts->alloc_t(&ts->barrier, 4))
        return -1;
    HN_CUDA_OK(cudaStreamSynchronize(0));
    ts->B = B;
    ts->sized = true;
    return 0;
}

unsigned short* planes_of(const TrainState* ts, const Act& y) {
    return reinterpret_cast<unsigned short*>(ts->parena + (y.p - ts->yarena));
}

Act grad_of(const TrainState* ts, const Act& y) {
    Act g = y;
    g.p = ts->garena + (y.p - ts->yarena);
    return g;
}

// ---- data gradient on the tensor cores: the transposed convolution as a stride-1 convolution of dz (zero-dilated for a
// strided conv) with the flipped weights, fp32 result added to din
struct DgradTc {
    ConvDesc t;               // the transposed convolution: Cin <-> Cout, padding kh-1-ph, kw-1-pw
    Act src;                  // its input: dz, or the dilated copy in din's geometry with Cout channels
    Act landing;              // its fp32 output, din's geometry
};

DgradTc dgrad_tc_geometry(const ConvDesc& d, const Act& dz, const Act& din, float* dil, float* landing) {
    DgradTc g;
    g.t.Cin = d.Cout; g.t.Cout = d.Cin; g.t.kh = d.kh; g.t.kw = d.kw;
    g.t.ph = d.kh - 1 - d.ph; g.t.pw = d.kw - 1 - d.pw;
    g.src = dz;
    if (d.sh != 1 || d.sw != 1) { g.src = din; g.src.C = d.Cout; g.src.p = dil; }
    g.landing = din; g.landing.p = landing;
    return g;
}

bool dgrad_tc_supported(const ConvDesc& d, const Act& dz, const Act& din) {
    const DgradTc g = dgrad_tc_geometry(d, dz, din, nullptr, nullptr);
    return conv_tc_supported(g.t, g.src, g.landing);
}

struct DgradScratch {
    float* dil;               // strided convs: din's pixels x Cout
    float* landing;           // din.numel()
    unsigned short* sp;       // planes of the (dilated) dz: 2 x its numel
    float* wflip;             // Cout*Cin*kh*kw
    unsigned short* wq;       // 2 x Cout*Cin*kh*kw
    float* aux;               // 3*Cin + 1 (epilogue constants, weight absmax)
    float* amax;              // 1: absmax of the (dilated) dz
    const float* zeros;       // Cin zeros: the epilogue shift
};

// din += dgrad(dz; w).  sp_is_dz: sp / amax already hold the planes of dz (a stride-1 unit whose weight gradient split them).
int dgrad_tc(const ConvDesc& d, const float* w_oihw, const Act& dz, const Act& din, const DgradScratch& s, bool sp_is_dz,
             cudaStream_t st) {
    DgradTc g = dgrad_tc_geometry(d, dz, din, s.dil, s.landing);
    g.t.shift = s.zeros;
    const bool strided = d.sh != 1 || d.sw != 1;
    if (strided && dilate_for_dgrad(dz, g.src, d.sh, d.sw, st)) return -1;
    if (!sp_is_dz && split_planes_pow2(g.src.p, s.sp, g.src.numel(), s.amax, st)) return -1;
    if (flip_oihw(w_oihw, s.wflip, d.Cout, d.Cin, d.kh, d.kw, st)) return -1;
    if (pack_weight_tc(s.wflip, s.wq, nullptr, nullptr, s.aux, s.aux + 3 * g.t.Cout, g.t.Cout, g.t.Cin, g.t.kh, g.t.kw, st))
        return -1;
    if (tc_aux_div_pow2(s.aux, g.t.Cout, s.amax, st)) return -1;      // planes of dz carry pow2_factor: divide it out
    if (conv_tc_planes(g.t, s.wq, s.aux, g.src, s.sp, g.landing, nullptr, g.landing.p, nullptr, st)) return -1;
    return add_inplace(din.p, g.landing.p, din.numel(), st);
}

#define GRAD(key) grad_buffer(m, ts, key)
// MLP head (model.py:238-243, :270-275): from the scatter back to d(sequence), left in *dseq
int mlp_backward(hn_model* m, TrainState* ts, const float* dbon, const float* dcor, cudaStream_t st, float** dseq) {
    const int B = ts->units.front().z.B;
    const size_t rows = (size_t)T_STEPS * B;
    const TrainCtx& tr = ts->ctx;
    const size_t nh = rows * 512;
    float* dh = ts->da;               // d(hidden), [rows][512]
    if (head_bwd(dbon, dcor, ts->mhd, m->T("linear.3.weight"), dh, GRAD("linear.3.weight"), GRAD("linear.3.bias"), T_STEPS,
                 B, 512, st))
        return -1;
    if (tr.head_p > 0.0 && (tr.mask[1] ? multiply_inplace(dh, tr.mask[1], nh, st)
                                       : dropout_inplace(dh, nh, tr.head_p, tr.seed, 1, false, st)))
        return -1;
    if (relu_bwd_inplace(dh, ts->mh, nh, st)) return -1;
    if (col_sum(dh, rows, 512, GRAD("linear.0.bias"), st)) return -1;
    // dW1 = dH^T SEQ: the weight gradient of a 1x1 "convolution" over the T*B rows, like W_ih of the LSTM
    const int CL = m->c_last;
    const Act xa = mk(ts->seq, 1, 1, (int)rows, CL, 0);
    const Act dg = mk(dh, 1, 1, (int)rows, 512, 0);
    ConvDesc wi; wi.Cin = CL; wi.Cout = 512;
    if (m->use_tc && wgrad_tc_on() && conv_wgrad_tc_supported(wi, xa, dg)) {
        unsigned short* xpl = reinterpret_cast<unsigned short*>(ts->pl_scratch);
        unsigned short* gpl = reinterpret_cast<unsigned short*>(ts->pl_scratch + rows * 1024);
        float* gmax = ts->aux_tmp + 3 * 4096 + 1;
        if (split_planes(ts->seq, xpl, rows * CL, st) || split_planes_pow2(dh, gpl, nh, gmax, st)) return -1;
        if (conv_wgrad_tc(wi, xa, xpl, dg, gpl, gmax, GRAD("linear.0.weight"), st)) return -1;
    } else if (conv_wgrad_f32(wi, xa, dg, GRAD("linear.0.weight"), st)) return -1;
    // d(sequence) = dH W1      (W1 [512][c_last] is already conv_f32's [K][N] packing)
    ConvDesc di; di.Cin = 512; di.Cout = CL; di.w = m->T("linear.0.weight"); di.scale = ts->ones; di.shift = ts->zeros;
    if (conv_f32(di, dg, mk(ts->db, 1, 1, (int)rows, CL, 0), nullptr, st)) return -1;
    *dseq = ts->db;
    HN_CUDA_OK(cudaEventRecord(ts->ev[1], st));
    HN_CUDA_OK(cudaEventRecord(ts->ev[2], st));          // no recurrence: the bi-LSTM phase is empty
    return 0;
}

// linear head and bi-LSTM BPTT: from the scatter back to d(sequence), left in *dseq
int rnn_backward(hn_model* m, TrainState* ts, const float* dbon, const float* dcor, cudaStream_t st, float** dseq) {
    const int B = ts->units.front().z.B;
    const size_t rows = (size_t)T_STEPS * B, nseq = rows * 1024;
    const TrainCtx& tr = ts->ctx;
    // ---- linear head (model.py:266) and its dropout (:265)
    float* dout = ts->da;
    float* dnext = ts->db;
    if (head_bwd(dbon, dcor, ts->rm[1], m->T("linear.weight"), dout, GRAD("linear.weight"), GRAD("linear.bias"), T_STEPS, B,
                 1024, st))
        return -1;
    if (tr.head_p > 0.0 && (tr.mask[1] ? multiply_inplace(dout, tr.mask[1], nseq, st)
                                       : dropout_inplace(dout, nseq, tr.head_p, tr.seed, 1, false, st)))
        return -1;
    HN_CUDA_OK(cudaEventRecord(ts->ev[1], st));
    // ---- bi-LSTM, layer 1 then layer 0 (model.py:264)
    for (int layer = 1; layer >= 0; --layer) {
        const std::string l = "_l" + std::to_string(layer);
        const float* X = layer == 0 ? ts->seq : ts->rm[0];
        const int K = m->xproj[layer].d.Cin;             // layer input width: c_last, then 1024
        if (lstm_gather(ts->r[layer], ts->xp[layer], ts->hprev, ts->gates, T_STEPS, B, st)) return -1;
        for (int dir = 0; dir < 2; ++dir) {
            // gate pre-activations of every step at once: XP + H_prev * W_hh^T
            if (transpose_f32(m->whh[layer][dir], ts->whh_t + (size_t)dir * 512 * 2048, 2048, 512, st)) return -1;
            ConvDesc g;
            g.Cin = 512; g.Cout = 2048; g.w = ts->whh_t + (size_t)dir * 512 * 2048; g.scale = ts->ones; g.shift = ts->zeros;
            Act a = mk(ts->hprev + dir * rows * 512, 1, 1, (int)rows, 512, 0);
            Act o = mk(ts->gates + dir * rows * 2048, 1, 1, (int)rows, 2048, 0);
            if (conv_f32(g, a, o, o.p, st)) return -1;
        }
        if (lstm_cell_scan(ts->gates, ts->cell, T_STEPS, B, st)) return -1;
        if (lstm_bwd_steps(dout, ts->gates, ts->cell, ts->whh_t, ts->whh_t + (size_t)512 * 2048, ts->dgates, ts->dc, T_STEPS, B,
                           ts->barrier, m->error_flag, st))
            return -1;
        // weight gradients = 1x1 "convolutions" over the T*B rows: dW_ih = dG^T X, dW_hh = dG^T H_prev
        const Act xa = mk(const_cast<float*>(X), 1, 1, (int)rows, K, 0);
        ConvDesc wi; wi.Cin = K; wi.Cout = 2048;
        ConvDesc wh; wh.Cin = 512; wh.Cout = 2048;
        const bool lstm_wg_tc = m->use_tc && wgrad_tc_on() &&
                                conv_wgrad_tc_supported(wi, xa, mk(ts->dgates, 1, 1, (int)rows, 2048, 0)) &&
                                conv_wgrad_tc_supported(wh, mk(ts->hprev, 1, 1, (int)rows, 512, 0), mk(ts->dgates, 1, 1, (int)rows, 2048, 0));
        // tensor-core kernel: planes of X, of this direction's H_prev and dG in the plane scratch (3584 floats' worth per row)
        unsigned short* xpl = reinterpret_cast<unsigned short*>(ts->pl_scratch);
        unsigned short* hpl = reinterpret_cast<unsigned short*>(ts->pl_scratch + rows * 1024);
        unsigned short* gpl = reinterpret_cast<unsigned short*>(ts->pl_scratch + rows * 1536);
        float* gmax = ts->aux_tmp + 3 * 4096 + 1;
        if (lstm_wg_tc && split_planes(X, xpl, rows * K, st)) return -1;
        for (int dir = 0; dir < 2; ++dir) {
            const std::string sfx = l + (dir ? "_reverse" : "");
            Act dg = mk(ts->dgates + dir * rows * 2048, 1, 1, (int)rows, 2048, 0);
            const Act ha = mk(ts->hprev + dir * rows * 512, 1, 1, (int)rows, 512, 0);
            if (lstm_wg_tc) {
                if (split_planes(ha.p, hpl, rows * 512, st) || split_planes_pow2(dg.p, gpl, rows * 2048, gmax, st)) return -1;
                if (conv_wgrad_tc(wi, xa, xpl, dg, gpl, gmax, GRAD("bi_rnn.weight_ih" + sfx), st)) return -1;
                if (conv_wgrad_tc(wh, ha, hpl, dg, gpl, gmax, GRAD("bi_rnn.weight_hh" + sfx), st)) return -1;
            } else {
                if (conv_wgrad_f32(wi, xa, dg, GRAD("bi_rnn.weight_ih" + sfx), st)) return -1;
                if (conv_wgrad_f32(wh, ha, dg, GRAD("bi_rnn.weight_hh" + sfx), st)) return -1;
            }
            float* bi = GRAD("bi_rnn.bias_ih" + sfx);
            if (col_sum(dg.p, rows, 2048, bi, st)) return -1;
            HN_CUDA_OK(cudaMemcpyAsync(GRAD("bi_rnn.bias_hh" + sfx), bi, 2048 * sizeof(float), cudaMemcpyDeviceToDevice, st));
            // d(layer input) (+)= dG * W_ih      (W_ih [2048][K] is already conv_f32's [K][N] packing)
            ConvDesc di; di.Cin = 2048; di.Cout = K; di.w = m->T("bi_rnn.weight_ih" + sfx); di.scale = ts->ones;
            di.shift = ts->zeros;
            Act dx = mk(dnext, 1, 1, (int)rows, K, 0);
            if (conv_f32(di, dg, dx, dir ? dnext : nullptr, st)) return -1;
        }
        if (layer == 1 && tr.rnn_p > 0.0 && (tr.mask[0] ? multiply_inplace(dnext, tr.mask[0], nseq, st)
                                                        : dropout_inplace(dnext, nseq, tr.rnn_p, tr.seed, 0, false, st)))
            return -1;
        std::swap(dout, dnext);
    }
    HN_CUDA_OK(cudaEventRecord(ts->ev[2], st));
    *dseq = dout;
    return 0;
}
#undef GRAD

int walk_backward(hn_model* m, TrainState* ts, const float* dbon, const float* dcor, cudaStream_t st) {
    for (auto& e : ts->ev) if (!e) HN_CUDA_OK(cudaEventCreate(&e));
    HN_CUDA_OK(cudaEventRecord(ts->ev[0], st));
    HN_CUDA_OK(cudaMemsetAsync(ts->garena, 0, ts->ysize * sizeof(float), st));
#define GRAD(key) grad_buffer(m, ts, key)
    float* dout = nullptr;
    if (m->use_rnn ? rnn_backward(m, ts, dbon, dcor, st, &dout) : mlp_backward(m, ts, dbon, dcor, st, &dout)) return -1;
    // dout = d(sequence) -> the four height-reduction outputs (model.py:152-155, 175-178, 263)
    Act dg[4];
    for (int s = 0; s < 4; ++s) dg[s] = grad_of(ts, ts->gout[s]);
    if (ghc_to_sequence_bwd(dout, dg, st)) return -1;
    HN_CUDA_OK(cudaEventRecord(ts->ev[3], st));

    // ---- conv units in reverse
    const bool prof = [] { const char* e = getenv("HN_TRAIN_PROF"); return e && atoi(e) != 0; }();
    if (prof && ts->uev.size() != 4 * ts->units.size()) {
        for (auto e : ts->uev) cudaEventDestroy(e);
        ts->uev.assign(4 * ts->units.size(), nullptr);
        for (auto& e : ts->uev) HN_CUDA_OK(cudaEventCreate(&e));
    }
    ts->units_timed = prof;
#define MARK(k) do { if (prof) HN_CUDA_OK(cudaEventRecord(ts->uev[4 * ui + (k)], st)); } while (0)
    for (size_t ui = ts->units.size(); ui-- > 0;) {
        const Unit& u = ts->units[ui];
        const ConvLayer& c = *u.c;
        MARK(0);
        if (u.is_stem && maxpool_bwd(ts->stem_y, grad_of(ts, ts->pool_y), grad_of(ts, ts->stem_y).p, st)) return -1;
        Act dz = u.z; dz.p = ts->dz_scratch;
        float* dres = nullptr;
        if (u.res) dres = ts->garena + (u.res - ts->yarena);
        if (bn_bwd(grad_of(ts, u.y), u.y, u.z, u.bn, u.train, u.relu, ts->sums, dz, dres, GRAD(c.bnprefix + ".weight"),
                   GRAD(c.bnprefix + ".bias"), c.biaskey.empty() ? nullptr : GRAD(c.biaskey), st))
            return -1;
        MARK(1);
        // planes of dz (gradients are tiny: power-of-two scaling around the split, see split_planes_pow2); a stride-1 unit
        // shares them between its weight gradient and its data gradient
        unsigned short* sp = reinterpret_cast<unsigned short*>(ts->pl_scratch);
        float* amax = ts->aux_tmp + 3 * 4096 + 1;
        const bool strided = u.d.sh != 1 || u.d.sw != 1;
        bool sp_is_dz = false;
        if (m->use_tc && !u.is_stem && wgrad_tc_on() && conv_wgrad_tc_supported(u.d, u.in, dz)) {
            unsigned short* zp = strided ? reinterpret_cast<unsigned short*>(ts->pl2_scratch) : sp;
            float* zmax = strided ? amax + 1 : amax;
            if (split_planes_pow2(dz.p, zp, dz.numel(), zmax, st)) return -1;
            if (conv_wgrad_tc(u.d, u.in, planes_of(ts, u.in), dz, zp, zmax, ts->dw_scratch, st)) return -1;
            sp_is_dz = !strided;
        } else if (conv_wgrad_f32(u.d, u.in, dz, ts->dw_scratch, st)) return -1;
        if (ohwi_to_oihw(ts->dw_scratch, GRAD(c.wkey), u.d.Cout, u.d.Cin, u.d.kh, u.d.kw, st)) return -1;
        MARK(2);
        if (u.is_stem) { MARK(3); continue; }                      // the image needs no gradient
        const Act din = grad_of(ts, u.in);
        if (m->use_tc && dgrad_tc_supported(u.d, dz, din)) {
            // tensor cores: planes of the (dilated) dz, flipped weights packed as planes, fp32 result added to the gradient
            const DgradScratch s = {ts->dil_scratch, ts->dtmp, sp, ts->dw_scratch,
                                    reinterpret_cast<unsigned short*>(ts->wd_scratch), ts->aux_tmp, amax, ts->zeros};
            if (dgrad_tc(u.d, m->T(c.wkey), dz, din, s, sp_is_dz, st)) return -1;
        } else if (u.d.Cout % 16 != 0) {
            // resnet18's ghc0.3 (16 -> 8): conv_dgrad_f32 takes Cout in steps of 16, so dz and the weights get zero channels
            // up to 16 (OIHW: the extra output channels are zero rows after the real ones).  dw_scratch and pl2_scratch are
            // free here: the weight gradient is already in its OIHW buffer and took the fp32 kernel
            ConvDesc dp = u.d;
            dp.Cout = (u.d.Cout + 15) / 16 * 16;
            Act dzp = dz;
            dzp.C = dp.Cout; dzp.p = ts->pl2_scratch;
            const size_t nw = (size_t)u.d.Cout * u.d.Cin * u.d.kh * u.d.kw, nwp = (size_t)dp.Cout * u.d.Cin * u.d.kh * u.d.kw;
            HN_CUDA_OK(cudaMemsetAsync(ts->dw_scratch, 0, nwp * sizeof(float), st));
            HN_CUDA_OK(cudaMemcpyAsync(ts->dw_scratch, m->T(c.wkey), nw * sizeof(float), cudaMemcpyDeviceToDevice, st));
            HN_CUDA_OK(cudaMemsetAsync(dzp.p, 0, dzp.numel() * sizeof(float), st));
            HN_CUDA_OK(cudaMemcpy2DAsync(dzp.p, dp.Cout * sizeof(float), dz.p, u.d.Cout * sizeof(float), u.d.Cout * sizeof(float),
                                         dz.numel() / u.d.Cout, cudaMemcpyDeviceToDevice, st));
            if (pack_dgrad_weight(ts->dw_scratch, ts->wd_scratch, dp.Cout, u.d.Cin, u.d.kh, u.d.kw, st)) return -1;
            if (conv_dgrad_f32(dp, ts->wd_scratch, dzp, din, true, ts->dil_scratch, ts->ones, ts->zeros, st)) return -1;
        } else {
            if (pack_dgrad_weight(m->T(c.wkey), ts->wd_scratch, u.d.Cout, u.d.Cin, u.d.kh, u.d.kw, st)) return -1;
            if (conv_dgrad_f32(u.d, ts->wd_scratch, dz, din, true, ts->dil_scratch, ts->ones, ts->zeros, st)) return -1;
        }
        MARK(3);
    }
#undef MARK
#undef GRAD
    HN_CUDA_OK(cudaEventRecord(ts->ev[4], st));
    ts->timed = true;
    return 0;
}

}  // namespace
}  // namespace hn

extern "C" {

int hn_train_forward(hn_model* m, const float* x, int B, int in_channels, float* bon, float* cor,
                     const unsigned char* bn_train, const double* bn_factor, int n_bn, unsigned long long seed,
                     double rnn_dropout, double head_dropout, const float* rnn_mask, const float* head_mask, void* stream) {
    HN_CHECK(m && x && bon && cor && bn_train && bn_factor, "hn_train_forward: NULL argument");
    HN_CHECK(m->finalized, "hn_train_forward: call hn_model_finalize after setting all tensors");
    HN_CHECK(B >= 1 && B <= m->max_batch && B <= 64, "hn_train_forward: batch exceeds max_batch (or 64)");
    HN_CHECK(in_channels >= 3 && n_bn == (int)m->bn_names.size(), "hn_train_forward: bad in_channels / n_bn");
    HN_CHECK(rnn_dropout >= 0.0 && rnn_dropout < 1.0 && head_dropout >= 0.0 && head_dropout < 1.0,
             "hn_train_forward: dropout probabilities must be in [0, 1)");
    HN_CHECK(m->use_rnn || (rnn_dropout == 0.0 && !rnn_mask),
             "hn_train_forward: the MLP head (use_rnn = 0) has no LSTM: rnn_dropout must be 0 and rnn_mask NULL");
    HN_ON_DEVICE(m->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (m->rnn_inflight) {
        HN_CUDA_OK(cudaStreamWaitEvent(st, m->ev_rnn_last, 0));
        m->rnn_inflight = false;
    }
    TrainState* ts = state_of(m);
    const TrainCtx tr{bn_train, bn_factor, seed, rnn_dropout, head_dropout, {rnn_mask, head_mask}};
    if (ensure_buffers(m, ts, B, tr)) return -1;
    ts->have_tape = false;
    if (walk_forward(m, ts, x, B, in_channels, bon, cor, tr, st, true)) return -1;
    ts->ctx = tr;                       // the backward needs seed / p / mask pointers (the caller keeps the masks alive)
    ts->ctx.bn_train = nullptr; ts->ctx.bn_factor = nullptr;
    ts->have_tape = true;
    for (int i = 0; i < n_bn; ++i) m->bn_stale = m->bn_stale || (bn_train[i] && bn_factor[i] >= 0.0);
    m->last_batch = B;
    return 0;
}

int hn_train_backward(hn_model* m, const float* dbon, const float* dcor, void* stream) {
    HN_CHECK(m && dbon && dcor, "hn_train_backward: NULL argument");
    TrainState* ts = state_of(m);
    HN_CHECK(ts->have_tape, "hn_train_backward: no tape -- call hn_train_forward first (one backward per forward)");
    HN_ON_DEVICE(m->device);
    ts->have_tape = false;
    return walk_backward(m, ts, dbon, dcor, (cudaStream_t)stream);
}

int hn_model_get_grad(hn_model* m, const char* key, float* out, long long numel, void* stream) {
    HN_CHECK(m && key && out, "hn_model_get_grad: NULL argument");
    auto it = m->index.find(key);
    if (it == m->index.end()) return fail(std::string("hn_model_get_grad: unknown key '") + key + "'");
    TrainState* ts = state_of(m);
    HN_CHECK(ts->grads.size() == m->slots.size() && ts->grads[it->second], "hn_model_get_grad: no gradient for this key yet");
    HN_CHECK(numel == m->slots[it->second].numel, "hn_model_get_grad: element count differs from the tensor's");
    HN_ON_DEVICE(m->device);
    HN_CUDA_OK(cudaMemcpyAsync(out, ts->grads[it->second], (size_t)numel * sizeof(float), cudaMemcpyDeviceToDevice,
                               (cudaStream_t)stream));
    return 0;
}

// Device time of the phases of the last hn_train_backward: ms[0] linear head, [1] bi-LSTM BPTT (both layers),
// [2] sequence -> height-reduction outputs, [3] the 69 conv units (BN backward + weight gradient + data gradient).
// MLP head: ms[0] is the whole MLP backward and ms[1] is 0.  Synchronises with the backward's stream.
int hn_train_profile(hn_model* m, double ms[4]) {
    HN_CHECK(m && ms, "hn_train_profile: NULL argument");
    TrainState* ts = state_of(m);
    HN_CHECK(ts->timed, "hn_train_profile: no backward has run");
    HN_ON_DEVICE(m->device);
    HN_CUDA_OK(cudaEventSynchronize(ts->ev[4]));
    for (int i = 0; i < 4; ++i) {
        float t = 0.f;
        HN_CUDA_OK(cudaEventElapsedTime(&t, ts->ev[i], ts->ev[i + 1]));
        ms[i] = (i == 1 && !m->use_rnn) ? 0.0 : t;          // the MLP head has no recurrence phase
    }
    return 0;
}

// With HN_TRAIN_PROF=1 set during the last hn_train_backward: the conv-unit phase split into ms[0] BatchNorm backward,
// ms[1] weight gradients (incl. the dz plane split of the tensor-core kernel and the OHWI -> OIHW pass), ms[2] data gradients,
// summed over the units.  Returns -1 when that backward was not profiled.
int hn_train_profile_units(hn_model* m, double ms[3]) {
    HN_CHECK(m && ms, "hn_train_profile_units: NULL argument");
    TrainState* ts = state_of(m);
    HN_CHECK(ts->timed && ts->units_timed && ts->uev.size() == 4 * ts->units.size(),
             "hn_train_profile_units: the last backward ran without HN_TRAIN_PROF=1");
    HN_ON_DEVICE(m->device);
    HN_CUDA_OK(cudaEventSynchronize(ts->ev[4]));
    ms[0] = ms[1] = ms[2] = 0.0;
    for (size_t ui = 0; ui < ts->units.size(); ++ui)
        for (int k = 0; k < 3; ++k) {
            float t = 0.f;
            HN_CUDA_OK(cudaEventElapsedTime(&t, ts->uev[4 * ui + k], ts->uev[4 * ui + k + 1]));
            ms[k] += t;
        }
    return 0;
}

// Tape inspection (debugging / tests): unit i of the last hn_train_forward; what = 0 activation y, 1 raw conv output z,
// 2 gradient of y (after hn_train_backward).  Copies the halo-1 NHWC buffer; dims = {B, H, W, C}.
int hn_train_debug_unit(hn_model* m, int i, int what, float* out, long long capacity, int dims[4], char* name, int name_cap,
                        void* stream) {
    HN_CHECK(m && out && dims, "hn_train_debug_unit: NULL argument");
    TrainState* ts = state_of(m);
    HN_CHECK(i >= 0 && i < (int)ts->units.size(), "hn_train_debug_unit: no such unit");
    const Unit& u = ts->units[i];
    const Act a = what == 1 ? u.z : (what == 2 ? grad_of(ts, u.y) : u.y);
    HN_CHECK((long long)a.numel() <= capacity, "hn_train_debug_unit: output buffer too small");
    dims[0] = a.B; dims[1] = a.H; dims[2] = a.W; dims[3] = a.C;
    if (name && name_cap > 0) { strncpy(name, u.c->bnprefix.c_str(), name_cap - 1); name[name_cap - 1] = 0; }
    HN_ON_DEVICE(m->device);
    HN_CUDA_OK(cudaMemcpyAsync(out, a.p, a.numel() * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return 0;
}

// ---- unit-test entry points (tests/test_gpu_parity.py compares them with torch.autograd) -------------------------------
int hn_conv2d_backward(const float* in, int B, int H, int W, int Cin, int in_halo, const float* w_oihw, const float* dz,
                       int Cout, int kh, int kw, int sh, int sw, int ph, int pw, float* din, float* dw_oihw, void* stream) {
    HN_CHECK(in && w_oihw && dz && dw_oihw, "hn_conv2d_backward: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    ConvDesc d;
    d.Cin = Cin; d.Cout = Cout; d.kh = kh; d.kw = kw; d.sh = sh; d.sw = sw; d.ph = ph; d.pw = pw;
    Act a = mk(const_cast<float*>(in), B, H, W, Cin, in_halo);
    const int Ho = (H + 2 * ph - kh) / sh + 1, Wo = (W + 2 * pw - kw) / sw + 1;
    Act z = mk(const_cast<float*>(dz), B, Ho, Wo, Cout, 1);
    const size_t nw = (size_t)Cout * Cin * kh * kw;
    float *tmp = nullptr, *ones = nullptr, *dil = nullptr;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&tmp), nw * sizeof(float), st));
    int rc = conv_wgrad_f32(d, a, z, tmp, st);
    if (!rc) rc = ohwi_to_oihw(tmp, dw_oihw, Cout, Cin, kh, kw, st);
    if (!rc && din) {
        Act di = mk(din, B, H, W, Cin, 1);
        HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ones), 2 * 4096 * sizeof(float), st));
        HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&dil), (size_t)B * H * (W + 2) * Cout * sizeof(float), st));
        rc = fill_f32(ones, 4096, 1.f, st) || fill_f32(ones + 4096, 4096, 0.f, st) ||
             pack_dgrad_weight(w_oihw, tmp, Cout, Cin, kh, kw, st) ||
             conv_dgrad_f32(d, tmp, z, di, false, dil, ones, ones + 4096, st);
        cudaFreeAsync(ones, st); cudaFreeAsync(dil, st);
    }
    cudaFreeAsync(tmp, st);
    return rc;
}

// Host-side plan of the tensor-core weight-gradient kernel for one convolution shape (halo-1 tensors; no GPU needed): plan[10] =
// tile columns, rows per tile, tiles per row, box rows, images per tile, pixel tiles, tiles per slice, slices, work items
// per slice, CTAs.  -1 for a shape the kernel does not take.
int hn_wgrad_tc_plan(int B, int H, int W, int Cin, int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int sms, int plan[10]) {
    HN_CHECK(plan, "hn_wgrad_tc_plan: NULL argument");
    ConvDesc d;
    d.Cin = Cin; d.Cout = Cout; d.kh = kh; d.kw = kw; d.sh = sh; d.sw = sw; d.ph = ph; d.pw = pw;
    HN_CHECK(B >= 1 && H >= 1 && W >= 1 && kh >= 1 && kw >= 1 && sh >= 1 && sw >= 1, "hn_wgrad_tc_plan: bad geometry");
    const Act a = mk(nullptr, B, H, W, Cin, 1);
    const Act z = mk(nullptr, B, (H + 2 * ph - kh) / sh + 1, (W + 2 * pw - kw) / sw + 1, Cout, 1);
    return conv_wgrad_tc_plan(d, a, z, sms, plan);
}

// 1 when the training step routes the weight gradients the tensor-core kernel supports through it (HN_WGRAD_TC or the built-in default)
int hn_wgrad_tc_enabled(void) { return wgrad_tc_on() ? 1 : 0; }

// Weight gradient on the tensor-core kernel (wgrad_tc.cu) from fp32 halo-1 NHWC tensors: splits both operands into planes
// (the training step has them already), runs conv_wgrad_tc, returns dW in OIHW.  Fails for shapes the kernel does not take.
int hn_conv2d_wgrad_tc(const float* in, int B, int H, int W, int Cin, const float* dz, int Cout, int kh, int kw, int sh,
                       int sw, int ph, int pw, float* dw_oihw, void* stream) {
    HN_CHECK(in && dz && dw_oihw, "hn_conv2d_wgrad_tc: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    ConvDesc d;
    d.Cin = Cin; d.Cout = Cout; d.kh = kh; d.kw = kw; d.sh = sh; d.sw = sw; d.ph = ph; d.pw = pw;
    Act a = mk(const_cast<float*>(in), B, H, W, Cin, 1);
    const int Ho = (H + 2 * ph - kh) / sh + 1, Wo = (W + 2 * pw - kw) / sw + 1;
    Act z = mk(const_cast<float*>(dz), B, Ho, Wo, Cout, 1);
    HN_CHECK(conv_wgrad_tc_supported(d, a, z), "hn_conv2d_wgrad_tc: shape not supported by the tensor-core weight-gradient kernel");
    const size_t nw = (size_t)Cout * Cin * kh * kw;
    float *tmp = nullptr, *amax = nullptr;
    unsigned short *ap = nullptr, *zp = nullptr;
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&tmp), nw * sizeof(float), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&amax), sizeof(float), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ap), a.numel() * 2 * sizeof(unsigned short), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&zp), z.numel() * 2 * sizeof(unsigned short), st));
    int rc = split_planes(a.p, ap, a.numel(), st) || split_planes_pow2(z.p, zp, z.numel(), amax, st) ||
             conv_wgrad_tc(d, a, ap, z, zp, amax, tmp, st) || ohwi_to_oihw(tmp, dw_oihw, Cout, Cin, kh, kw, st);
    cudaFreeAsync(tmp, st); cudaFreeAsync(amax, st); cudaFreeAsync(ap, st); cudaFreeAsync(zp, st);
    return rc;
}

// Data gradient on the tensor cores through the training step's own dgrad_tc, added to din; the scratch TrainState
// provides there is allocated here.  Fails for shapes the kernel does not take.
int hn_conv2d_dgrad_tc(int B, int H, int W, int Cin, const float* w_oihw, const float* dz, int Cout, int kh, int kw, int sh,
                       int sw, int ph, int pw, float* din, void* stream) {
    HN_CHECK(w_oihw && dz && din, "hn_conv2d_dgrad_tc: NULL argument");
    HN_CHECK(B >= 1 && H >= 1 && W >= 1 && kh >= 1 && kw >= 1 && sh >= 1 && sw >= 1, "hn_conv2d_dgrad_tc: bad geometry");
    cudaStream_t st = (cudaStream_t)stream;
    ConvDesc d;
    d.Cin = Cin; d.Cout = Cout; d.kh = kh; d.kw = kw; d.sh = sh; d.sw = sw; d.ph = ph; d.pw = pw;
    const int Ho = (H + 2 * ph - kh) / sh + 1, Wo = (W + 2 * pw - kw) / sw + 1;
    const Act z = mk(const_cast<float*>(dz), B, Ho, Wo, Cout, 1);
    const Act di = mk(din, B, H, W, Cin, 1);
    HN_CHECK(dgrad_tc_supported(d, z, di), "hn_conv2d_dgrad_tc: shape not supported by the tensor-core kernel");
    const bool strided = sh != 1 || sw != 1;
    const size_t nw = (size_t)Cout * Cin * kh * kw, ndil = strided ? (size_t)B * H * (W + 2) * Cout : 0;
    const size_t nsrc = strided ? ndil : z.numel();
    float *dil = nullptr, *landing = nullptr, *wflip = nullptr, *aux = nullptr, *zeros = nullptr;
    unsigned short *sp = nullptr, *wq = nullptr;
    if (strided) HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&dil), ndil * sizeof(float), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&landing), di.numel() * sizeof(float), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&sp), nsrc * 2 * sizeof(unsigned short), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&wflip), nw * sizeof(float), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&wq), nw * 2 * sizeof(unsigned short), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&aux), (3 * (size_t)Cin + 2) * sizeof(float), st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&zeros), (size_t)Cin * sizeof(float), st));
    const DgradScratch s = {dil, landing, sp, wflip, wq, aux, aux + 3 * Cin + 1, zeros};
    int rc = fill_f32(zeros, Cin, 0.f, st);
    if (!rc) rc = dgrad_tc(d, w_oihw, z, di, s, false, st);
    if (dil) cudaFreeAsync(dil, st);
    cudaFreeAsync(landing, st); cudaFreeAsync(sp, st); cudaFreeAsync(wflip, st); cudaFreeAsync(wq, st);
    cudaFreeAsync(aux, st); cudaFreeAsync(zeros, st);
    return rc;
}

// BatchNorm2d (+ identity, ReLU) forward and backward on halo-1 NHWC tensors; bn_scratch: 4*C floats, sums: 3*C doubles
int hn_bn_forward_backward(const float* z, int B, int H, int W, int C, const float* gamma, const float* beta,
                           float* running_mean, float* running_var, double factor, int train, int relu, const float* res,
                           float* y, const float* dy, float* dz, float* dres, float* dgamma, float* dbeta, float* bn_scratch,
                           double* sums, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    Act za = mk(const_cast<float*>(z), B, H, W, C), ya = mk(y, B, H, W, C);
    if (train && bn_batch_stats(za, false, sums, st)) return -1;
    if (bn_finalize_full(sums, (long long)B * H * W, gamma, beta, nullptr, running_mean, running_var, factor, train != 0,
                         bn_scratch, C, st))
        return -1;
    if (bn_apply_fwd(za, bn_scratch, res, relu != 0, ya, nullptr, st)) return -1;
    return bn_bwd(mk(const_cast<float*>(dy), B, H, W, C), ya, za, bn_scratch, train != 0, relu != 0, sums, mk(dz, B, H, W, C),
                  dres, dgamma, dbeta, nullptr, st);
}

// One bidirectional LSTM layer backward from its saved forward tensors: xp [T][B][4096] (input projection + biases),
// hout [T][B][1024], dout [T][B][1024] -> dgates [2][T][B][2048] (= d xp, per direction).  Scratch layout: see the header.
int hn_lstm_layer_backward(const float* xp, const float* hout, const float* whf, const float* whb, const float* dout, int T,
                           int B, int persistent, float* dgates, float* scratch, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const size_t rows = (size_t)T * B;
    float* hprev = scratch;                         // 2*rows*512
    float* gates = hprev + 2 * rows * 512;          // 2*rows*2048
    float* cell = gates + 2 * rows * 2048;          // 2*rows*512
    float* dc = cell + 2 * rows * 512;              // 2*B*512
    float* wt = dc + (size_t)2 * B * 512;           // 2*512*2048
    float* ones = wt + (size_t)2 * 512 * 2048;      // 4096 + 4096
    unsigned int* barrier = reinterpret_cast<unsigned int*>(ones + 8192);
    int* error_flag = reinterpret_cast<int*>(ones + 8193);
    if (persistent) {
        bool fits = false;
        if (lstm_bwd_persistent_fits(B, &fits)) return -1;
        HN_CHECK(fits, "hn_lstm_layer_backward: cooperative BPTT kernel not supported on this device (its 128 CTAs cannot be "
                       "co-resident)");
        HN_CUDA_OK(cudaMemsetAsync(error_flag, 0, sizeof(int), st));
    }
    if (fill_f32(ones, 4096, 1.f, st) || fill_f32(ones + 4096, 4096, 0.f, st)) return -1;
    if (lstm_gather(hout, xp, hprev, gates, T, B, st)) return -1;
    for (int dir = 0; dir < 2; ++dir) {
        if (transpose_f32(dir ? whb : whf, wt + (size_t)dir * 512 * 2048, 2048, 512, st)) return -1;
        ConvDesc g;
        g.Cin = 512; g.Cout = 2048; g.w = wt + (size_t)dir * 512 * 2048; g.scale = ones; g.shift = ones + 4096;
        Act a = mk(hprev + dir * rows * 512, 1, 1, (int)rows, 512, 0);
        Act o = mk(gates + dir * rows * 2048, 1, 1, (int)rows, 2048, 0);
        if (conv_f32(g, a, o, o.p, st)) return -1;
    }
    if (lstm_cell_scan(gates, cell, T, B, st)) return -1;
    // persistent: the cooperative kernel the training step launches (checked above to fit, so lstm_bwd_steps takes it)
    return lstm_bwd_steps(dout, gates, cell, wt, wt + (size_t)512 * 2048, dgates, dc, T, B, persistent ? barrier : nullptr,
                          persistent ? error_flag : nullptr, st);
}

}  // extern "C"
