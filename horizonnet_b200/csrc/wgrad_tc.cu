// Tensor-core (wgmma) weight gradient of a convolution (training step, SURVEY 8 row f1; reference train.py:278
// `loss.backward()` through every nn.Conv2d of model.py:73-81, 129):
//     dW[co][dy][dx][ci] = sum over output pixels (b, ho, wo) of  dz[b][ho][wo][co] * in[b][ho*sh - ph + dy][wo*sw - pw + dx][ci]
// i.e. a GEMM  D[Cout x Cin] = dz^T * in_shifted  per filter tap whose reduction dimension is the PIXEL axis.  Both
// operands are halo-NHWC split planes (fp16 hi / lo of the 2^-4-scaled value, conv_tc.cuh; dz additionally scaled by a
// power of two, split_planes_pow2), so a TMA box of {64 channels, pixels} lands in shared memory as 128-byte rows, one
// per pixel: exactly the forward kernel's activation tile.  Read as an **MN-major** wgmma operand (transpose flags set;
// canonical 128B-swizzle layout: 128 B of channels contiguous, 8 pixel rows per swizzle atom, SBO = 1024 B between
// 8-pixel groups, LBO = the distance between two 64-channel atoms) the same tile is the [channels x pixels] operand the
// weight gradient needs -- no transposed copy of any activation is ever made.
//
// One CTA = one work item (128 output channels x <=128 input channels x one tap x one slice of the pixel axis):
//   warp 0     TMA producer: per 64-pixel K tile the dz atoms (hi, lo) and the tap-shifted input atoms (hi, lo); the
//              pixel tile is {tw columns, rows, images} like the forward kernel's row boxes (zero H padding = TMA
//              out-of-bounds fill, circular W padding = the halo column, stride 2 along H = TMA traversal stride,
//              stride 2 along W = the parity view); 3-stage mbarrier ring of 64 KB stages
//   warps 4-11 two consumer warpgroups, warpgroup g = output channels [64g, 64g + 64) of the tile: 4 K-steps of 16
//              pixels x 3 products per tile (hi*hi -> main accumulator; hi*lo, lo*hi -> cross accumulator, both in
//              registers), then main + cross, power-of-two rescale and fp32 reductions (red.global.add.v2) into
//              dW[Cout][taps][Cin] (several pixel slices and the CTAs of different images add into the same tile)
#include <cuda.h>
#include <cstring>

#include "hn_common.cuh"
#include "conv_tc.cuh"
#include "ptx.cuh"
#include "tc_common.cuh"
#include "bwd_kernels.cuh"

namespace hn {

namespace {

using namespace tc;

constexpr int KT = 64;                    // pixels per pipeline stage (the GEMM's K dimension)
constexpr int ATOM = KT * 128;            // one operand atom: 64 pixels x 64 fp16 channels = 8 KB
constexpr int PLANE = 2 * ATOM;           // up to two 64-channel atoms per operand plane
constexpr int STAGE = 4 * PLANE;          // dz hi, dz lo, in hi, in lo = 64 KB
constexpr int NST = 3;
constexpr int BAR_OFF = NST * STAGE;
constexpr int SMEM_TOTAL = BAR_OFF + 256 + 1024;       // barriers + alignment slack
constexpr int CONS_WARP0 = 4;
constexpr int CONS_WARPS = 8;

struct WgArgs {
    float* dw;                // [Cout][taps][Cin], accumulated
    const float* absmax;      // of dz: its planes hold dz * pow2_factor(*absmax) * 2^-4
    int Cout, Cin, taps, kw;
    int n_tiles;              // 128-channel tiles along Cin (the 128-channel tiles along Cout come from the grid size)
    int tw, rpt, wsegs, Ho;   // K tile = rpt output rows x tw columns (rows of one image, or rpt / Ho whole images)
    int out_halo;
    int sh, ph, woff, parity; // woff = in_halo - pw; parity = 1: stride 2 along W through the [Wp/2][2] view
    int num_kt, kt_per_slice, items_per_slice;
};

__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// the 12 wgmma of one 64-pixel K tile for N = 64 * n_atoms input channels; both operands MN-major
template <int R>
__device__ __forceinline__ void tile_mma(float (&mn)[R], float (&cr)[R], uint64_t z_hi, uint64_t z_lo, uint64_t i_hi,
                                         uint64_t i_lo, bool fresh) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KT / 16; ++k) {
        const uint64_t ko = (uint64_t)((k * 16 * 128) >> 4);     // 16 pixel rows of 128 B further on
        const uint32_t acc = (fresh && k == 0) ? 0u : 1u;        // the slice's first K-step overwrites
        wgmma_f16<1, 1>(mn, z_hi + ko, i_hi + ko, acc);
        wgmma_f16<1, 1>(cr, z_hi + ko, i_lo + ko, acc);
        wgmma_f16<1, 1>(cr, z_lo + ko, i_hi + ko, 1u);
    }
    wgmma_commit();
    wgmma_wait0();
    reg_fence(mn);
    reg_fence(cr);
}

// consumer warpgroup: K tiles [kt0, kt1) of the ring, then the reduction of its 64 x 64*NA block into dW
template <int NA>
__device__ __forceinline__ void wgrad_consume(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, const WgArgs& a,
                                              bool active, int wg, int kt0, int kt1, int co0, int ci0, int tap, int m_atoms) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float mn[32 * NA], cr[32 * NA];
    int stage = 0;
    uint32_t phase = 0;
    for (int kt = kt0; kt < kt1; ++kt) {
        mbar_wait(full_bar + stage, phase);
        if (active) {
            const uint32_t sZ = smem_u32(smem + stage * STAGE) + wg * ATOM;     // this warpgroup's 64 output channels
            const uint32_t sI = smem_u32(smem + stage * STAGE) + 2 * PLANE;
            tile_mma(mn, cr, gmma_desc_sw128(sZ, ATOM, 1024), gmma_desc_sw128(sZ + PLANE, ATOM, 1024),
                     gmma_desc_sw128(sI, ATOM, 1024), gmma_desc_sw128(sI + PLANE, ATOM, 1024), kt == kt0);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar + stage);          // the smem stage is free again
        if (++stage == NST) { stage = 0; phase ^= 1; }
    }
    if (!active || kt1 <= kt0) return;
    const float factor = 256.f / pow2_factor(__ldg(a.absmax));     // both operands carry 2^-4; dz also the power of two
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);       // output channel of the tile (and row + 8)
    (void)m_atoms;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float* drow = a.dw + ((size_t)(co0 + row + 8 * h) * a.taps + tap) * a.Cin + ci0 + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 8 * NA; ++j)
            red_add_v2(drow + 8 * j, (mn[4 * j + 2 * h] + cr[4 * j + 2 * h]) * factor,
                       (mn[4 * j + 2 * h + 1] + cr[4 * j + 2 * h + 1]) * factor);
    }
}

__global__ void __launch_bounds__(NTHREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmZh, const __grid_constant__ CUtensorMap tmZl,
                const __grid_constant__ CUtensorMap tmIh, const __grid_constant__ CUtensorMap tmIl, const WgArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + BAR_OFF);
    uint64_t* empty_bar = full_bar + NST;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // ---- which work item is this CTA's?  Items of one pixel slice are adjacent in the grid: they share their operand
    // tiles through L2.
    const int slice = (int)blockIdx.x / a.items_per_slice;
    int rem = (int)blockIdx.x - slice * a.items_per_slice;
    const int tap = rem % a.taps;
    rem /= a.taps;
    const int nt = rem % a.n_tiles, mt = rem / a.n_tiles;
    const int co0 = mt * 128, ci0 = nt * 128;
    const int m_atoms = min(2, (a.Cout - co0) / 64), n_atoms = min(2, (a.Cin - ci0) / 64);
    const int kt0 = slice * a.kt_per_slice, kt1 = min(a.num_kt, kt0 + a.kt_per_slice);
    const int dy = tap / a.kw, dx = tap - dy * a.kw;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmZh)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmZl)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmIh)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmIl)) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < NST; ++i) { mbar_init(full_bar + i, 1); mbar_init(empty_bar + i, CONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            const uint32_t bytes = (uint32_t)(2 * (m_atoms + n_atoms) * ATOM);
            for (int kt = kt0; kt < kt1; ++kt) {
                const int rg = kt / a.wsegs;
                const int wo0 = (kt - rg * a.wsegs) * a.tw;
                const int row0 = rg * a.rpt;
                const int b = row0 / a.Ho, ho = row0 - b * a.Ho;
                const int hin = ho * a.sh + dy - a.ph;
                mbar_wait(empty_bar + stage, phase ^ 1);
                uint8_t* sZ = smem + stage * STAGE;
                uint8_t* sI = sZ + 2 * PLANE;
                mbar_expect_tx(full_bar + stage, bytes);
                for (int j = 0; j < m_atoms; ++j) {
                    tma_load_4d(sZ + j * ATOM, &tmZh, full_bar + stage, co0 + 64 * j, wo0 + a.out_halo, ho, b);
                    tma_load_4d(sZ + PLANE + j * ATOM, &tmZl, full_bar + stage, co0 + 64 * j, wo0 + a.out_halo, ho, b);
                }
                for (int j = 0; j < n_atoms; ++j) {
                    if (a.parity) {
                        const int p = dx + a.woff;
                        tma_load_5d(sI + j * ATOM, &tmIh, full_bar + stage, ci0 + 64 * j, p & 1, wo0 + (p >> 1), hin, b);
                        tma_load_5d(sI + PLANE + j * ATOM, &tmIl, full_bar + stage, ci0 + 64 * j, p & 1, wo0 + (p >> 1), hin, b);
                    } else {
                        tma_load_4d(sI + j * ATOM, &tmIh, full_bar + stage, ci0 + 64 * j, wo0 + dx + a.woff, hin, b);
                        tma_load_4d(sI + PLANE + j * ATOM, &tmIl, full_bar + stage, ci0 + 64 * j, wo0 + dx + a.woff, hin, b);
                    }
                }
                if (++stage == NST) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp >= CONS_WARP0) {
        // =============================== consumers ===============================
        const int wg = (warp - CONS_WARP0) >> 2;
        const bool active = wg < m_atoms;
        if (n_atoms == 2) wgrad_consume<2>(smem, full_bar, empty_bar, a, active, wg, kt0, kt1, co0, ci0, tap, m_atoms);
        else wgrad_consume<1>(smem, full_bar, empty_bar, a, active, wg, kt0, kt1, co0, ci0, tap, m_atoms);
    }
}

struct Geometry {
    int tw, rpt, wsegs, box_rows, imgs;
    long long num_kt;
};

// pixel tiling of the output (= dz) geometry: 64 pixels per tile as {tw columns, box_rows rows, imgs images}
bool tile_geometry(const Act& dz, Geometry* g) {
    const int tw = dz.W < KT ? dz.W : KT;
    if (tw < 8 || (tw & (tw - 1)) != 0 || dz.W % tw != 0) return false;
    const int rpt = KT / tw;
    g->tw = tw; g->rpt = rpt; g->wsegs = dz.W / tw;
    if (dz.H % rpt == 0) { g->box_rows = rpt; g->imgs = 1; }
    else if (rpt % dz.H == 0) { g->box_rows = dz.H; g->imgs = rpt / dz.H; }
    else return false;
    const long long rows = (long long)dz.B * dz.H;
    g->num_kt = ((rows + rpt - 1) / rpt) * g->wsegs;
    return true;
}

// pixel slices: at most 64 tiles (4096 pixels, 256 accumulation steps) and at least 8 tiles per CTA; among those the
// slice count whose CTA total fills whole waves of the SMs best (one CTA per SM), fewer slices on a tie (fewer reductions).
// Returns the tiles per slice, *slices_out = the slice count that follows from it.
int choose_slices(long long num_kt, long long items, int sms, long long* slices_out) {
    const long long smin = (num_kt + 63) / 64;
    long long smax = num_kt / 8;
    if (smax < smin) smax = smin;
    long long slices = smin;
    double best = 0.0;
    for (long long s = smin; s <= smax; ++s) {
        const long long total = items * s, waves = (total + sms - 1) / sms;
        const double fill = (double)total / (double)(waves * sms);
        if (fill > best + 0.02) { best = fill; slices = s; }
        if (total >= 16ll * sms) break;
    }
    const int kt_per_slice = (int)((num_kt + slices - 1) / slices);
    *slices_out = (num_kt + kt_per_slice - 1) / kt_per_slice;
    return kt_per_slice;
}

}  // namespace

bool conv_wgrad_tc_supported(const ConvDesc& d, const Act& in, const Act& dz) {
    if (d.Cin % 64 != 0 || d.Cout % 64 != 0) return false;
    if (d.pw > in.halo || in.halo > 1 || dz.halo > 1) return false;
    if (in.C != d.Cin || dz.C != d.Cout || in.B != dz.B) return false;
    if (d.sh != 1 && d.sh != 2) return false;
    if (d.sw != 1 && d.sw != 2) return false;
    if (d.sw == 2 && (in.Wp() % 2) != 0) return false;
    if ((in.H + 2 * d.ph - d.kh) / d.sh + 1 != dz.H || (in.W + 2 * d.pw - d.kw) / d.sw + 1 != dz.W) return false;
    Geometry g;
    if (!tile_geometry(dz, &g)) return false;
    if (g.box_rows * d.sh > 256 || g.imgs > 256) return false;
    return g.num_kt > 0 && g.num_kt < (1ll << 24);
}

// The host-side plan of conv_wgrad_tc for a shape (no device work; `sms` = SM count to plan for):
// plan[0..9] = tw, rows per tile, tiles per row, box rows, images per tile, pixel tiles, tiles per slice, slices,
// work items per slice (Cout tiles x Cin tiles x taps), CTAs.
int conv_wgrad_tc_plan(const ConvDesc& d, const Act& in, const Act& dz, int sms, int plan[10]) {
    HN_CHECK(conv_wgrad_tc_supported(d, in, dz), "conv_wgrad_tc: unsupported shape");
    HN_CHECK(sms >= 1, "conv_wgrad_tc_plan: sms must be positive");
    Geometry g;
    tile_geometry(dz, &g);
    const long long items = (long long)((d.Cout + 127) / 128) * ((d.Cin + 127) / 128) * d.kh * d.kw;
    long long slices = 0;
    const int kps = choose_slices(g.num_kt, items, sms, &slices);
    HN_CHECK(items * slices < (1ll << 31), "conv_wgrad_tc: too many work items");
    const int v[10] = {g.tw, g.rpt, g.wsegs, g.box_rows, g.imgs, (int)g.num_kt, kps, (int)slices, (int)items, (int)(items * slices)};
    for (int i = 0; i < 10; ++i) plan[i] = v[i];
    return 0;
}

int conv_wgrad_tc(const ConvDesc& d, const Act& in, const unsigned short* in_planes, const Act& dz,
                  const unsigned short* dz_planes, const float* dz_absmax, float* dw_ohwi, cudaStream_t st) {
    HN_CHECK(conv_wgrad_tc_supported(d, in, dz), "conv_wgrad_tc: unsupported shape");
    Geometry g;
    tile_geometry(dz, &g);
    WgArgs a;
    memset(&a, 0, sizeof(a));
    a.dw = dw_ohwi; a.absmax = dz_absmax;
    a.Cout = d.Cout; a.Cin = d.Cin; a.taps = d.kh * d.kw; a.kw = d.kw;
    a.n_tiles = (d.Cin + 127) / 128;
    const int m_tiles = (d.Cout + 127) / 128;
    a.tw = g.tw; a.rpt = g.rpt; a.wsegs = g.wsegs; a.Ho = dz.H; a.out_halo = dz.halo;
    a.sh = d.sh; a.ph = d.ph; a.woff = in.halo - d.pw; a.parity = (d.sw == 2);
    a.num_kt = (int)g.num_kt;
    HN_CUDA_OK(cudaMemsetAsync(dw_ohwi, 0, (size_t)d.Cout * a.taps * d.Cin * sizeof(float), st));

    int dev = 0, sms = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    HN_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long items = (long long)m_tiles * a.n_tiles * a.taps;
    long long slices = 0;
    a.kt_per_slice = choose_slices(g.num_kt, items, sms, &slices);
    a.items_per_slice = (int)items;
    HN_CHECK(items * slices < (1ll << 31), "conv_wgrad_tc: too many work items");

    CUtensorMap tmZ[2], tmI[2];
    const size_t in_plane = in.numel(), dz_plane = dz.numel();
    for (int p = 0; p < 2; ++p) {
        {   // dz planes: {Cout, Wop, Ho, B}, interior columns only (the box starts at out_halo)
            const cuuint64_t C2 = (cuuint64_t)d.Cout * 2, Wp = dz.Wp();
            cuuint64_t dims[4] = {(cuuint64_t)d.Cout, Wp, (cuuint64_t)dz.H, (cuuint64_t)dz.B};
            cuuint64_t str[3] = {C2, C2 * Wp, C2 * Wp * dz.H};
            cuuint32_t box[4] = {64, (cuuint32_t)g.tw, (cuuint32_t)g.box_rows, (cuuint32_t)g.imgs};
            if (make_map(&tmZ[p], dz_planes + p * dz_plane, 4, dims, str, box)) return -1;
        }
        // input planes: the rows a tile's output rows read under tap dy are box_rows rows sh apart (traversal stride)
        const bool strided_rows = d.sh == 2 && g.box_rows * g.imgs > 1;
        const cuuint32_t boxrows = strided_rows ? (cuuint32_t)(g.box_rows * 2) : (cuuint32_t)g.box_rows;
        const cuuint64_t C2 = (cuuint64_t)d.Cin * 2, Wp = in.Wp();
        if (!a.parity) {
            cuuint64_t dims[4] = {(cuuint64_t)d.Cin, Wp, (cuuint64_t)in.H, (cuuint64_t)in.B};
            cuuint64_t str[3] = {C2, C2 * Wp, C2 * Wp * in.H};
            cuuint32_t box[4] = {64, (cuuint32_t)g.tw, boxrows, (cuuint32_t)g.imgs};
            if (make_map(&tmI[p], in_planes + p * in_plane, 4, dims, str, box, strided_rows ? 2 : -1, 2)) return -1;
        } else {
            cuuint64_t dims[5] = {(cuuint64_t)d.Cin, 2, Wp / 2, (cuuint64_t)in.H, (cuuint64_t)in.B};
            cuuint64_t str[4] = {C2, 2 * C2, C2 * Wp, C2 * Wp * in.H};
            cuuint32_t box[5] = {64, 1, (cuuint32_t)g.tw, boxrows, (cuuint32_t)g.imgs};
            if (make_map(&tmI[p], in_planes + p * in_plane, 5, dims, str, box, strided_rows ? 3 : -1, 2)) return -1;
        }
    }
    HN_CUDA_OK(cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
    wgrad_tc_kernel<<<(unsigned)(items * slices), NTHREADS, SMEM_TOTAL, st>>>(tmZ[0], tmZ[1], tmI[0], tmI[1], a);
    HN_LAUNCH_OK();
    return 0;
}

}  // namespace hn
