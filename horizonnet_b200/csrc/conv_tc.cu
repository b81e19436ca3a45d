// wgmma tensor-core convolution / GEMM for sm_90a: split precision, three products, fp32 accumulate.
//
// Why split precision: the contract is <= 1e-4 max-abs against the fp32 reference on random-init
// weights; single-pass bf16 (1.4e-2) or tf32 (1.5e-3) miss it (SURVEY hard-part 1), and a
// bf16+bf16 split keeps only 8 + 8 significant bits per operand.  Every fp32 value
// is carried as two fp16 planes of its 2^-4-scaled value:  hi = fp16(s), lo = fp16(s - hi)
// (11 + 11 significant bits, same 4 B/element as fp32, see conv_tc.cuh), and the product is
//     Ahi*Bhi + Ahi*Blo + Alo*Bhi            (the dropped Alo*Blo term is 2^-22 relative)
// accumulated in fp32 registers, segmented (see below).  The planes are written by the producing kernel's epilogue,
// so every operand tile is MMA-ready when TMA drops it into shared memory (no in-kernel conversion pass).
//
// conv_tc_kernel<BN> (persistent, one CTA per SM, 384 threads, launched with programmatic stream serialisation:
// griddepcontrol.launch_dependents at entry, griddepcontrol.wait after the prologue) runs every convolution of the
// tensor-core path (3x3 / strided / 1x1, the LSTM input projections, the data gradients of the training step).
// Like every persistent kernel of this file it takes its tiles one at a time from the stream's tile counter (the
// producer claims, the other roles read the index from a TileQueue, tc_common.cuh):
//   warp 0     TMA producer: per 64-channel K chunk it loads A (hi, lo: 128 pixels x 64 ch, 128B swizzle) from the
//              halo-NHWC planes with ONE box per plane -- {64 ch, tw pixels, R rows} for multi-row tiles (traversal
//              stride 2 along H for the stride-(2,1) convs, whole images when an image has fewer rows than a tile);
//              the 3x3 taps are shifted box coordinates, zero H padding is TMA out-of-bounds fill, circular W padding
//              is the halo column, stride-2 in W reads a parity view -- and B (hi, lo: BN x 64 weights, K-major);
//              3-stage mbarrier ring of 64 KB stages (4 stages of 48 KB for BN <= 64).  After a tile's last K chunk it
//              claims the next stage as the tile's epilogue slot (one stage holds exactly one output tile, BM x BN x 4 B)
//              and TMA-loads the residual tile into it, so the residual lands while the last chunks compute.
//              A block-0 conv3 with its downsample folded in reads two A sources: its K chunks over t2, then its K
//              chunks over the block input x (1x1, stride 1 or 2 through the parity view), each as the same 128-pixel box.
//              "dxr" mode (3x3, one 128-pixel row per tile): one 130-pixel box per (dy, chunk) feeds all three dx taps
//              through wgmma descriptors whose start address is shifted by dx rows (the swizzle is a function of the
//              absolute shared-memory address), so each input row crosses L2 -> SM once instead of three times.  The
//              ring then holds two input-row slots and NST weight slots; a weight slot holds exactly half an output tile,
//              so the epilogue slot is the next two weight slots (hi plane in the first, lo plane in the second).
//   warps 4-7, 8-11   two consumer warpgroups; warpgroup g owns tile rows [64g, 64g + 64) x all BN columns: per chunk
//              12 wgmma m64nBNk16 (3 products x 4 K-steps of 16, one wgmma group; the group of the previous chunk stays in
//              flight until this one is issued) into a register accumulator that is restarted every
//              SEG chunks and added into a second register sum with round-to-nearest fp32 adds (bounds whatever
//              rounding the tensor-core accumulation applies over K up to 18432); then the epilogue in the slot:
//              folded BN scale/shift, + the residual the slot holds, ReLU, re-split into hi/lo planes (or fp32) written
//              in place, the circular halo columns stored directly.  The consumers go straight on to the next tile.
//   warp 3     store warp: TMA-stores each finished output tile from its slot and hands the stage back to the producer
//              once the TMA engine has read it.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "hn_common.cuh"
#include "conv_tc.cuh"
#include "ptx.cuh"
#include "tc_common.cuh"

namespace hn {

namespace {

using namespace tc;                // BM = 128 pixels per tile, NTHREADS, PTX wrappers, make_map, launch_tc
constexpr int BKC = 64;            // fp16 channels per K chunk = one 128-byte swizzle row
constexpr int STAGES = 3;
constexpr int CONS_WARP0 = 4;      // first consumer warp
constexpr int CONS_WARPS = 8;
// K chunks accumulated by the tensor cores before the sum is promoted to the fp32 register sum, in every kernel of this
// file; one constant keeps bott_tc_kernel's conv2 bit-identical to conv_tc_kernel<64>
constexpr int SEG = 4;

struct TcArgs {
    int mode;                 // 0: GEMM rows (1x1 stride-1 conv over all halo-NHWC pixels, or plain GEMM); 1: conv rows
    int M;                    // mode 0: rows; mode 1: B*Ho output rows
    int Ho, Wo, Wop;          // mode 1 output geometry (Wop = Wo + 2*out_halo)
    int out_halo;
    int tw, rows_per_tile, wsegs;
    int sh, ph, parity, woff; // parity = 1: stride 2 along W through the [Wp/2][2] view; woff = in_halo - pw
    int kw, kc_per_tap, num_kc;
    // mode 1, two A sources (a block-0 conv3 with the downsample folded in): chunks [0, k1) come from tmA as described
    // above, chunks [k1, num_kc) from tmA2, a 1x1 conv without padding with its own row stride, parity and woff.
    // k1 = num_kc: one source
    int k1, sh2, parity2, woff2;
    int Bimg;                 // images per plane (plane p of image b sits at index p*Bimg + b of the outer TMA dim)
    int Cout, n_tiles, num_tiles;
    const float* scale;
    const float* shift;
    const unsigned short* res; // residual planes in the OUTPUT geometry (hi at res, lo at res + out_plane), or null
    unsigned short* out;       // split output planes (hi at out, lo at out + out_plane)
    float* out_f32;           // fp32 output instead of planes (LSTM projections)
    size_t out_plane;         // elements per plane
    int relu;
    int dxr;                  // 1: 3x3 single-row tiles load each (dy, channel chunk) input row ONCE (130 pixels) and the three
                              //    dx taps read it through row-shifted descriptors (L2->SM traffic per tap: 64 -> 43 KB)
    int pf;                   // gemm_tc_kernel: L2 prefetch distance (in tiles) of the residual / activation boxes, 0 = off
};

template <int BN>
struct Smem {
    static constexpr int NST = (BN <= 64) ? 4 : STAGES;   // 48 KB stages (BN <= 64) leave room for a 4th
    static constexpr int A_PLANE = BM * BKC * 2;          // 16 KB
    static constexpr int B_PLANE = BN * BKC * 2;
    static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
    static constexpr int BAR_OFF = NST * STAGE;
    static constexpr int CST_OFF = BAR_OFF + 256;         // epilogue constants scale[Cout], shift[Cout]
    static constexpr int TOTAL = CST_OFF + 1024;          // + alignment slack; the launch adds 8 * Cout bytes of constants
};
constexpr int MAX_SMEM = 227 * 1024;
// dynamic shared memory of conv_tc_kernel<BN> for Cout output channels
template <int BN>
constexpr int conv_smem_bytes(int cout) { return Smem<BN>::TOTAL + 8 * cout; }

// 12 wgmma of one 64-channel K chunk as one wgmma group: hi*hi (overwrites the accumulator when `fresh`), hi*lo, lo*hi
template <int R>
__device__ __forceinline__ void chunk_issue(float (&acc)[R], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                            bool fresh) {
    const uint64_t dah = gmma_desc_sw128(a_hi), dal = gmma_desc_sw128(a_lo);
    const uint64_t dbh = gmma_desc_sw128(b_hi), dbl = gmma_desc_sw128(b_lo);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BKC / 16; ++k) {
        const uint64_t ko = (uint64_t)((k * 16 * 2) >> 4);     // advance 32 B inside the swizzle row
        wgmma_f16<0, 0>(acc, dah + ko, dbh + ko, (fresh && k == 0) ? 0u : 1u);
        wgmma_f16<0, 0>(acc, dah + ko, dbl + ko, 1u);
        wgmma_f16<0, 0>(acc, dal + ko, dbh + ko, 1u);
    }
    wgmma_commit();
}
// the same, completed before it returns
template <int R>
__device__ __forceinline__ void chunk_mma(float (&acc)[R], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                          bool fresh) {
    chunk_issue(acc, a_hi, a_lo, b_hi, b_lo, fresh);
    wgmma_wait0();
    reg_fence(acc);
}

// Consumer side of an operand ring.  Per K chunk: the weight tile (hi plane, lo plane b_plane bytes on) of ring stage
// `stage`, and the A operand (hi, lo a_plane bytes on) -- from the same stage, or in dxr mode from one of two input-row
// slots that three consecutive chunks (taps dx = 0, 1, 2) read at a start address shifted by dx rows of 128 B.  Chunks
// are acquired and released in ring order; the release cursor trails the acquire cursor by the chunks whose wgmma
// group may still be in flight.
struct RingPos {
    int stage = 0, ast = 0, dx = 0;        // weight stage; dxr: input-row slot and tap
    uint32_t phase = 0, aph = 0;
    // one chunk on; selects, no branches
    template <bool DXR>
    __device__ __forceinline__ void step(int nst) {
        const bool wrap = stage + 1 == nst;
        stage = wrap ? 0 : stage + 1;
        phase ^= (uint32_t)wrap;
        if (DXR) {
            const bool row_end = dx == 2;
            dx = row_end ? 0 : dx + 1;
            aph ^= (uint32_t)(row_end && ast == 1);
            ast ^= (int)row_end;
        }
    }
};
struct ConsRing {
    uint32_t a0, a_step, a_plane, b0, b_step, b_plane;     // shared addresses: slot i at a0 + i * a_step (likewise b)
    uint64_t* full;
    uint64_t* empty;
    uint64_t* afull;           // dxr: input-row slot filled / read by its three taps
    uint64_t* aempty;
    int nst;
    RingPos get, rel;
};
// hand the oldest unreleased chunk's weight stage (and, after its third tap, its input-row slot) back to the producer;
// only once the chunk's wgmma group has completed
template <bool DXR>
__device__ __forceinline__ void ring_release(ConsRing& q, int lane) {
    __syncwarp();
    mbar_arrive_if(q.empty + q.rel.stage, lane == 0);
    if (DXR) mbar_arrive_if(q.aempty + q.rel.ast, lane == 0 && q.rel.dx == 2);
    q.rel.step<DXR>(q.nst);
}
// One segment of N chunks: the accumulator restarts at its first chunk and is added into `sum` (round-to-nearest fp32)
// after its last.  Straight-line code with compile-time wgmma wait counts: chunk i + 1 is issued while chunk i's group
// is in flight, and nothing between an issue and its wait branches (see mbar_arrive_if).
template <int N, bool DXR, int R>
__device__ __forceinline__ void mma_segment(float (&acc)[R], float (&sum)[R], ConsRing& q, uint32_t a_row_off, int lane) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const RingPos& g = q.get;
        if (DXR) mbar_wait(q.afull + g.ast, g.aph);   // returns at once for dx = 1, 2: the slot is held until dx = 2 retires
        mbar_wait(q.full + g.stage, g.phase);
        const uint32_t a = DXR ? q.a0 + g.ast * q.a_step + g.dx * 128 : q.a0 + g.stage * q.a_step;
        const uint32_t b = q.b0 + g.stage * q.b_step;
        chunk_issue(acc, a + a_row_off, a + q.a_plane + a_row_off, b, b + q.b_plane, i == 0);
        q.get.step<DXR>(q.nst);
        if (i > 0) {
            wgmma_wait1();
            ring_release<DXR>(q, lane);
        }
    }
    wgmma_wait0();
    reg_fence(acc);
    ring_release<DXR>(q, lane);
#pragma unroll
    for (int j = 0; j < R; ++j) sum[j] += acc[j];
}
// sum = the num_kc chunks of one tile in segments of SEG; the last segment takes the K tail.  Nothing is in flight
// between segments, so the choice of the tail's length branches freely.
template <bool DXR, int R>
__device__ __forceinline__ void mma_chunks(float (&acc)[R], float (&sum)[R], ConsRing& q, int num_kc, uint32_t a_row_off,
                                           int lane) {
    static_assert(SEG == 4, "mma_chunks: tail segments of 1 to 3 chunks");
#pragma unroll
    for (int j = 0; j < R; ++j) sum[j] = 0.f;
    int kc = 0;
    for (; kc + SEG <= num_kc; kc += SEG) mma_segment<SEG, DXR>(acc, sum, q, a_row_off, lane);
    switch (num_kc - kc) {
        case 3: mma_segment<3, DXR>(acc, sum, q, a_row_off, lane); break;
        case 2: mma_segment<2, DXR>(acc, sum, q, a_row_off, lane); break;
        case 1: mma_segment<1, DXR>(acc, sum, q, a_row_off, lane); break;
        default: break;
    }
}

// tile row of accumulator element pair h (0: d[4j], d[4j+1]; 1: d[4j+2], d[4j+3]) of this thread's wgmma fragment
__device__ __forceinline__ int frag_row(int wg, int warp, int lane, int h) {
    return wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
}
// byte offset of the column pair (c, c + 1), c even, of tile row r in a [rows][64 fp16] buffer with 128-byte swizzle
__device__ __forceinline__ uint32_t swz_pair_off(int r, int c) {
    return (uint32_t)(r * 128 + ((((c >> 3) ^ (r & 7)) << 4)) + (c & 7) * 2);
}
__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_shared_f2(uint32_t addr, float a, float b) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
// named barrier of one consumer warpgroup (ids 1, 2; id 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, const void* src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(tm)),
                 "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* tm, const void* src, int c0, int c1, int c2, int c3, int c4) {
    asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(tm)),
                 "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive_cnt(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

// circular halo columns of output rows (hn_common.cuh): wp = Wo + 1 copies wo = 0, wp = 0 copies wo = Wo - 1.
// Halo pixel that tile row r is copied to, or -1: rowbase = pixel index of wp = 0 of the tile's first output row, Wop
// pixels per output row, tw tile columns per output row starting at column wo0, `rows` output rows of the tile that exist
__device__ __forceinline__ long long halo_pixel(int r, long long rowbase, int Wop, int tw, int rows, int wo0, int Wo) {
    const unsigned rr = (unsigned)r / (unsigned)tw;
    const int wo = wo0 + (r - (int)rr * tw);
    if ((int)rr >= rows) return -1;
    const long long base = rowbase + (long long)rr * Wop;
    return wo == 0 ? base + Wo + 1 : (wo == Wo - 1 ? base : -1);
}
struct HaloStore {
    void* out;                // output planes (hi; lo at + out_plane) or fp32 output
    size_t out_plane;
    int C, n0;                // channels, first channel of the buffer
    long long pix[2];         // halo_pixel of this thread's fragment rows (frag_row h = 0, 1)
};

// In-place epilogue of a C-channel output tile held as fragments `acc` (rows of this warpgroup): y = acc*sc + sf
// (+ the residual the buffer holds) (ReLU), re-split into the hi / lo planes e_hi / e_lo of the buffer: [128][64] fp16
// with 128-byte swizzle for C = 64, unswizzled [128][32] fp16 for C = 32.  conv_tc_kernel, gemm_tc_kernel and the conv3
// stage of bott_tc_kernel share it, so their results agree bit for bit.
template <int C>
__device__ __forceinline__ void epi_inplace(const float (&acc)[C / 2], const float* sc, const float* sf, uint32_t e_hi,
                                            uint32_t e_lo, bool has_res, bool relu, int wg, int warp, int lane,
                                            const HaloStore* halo = nullptr) {
    static_assert(C == 64 || C == 32, "epi_inplace: 64 or 32 channels");
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = frag_row(wg, warp, lane, h);
        const long long hp = halo ? halo->pix[h] : -1;
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            const float2 k = *reinterpret_cast<const float2*>(sc + c);
            const float2 f = *reinterpret_cast<const float2*>(sf + c);
            float y0 = fmaf(acc[4 * j + 2 * h], k.x, f.x);
            float y1 = fmaf(acc[4 * j + 2 * h + 1], k.y, f.y);
            const uint32_t off = C == 64 ? swz_pair_off(r, c) : (uint32_t)(r * 64 + c * 2);
            if (has_res) {                                    // y is in plane units here: no rescaling needed
                const float2 fh = unpack_half2(ld_shared_u32(e_hi + off)), fl = unpack_half2(ld_shared_u32(e_lo + off));
                y0 += fh.x + fl.x;
                y1 += fh.y + fl.y;
            }
            if (relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
            uint32_t ph, pl;
            split2_scaled(y0, y1, ph, pl);
            st_shared_u32(e_hi + off, ph);
            st_shared_u32(e_lo + off, pl);
            if (hp >= 0) {
                unsigned short* o = static_cast<unsigned short*>(halo->out) + (size_t)hp * halo->C + halo->n0 + c;
                *reinterpret_cast<uint32_t*>(o) = ph;
                *reinterpret_cast<uint32_t*>(o + halo->out_plane) = pl;
            }
        }
    }
}
// the same for fp32 output (no residual): 32 channels into a [128][32] fp32 buffer with 128-byte swizzle
__device__ __forceinline__ void epi_f32(const float (&acc)[16], const float* sc, const float* sf, uint32_t e, bool relu,
                                        int wg, int warp, int lane, const HaloStore* halo) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = frag_row(wg, warp, lane, h);
        const long long hp = halo->pix[h];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            const float2 k = *reinterpret_cast<const float2*>(sc + c);
            const float2 f = *reinterpret_cast<const float2*>(sf + c);
            float y0 = fmaf(acc[4 * j + 2 * h], k.x, f.x);
            float y1 = fmaf(acc[4 * j + 2 * h + 1], k.y, f.y);
            if (relu) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
            st_shared_f2(e + (uint32_t)(r * 128 + ((((c >> 2) ^ (r & 7)) << 4)) + (c & 3) * 4), y0, y1);
            if (hp >= 0) *reinterpret_cast<float2*>(static_cast<float*>(halo->out) + (size_t)hp * halo->C + halo->n0 + c) = make_float2(y0, y1);
        }
    }
}

// Output tile of conv_tc_kernel in its epilogue slot: NPART parts of 128 rows x CW channels, `row_bytes` per row --
// planes: hi plane then lo plane, each as BN / CW channel boxes (CW = 64, 128-byte swizzle; CW = 32 for BN = 32,
// unswizzled); fp32: BN / 32 boxes of 32 channels (128-byte swizzle).  Every layout is BM * BN * 4 bytes, in two halves
// of BM * BN * 2 bytes (the planes, or the first and last fp32 boxes) that may sit apart: the first half at `x`, the
// second at `y`.
template <int BN>
struct EpiLayout {
    int cw, nj, npart, row_bytes;
    __device__ __forceinline__ explicit EpiLayout(bool f32)
        : cw(f32 ? 32 : (BN < 64 ? BN : 64)), nj(BN / cw), npart(f32 ? BN / 32 : 2 * (BN / cw)), row_bytes(f32 ? 128 : 2 * cw) {}
    __device__ __forceinline__ uint8_t* part(uint8_t* x, uint8_t* y, int k) const {
        const int half = npart > 1 ? npart / 2 : 1;
        return (k < half ? x : y) + (k % half) * BM * row_bytes;
    }
};

// Output rows of M tile mt (mode 1): the first output row R0, how many of its rows_per_tile rows exist, first column
__device__ __forceinline__ void tile_rows(const TcArgs& a, int mt, int& R0, int& valid_rows, int& wo0) {
    const int rg = mt / a.wsegs;
    wo0 = (mt - rg * a.wsegs) * a.tw;
    R0 = rg * a.rows_per_tile;
    valid_rows = min(a.rows_per_tile, a.M - R0);
}

// Residual load (`bar` counts the bytes) or output store of part k of tile (mt, nt) through tensor map tm (conv_tc_map):
// mode 0 one box {cw, 128 rows}; mode 1 one box of all the tile's rows
template <int BN, bool STORE>
__device__ __forceinline__ void tile_boxes(const TcArgs& a, const EpiLayout<BN>& L, const CUtensorMap* tm, uint8_t* x,
                                           uint8_t* y, uint64_t* bar, int mt, int nt, int k) {
    const int c0 = nt * BN + (k % L.nj) * L.cw, plane = k / L.nj;
    uint8_t* dst = L.part(x, y, k);
    if (a.mode == 0) {
        if (STORE) tma_store_3d(tm, dst, c0, mt * BM, plane);
        else tma_load_3d(dst, tm, bar, c0, mt * BM, plane);
        return;
    }
    int R0, valid_rows, wo0;
    tile_rows(a, mt, R0, valid_rows, wo0);
    const int b = R0 / a.Ho, ho = R0 - b * a.Ho;
    if (STORE) tma_store_5d(tm, dst, c0, wo0 + a.out_halo, ho, b, plane);
    else tma_load_5d(dst, tm, bar, c0, wo0 + a.out_halo, ho, b, plane);
}

template <int BN>
__global__ void __launch_bounds__(NTHREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmR,
               const __grid_constant__ CUtensorMap tmO, const TcArgs a, unsigned* sched) {
    using S = Smem<BN>;
    constexpr int NST = S::NST;
    constexpr int HALF_TILE = BM * BN * 2;     // one output plane; half an output tile
    static_assert(2 * HALF_TILE <= S::STAGE, "an output tile must fit one ring stage");
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::BAR_OFF);
    uint64_t* empty_bar = full_bar + NST;
    uint64_t* oready_bar = empty_bar + NST;          // [NST] all 8 consumer warps have written the output tile in that stage
    uint64_t* afull_bar = oready_bar + NST;         // [2] dxr mode: input-row slot filled
    uint64_t* aempty_bar = afull_bar + 2;           // [2] dxr mode: the three taps have read the input-row slot
    TileQueue* tq = reinterpret_cast<TileQueue*>(smem + S::BAR_OFF + 128);
    // dxr mode re-partitions the operand ring: two input-row slots (hi + lo plane, 136 rows of 128 B each, 130 used)
    // followed by NST weight-tile slots
    constexpr int AX_PLANE = 17 * 1024;
    constexpr int AX_SLOT = 2 * AX_PLANE;
    constexpr int BX_OFF = 2 * AX_SLOT;
    constexpr int BX_SLOT = 2 * S::B_PLANE;
    static_assert(BX_OFF + NST * BX_SLOT <= NST * S::STAGE, "dxr layout does not fit the operand ring");
    static_assert(BX_SLOT == HALF_TILE, "a dxr weight slot holds half an output tile");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool has_res = a.res != nullptr;
    // Ring sequence per tile: the tile's K chunks, then its epilogue slot -- one ring stage, which holds exactly one output
    // tile, or in dxr mode two consecutive weight slots, each holding half of one (x: first half, y: second half).
    // The producer fills the slot with the residual tile, the consumers turn it into the output tile in place, the store
    // warp hands it to the TMA engine and releases the slot's stages to the producer.
    const int epi_stages = a.dxr ? 2 : 1;
    auto slot_x = [&](int st) { return smem + (a.dxr ? BX_OFF + st * BX_SLOT : st * S::STAGE); };
    auto slot_y = [&](int st) { return a.dxr ? slot_x(st + 1 == NST ? 0 : st + 1) : slot_x(st) + HALF_TILE; };

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        if (a.k1 < a.num_kc) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA2)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmO)) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < NST; ++i) {
            mbar_init(full_bar + i, 1);
            mbar_init(empty_bar + i, CONS_WARPS);
            mbar_init(oready_bar + i, CONS_WARPS);
        }
        for (int i = 0; i < 2; ++i) { mbar_init(afull_bar + i, 1); mbar_init(aempty_bar + i, CONS_WARPS); }
        tq->init(CONS_WARPS + 1);                    // readers: the consumer warps and the store warp
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_wait();                                              // everything below reads / writes activations
    // the epilogue constants, loaded after pdl_wait: in the training step the kernel before this one may have written them
    float* cst = reinterpret_cast<float*>(smem + S::CST_OFF);
    for (int i = threadIdx.x; i < 2 * a.Cout; i += NTHREADS) cst[i] = (i < a.Cout) ? a.scale[i] : a.shift[i - a.Cout];
    __syncthreads();

    if (warp == 0) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
            int stage = 0, ast = 0;
            uint32_t phase = 0, aph = 0;
            for (int it = 0;; ++it) {
                const int tile = tq->claim(it, sched);
                if (tile >= a.num_tiles) { sched_retire(sched); break; }
                const int mt = tile / a.n_tiles, nt = tile - mt * a.n_tiles;
                int valid_rows = 1, row0 = 0, wo0 = 0;
                if (a.mode == 1) tile_rows(a, mt, row0, valid_rows, wo0);
                if (a.dxr) {
                    // 3x3 conv, one output row of 128 pixels per tile: per (dy, channel chunk) ONE box of 130 input pixels,
                    // then the three weight tiles of that (dy, chunk)
                    const int ndyc = a.num_kc / a.kw;
                    const int b = row0 / a.Ho, ho = row0 - b * a.Ho;
                    for (int dyc = 0; dyc < ndyc; ++dyc) {
                        const int dy = dyc / a.kc_per_tap, cc = dyc - dy * a.kc_per_tap;
                        const int hin = ho * a.sh + dy - a.ph;
                        mbar_wait(aempty_bar + ast, aph ^ 1);
                        uint8_t* sAx = smem + ast * AX_SLOT;
                        mbar_expect_tx(afull_bar + ast, 2u * 130u * 128u);
                        tma_load_4d(sAx, &tmA, afull_bar + ast, cc * BKC, wo0 + a.woff, hin, b);
                        tma_load_4d(sAx + AX_PLANE, &tmA, afull_bar + ast, cc * BKC, wo0 + a.woff, hin, a.Bimg + b);
                        if (++ast == 2) { ast = 0; aph ^= 1; }
                        for (int dx = 0; dx < 3; ++dx) {
                            mbar_wait(empty_bar + stage, phase ^ 1);
                            uint8_t* sB = smem + BX_OFF + stage * BX_SLOT;
                            mbar_expect_tx(full_bar + stage, 2u * S::B_PLANE);
                            const int kb = ((dy * a.kw + dx) * a.kc_per_tap + cc) * BKC;
                            tma_load_3d(sB, &tmB, full_bar + stage, kb, nt * BN, 0);
                            tma_load_3d(sB + S::B_PLANE, &tmB, full_bar + stage, kb, nt * BN, 1);
                            if (++stage == NST) { stage = 0; phase ^= 1; }
                        }
                    }
                } else {
                    for (int kc = 0; kc < a.num_kc; ++kc) {
                        mbar_wait(empty_bar + stage, phase ^ 1);
                        uint8_t* sA = smem + stage * S::STAGE;
                        uint8_t* sB = sA + 2 * S::A_PLANE;
                        const bool src2 = kc >= a.k1;
                        const int tap = src2 ? 0 : kc / a.kc_per_tap;
                        const int c0 = (src2 ? kc - a.k1 : kc - tap * a.kc_per_tap) * BKC;
                        // one box per plane always delivers the full tile (rows past the end are out-of-bounds zero fill)
                        mbar_expect_tx(full_bar + stage, 2u * S::A_PLANE + 2u * S::B_PLANE);
                        if (a.mode == 0) {
                            tma_load_3d(sA, &tmA, full_bar + stage, c0, mt * BM, 0);
                            tma_load_3d(sA + S::A_PLANE, &tmA, full_bar + stage, c0, mt * BM, 1);
                        } else {
                            // the tile's output rows are consecutive rows of one image, or whole images (conv_tc_plan)
                            const CUtensorMap* tm = src2 ? &tmA2 : &tmA;
                            const int dy = tap / a.kw, dx = tap - dy * a.kw;
                            const int b = row0 / a.Ho, ho = row0 - b * a.Ho;
                            const int hin = src2 ? ho * a.sh2 : ho * a.sh + dy - a.ph;
                            const int woff = src2 ? a.woff2 : a.woff;
                            if (src2 ? a.parity2 : a.parity) {
                                const int p = dx + woff;
                                tma_load_5d(sA, tm, full_bar + stage, c0, p & 1, wo0 + (p >> 1), hin, b);
                                tma_load_5d(sA + S::A_PLANE, tm, full_bar + stage, c0, p & 1, wo0 + (p >> 1), hin,
                                            a.Bimg + b);
                            } else {
                                tma_load_4d(sA, tm, full_bar + stage, c0, wo0 + dx + woff, hin, b);
                                tma_load_4d(sA + S::A_PLANE, tm, full_bar + stage, c0, wo0 + dx + woff, hin, a.Bimg + b);
                            }
                        }
                        tma_load_3d(sB, &tmB, full_bar + stage, kc * BKC, nt * BN, 0);
                        tma_load_3d(sB + S::B_PLANE, &tmB, full_bar + stage, kc * BKC, nt * BN, 1);
                        if (++stage == NST) { stage = 0; phase ^= 1; }
                    }
                }
                // epilogue slot: the residual tile lands while the tile's last chunks compute
                const int st0 = stage;
                for (int e = 0; e < epi_stages; ++e) {
                    mbar_wait(empty_bar + stage, phase ^ 1);
                    if (e > 0 || !has_res) mbar_arrive(full_bar + stage);
                    if (++stage == NST) { stage = 0; phase ^= 1; }
                }
                if (has_res) {
                    const EpiLayout<BN> L(false);
                    mbar_expect_tx(full_bar + st0, (uint32_t)(BM * BN * 4));
                    for (int k = 0; k < L.npart; ++k)
                        tile_boxes<BN, false>(a, L, &tmR, slot_x(st0), slot_y(st0), full_bar + st0, mt, nt, k);
                }
            }
        }
    } else if (warp >= CONS_WARP0) {
        // =============================== consumers: MMA + in-place epilogue ===============================
        const int wg = (warp - CONS_WARP0) >> 2;         // tile rows [64 wg, 64 wg + 64)
        const uint32_t a_row_off = (uint32_t)(wg * 64 * 128);
        float acc[BN / 2], sum[BN / 2];
        // dxr: the two input-row slots, then the weight slots; otherwise A and B planes of each ring stage
        const uint32_t s0 = smem_u32(smem);
        ConsRing ring = a.dxr ? ConsRing{s0, AX_SLOT, AX_PLANE, s0 + BX_OFF, BX_SLOT, S::B_PLANE,
                                         full_bar, empty_bar, afull_bar, aempty_bar, NST}
                              : ConsRing{s0, S::STAGE, S::A_PLANE, s0 + 2 * S::A_PLANE, S::STAGE, S::B_PLANE,
                                         full_bar, empty_bar, afull_bar, aempty_bar, NST};
        for (int it = 0;; ++it) {
            const int tile = tq->next(it);
            __syncwarp();
            if (lane == 0) tq->release(it);
            if (tile >= a.num_tiles) break;
            const int mt = tile / a.n_tiles, nt = tile - mt * a.n_tiles;
            if (a.dxr) mma_chunks<true>(acc, sum, ring, a.num_kc, a_row_off, lane);
            else mma_chunks<false>(acc, sum, ring, a.num_kc, a_row_off, lane);

            // ---- epilogue in the slot
            HaloStore halo = {a.out_f32 ? static_cast<void*>(a.out_f32) : a.out, a.out_plane, a.Cout, 0, {-1, -1}};
            if (a.mode == 1 && a.out_halo) {
                int R0, rows, wo0;
                tile_rows(a, mt, R0, rows, wo0);
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    halo.pix[h] = halo_pixel(frag_row(wg, warp, lane, h), (long long)R0 * a.Wop, a.Wop, a.tw, rows, wo0, a.Wo);
            }
            // the slot's stages go back to the producer through the store warp
            const int st0 = ring.get.stage;
            const uint32_t x = smem_u32(slot_x(st0)), y = smem_u32(slot_y(st0));
            for (int e = 0; e < epi_stages; ++e) {
                mbar_wait(full_bar + ring.get.stage, ring.get.phase);
                ring.get.step<false>(NST);
                ring.rel.step<false>(NST);
            }
            const float* sc = cst + nt * BN;
            const float* sf = cst + a.Cout + nt * BN;
            if (a.out_f32) {
                // fp32 boxes of 32 channels, the first half at x (BN = 32: its one box; the plan keeps that out of dxr)
                constexpr int HQ = BN / 64 > 0 ? BN / 64 : 1;
#pragma unroll
                for (int q = 0; q < BN / 32; ++q) {
                    halo.n0 = nt * BN + 32 * q;
                    epi_f32(*reinterpret_cast<const float(*)[16]>(sum + 16 * q), sc + 32 * q, sf + 32 * q,
                            (q < HQ ? x : y) + (q % HQ) * BM * 128, a.relu != 0, wg, warp, lane, &halo);
                }
            } else if (BN == 32) {
                halo.n0 = nt * BN;
                epi_inplace<32>(*reinterpret_cast<const float(*)[16]>(sum), sc, sf, x, y, has_res, a.relu != 0, wg, warp,
                                lane, &halo);
            } else {
#pragma unroll
                for (int j = 0; j < BN / 64; ++j) {
                    halo.n0 = nt * BN + 64 * j;
                    epi_inplace<64>(*reinterpret_cast<const float(*)[32]>(sum + 32 * j), sc + 64 * j, sf + 64 * j,
                                    x + j * BM * 128, y + j * BM * 128, has_res, a.relu != 0, wg, warp, lane, &halo);
                }
            }
            // make the generic-proxy writes visible to the TMA engine and tell the store warp
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(oready_bar + st0);
        }
    } else if (warp == 3) {
        // =============================== store warp ===============================
        // one thread follows the ring to each tile's epilogue slot, stores the output tile from it with TMA and
        // releases the slot's stages to the producer once the engine has read it
        if (lane == 0) {
            int stage = 0;
            uint32_t ophase = 0;                   // bit s: phase of oready_bar[s]
            for (int it = 0;; ++it) {
                const int tile = tq->next(it);
                tq->release(it);
                if (tile >= a.num_tiles) break;
                const int mt = tile / a.n_tiles, nt = tile - mt * a.n_tiles;
                stage = (stage + a.num_kc) % NST;
                mbar_wait(oready_bar + stage, (ophase >> stage) & 1);
                ophase ^= 1u << stage;
                const EpiLayout<BN> L(a.out_f32 != nullptr);
                for (int k = 0; k < L.npart; ++k)
                    tile_boxes<BN, true>(a, L, &tmO, slot_x(stage), slot_y(stage), nullptr, mt, nt, k);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                for (int e = 0; e < epi_stages; ++e) {
                    mbar_arrive_cnt(empty_bar + stage, CONS_WARPS);
                    if (++stage == NST) stage = 0;
                }
            }
            asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");          // all stores have landed
        }
    }
}

// ================================================================================================
// gemm_tc_kernel: 1x1 stride-1 convolutions in GEMM mode with K <= 256 (conv3 / conv1 of layer1-3: the
// bottlenecks).  These layers are bound by the epilogue, not by the MMAs.  Like conv_tc_kernel's, all epilogue
// traffic is asynchronous, but with two dedicated epilogue buffers instead of a ring stage per tile (measured faster
// than conv_tc_kernel<128> on 7 of these 15 launches of the batch-32 forward, DESIGN section 3): the producer warp
// TMA-loads the residual tile (hi, lo planes, 128 rows x 64 channels, 128-byte
// swizzle) into one of two epilogue buffers a whole tile ahead, the consumer warpgroups update it IN PLACE from their
// accumulator fragments (BN scale/shift, + residual, ReLU, re-split) and one thread (warp 3) hands the buffer to the
// TMA engine for the store.  Tiles are 128 x 64 so that a 3-stage operand ring (48 KB/stage) and the two 32 KB
// epilogue buffers fit into shared memory together.
constexpr int GBN = 64;

struct GSmem {
    static constexpr int A_PLANE = BM * BKC * 2;          // 16 KB
    static constexpr int B_PLANE = GBN * BKC * 2;         // 8 KB
    static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;            // 48 KB
    static constexpr int E_PLANE = BM * GBN * 2;          // 16 KB: 128 rows x 64 channels fp16
    static constexpr int EBUF = 2 * E_PLANE;              // hi + lo
    static constexpr int EPI_OFF = STAGES * STAGE;        // 144 KB
    static constexpr int BAR_OFF = EPI_OFF + 2 * EBUF;    // 208 KB
    static constexpr int CST_OFF = BAR_OFF + 256;         // epilogue constants scale[Cout] shift[Cout], Cout <= 1024
    static constexpr int MAX_COUT = 1024;
    static constexpr int TOTAL = CST_OFF + 2 * MAX_COUT * 4 + 1024;
};

__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* tm, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(reinterpret_cast<uint64_t>(tm)),
                 "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}


__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmO, const TcArgs a,
               unsigned* sched) {
    using S = GSmem;
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::BAR_OFF);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* rfull_bar = empty_bar + STAGES;       // [2] epilogue buffer holds the residual tile (or is simply free)
    uint64_t* efree_bar = rfull_bar + 2;            // [2] the TMA store has finished reading the epilogue buffer
    uint64_t* oready_bar = efree_bar + 2;           // [2] all 8 consumer warps have written their part of the output tile
    TileQueue* tq = reinterpret_cast<TileQueue*>(smem + S::BAR_OFF + 128);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool has_res = a.res != nullptr;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmO)) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(full_bar + i, 1); mbar_init(empty_bar + i, CONS_WARPS); }
        for (int i = 0; i < 2; ++i) { mbar_init(rfull_bar + i, 1); mbar_init(efree_bar + i, 1); mbar_init(oready_bar + i, CONS_WARPS); }
        tq->init(CONS_WARPS + 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // epilogue constants -> shared memory (weights-side data, safe to read before pdl_wait)
    float* cst = reinterpret_cast<float*>(smem + S::CST_OFF);
    for (int i = threadIdx.x; i < 2 * a.Cout; i += NTHREADS) cst[i] = (i < a.Cout) ? a.scale[i] : a.shift[i - a.Cout];
    __syncthreads();
    pdl_wait();

    if (warp == 0) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int it = 0;; ++it) {
                const int tile = tq->claim(it, sched);
                if (tile >= a.num_tiles) { sched_retire(sched); break; }
                const int mt = tile / a.n_tiles, nt = tile - mt * a.n_tiles;
                // residual and activation boxes -> L2 of the tile claimed about a.pf rounds ahead (tiles are claimed in
                // order, about gridDim.x per round)
                if (a.pf > 0) {
                    const int ta = tile + a.pf * (int)gridDim.x;
                    if (ta < a.num_tiles) {
                        const int mta = ta / a.n_tiles, nta = ta - mta * a.n_tiles;
                        if (has_res) {
                            tma_prefetch_3d(&tmR, nta * GBN, mta * BM, 0);
                            tma_prefetch_3d(&tmR, nta * GBN, mta * BM, 1);
                        }
                        for (int kc = 0; kc < a.num_kc; ++kc) {
                            tma_prefetch_3d(&tmA, kc * BKC, mta * BM, 0);
                            tma_prefetch_3d(&tmA, kc * BKC, mta * BM, 1);
                        }
                    }
                }
                for (int kc = 0; kc < a.num_kc; ++kc) {
                    mbar_wait(empty_bar + stage, phase ^ 1);
                    uint8_t* sA = smem + stage * S::STAGE;
                    uint8_t* sB = sA + 2 * S::A_PLANE;
                    mbar_expect_tx(full_bar + stage, 2u * S::A_PLANE + 2u * S::B_PLANE);
                    tma_load_3d(sA, &tmA, full_bar + stage, kc * BKC, mt * BM, 0);
                    tma_load_3d(sA + S::A_PLANE, &tmA, full_bar + stage, kc * BKC, mt * BM, 1);
                    tma_load_3d(sB, &tmB, full_bar + stage, kc * BKC, nt * GBN, 0);
                    tma_load_3d(sB + S::B_PLANE, &tmB, full_bar + stage, kc * BKC, nt * GBN, 1);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
                // epilogue buffer of this tile: wait until its previous store is done, then load the residual
                const int eb = it & 1;
                mbar_wait(efree_bar + eb, ((it >> 1) & 1) ^ 1);
                uint8_t* ebuf = smem + S::EPI_OFF + eb * S::EBUF;
                if (has_res) {
                    mbar_expect_tx(rfull_bar + eb, 2u * S::E_PLANE);
                    tma_load_3d(ebuf, &tmR, rfull_bar + eb, nt * GBN, mt * BM, 0);
                    tma_load_3d(ebuf + S::E_PLANE, &tmR, rfull_bar + eb, nt * GBN, mt * BM, 1);
                } else {
                    mbar_arrive(rfull_bar + eb);
                }
            }
        }
    } else if (warp >= CONS_WARP0) {
        // =============================== consumers: MMA + in-place epilogue ===============================
        const int wg = (warp - CONS_WARP0) >> 2;
        const uint32_t a_row_off = (uint32_t)(wg * 64 * 128);
        float acc[GBN / 2], sum[GBN / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int it = 0;; ++it) {
            const int tile = tq->next(it);
            __syncwarp();
            if (lane == 0) tq->release(it);
            if (tile >= a.num_tiles) break;
            const int nt = tile % a.n_tiles;
#pragma unroll
            for (int j = 0; j < GBN / 2; ++j) sum[j] = 0.f;
            int seg_pos = 0;
            for (int kc = 0; kc < a.num_kc; ++kc) {
                mbar_wait(full_bar + stage, phase);
                const uint32_t sA = smem_u32(smem + stage * S::STAGE);
                const uint32_t sB = sA + 2 * S::A_PLANE;
                chunk_mma(acc, sA + a_row_off, sA + S::A_PLANE + a_row_off, sB, sB + S::B_PLANE, seg_pos == 0);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar + stage);
                if (++seg_pos == SEG || kc == a.num_kc - 1) {
#pragma unroll
                    for (int j = 0; j < GBN / 2; ++j) sum[j] += acc[j];
                    seg_pos = 0;
                }
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            const int eb = it & 1;
            mbar_wait(rfull_bar + eb, (it >> 1) & 1);
            const uint32_t e_hi = smem_u32(smem + S::EPI_OFF + eb * S::EBUF);
            epi_inplace<64>(sum, cst + nt * GBN, cst + a.Cout + nt * GBN, e_hi, e_hi + S::E_PLANE, has_res, a.relu != 0, wg,
                          warp, lane);
            // make the generic-proxy writes visible to the TMA engine and tell the store warp
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(oready_bar + eb);
        }
    } else if (warp == 3) {
        // =============================== store warp ===============================
        // one thread hands finished output tiles to the TMA engine and returns the buffer to the producer
        // as soon as the engine has read it, so the residual of tile it+2 is prefetched a whole tile ahead
        if (lane == 0) {
            for (int it = 0;; ++it) {
                const int tile = tq->next(it);
                tq->release(it);
                if (tile >= a.num_tiles) break;
                const int mt = tile / a.n_tiles, nt = tile - mt * a.n_tiles;
                const int eb = it & 1;
                mbar_wait(oready_bar + eb, (it >> 1) & 1);
                const uint8_t* ebuf = smem + S::EPI_OFF + eb * S::EBUF;
                tma_store_3d(&tmO, ebuf, nt * GBN, mt * BM, 0);
                tma_store_3d(&tmO, ebuf + S::E_PLANE, nt * GBN, mt * BM, 1);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                mbar_arrive(efree_bar + eb);
            }
            asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");          // all stores have landed
        }
    }
}


// ================================================================================================
// stem_tc_kernel: the 7x7 stride-2 stem (3 -> 64 channels, model.py:73-75) as an implicit GEMM on wgmma.
//
// Cin = 3 does not give a K-major operand by itself, so a pre-pass (stem_pack_kernel) writes the normalised
// input as split planes of PIXEL PAIRS:  P[plane][b][h][j][8] fp16,  element e of pair j = channel e&3 (channel 3
// is zero) of input column 2j + (e>>2) - 3 (circular in W), h = input row + 3 (rows outside the image are zero:
// the zero H padding of the normalised input).  With K ordered (dy, pair p, e) -- i.e. an 8-wide dx window whose
// 8th tap has zero weight -- the A row of output pixel xo for (dy, p) is pair xo + p of row 2*yo + dy: for a tile
// of 128 consecutive output pixels all four p are the SAME shared-memory bytes shifted by p*16 B.  That is exactly
// the no-swizzle K-major wgmma layout (core matrix = 8 rows x 16 B contiguous, SBO = 128 B) with a leading-dimension
// offset of one row (LBO = 16 B): a tile needs ONE TMA box per plane (7 rows x 136 pairs, 15 KB) and the MMAs read
// overlapping operands straight out of it.  K = 7 x 32 = 224 (147 useful), 14 K-steps x 3 products per tile.
// The weights ([2][64][224] fp16 planes, 128-byte swizzle) stay resident in shared memory for the whole kernel.
// Epilogue: accumulator fragments -> BN scale/shift -> ReLU -> fp32 [128 px][64 ch] tile in shared memory (2 x 16 KB, swizzled)
// -> two TMA stores into the halo-NHWC fp32 stem output (the max-pool does not read the halo columns).
constexpr int SP_ROWS = 517;                 // input rows -3 .. 513
constexpr int SP_PAIRS = 520;                // pixel pairs per row (516 used, padded to a multiple of 8)
constexpr int SP_K = 224;                    // 7 dy x 4 pairs x 8
constexpr float STEM_IN_SCALE = 16.f;        // planes hold 16 * normalised input: keeps the lo plane a normal fp16

struct StSmem {
    static constexpr int B_CHUNK = 64 * BKC * 2;              // 8 KB: 64 couts x 64 k
    static constexpr int B_BYTES = 2 * 4 * B_CHUNK;           // hi/lo x 4 chunks = 64 KB
    static constexpr int A_ROW = 136 * 16;                    // one dy: 136 pairs x 16 B
    static constexpr int A_PLANE = 7 * A_ROW;                 // 15232 B
    static constexpr int A_STAGE = 30 * 1024;                 // hi + lo (30464 B) rounded up
    static constexpr int NSTAGE = 3;
    static constexpr int A_OFF = B_BYTES;
    static constexpr int E_HALF = 128 * 128;                  // 128 px x 32 ch fp32
    static constexpr int EBUF = 2 * E_HALF;
    static constexpr int EPI_OFF = A_OFF + NSTAGE * A_STAGE;  // 154 KB
    static constexpr int BAR_OFF = EPI_OFF + 2 * EBUF;        // 218 KB
    static constexpr int TOTAL = BAR_OFF + 256 + 1024;
};

struct StemArgs {
    int B, num_tiles;
    const float* scale;       // accumulator -> true units for an input scaled by 2^-4 (tc_aux[0..64))
    const float* shift;       // folded BN shift
    float floor;              // 0: ReLU (model.py:75); -inf: none
};

// K-major operand without swizzle: 8-row x 16-byte core matrices, `lbo` bytes between the two core matrices of a
// K=16 step, `sbo` bytes between 8-row groups
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(tm)),
                 "r"(smem_u32(src)), "r"(c0), "r"(c1)
                 : "memory");
}

__global__ void __launch_bounds__(256) stem_pack_kernel(const float* __restrict__ x, int Cx,
                                                        unsigned short* __restrict__ out, int B) {
    const size_t total = (size_t)B * SP_ROWS * SP_PAIRS;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int j = (int)(i % SP_PAIRS);
    const size_t t = i / SP_PAIRS;
    const int h = (int)(t % SP_ROWS);
    const int b = (int)(t / SP_ROWS);
    const int row = h - 3;
    uint32_t hi[4] = {0u, 0u, 0u, 0u}, lo[4] = {0u, 0u, 0u, 0u};
    if (row >= 0 && row < 512 && j < 516) {
        const float mean[3] = {0.485f, 0.456f, 0.406f};       // reference model.py:186
        const float stdv[3] = {0.229f, 0.224f, 0.225f};       // reference model.py:187
        unsigned short hs[8], ls[8];
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            int px = 2 * j + e2 - 3;
            px = px < 0 ? px + 1024 : (px >= 1024 ? px - 1024 : px);        // circular W (model.py:27-29)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float v = 0.f;
                if (c < 3) v = (__ldg(x + (((size_t)b * Cx + c) * 512 + row) * 1024 + px) - mean[c]) / stdv[c] * STEM_IN_SCALE;
                const __half hh = __float2half_rn(v);
                hs[e2 * 4 + c] = __half_as_ushort(hh);
                ls[e2 * 4 + c] = __half_as_ushort(__float2half_rn(v - __half2float(hh)));
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) { hi[q] = pack2(hs[2 * q], hs[2 * q + 1]); lo[q] = pack2(ls[2 * q], ls[2 * q + 1]); }
    }
    *reinterpret_cast<uint4*>(out + i * 8) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(out + (total + i) * 8) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// OIHW [64][3][7][7] -> OIHW [64][4][7][8] with zero 4th channel / 8th column (so that pack_weight_tc's K order
// (dy, dx, c) becomes the kernel's (dy, pair, e) order)
__global__ void stem_weight_pad_kernel(const float* __restrict__ w, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 64 * 4 * 7 * 8) return;
    const int dx = i % 8, dy = (i / 8) % 7, c = (i / 56) % 4, n = i / 224;
    out[i] = (c < 3 && dx < 7) ? w[((n * 3 + c) * 7 + dy) * 7 + dx] : 0.f;
}


__global__ void __launch_bounds__(NTHREADS, 1)
stem_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmO, const StemArgs a, unsigned* sched) {
    using S = StSmem;
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::BAR_OFF);
    uint64_t* empty_bar = full_bar + S::NSTAGE;
    uint64_t* bfull_bar = empty_bar + S::NSTAGE;   // weights resident
    uint64_t* oready_bar = bfull_bar + 1;          // [2] output tile staged by all 8 consumer warps
    uint64_t* efree_bar = oready_bar + 2;          // [2] the TMA store has read the staging buffer
    TileQueue* tq = reinterpret_cast<TileQueue*>(smem + S::BAR_OFF + 128);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmO)) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < S::NSTAGE; ++i) { mbar_init(full_bar + i, 1); mbar_init(empty_bar + i, CONS_WARPS); }
        mbar_init(bfull_bar, 1);
        for (int i = 0; i < 2; ++i) { mbar_init(oready_bar + i, CONS_WARPS); mbar_init(efree_bar + i, 1); }
        tq->init(CONS_WARPS + 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_wait();

    // tile -> (image b, output row yo, 128-pixel segment sg): 4 segments per row, 256 rows per image
    if (warp == 0) {
        if (lane == 0) {
            mbar_expect_tx(bfull_bar, (uint32_t)S::B_BYTES);
            for (int pl = 0; pl < 2; ++pl)
                for (int c = 0; c < 4; ++c)
                    tma_load_3d(smem + (pl * 4 + c) * S::B_CHUNK, &tmB, bfull_bar, c * BKC, 0, pl);
            int stage = 0;
            uint32_t phase = 0;
            for (int it = 0;; ++it) {
                const int tile = tq->claim(it, sched);
                if (tile >= a.num_tiles) { sched_retire(sched); break; }
                const int b = tile >> 10, yo = (tile >> 2) & 255, sg = tile & 3;
                mbar_wait(empty_bar + stage, phase ^ 1);
                uint8_t* sA = smem + S::A_OFF + stage * S::A_STAGE;
                mbar_expect_tx(full_bar + stage, 2u * S::A_PLANE);
                tma_load_4d(sA, &tmA, full_bar + stage, 0, sg * 16, 2 * yo, b);
                tma_load_4d(sA + S::A_PLANE, &tmA, full_bar + stage, 0, sg * 16, 2 * yo, a.B + b);
                if (++stage == S::NSTAGE) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp >= CONS_WARP0) {
        // consumer warpgroup wg: output pixels [64 wg, 64 wg + 64) of the tile x all 64 channels
        const int wg = (warp - CONS_WARP0) >> 2;
        float sc[16], sf[16];                     // columns 8j + 2(lane%4) + e -> [2j + e]
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = 8 * j + 2 * (lane & 3) + e;
                sc[2 * j + e] = __ldg(a.scale + c) * (ACT_SCALE / STEM_IN_SCALE);   // tc_aux assumes 2^-4-scaled inputs
                sf[2 * j + e] = __ldg(a.shift + c);
            }
        mbar_wait(bfull_bar, 0);
        const uint32_t sB = smem_u32(smem);
        int stage = 0;
        uint32_t phase = 0;
        float acc[32];
        for (int it = 0;; ++it) {
            const int tile = tq->next(it);
            __syncwarp();
            if (lane == 0) tq->release(it);
            if (tile >= a.num_tiles) break;
            const int eb = it & 1;
            mbar_wait(full_bar + stage, phase);
            const uint32_t sA = smem_u32(smem + S::A_OFF + stage * S::A_STAGE) + (uint32_t)(wg * 64 * 16);
            wgmma_fence();
#pragma unroll
            for (int prod = 0; prod < 3; ++prod) {            // hi*hi, hi*lo, lo*hi
                const uint32_t pa = sA + (prod == 2 ? S::A_PLANE : 0);
                const uint32_t pb = sB + (prod == 1 ? 4 * S::B_CHUNK : 0);
#pragma unroll
                for (int dy = 0; dy < 7; ++dy)
#pragma unroll
                    for (int h2 = 0; h2 < 2; ++h2) {
                        const uint64_t ad = gmma_desc_interleave(pa + dy * S::A_ROW + h2 * 32, 16, 128);
                        const uint64_t bd = gmma_desc_sw128(pb + (dy >> 1) * S::B_CHUNK) +
                                            (uint64_t)((((dy & 1) * 32 + h2 * 16) * 2) >> 4);
                        wgmma_f16<0, 0>(acc, ad, bd, (prod | dy | h2) != 0 ? 1u : 0u);
                    }
            }
            wgmma_commit();
            wgmma_wait0();
            reg_fence(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar + stage);
            if (++stage == S::NSTAGE) { stage = 0; phase ^= 1; }
            // fp32 [128 px][64 ch] tile as two [128][32] halves of 128-byte swizzled rows
            mbar_wait(efree_bar + eb, ((it >> 1) & 1) ^ 1);
            const uint32_t e = smem_u32(smem + S::EPI_OFF + eb * S::EBUF);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = frag_row(wg, warp, lane, h);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3), cc = c & 31;
                    const float y0 = fmaxf(fmaf(acc[4 * j + 2 * h], sc[2 * j], sf[2 * j]), a.floor);
                    const float y1 = fmaxf(fmaf(acc[4 * j + 2 * h + 1], sc[2 * j + 1], sf[2 * j + 1]), a.floor);
                    st_shared_f2(e + (uint32_t)((c >> 5) * S::E_HALF + r * 128 + ((((cc >> 2) ^ (r & 7))) << 4) + (cc & 3) * 4),
                                 y0, y1);
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(oready_bar + eb);
        }
    } else if (warp == 3) {
        if (lane == 0) {
            for (int it = 0;; ++it) {
                const int tile = tq->next(it);
                tq->release(it);
                if (tile >= a.num_tiles) break;
                const int b = tile >> 10, yo = (tile >> 2) & 255, sg = tile & 3;
                const int eb = it & 1;
                mbar_wait(oready_bar + eb, (it >> 1) & 1);
                const uint8_t* ebuf = smem + S::EPI_OFF + eb * S::EBUF;
                const int pix = (b * 256 + yo) * 514 + sg * 128 + 1;
                tma_store_2d(&tmO, ebuf, 0, pix);
                tma_store_2d(&tmO, ebuf + S::E_HALF, 32, pix);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                mbar_arrive(efree_bar + eb);
            }
            asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        }
    }
}

// ================================================================================================
// bott_tc_kernel: conv2 (3x3, stride 1, 64 -> 64) + BN + ReLU  FUSED WITH  conv3 (1x1, 64 -> C3) + BN + identity + ReLU
// of a layer1 bottleneck (torchvision Bottleneck.forward; reference model.py:78).  Per tile of 128 pixels of one
// output row, each consumer warpgroup (64 of the pixels):
//   stage 1   computes the conv2 tile exactly as conv_tc_kernel<64> does (same wgmma order, segments,
//             epilogue maths), but writes the BN+ReLU'd result as hi/lo planes into SHARED memory (t2, [128 px][64 ch]
//             rows of 128 B, 128-byte swizzle: exactly a K-major wgmma A operand) instead of HBM;
//   stage 2   runs conv3 as C3 / 64 tiles of 128 x 64 with A = t2, B = conv3 weights, the residual tile TMA-loaded into
//             an epilogue buffer ahead of use, updated in place and TMA-stored (the epilogue of gemm_tc_kernel),
//             halo columns by direct stores.
// The 64-channel intermediate never visits HBM, and the TMA engine streams the residual and the output of one
// conv3 tile while the next one computes.
// With the downsample folded in (`fold`, layer1.0) conv3 has no residual: the producer loads the tile's 128 pixels of
// the block input x once, into the next input-row slot, and every conv3 n-tile accumulates two K chunks, t2 and that x
// tile, against the folded weights [s3 W3 ; sd Wd] -- the same products in the same order as conv_tc_kernel's two-source
// conv3.
//   warp 0      TMA producer (input rows, the x tile, then the conv2 and conv3 weight tiles of the tile through one ring)
//   warp 2      residual-tile loader          warp 3   TMA store          warps 4-11   two consumer warpgroups
struct BottArgs {
    int Ho, Wo, Wop, wsegs, Bimg;
    int num_tiles;
    int n3;                              // conv3 n-tiles of 64 channels (Cout3 / 64)
    int C3;                              // conv3 output channels
    int fold;                            // 1: conv3 K = [t2 | x] (downsample folded in), no residual
    const float* scale2; const float* shift2;     // conv2: accumulator -> plane units, shift in plane units
    const float* scale3; const float* shift3;     // conv3
    unsigned short* out; size_t out_plane;        // output planes (halo-column stores)
};

struct BtSmem {
    static constexpr int AX_PLANE = 17 * 1024;            // 130 input pixels x 128 B (136 rows reserved)
    static constexpr int AX_SLOT = 2 * AX_PLANE;          // hi + lo
    static constexpr int NB = 3;                          // weight-tile ring
    static constexpr int B_PLANE = 64 * BKC * 2;          // 8 KB
    static constexpr int B_STAGE = 2 * B_PLANE;           // 16 KB
    static constexpr int B_OFF = 2 * AX_SLOT;             // 68 KB
    static constexpr int T2_OFF = B_OFF + NB * B_STAGE;   // 116 KB (1024-aligned)
    static constexpr int T_PLANE = BM * BKC * 2;          // 16 KB
    static constexpr int E_OFF = T2_OFF + 2 * T_PLANE;    // 148 KB
    static constexpr int E_PLANE = BM * 64 * 2;           // 16 KB
    static constexpr int EBUF = 2 * E_PLANE;
    static constexpr int BAR_OFF = E_OFF + 2 * EBUF;      // 212 KB
    static constexpr int CST_OFF = BAR_OFF + 512;         // epilogue constants: scale2[64] shift2[64] scale3[C3] shift3[C3] (C3 <= 512)
    static constexpr int TOTAL = CST_OFF + (128 + 2 * 512) * 4 + 1024;
};
static_assert(BtSmem::T2_OFF % 1024 == 0 && BtSmem::E_OFF % 1024 == 0 && BtSmem::B_OFF % 1024 == 0, "swizzle atoms need 1024-byte alignment");
__global__ void __launch_bounds__(NTHREADS, 1)
bott_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB2,
               const __grid_constant__ CUtensorMap tmB3, const __grid_constant__ CUtensorMap tmR,
               const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmO, const BottArgs a,
               unsigned* sched) {
    using S = BtSmem;
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::BAR_OFF);   // [NB] weight tile landed
    uint64_t* empty_bar = full_bar + S::NB;         // [NB] weight tile consumed
    uint64_t* afull_bar = empty_bar + S::NB;        // [2] input-row slot filled
    uint64_t* aempty_bar = afull_bar + 2;           // [2] input-row slot consumed
    uint64_t* rfull_bar = aempty_bar + 2;           // [2] residual tile landed in the epilogue buffer
    uint64_t* oready_bar = rfull_bar + 2;           // [2] output tile complete in the epilogue buffer
    uint64_t* efree_bar = oready_bar + 2;           // [2] TMA store has read the epilogue buffer
    TileQueue* tq = reinterpret_cast<TileQueue*>(smem + S::BAR_OFF + 128);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB2)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB3)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(a.fold ? &tmX : &tmR)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmO)) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < S::NB; ++i) { mbar_init(full_bar + i, 1); mbar_init(empty_bar + i, CONS_WARPS); }
        for (int i = 0; i < 2; ++i) {
            mbar_init(afull_bar + i, 1); mbar_init(aempty_bar + i, CONS_WARPS);
            mbar_init(rfull_bar + i, 1); mbar_init(oready_bar + i, CONS_WARPS); mbar_init(efree_bar + i, 1);
        }
        tq->init(CONS_WARPS + 2);                    // readers: the consumer warps, the residual loader, the store warp
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // epilogue constants -> shared memory (weights-side data, safe to read before pdl_wait)
    float* cst = reinterpret_cast<float*>(smem + S::CST_OFF);
    for (int i = threadIdx.x; i < 128 + 2 * a.C3; i += NTHREADS)
        cst[i] = (i < 64) ? a.scale2[i] : (i < 128) ? a.shift2[i - 64] : (i < 128 + a.C3) ? a.scale3[i - 128] : a.shift3[i - 128 - a.C3];
    __syncthreads();
    pdl_wait();
    const int n3 = a.n3;

    if (warp == 0) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
            int ast = 0, bst = 0;
            uint32_t aph = 0, bph = 0;
            for (int it = 0;; ++it) {
                const int tile = tq->claim(it, sched);
                if (tile >= a.num_tiles) { sched_retire(sched); break; }
                const int rg = tile / a.wsegs;
                const int wo0 = (tile - rg * a.wsegs) * BM;
                const int b = rg / a.Ho, ho = rg - b * a.Ho;
                for (int dy = 0; dy < 3; ++dy) {
                    const int hin = ho + dy - 1;
                    mbar_wait(aempty_bar + ast, aph ^ 1);
                    uint8_t* sAx = smem + ast * S::AX_SLOT;
                    mbar_expect_tx(afull_bar + ast, 2u * 130u * 128u);
                    tma_load_4d(sAx, &tmA, afull_bar + ast, 0, wo0, hin, b);
                    tma_load_4d(sAx + S::AX_PLANE, &tmA, afull_bar + ast, 0, wo0, hin, a.Bimg + b);
                    if (++ast == 2) { ast = 0; aph ^= 1; }
                    for (int dx = 0; dx < 3; ++dx) {
                        mbar_wait(empty_bar + bst, bph ^ 1);
                        uint8_t* sB = smem + S::B_OFF + bst * S::B_STAGE;
                        mbar_expect_tx(full_bar + bst, (uint32_t)S::B_STAGE);
                        const int kb = (dy * 3 + dx) * BKC;
                        tma_load_3d(sB, &tmB2, full_bar + bst, kb, 0, 0);
                        tma_load_3d(sB + S::B_PLANE, &tmB2, full_bar + bst, kb, 0, 1);
                        if (++bst == S::NB) { bst = 0; bph ^= 1; }
                    }
                }
                if (a.fold) {                           // the tile's 128 pixels of x, read by every conv3 n-tile
                    mbar_wait(aempty_bar + ast, aph ^ 1);
                    uint8_t* sX = smem + ast * S::AX_SLOT;
                    const int pix0 = rg * a.Wop + 1 + wo0;
                    mbar_expect_tx(afull_bar + ast, 2u * BM * 128u);
                    tma_load_3d(sX, &tmX, afull_bar + ast, 0, pix0, 0);
                    tma_load_3d(sX + S::AX_PLANE, &tmX, afull_bar + ast, 0, pix0, 1);
                    if (++ast == 2) { ast = 0; aph ^= 1; }
                }
                for (int j = 0; j < n3; ++j) {          // conv3 weight tiles (the same for every tile: L2 hits)
                    for (int kc = 0; kc <= a.fold; ++kc) {
                        mbar_wait(empty_bar + bst, bph ^ 1);
                        uint8_t* sB = smem + S::B_OFF + bst * S::B_STAGE;
                        mbar_expect_tx(full_bar + bst, (uint32_t)S::B_STAGE);
                        tma_load_3d(sB, &tmB3, full_bar + bst, kc * BKC, j * 64, 0);
                        tma_load_3d(sB + S::B_PLANE, &tmB3, full_bar + bst, kc * BKC, j * 64, 1);
                        if (++bst == S::NB) { bst = 0; bph ^= 1; }
                    }
                }
            }
        }
    } else if (warp == 2) {
        // =============================== residual loader ===============================
        // its own thread, so that the identity tile of n-tile j is requested the moment its epilogue buffer is released
        if (lane == 0) {
            int g3 = 0;
            for (int it = 0;; ++it) {
                const int tile = tq->next(it);
                tq->release(it);
                if (tile >= a.num_tiles) break;
                const int rg = tile / a.wsegs;
                const int pix0 = rg * a.Wop + 1 + (tile - rg * a.wsegs) * BM;
                for (int j = 0; j < n3; ++j, ++g3) {
                    const int eb = g3 & 1;
                    mbar_wait(efree_bar + eb, ((g3 >> 1) & 1) ^ 1);
                    if (a.fold) { mbar_arrive(rfull_bar + eb); continue; }      // no residual: the buffer is just free
                    uint8_t* ebuf = smem + S::E_OFF + eb * S::EBUF;
                    mbar_expect_tx(rfull_bar + eb, 2u * S::E_PLANE);
                    tma_load_3d(ebuf, &tmR, rfull_bar + eb, j * 64, pix0, 0);
                    tma_load_3d(ebuf + S::E_PLANE, &tmR, rfull_bar + eb, j * 64, pix0, 1);
                }
            }
        }
    } else if (warp == 3) {
        // =============================== store warp ===============================
        if (lane == 0) {
            int g3 = 0;
            for (int it = 0;; ++it) {
                const int tile = tq->next(it);
                tq->release(it);
                if (tile >= a.num_tiles) break;
                const int rg = tile / a.wsegs;
                const int pix0 = rg * a.Wop + 1 + (tile - rg * a.wsegs) * BM;
                for (int j = 0; j < n3; ++j, ++g3) {
                    const int eb = g3 & 1;
                    mbar_wait(oready_bar + eb, (g3 >> 1) & 1);
                    const uint8_t* ebuf = smem + S::E_OFF + eb * S::EBUF;
                    tma_store_3d(&tmO, ebuf, j * 64, pix0, 0);
                    tma_store_3d(&tmO, ebuf + S::E_PLANE, j * 64, pix0, 1);
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    mbar_arrive(efree_bar + eb);
                }
            }
            asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        }
    } else if (warp >= CONS_WARP0) {
        // =============================== consumers: conv2 -> t2 -> conv3 ===============================
        const int wg = (warp - CONS_WARP0) >> 2;
        const uint32_t a_row_off = (uint32_t)(wg * 64 * 128);
        const uint32_t t_hi = smem_u32(smem + S::T2_OFF), t_lo = t_hi + S::T_PLANE;
        int ast = 0, bst = 0, g3 = 0;
        uint32_t aph = 0, bph = 0;
        float acc[32], sum[32];
        auto release_b = [&]() {
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar + bst);
            if (++bst == S::NB) { bst = 0; bph ^= 1; }
        };
        for (int it = 0;; ++it) {
            const int tile = tq->next(it);
            __syncwarp();
            if (lane == 0) tq->release(it);
            if (tile >= a.num_tiles) break;
            const int rg = tile / a.wsegs;
            const int wo0 = (tile - rg * a.wsegs) * BM;
            // ---- conv2 (identical to conv_tc_kernel<64>)
#pragma unroll
            for (int j = 0; j < 32; ++j) sum[j] = 0.f;
            int seg_pos = 0, kc = 0;
            for (int dy = 0; dy < 3; ++dy) {
                mbar_wait(afull_bar + ast, aph);
                const uint32_t sAx = smem_u32(smem + ast * S::AX_SLOT);
                for (int dx = 0; dx < 3; ++dx, ++kc) {
                    mbar_wait(full_bar + bst, bph);
                    const uint32_t sB = smem_u32(smem + S::B_OFF + bst * S::B_STAGE);
                    chunk_mma(acc, sAx + dx * 128 + a_row_off, sAx + S::AX_PLANE + dx * 128 + a_row_off, sB, sB + S::B_PLANE,
                              seg_pos == 0);
                    release_b();
                    if (++seg_pos == SEG || kc == 8) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) sum[j] += acc[j];
                        seg_pos = 0;
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(aempty_bar + ast);
                if (++ast == 2) { ast = 0; aph ^= 1; }
            }
            // ---- BN + ReLU -> t2 rows of this warpgroup (its previous conv3 wgmmas, the only readers, have completed)
            wg_sync(wg);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = frag_row(wg, warp, lane, h);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3);
                    const float y0 = fmaxf(fmaf(sum[4 * j + 2 * h], cst[c], cst[64 + c]), 0.f);
                    const float y1 = fmaxf(fmaf(sum[4 * j + 2 * h + 1], cst[c + 1], cst[64 + c + 1]), 0.f);
                    uint32_t ph, pl;
                    split2_scaled(y0, y1, ph, pl);
                    st_shared_u32(t_hi + swz_pair_off(r, c), ph);
                    st_shared_u32(t_lo + swz_pair_off(r, c), pl);
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> wgmma operand reads
            wg_sync(wg);
            // ---- conv3: one 128 x 64 tile per 64 output channels, in-place epilogue on the residual tile
            HaloStore halo = {a.out, a.out_plane, a.C3, 0, {-1, -1}};
#pragma unroll
            for (int h = 0; h < 2; ++h)
                halo.pix[h] = halo_pixel(frag_row(wg, warp, lane, h), (long long)rg * a.Wop, a.Wop, BM, 1, wo0, a.Wo);
            uint32_t x_hi = 0;
            if (a.fold) {
                mbar_wait(afull_bar + ast, aph);
                x_hi = smem_u32(smem + ast * S::AX_SLOT) + a_row_off;
            }
            for (int j = 0; j < n3; ++j, ++g3) {
                mbar_wait(full_bar + bst, bph);
                const uint32_t sB = smem_u32(smem + S::B_OFF + bst * S::B_STAGE);
                chunk_issue(acc, t_hi + a_row_off, t_lo + a_row_off, sB, sB + S::B_PLANE, true);
                if (a.fold) {                         // + the x chunk against the next weight tile, one segment
                    const int b1 = bst + 1 == S::NB ? 0 : bst + 1;
                    mbar_wait(full_bar + b1, b1 == 0 ? bph ^ 1 : bph);
                    const uint32_t sB1 = smem_u32(smem + S::B_OFF + b1 * S::B_STAGE);
                    chunk_issue(acc, x_hi, x_hi + S::AX_PLANE, sB1, sB1 + S::B_PLANE, false);
                }
                wgmma_wait0();
                reg_fence(acc);
                release_b();
                if (a.fold) release_b();
#pragma unroll
                for (int q = 0; q < 32; ++q) sum[q] = 0.f + acc[q];      // as gemm_tc_kernel's single segment
                const int eb = g3 & 1;
                mbar_wait(rfull_bar + eb, (g3 >> 1) & 1);
                const uint32_t e_hi = smem_u32(smem + S::E_OFF + eb * S::EBUF);
                HaloStore hj = halo;
                hj.n0 = j * 64;
                epi_inplace<64>(sum, cst + 128 + j * 64, cst + 128 + a.C3 + j * 64, e_hi, e_hi + S::E_PLANE, !a.fold, true,
                                wg, warp, lane, &hj);
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane == 0) mbar_arrive(oready_bar + eb);
            }
            if (a.fold) {                             // every n-tile has read the x tile
                __syncwarp();
                if (lane == 0) mbar_arrive(aempty_bar + ast);
                if (++ast == 2) { ast = 0; aph ^= 1; }
            }
        }
    }
}

// -------------------------------------------------------------------------------- host side
template <int BN>
int launch(const CUtensorMap& tmA, const CUtensorMap& tmA2, const CUtensorMap& tmB, const CUtensorMap& tmR,
           const CUtensorMap& tmO, const TcArgs& a, int grid, cudaStream_t st) {
    const int bytes = conv_smem_bytes<BN>(a.Cout);
    HN_CHECK(bytes <= MAX_SMEM, "conv_tc: too many output channels for the epilogue constants in shared memory");
    HN_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    HN_CUDA_OK(launch_tc(conv_tc_kernel<BN>, grid, bytes, st, tmA, tmA2, tmB, tmR, tmO, a));
    HN_LAUNCH_OK();
    return 0;
}

int launch_bn(int BN, const CUtensorMap& tmA, const CUtensorMap& tmA2, const CUtensorMap& tmB, const CUtensorMap& tmR,
              const CUtensorMap& tmO, const TcArgs& a, int grid, cudaStream_t st) {
    switch (BN) {
        case 128: return launch<128>(tmA, tmA2, tmB, tmR, tmO, a, grid, st);
        case 64: return launch<64>(tmA, tmA2, tmB, tmR, tmO, a, grid, st);
        default: return launch<32>(tmA, tmA2, tmB, tmR, tmO, a, grid, st);
    }
}

// Conv-row (mode 1) A operand map of a 1x1 or kxk conv over `in` for the tiles of plan pl: {C, Wp, H, 2B} (or with
// stride 2 along W the parity view {C, 2, Wp/2, H, 2B}), one box per plane of a tile's 128 pixels x 64 channels
int conv_rows_map(CUtensorMap* tm, const unsigned short* in_planes, const Act& in, int Cin, int sh, bool parity,
                  bool dxr, const TcPlan& pl) {
    // stride 2 along H (height-reduction convs): a box of several rows spans 2*rows input rows and takes every second
    // one; a one-row tile reads its input row without a traversal stride
    const int hs = pl.rows_per_tile > 1 ? sh : 1;
    const cuuint32_t boxrows = (cuuint32_t)(pl.box_rows * hs);
    const cuuint64_t C2 = (cuuint64_t)Cin * 2, Wp = in.Wp();
    if (!parity) {
        cuuint64_t dims[4] = {(cuuint64_t)Cin, Wp, (cuuint64_t)in.H, (cuuint64_t)2 * in.B};
        cuuint64_t str[3] = {C2, C2 * Wp, C2 * Wp * in.H};
        cuuint32_t box[4] = {BKC, dxr ? 130u : (cuuint32_t)pl.tw, boxrows, (cuuint32_t)pl.box_imgs};
        return make_map(tm, in_planes, 4, dims, str, box, 2, hs);
    }
    cuuint64_t dims[5] = {(cuuint64_t)Cin, 2, Wp / 2, (cuuint64_t)in.H, (cuuint64_t)2 * in.B};
    cuuint64_t str[4] = {C2, 2 * C2, C2 * Wp, C2 * Wp * in.H};
    cuuint32_t box[5] = {BKC, 1, (cuuint32_t)pl.tw, boxrows, (cuuint32_t)pl.box_imgs};
    return make_map(tm, in_planes, 5, dims, str, box, 3, hs);
}

// Tensor map of an output-geometry tensor (output or residual) as the epilogue of a tile with BN channels moves it (see
// EpiLayout): planes (hi, lo: an outer dimension of 2) or fp32 (an outer dimension of 1).  Mode 0 {Cout, M pixels,
// plane}, box {cw, 128}; mode 1 {Cout, Wop, Ho, B, plane} -- the plane has its own dimension, so a box clipped past the
// last image never spills into the lo plane -- box {cw, tw, box rows, box images}.
int conv_tc_map(CUtensorMap* tm, const void* base, const TcPlan& pl, const Act& out, int Cout, bool f32) {
    const cuuint64_t es = f32 ? 4 : 2, C = (cuuint64_t)Cout, plane_bytes = (cuuint64_t)out.numel() * es;
    const cuuint32_t cw = f32 ? 32u : (pl.BN < 64 ? (cuuint32_t)pl.BN : 64u);
    const CUtensorMapDataType dt = f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const CUtensorMapSwizzle sw = (cw * es == 128) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE;
    const cuuint64_t planes = f32 ? 1 : 2;
    if (pl.mode == 0) {
        cuuint64_t dims[3] = {C, (cuuint64_t)pl.M, planes};
        cuuint64_t str[2] = {C * es, plane_bytes};
        cuuint32_t box[3] = {cw, (cuuint32_t)BM, 1};
        return make_map(tm, base, 3, dims, str, box, -1, 1, dt, sw);
    }
    const cuuint64_t Wop = out.Wp();
    cuuint64_t dims[5] = {C, Wop, (cuuint64_t)out.H, (cuuint64_t)out.B, planes};
    cuuint64_t str[4] = {C * es, C * es * Wop, C * es * Wop * out.H, plane_bytes};
    cuuint32_t box[5] = {cw, (cuuint32_t)pl.tw, (cuuint32_t)pl.box_rows, (cuuint32_t)pl.box_imgs, 1};
    return make_map(tm, base, 5, dims, str, box, -1, 1, dt, sw);
}

}  // namespace

// channel and padding limits of both modes
static bool conv_channels_supported(const ConvDesc& d, const Act& in) {
    if (d.Cin % 64 != 0 || d.Cout % 32 != 0) return false;
    if (d.Cout > 64 && d.Cout % 128 != 0) return false;
    if (d.Cout < 64 && d.Cout != 32) return false;
    return d.pw <= in.halo;
}

// the conv-row (mode 1) tiling
static bool conv_rows_supported(const ConvDesc& d, const Act& in, const Act& out) {
    if (d.sw != 1 && d.sw != 2) return false;
    if (d.sw == 2 && (in.Wp() % 2) != 0) return false;
    const int tw = out.W < 128 ? out.W : 128;
    if (tw < 8 || (tw & (tw - 1)) != 0 || out.W % tw != 0) return false;       // 8-row swizzle atoms, exact W tiling
    // one TMA box per plane loads a tile: its BM / tw output rows are consecutive rows of one image or whole images, and
    // their input rows are 1 or 2 apart (a traversal stride along H)
    const int rows_per_tile = BM / tw;
    if (d.sh != 1 && d.sh != 2) return false;
    return out.H % rows_per_tile == 0 || rows_per_tile % out.H == 0;
}

bool conv_tc_supported(const ConvDesc& d, const Act& in, const Act& out) {
    if (!conv_channels_supported(d, in)) return false;
    const bool gemm = (d.kh == 1 && d.kw == 1 && d.sh == 1 && d.sw == 1 && in.halo == out.halo);
    return gemm || conv_rows_supported(d, in, out);
}

// output channels per tile for `rows` output pixels
static int tile_bn(int Cout, long long rows) {
    const int BN = Cout >= 128 ? 128 : Cout;
    // layers with too few 128x128 tiles to fill the SMs (the tail of the height-reduction convs): halve the tile width
    const long long tiles128 = ((rows + BM - 1) / BM) * (Cout / 128 > 0 ? Cout / 128 : 1);
    return (BN == 128 && tiles128 < 110) ? 64 : BN;
}

// conv-row (mode 1) fields of the plan; returns the number of M tiles
static long long plan_rows(const ConvDesc& d, const Act& in, const Act& out, bool out_f32, TcPlan* p) {
    p->mode = 1;
    p->M = out.B * out.H;
    p->tw = out.W < 128 ? out.W : 128;
    p->rows_per_tile = BM / p->tw;
    p->wsegs = out.W / p->tw;
    p->parity = (d.sw == 2);
    // one box for all rows of a tile: consecutive output rows of one image, or whole images when an image has fewer
    // output rows than a tile (the last height-reduction convs) -- the box then spans R / Ho consecutive images
    p->box_rows = p->box_imgs = 1;
    if (out.H % p->rows_per_tile == 0) p->box_rows = p->rows_per_tile;
    else { p->box_rows = out.H; p->box_imgs = p->rows_per_tile / out.H; }
    // dx reuse.  Its epilogue slot is two weight slots, each half an output tile: a plane, or half of the fp32 boxes --
    // which needs two of them (BN >= 64)
    p->dxr = (!p->parity && d.kw == 3 && p->rows_per_tile == 1 && p->tw == BM &&
              !(out_f32 && p->BN < 64) &&
              (long long)p->wsegs * BM + (in.halo - d.pw) + 2 <= (long long)in.Wp()) ? 1 : 0;
    return (long long)((p->M + p->rows_per_tile - 1) / p->rows_per_tile) * p->wsegs;
}

int conv_tc_plan(const ConvDesc& d, const Act& in, const Act& out, bool out_f32, bool has_residual, int sms, TcPlan* p) {
    HN_CHECK(conv_tc_supported(d, in, out), "conv_tc: unsupported shape");
    HN_CHECK(!(out_f32 && has_residual), "conv_tc: residual with fp32 output is not supported");
    HN_CHECK(sms >= 1, "conv_tc_plan: sms must be positive");
    memset(p, 0, sizeof(*p));
    const bool gemm = (d.kh == 1 && d.kw == 1 && d.sh == 1 && d.sw == 1 && in.halo == out.halo);
    const int BN = tile_bn(d.Cout, gemm ? (long long)in.B * in.H * in.Wp() : (long long)out.B * out.H * out.W);
    p->num_kc = d.kh * d.kw * (d.Cin / BKC);
    p->seg = SEG;
    p->box_rows = p->box_imgs = 1;
    long long m_tiles;
    // asynchronous-epilogue GEMM kernel: plane output, Cin <= 256, Cout a multiple of 64
    if (gemm && !out_f32 && d.Cin <= 256 && d.Cout % GBN == 0 && d.Cout <= GSmem::MAX_COUT) {
        const long long Mtot = (long long)in.B * in.H * in.Wp();
        p->gemm_kernel = 1;
        p->BN = GBN;
        p->mode = 0;
        p->M = (int)Mtot;
        // L2 prefetch two tile rounds ahead for the K = 64 layers (one activation box per tile); the K = 256 layers
        // already keep 8 boxes per tile in flight
        p->pf = p->num_kc == 1 ? 2 : 0;
        m_tiles = (Mtot + BM - 1) / BM;
    } else if (gemm) {
        p->BN = BN;
        p->mode = 0;
        p->M = (int)((long long)in.B * in.H * in.Wp());
        m_tiles = ((long long)p->M + BM - 1) / BM;
    } else {
        p->BN = BN;
        m_tiles = plan_rows(d, in, out, out_f32, p);
    }
    p->n_tiles = d.Cout / p->BN;
    HN_CHECK(m_tiles * p->n_tiles < (1ll << 31), "conv_tc: too many tiles");
    p->num_tiles = (int)(m_tiles * p->n_tiles);
    p->grid = p->num_tiles < sms ? p->num_tiles : sms;
    return 0;
}

// in / out / residual are split plane pairs in halo-NHWC geometry (hi plane, then lo plane).
// wq: [2][Cout][K] weight planes, K = (dy*kw+dx)*Cin + c; tc_scale folds BN scale and the plane scales.
int conv_tc_planes(const ConvDesc& d, const unsigned short* wq, const float* tc_aux, const Act& in,
                   const unsigned short* in_planes, const Act& out, unsigned short* out_planes, float* out_f32,
                   const unsigned short* res_planes, cudaStream_t st) {
    TcPlan pl;
    if (conv_tc_plan(d, in, out, out_f32 != nullptr, res_planes != nullptr, num_sms(), &pl)) return -1;
    const int K = d.kh * d.kw * d.Cin;
    const int BN = pl.BN;
    TcArgs a;
    memset(&a, 0, sizeof(a));
    const size_t in_plane = in.numel(), out_plane = out.numel();
    CUtensorMap tmA, tmB;
    {   // weights: {K, Cout, 2}
        cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)d.Cout, 2};
        cuuint64_t str[2] = {(cuuint64_t)K * 2, (cuuint64_t)K * d.Cout * 2};
        cuuint32_t box[3] = {BKC, (cuuint32_t)BN, 1};
        if (make_map(&tmB, wq, 3, dims, str, box)) return -1;
    }
    a.Cout = d.Cout;
    a.n_tiles = pl.n_tiles;
    a.num_tiles = pl.num_tiles;
    a.kw = d.kw;
    a.kc_per_tap = d.Cin / BKC;
    a.num_kc = pl.num_kc;
    a.scale = out_f32 ? tc_aux : tc_aux + d.Cout;            // fp32 outputs in true units, planes in plane units
    a.shift = out_f32 ? d.shift : tc_aux + 2 * d.Cout;
    a.res = res_planes; a.out = out_planes; a.out_f32 = out_f32; a.out_plane = out_plane; a.relu = d.relu;
    a.Bimg = in.B;
    a.mode = pl.mode;
    a.M = pl.M;
    if (pl.gemm_kernel) {
        const long long Mtot = pl.M;
        a.pf = pl.pf;
        CUtensorMap tmR, tmO;
        {
            cuuint64_t dims[3] = {(cuuint64_t)d.Cin, (cuuint64_t)Mtot, 2};
            cuuint64_t str[2] = {(cuuint64_t)d.Cin * 2, (cuuint64_t)in_plane * 2};
            cuuint32_t box[3] = {BKC, BM, 1};
            if (make_map(&tmA, in_planes, 3, dims, str, box)) return -1;
        }
        if (conv_tc_map(&tmO, out_planes, pl, out, d.Cout, false)) return -1;
        if (conv_tc_map(&tmR, res_planes ? res_planes : out_planes, pl, out, d.Cout, false)) return -1;
        HN_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GSmem::TOTAL));
        HN_CUDA_OK(launch_tc(gemm_tc_kernel, pl.grid, GSmem::TOTAL, st, tmA, tmB, tmR, tmO, a));
        HN_LAUNCH_OK();
        return 0;
    }
    a.k1 = a.num_kc;
    if (pl.mode == 0) {
        cuuint64_t dims[3] = {(cuuint64_t)d.Cin, (cuuint64_t)pl.M, 2};
        cuuint64_t str[2] = {(cuuint64_t)d.Cin * 2, (cuuint64_t)in_plane * 2};
        cuuint32_t box[3] = {BKC, BM, 1};
        if (make_map(&tmA, in_planes, 3, dims, str, box)) return -1;
    } else {
        a.Ho = out.H; a.Wo = out.W; a.Wop = out.Wp(); a.out_halo = out.halo;
        a.tw = pl.tw;
        a.rows_per_tile = pl.rows_per_tile;
        a.wsegs = pl.wsegs;
        a.sh = d.sh; a.ph = d.ph; a.woff = in.halo - d.pw;
        a.parity = pl.parity;
        a.dxr = pl.dxr;
        if (conv_rows_map(&tmA, in_planes, in, d.Cin, d.sh, a.parity != 0, a.dxr != 0, pl)) return -1;
    }
    if (a.num_tiles == 0) return 0;
    CUtensorMap tmR, tmO;
    const bool f32 = out_f32 != nullptr;
    const void* obase = f32 ? static_cast<const void*>(out_f32) : static_cast<const void*>(out_planes);
    if (conv_tc_map(&tmO, obase, pl, out, d.Cout, f32)) return -1;
    if (conv_tc_map(&tmR, res_planes ? static_cast<const void*>(res_planes) : obase, pl, out, d.Cout, f32)) return -1;
    return launch_bn(BN, tmA, tmA, tmB, tmR, tmO, a, pl.grid, st);
}

// ---------------------------------------------------------------------- block-0 conv3 with the downsample folded in
// Plan of conv_tc_fold_planes: conv rows over the output geometry (the downsample's plan, stride 1 or 2), K chunks of t2
// then of x
int conv_tc_fold_plan(const Act& t2, const Act& x, int stride, const Act& out, int sms, TcPlan* p) {
    ConvDesc dd;
    memset(&dd, 0, sizeof(dd));
    dd.Cin = x.C; dd.Cout = out.C; dd.kh = dd.kw = 1; dd.sh = dd.sw = stride;
    HN_CHECK(stride == 1 || stride == 2, "conv_tc_fold: stride must be 1 or 2");
    HN_CHECK(t2.B == out.B && t2.H == out.H && t2.W == out.W && t2.halo == out.halo && x.B == out.B &&
             x.H == out.H * stride && x.W == out.W * stride && t2.C % 64 == 0,
             "conv_tc_fold: t2 must have the output geometry and x stride times its size");
    HN_CHECK(conv_channels_supported(dd, x) && conv_rows_supported(dd, x, out), "conv_tc_fold: unsupported shape");
    HN_CHECK(sms >= 1, "conv_tc_fold_plan: sms must be positive");
    memset(p, 0, sizeof(*p));
    p->BN = tile_bn(out.C, (long long)out.B * out.H * out.W);
    p->num_kc = (t2.C + x.C) / BKC;
    p->seg = SEG;
    const long long m_tiles = plan_rows(dd, x, out, false, p);
    p->n_tiles = out.C / p->BN;
    HN_CHECK(m_tiles * p->n_tiles < (1ll << 31), "conv_tc: too many tiles");
    p->num_tiles = (int)(m_tiles * p->n_tiles);
    p->grid = p->num_tiles < sms ? p->num_tiles : sms;
    return 0;
}

int conv_tc_fold_planes(const unsigned short* wq, const float* tc_aux, const Act& t2, const unsigned short* t2_planes,
                        const Act& x, const unsigned short* x_planes, int stride, const Act& out, unsigned short* out_planes,
                        cudaStream_t st) {
    TcPlan pl;
    if (conv_tc_fold_plan(t2, x, stride, out, num_sms(), &pl)) return -1;
    const int K = t2.C + x.C, Cout = out.C;
    TcArgs a;
    memset(&a, 0, sizeof(a));
    CUtensorMap tmA, tmA2, tmB, tmR, tmO;
    {   // folded weights: {K, Cout, 2}
        cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)Cout, 2};
        cuuint64_t str[2] = {(cuuint64_t)K * 2, (cuuint64_t)K * Cout * 2};
        cuuint32_t box[3] = {BKC, (cuuint32_t)pl.BN, 1};
        if (make_map(&tmB, wq, 3, dims, str, box)) return -1;
    }
    a.mode = 1; a.M = pl.M;
    a.Cout = Cout; a.n_tiles = pl.n_tiles; a.num_tiles = pl.num_tiles;
    a.kw = 1; a.kc_per_tap = t2.C / BKC; a.num_kc = pl.num_kc; a.k1 = t2.C / BKC;
    a.scale = tc_aux + Cout; a.shift = tc_aux + 2 * Cout;                // plane units
    a.out = out_planes; a.out_plane = out.numel(); a.relu = 1;
    a.Bimg = out.B;
    a.Ho = out.H; a.Wo = out.W; a.Wop = out.Wp(); a.out_halo = out.halo;
    a.tw = pl.tw; a.rows_per_tile = pl.rows_per_tile; a.wsegs = pl.wsegs;
    a.sh = 1; a.ph = 0; a.parity = 0; a.woff = t2.halo;
    a.sh2 = stride; a.parity2 = pl.parity; a.woff2 = x.halo;
    if (conv_rows_map(&tmA, t2_planes, t2, t2.C, 1, false, false, pl)) return -1;
    if (conv_rows_map(&tmA2, x_planes, x, x.C, stride, pl.parity != 0, false, pl)) return -1;
    if (a.num_tiles == 0) return 0;
    if (conv_tc_map(&tmO, out_planes, pl, out, Cout, false)) return -1;
    if (conv_tc_map(&tmR, out_planes, pl, out, Cout, false)) return -1;
    return launch_bn(pl.BN, tmA, tmA2, tmB, tmR, tmO, a, pl.grid, st);
}


// ---------------------------------------------------------------------- fused conv2 + conv3 of a bottleneck (host side)
bool bott_tc_supported(const ConvDesc& d2, const ConvDesc& d3, const Act& in, const Act& out) {
    return d2.kh == 3 && d2.kw == 3 && d2.sh == 1 && d2.sw == 1 && d2.ph == 1 && d2.pw == 1 && d2.Cin == 64 && d2.Cout == 64 &&
           d2.relu && d3.kh == 1 && d3.kw == 1 && d3.sh == 1 && d3.sw == 1 && d3.Cin == 64 && d3.Cout % 64 == 0 && d3.relu &&
           in.halo == 1 && out.halo == 1 && in.H == out.H && in.W == out.W && in.B == out.B && out.W % BM == 0 &&
           in.C == 64 && out.C == d3.Cout;
}

// in: conv2 input planes [B][H][W+2][64]; res / out: [B][H][W+2][C3] planes (res = the block's identity); wq2 / aux2, wq3 / aux3
// as produced by pack_weight_tc for the two convolutions.  Folded downsample instead of an identity (res_planes null):
// x_planes = the block input, in `in`'s geometry, and wq3 / aux3 the folded pack [2][C3][64 + 64] (conv_tc_fold_planes).
int bott_tc_planes(const ConvDesc& d2, const unsigned short* wq2, const float* aux2, const ConvDesc& d3,
                   const unsigned short* wq3, const float* aux3, const Act& in, const unsigned short* in_planes, const Act& out,
                   unsigned short* out_planes, const unsigned short* res_planes, const unsigned short* x_planes,
                   cudaStream_t st) {
    HN_CHECK(bott_tc_supported(d2, d3, in, out), "bott_tc: unsupported shape");
    HN_CHECK((res_planes != nullptr) != (x_planes != nullptr),
             "bott_tc: the fused kernel takes the block's identity or, folded, its input");
    const int fold = x_planes != nullptr;
    const int K3 = 64 * (1 + fold);
    const size_t in_plane = in.numel(), out_plane = out.numel();
    const cuuint64_t Wp = in.Wp();
    CUtensorMap tmA, tmB2, tmB3, tmR, tmX, tmO;
    {
        cuuint64_t dims[4] = {64, Wp, (cuuint64_t)in.H, (cuuint64_t)2 * in.B};
        cuuint64_t str[3] = {128, 128 * Wp, 128 * Wp * in.H};
        cuuint32_t box[4] = {BKC, 130, 1, 1};
        if (make_map(&tmA, in_planes, 4, dims, str, box)) return -1;
    }
    {
        cuuint64_t dims[3] = {576, 64, 2};
        cuuint64_t str[2] = {576 * 2, 576 * 64 * 2};
        cuuint32_t box[3] = {BKC, 64, 1};
        if (make_map(&tmB2, wq2, 3, dims, str, box)) return -1;
    }
    {
        cuuint64_t dims[3] = {(cuuint64_t)K3, (cuuint64_t)d3.Cout, 2};
        cuuint64_t str[2] = {(cuuint64_t)K3 * 2, (cuuint64_t)K3 * d3.Cout * 2};
        cuuint32_t box[3] = {BKC, 64, 1};
        if (make_map(&tmB3, wq3, 3, dims, str, box)) return -1;
    }
    {
        const cuuint64_t Mtot = (cuuint64_t)out.B * out.H * out.Wp();
        cuuint64_t dims[3] = {(cuuint64_t)d3.Cout, Mtot, 2};
        cuuint64_t str[2] = {(cuuint64_t)d3.Cout * 2, (cuuint64_t)out_plane * 2};
        cuuint32_t box[3] = {64, BM, 1};
        if (make_map(&tmO, out_planes, 3, dims, str, box)) return -1;
        if (make_map(&tmR, fold ? out_planes : res_planes, 3, dims, str, box)) return -1;
        cuuint64_t xdims[3] = {64, Mtot, 2};
        cuuint64_t xstr[2] = {128, (cuuint64_t)in_plane * 2};
        if (make_map(&tmX, fold ? x_planes : in_planes, 3, xdims, xstr, box)) return -1;
    }
    BottArgs a;
    memset(&a, 0, sizeof(a));
    a.Ho = out.H; a.Wo = out.W; a.Wop = out.Wp(); a.wsegs = out.W / BM; a.Bimg = in.B;
    const long long tiles = (long long)out.B * out.H * a.wsegs;
    HN_CHECK(tiles < (1ll << 31) && (long long)out.B * out.H * out.Wp() < (1ll << 31), "bott_tc: too many tiles");
    a.num_tiles = (int)tiles;
    a.n3 = d3.Cout / 64; a.C3 = d3.Cout;
    a.fold = fold;
    a.scale2 = aux2 + 64; a.shift2 = aux2 + 2 * 64;                        // plane units (conv_tc.cuh: tc_aux)
    a.scale3 = aux3 + d3.Cout; a.shift3 = aux3 + 2 * d3.Cout;
    a.out = out_planes; a.out_plane = out_plane;
    if (a.num_tiles == 0) return 0;
    HN_CUDA_OK(cudaFuncSetAttribute(bott_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BtSmem::TOTAL));
    int dev = 0, sms = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    HN_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    HN_CUDA_OK(launch_tc(bott_tc_kernel, a.num_tiles < sms ? a.num_tiles : sms, BtSmem::TOTAL, st, tmA, tmB2, tmB3, tmR, tmX,
                         tmO, a));
    HN_LAUNCH_OK();
    return 0;
}

// ---------------------------------------------------------------------- stem on tensor cores (host side)
size_t stem_tc_scratch_bytes(int B) { return (size_t)2 * B * SP_ROWS * SP_PAIRS * 16; }

int stem_tc_pack_weights(const float* w_oihw, float* pad_scratch, unsigned short* wq, const float* scale,
                         const float* shift, float* tc_aux, cudaStream_t st) {
    stem_weight_pad_kernel<<<(64 * SP_K + 255) / 256, 256, 0, st>>>(w_oihw, pad_scratch);
    HN_LAUNCH_OK();
    return pack_weight_tc(pad_scratch, wq, scale, shift, tc_aux, tc_aux + 3 * 64, 64, 4, 7, 8, st);
}

int stem_tc(const float* x_nchw, int B, int in_channels, const unsigned short* wq, const float* tc_aux,
            const float* shift, unsigned short* scratch, const Act& out, cudaStream_t st, bool relu) {
    HN_CHECK(in_channels >= 3, "stem: input needs >= 3 channels (reference model.py:252 uses x[:, :3])");
    HN_CHECK(out.B == B && out.H == 256 && out.W == 512 && out.C == 64 && out.halo == 1, "stem: bad output tensor");
    HN_CHECK(B >= 1 && B <= 2048, "stem: bad batch");
    const size_t total = (size_t)B * SP_ROWS * SP_PAIRS;
    stem_pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x_nchw, in_channels, scratch, B);
    HN_LAUNCH_OK();
    CUtensorMap tmA, tmB, tmO;
    {   // packed input: {64 = 8 pairs x 8 elements, 65 pair groups, 517 rows, 2 planes x B}
        cuuint64_t dims[4] = {64, SP_PAIRS / 8, SP_ROWS, (cuuint64_t)2 * B};
        cuuint64_t str[3] = {128, (cuuint64_t)SP_PAIRS * 16, (cuuint64_t)SP_ROWS * SP_PAIRS * 16};
        cuuint32_t box[4] = {64, 17, 7, 1};
        if (make_map(&tmA, scratch, 4, dims, str, box, -1, 1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, CU_TENSOR_MAP_SWIZZLE_NONE))
            return -1;
    }
    {   // weights: {K = 224, 64, 2}; the last 64-wide chunk is half out of bounds (zero filled, never multiplied)
        cuuint64_t dims[3] = {SP_K, 64, 2};
        cuuint64_t str[2] = {SP_K * 2, SP_K * 64 * 2};
        cuuint32_t box[3] = {BKC, 64, 1};
        if (make_map(&tmB, wq, 3, dims, str, box)) return -1;
    }
    {   // fp32 halo-NHWC output as {64 channels, B*256*514 pixels}
        cuuint64_t dims[2] = {64, (cuuint64_t)B * 256 * 514};
        cuuint64_t str[1] = {256};
        cuuint32_t box[2] = {32, 128};
        if (make_map(&tmO, out.p, 2, dims, str, box, -1, 1, CU_TENSOR_MAP_DATA_TYPE_FLOAT32)) return -1;
    }
    StemArgs a;
    a.B = B;
    a.num_tiles = B * 1024;
    a.scale = tc_aux;
    a.shift = shift;
    a.floor = relu ? 0.f : -INFINITY;       // no ReLU: the raw output the train-mode batch statistics are taken from
    HN_CUDA_OK(cudaFuncSetAttribute(stem_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, StSmem::TOTAL));
    int dev = 0, sms = 0;
    HN_CUDA_OK(cudaGetDevice(&dev));
    HN_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    HN_CUDA_OK(launch_tc(stem_tc_kernel, a.num_tiles < sms ? a.num_tiles : sms, StSmem::TOTAL, st, tmA, tmB, tmO, a));
    HN_LAUNCH_OK();
    return 0;
}

// ---------------------------------------------------------------------- format conversion kernels
namespace {

__global__ void split_kernel(const float* __restrict__ in, unsigned short* __restrict__ out, size_t n) {
    const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= n) return;
    const float4 v = *reinterpret_cast<const float4*>(in + i);
    const float f[4] = {v.x, v.y, v.z, v.w};
    unsigned short h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split_scaled(f[j], h[j], l[j]);
    *reinterpret_cast<uint2*>(out + i) = make_uint2(pack2(h[0], h[1]), pack2(h[2], h[3]));
    *reinterpret_cast<uint2*>(out + n + i) = make_uint2(pack2(l[0], l[1]), pack2(l[2], l[3]));
}

__global__ void merge_kernel(const unsigned short* __restrict__ in, float* __restrict__ out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = merge_scaled(in[i], in[n + i]);
}

__global__ void absmax_kernel(const float* __restrict__ w, size_t n, float* __restrict__ out) {
    float m = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(w[i]));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));   // m >= 0: int order = float order
}

// weight scale exponent t: max|w| * 2^t lands in (2^13, 2^14]: inside fp16 range, lo plane normal
__device__ __forceinline__ float weight_scale(float absmax) {
    if (!(absmax > 0.f) || !isfinite(absmax)) return 1.f;
    int e;
    frexpf(16384.f / absmax, &e);
    return ldexpf(1.f, e - 1);
}

// fp32 weights -> [2][Cout][K] planes of w * 2^t (fp16 hi, fp16 lo); source index from (n, k)
template <bool OIHW>
__global__ void pack_weight_tc_kernel(const float* __restrict__ w, unsigned short* __restrict__ out,
                                      const float* __restrict__ absmax, int Cout, int Cin, int kh, int kw) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t K = (size_t)Cin * kh * kw;
    const size_t total = (size_t)Cout * K;
    if (i >= total) return;
    const int n = (int)(i / K);
    const size_t k = i - (size_t)n * K;
    float v;
    if (OIHW) {
        const int c = (int)(k % Cin);
        const int tap = (int)(k / Cin);
        const int dy = tap / kw, dx = tap % kw;
        v = w[(((size_t)n * Cin + c) * kh + dy) * kw + dx];
    } else {
        v = w[k * Cout + n];                 // packed [K][Cout] (unit-test entry point)
    }
    const float s = v * weight_scale(*absmax);
    const __half h = __float2half_rn(s);
    out[i] = __half_as_ushort(h);
    out[total + i] = __half_as_ushort(__float2half_rn(s - __half2float(h)));
}

__global__ void tc_scale_kernel(const float* __restrict__ scale, const float* __restrict__ shift,
                                const float* __restrict__ absmax, float* __restrict__ tc_aux, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C) return;
    const float s = (scale ? scale[i] : 1.f) * ACT_UNSCALE / weight_scale(*absmax);   // accumulator -> true units
    tc_aux[i] = s;
    tc_aux[C + i] = s * ACT_SCALE;                                                    // accumulator -> plane units
    tc_aux[2 * C + i] = (shift ? shift[i] : 0.f) * ACT_SCALE;
}

template <bool OIHW>
int pack_weight_impl(const float* w, unsigned short* wq, const float* scale, const float* shift, float* tc_aux,
                     float* scratch, int Cout, int Cin, int kh, int kw, cudaStream_t st) {
    const size_t total = (size_t)Cout * Cin * kh * kw;
    HN_CUDA_OK(cudaMemsetAsync(scratch, 0, sizeof(float), st));
    // 4 elements per thread (the first version's 64 serial loads per thread cost 32 us per layer: 4.4 ms per training step)
    absmax_kernel<<<(unsigned)((total + 256 * 4 - 1) / (256 * 4)), 256, 0, st>>>(w, total, scratch);
    HN_LAUNCH_OK();
    pack_weight_tc_kernel<OIHW><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w, wq, scratch, Cout, Cin, kh, kw);
    HN_LAUNCH_OK();
    tc_scale_kernel<<<(Cout + 255) / 256, 256, 0, st>>>(scale, shift, scratch, tc_aux, Cout);
    HN_LAUNCH_OK();
    return 0;
}

}  // namespace

int split_planes(const float* in, unsigned short* out, size_t n, cudaStream_t st) {
    HN_CHECK(n % 4 == 0, "split_planes: element count must be a multiple of 4");
    if (n == 0) return 0;
    split_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, st>>>(in, out, n);
    HN_LAUNCH_OK();
    return 0;
}

int merge_planes(const unsigned short* in, float* out, size_t n, cudaStream_t st) {
    if (n == 0) return 0;
    merge_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, out, n);
    HN_LAUNCH_OK();
    return 0;
}

int pack_weight_tc(const float* w_oihw, unsigned short* wq, const float* scale, const float* shift, float* tc_aux,
                   float* scratch, int Cout, int Cin, int kh, int kw, cudaStream_t st) {
    return pack_weight_impl<true>(w_oihw, wq, scale, shift, tc_aux, scratch, Cout, Cin, kh, kw, st);
}

int tc_aux_update(const float* scale, const float* shift, const float* absmax, float* tc_aux, int Cout, cudaStream_t st) {
    tc_scale_kernel<<<(Cout + 255) / 256, 256, 0, st>>>(scale, shift, absmax, tc_aux, Cout);
    HN_LAUNCH_OK();
    return 0;
}

// Unit-test convenience: fp32 halo-NHWC in and out, planes built on the fly; out_f32: the kernel's fp32 epilogue writes
// `out` directly (true-unit scale, d.shift) instead of planes that are merged afterwards.
int conv_tc(const ConvDesc& d, const Act& in, const Act& out, const float* residual, bool out_f32, cudaStream_t st) {
    HN_CHECK(conv_tc_supported(d, in, out), "conv_tc: unsupported shape");
    HN_CHECK(!(out_f32 && residual), "conv_tc: residual with fp32 output is not supported");
    const size_t K = (size_t)d.kh * d.kw * d.Cin;
    const size_t n_in = in.numel(), n_out = out.numel(), n_w = K * d.Cout;
    unsigned short *pin = nullptr, *pout = nullptr, *pres = nullptr, *pw = nullptr;
    float* aux = nullptr;          // [3*Cout] tc_aux + 1 scratch float
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&pin), n_in * 4, st));
    if (!out_f32) {   // all-ones fp16 = NaN: an output plane element the kernel leaves unwritten merges to NaN
        HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&pout), n_out * 4, st));
        HN_CUDA_OK(cudaMemsetAsync(pout, 0xff, n_out * 4, st));
    }
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&pw), n_w * 4, st));
    HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&aux), (3 * d.Cout + 1) * sizeof(float), st));
    if (residual) HN_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&pres), n_out * 4, st));
    int rc = split_planes(in.p, pin, n_in, st);
    if (!rc && residual) rc = split_planes(residual, pres, n_out, st);
    if (!rc) rc = pack_weight_impl<false>(d.w, pw, d.scale, d.shift, aux, aux + 3 * d.Cout, d.Cout, d.Cin, d.kh, d.kw, st);
    if (!rc) rc = conv_tc_planes(d, pw, aux, in, pin, out, pout, out_f32 ? out.p : nullptr, pres, st);
    if (!rc && !out_f32) rc = merge_planes(pout, out.p, n_out, st);
    cudaFreeAsync(pin, st); cudaFreeAsync(pw, st); cudaFreeAsync(aux, st);
    if (pout) cudaFreeAsync(pout, st);
    if (pres) cudaFreeAsync(pres, st);
    return rc;
}

// Unit-test conveniences of the folded conv3 and of the fused layer1 bottleneck: fp32 halo-NHWC tensors in and out,
// planes and packed weights built on the fly.  `bufs` holds the device allocations, freed on every path.
namespace {
struct DevBufs {
    cudaStream_t st;
    std::vector<void*> p;
    template <typename T>
    T* get(size_t n) {
        void* q = nullptr;
        if (cudaMallocAsync(&q, n * sizeof(T), st) != cudaSuccess) return nullptr;
        p.push_back(q);
        return static_cast<T*>(q);
    }
    ~DevBufs() { for (void* q : p) cudaFreeAsync(q, st); }
};
}  // namespace

int conv_tc_fold(const float* w, const float* shift, const Act& t2, const Act& x, int stride, const Act& out,
                 cudaStream_t st) {
    TcPlan pl;
    if (conv_tc_fold_plan(t2, x, stride, out, 1, &pl)) return -1;
    const int K = t2.C + x.C;
    DevBufs b{st, {}};
    unsigned short *pt = b.get<unsigned short>(2 * t2.numel()), *px = b.get<unsigned short>(2 * x.numel());
    unsigned short *po = b.get<unsigned short>(2 * out.numel()), *pw = b.get<unsigned short>((size_t)2 * K * out.C);
    float* aux = b.get<float>(3 * out.C + 1);
    HN_CHECK(pt && px && po && pw && aux, "conv_tc_fold: out of device memory");
    HN_CUDA_OK(cudaMemsetAsync(po, 0xff, out.numel() * 4, st));     // NaN: an element the kernel leaves unwritten
    if (split_planes(t2.p, pt, t2.numel(), st) || split_planes(x.p, px, x.numel(), st)) return -1;
    if (pack_weight_impl<true>(w, pw, nullptr, shift, aux, aux + 3 * out.C, out.C, K, 1, 1, st)) return -1;
    if (conv_tc_fold_planes(pw, aux, t2, pt, x, px, stride, out, po, st)) return -1;
    return merge_planes(po, out.p, out.numel(), st);
}

int bott_tc_f32(const float* w2, const float* scale2, const float* shift2, const float* w3, const float* scale3,
                const float* shift3, const Act& in, const float* res, const float* x, const Act& out, cudaStream_t st) {
    ConvDesc d2, d3;
    memset(&d2, 0, sizeof(d2));
    d2.Cin = d2.Cout = 64; d2.kh = d2.kw = 3; d2.sh = d2.sw = 1; d2.ph = d2.pw = 1; d2.relu = 1;
    d3 = d2;
    d3.Cout = out.C; d3.kh = d3.kw = 1; d3.ph = d3.pw = 0;
    HN_CHECK(bott_tc_supported(d2, d3, in, out), "bott_tc_f32: unsupported shape");
    HN_CHECK((res != nullptr) != (x != nullptr), "bott_tc_f32: pass the block's identity or, folded, its input");
    const size_t n2 = x ? in.numel() : out.numel();           // the second source: x in in's geometry, res in out's
    const int K3 = x ? 128 : 64;
    DevBufs b{st, {}};
    unsigned short *pi = b.get<unsigned short>(2 * in.numel()), *p2 = b.get<unsigned short>(2 * n2);
    unsigned short *po = b.get<unsigned short>(2 * out.numel());
    unsigned short *pw2 = b.get<unsigned short>(2 * 64 * 576), *pw3 = b.get<unsigned short>((size_t)2 * out.C * K3);
    float *aux2 = b.get<float>(3 * 64 + 1), *aux3 = b.get<float>(3 * out.C + 1);
    HN_CHECK(pi && p2 && po && pw2 && pw3 && aux2 && aux3, "bott_tc_f32: out of device memory");
    HN_CUDA_OK(cudaMemsetAsync(po, 0xff, out.numel() * 4, st));
    if (split_planes(in.p, pi, in.numel(), st) || split_planes(x ? x : res, p2, n2, st)) return -1;
    if (pack_weight_impl<true>(w2, pw2, scale2, shift2, aux2, aux2 + 3 * 64, 64, 64, 3, 3, st)) return -1;
    if (pack_weight_impl<true>(w3, pw3, scale3, shift3, aux3, aux3 + 3 * out.C, out.C, K3, 1, 1, st)) return -1;
    if (bott_tc_planes(d2, pw2, aux2, d3, pw3, aux3, in, pi, out, po, x ? nullptr : p2, x ? p2 : nullptr, st)) return -1;
    return merge_planes(po, out.p, out.numel(), st);
}

}  // namespace hn
