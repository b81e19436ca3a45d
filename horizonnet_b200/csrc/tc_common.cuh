// wgmma / TMA PTX wrappers and the host-side tensor-map + launch helpers shared by the tensor-core kernels of this
// library (conv_tc.cu: forward convolutions and data gradients; wgrad_tc.cu: weight gradients).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdlib>
#include <map>
#include <mutex>
#include <string>
#include <utility>

#include "hn_common.cuh"
#include "ptx.cuh"

namespace hn {
namespace tc {

constexpr int BM = 128;            // rows of an accumulator tile = two m64 wgmma blocks
constexpr int NTHREADS = 384;      // warp 0 TMA producer (warps 1-3 idle), warpgroups 1 and 2 MMA + epilogue

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
        "r"(c4)
        : "memory");
}

// Programmatic dependent launch: the next kernel of the stream may be scheduled while this one still runs (its CTAs take
// over an SM as soon as ours exit, set up barriers / tensor-map prefetch there) and blocks in pdl_wait() until this
// grid has completed and flushed: the kernel boundaries of a forward stop costing a launch latency + prologue each.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Dynamic tile scheduling of the persistent kernels.  A CTA does not own a fixed share of the tiles: its producer
// thread claims one tile at a time from a global counter (`sched`, see tile_counter) and hands the index to the other
// roles of the CTA through this queue, in claim order.  CTAs that become resident late -- while the LSTM recurrence of
// another stream holds part of the GPU -- therefore find less work left, and the launch ends when the tiles run out
// rather than when the last CTA has worked through a share fixed at launch.  The tile-to-CTA assignment changes no
// arithmetic: every tile is computed exactly as before.  The producer pushes one index past the last tile as the end
// marker.  Kept in the barrier area of the kernel's shared memory (80 bytes).
struct TileQueue {
    static constexpr int N = 4;
    uint64_t full[N];         // the index of slot i has been written
    uint64_t empty[N];        // every reader has taken it
    int tile[N];
    __device__ __forceinline__ void init(uint32_t readers) {
        for (int i = 0; i < N; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, readers); }
    }
    // producer, it-th claim: waits for a free slot, claims the next tile of the launch, publishes it
    __device__ __forceinline__ int claim(int it, unsigned* sched) {
        const int s = it % N;
        mbar_wait(empty + s, ((it / N) & 1) ^ 1);
        const int t = (int)atomicAdd(sched, 1u);
        tile[s] = t;
        mbar_arrive(full + s);
        return t;
    }
    // reader, it-th index; every reading warp then calls release(it) once (after __syncwarp)
    __device__ __forceinline__ int next(int it) {
        const int s = it % N;
        mbar_wait(full + s, (it / N) & 1);
        return *static_cast<volatile int*>(tile + s);
    }
    __device__ __forceinline__ void release(int it) { mbar_arrive(empty + it % N); }
};
static_assert(sizeof(TileQueue) <= 128, "the kernels keep the queue in the upper 128 bytes of a 256-byte barrier area");
// The producer of each CTA calls this once, after the claim that returned the end marker.  The last CTA to get
// there resets the counter for the next launch on the stream, which reads it only after pdl_wait(), i.e. after
// this grid has completed and flushed.
__device__ __forceinline__ void sched_retire(unsigned* sched) {
    __threadfence();          // this CTA's claims come before its retirement
    if (atomicAdd(sched + 1, 1u) == gridDim.x - 1) {
        atomicExch(sched, 0u);
        atomicExch(sched + 1, 0u);
    }
}

// 128-byte swizzle shared-memory matrix descriptor of wgmma (sm_90 layout: start address bits [0,14), leading byte
// offset [16,30), stride byte offset [32,46), layout type [62,64) = 1 for SWIZZLE_128B).  K-major operands: rows of
// 128 B, 8-row atoms 1024 B apart (sbo), lbo unused.  MN-major operands: lbo = distance between 64-element atoms along
// M/N, sbo = distance between 8-row groups along K.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo = 16, uint32_t sbo = 1024) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo & 0x3FFFF) >> 4) << 16;
    d |= (uint64_t)((sbo & 0x3FFFF) >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// K-major operand without swizzle (layout type 0): 8-row x 16-byte core matrices, `lbo` bytes between the two core
// matrices of a K = 16 step, `sbo` bytes between 8-row groups
__device__ __forceinline__ uint64_t gmma_desc_interleave(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo & 0x3FFFF) >> 4) << 16;
    d |= (uint64_t)((sbo & 0x3FFFF) >> 4) << 32;
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// the accumulator registers must not be touched by other instructions while a wgmma that writes them is in flight
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 operands from shared memory, fp32 accumulator fragment in registers
// (d[4j + e]: row lane/4 + 8*(e/2) of the warp's 16 rows, column 8j + 2*(lane%4) + e%2).  acc = 0 overwrites D.
// TA / TB = 1: the operand is MN-major (transposed).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}

__device__ __forceinline__ uint32_t pack2(unsigned short a, unsigned short b) {
    return (uint32_t)a | ((uint32_t)b << 16);
}

// -------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

inline int make_map(CUtensorMap* tm, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
             const cuuint32_t* box, int stride_dim = -1, int stride = 1,
             CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
             CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    EncodeTiledFn fn = encode_fn();
    HN_CHECK(fn != nullptr, "conv_tc: cuTensorMapEncodeTiled unavailable");
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    if (stride_dim >= 0) estr[stride_dim] = (cuuint32_t)stride;      // traversal stride: every stride-th element of the box span
    CUresult r = fn(tm, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes,
                    box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("conv_tc: cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return 0;
}

inline bool pdl_on() {
    static const bool on = [] { const char* e = getenv("HN_TC_PDL"); return !(e && atoi(e) == 0); }();
    return on;
}

// Tile counter (TileQueue::claim, sched_retire) of the persistent kernels launched on stream `st`: two unsigned ints,
// zero between launches.  One per (device, stream): launches on one stream run one after the other (the next one
// claims only after pdl_wait), launches on different streams -- the encoder and recurrence streams of the pipelined
// forward -- may run at the same time and must not share a counter.
inline cudaError_t tile_counter(cudaStream_t st, unsigned** out) {
    static std::mutex mu;
    static std::map<std::pair<int, unsigned long long>, unsigned*> counters;
    int dev = 0;
    unsigned long long id = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaStreamGetId(st, &id);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    unsigned*& c = counters[{dev, id}];
    if (!c) {
        e = cudaMalloc(reinterpret_cast<void**>(&c), 2 * sizeof(unsigned));
        if (e == cudaSuccess) e = cudaMemsetAsync(c, 0, 2 * sizeof(unsigned), st);
        if (e != cudaSuccess) { c = nullptr; return e; }
    }
    *out = c;
    return cudaSuccess;
}

// launch of a persistent tensor-core kernel with programmatic stream serialisation (see pdl_trigger / pdl_wait); the
// kernel's last parameter is the stream's tile counter
template <typename K, typename... Args>
inline cudaError_t launch_tc(K kernel, int grid, size_t smem_bytes, cudaStream_t st, Args... args) {
    unsigned* sched = nullptr;
    const cudaError_t e = tile_counter(st, &sched);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(NTHREADS);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl_on() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, args..., sched);
}

}  // namespace tc
}  // namespace hn
