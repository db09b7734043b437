// b200sd -- shared device/host helpers for the sm_90a kernels (inline PTX wrappers for
// mbarrier, TMA, wgmma; host-side tensor-map encoding; error plumbing).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace b200sd {

// ---------------------------------------------------------------------------------------
// error plumbing (C-ABI returns int status; message via b200sd_last_error)
// ---------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);

#define B200SD_CHECK_CUDA(expr)                                                            \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess) {                                                           \
            ::b200sd::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),    \
                                __FILE__, __LINE__);                                       \
            return 1;                                                                      \
        }                                                                                  \
    } while (0)

#define B200SD_REQUIRE(cond, ...)                                                          \
    do {                                                                                   \
        if (!(cond)) {                                                                     \
            ::b200sd::set_error(__VA_ARGS__);                                              \
            return 2;                                                                      \
        }                                                                                  \
    } while (0)

// Encodes a tiled fp16 tensor map (SWIZZLE_128B).  dims/strides innermost first; strides in
// bytes for dims 1..rank-1.  Returns 0 on success.  bf16 tensors use the same encoding: TMA only copies bytes, both
// types are two bytes wide and the out-of-bounds zero fill (0x0000) is +0 in both.
int encode_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides);
// The same encoding for any element type (UINT8 for the int8 convolution: its zero fill is 0 as well).
// swizzle: SWIZZLE_NONE for boxes that are not operand tiles (the packed palette indices of b200sd_gemm_lut).
int encode_tmap(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides,
                CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B);

int num_sms();

// Programmatic dependent launch (PDL): when enabled every kernel is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, so the next kernel's CTAs may start (and run their
// prologue: barrier init, tensor-map prefetch) while the previous grid drains; every kernel
// executes griddepcontrol.wait before it reads or writes global memory.
bool pdl_enabled();

// Launch classes (1 GEMM / convolution, 2 attention, 4 normalisation, 8 elementwise): bench.py captures graphs with only
// one class enabled to attribute the step time per kernel class without event gaps or profiler serialisation.
bool launch_class_enabled(int cls);

#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    if (pdl_enabled()) {
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
    }
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------
// griddepcontrol.wait: block until the preceding grid in the stream has completed and its memory is visible
// (no-op when the kernel was not launched as a programmatic dependent).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// griddepcontrol.launch_dependents: this CTA no longer objects to the next grid being scheduled.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

// L2 cache-policy constants (same encodings CUTLASS uses for createpolicy results)
static constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
static constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
static constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4, %5}], [%2], %6;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(hint)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(hint)
        : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA: 128 threads, fp32 accumulators in registers) ------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Register reallocation between warpgroups: a warpgroup returns registers to the CTA's pool (dec) or waits for them
// (inc).  Every warp of the warpgroup executes the same instruction; N is a multiple of 8 in [24, 256].
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define B200SD_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// D[64 x N] (+)= A[64 x 16] (smem, K-major) * B[N x 16]^T (smem, K-major) as ONE wgmma; 16-bit operands of type T
// (fp16, or bf16 for the VAEs whose activations overflow fp16), fp32 accumulate.
// N / 2 accumulators per thread (thread t of the warpgroup): d[4 j + e] = (row 16 (t / 32) + (t % 32) / 4 + 8 (e / 2),
// column 8 j + 2 (t % 4) + e % 2).  Specialised for the widths the kernels issue.
template <int N, typename T = __half>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db, uint32_t acc);
// one specialisation per (width, operand type): TY is the PTX type of both operands
#define B200SD_WGMMA_SS(N, T, TY, REGS, IP, IA, IB, ...)                                                             \
    template <>                                                                                                      \
    __device__ __forceinline__ void wgmma_ss<N, T>(float* d, uint64_t da, uint64_t db, uint32_t acc) {               \
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IP ", 0;\n\t"                                          \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " {" REGS "}, %" #IA ", %" #IB        \
                     ", p, 1, 1, 0, 0;\n\t}\n"                                                                         \
                     : __VA_ARGS__                                                                                   \
                     : "l"(da), "l"(db), "r"(acc)                                                                    \
                     : "memory");                                                                                    \
    }
#define B200SD_WGMMA_SS_BOTH(N, REGS, IP, IA, IB, ...)                  \
    B200SD_WGMMA_SS(N, __half, "f16", REGS, IP, IA, IB, __VA_ARGS__)   \
    B200SD_WGMMA_SS(N, __nv_bfloat16, "bf16", REGS, IP, IA, IB, __VA_ARGS__)
B200SD_WGMMA_SS_BOTH(16,
                     "%0, %1, %2, %3, %4, %5, %6, %7",
                     10, 8, 9, B200SD_F8(0))
B200SD_WGMMA_SS_BOTH(32,
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15",
                     18, 16, 17, B200SD_F8(0), B200SD_F8(8))
B200SD_WGMMA_SS_BOTH(64,
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31",
                     34, 32, 33, B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24))
B200SD_WGMMA_SS_BOTH(96,
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47",
                     50, 48, 49, B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24), B200SD_F8(32), B200SD_F8(40))
B200SD_WGMMA_SS_BOTH(128,
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63",
                     66, 64, 65, B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24), B200SD_F8(32), B200SD_F8(40), B200SD_F8(48), B200SD_F8(56))
B200SD_WGMMA_SS_BOTH(160,
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
                     "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79",
                     82, 80, 81, B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24), B200SD_F8(32), B200SD_F8(40), B200SD_F8(48), B200SD_F8(56), B200SD_F8(64), B200SD_F8(72))
B200SD_WGMMA_SS_BOTH(192,
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
                     "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
                     "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95",
                     98, 96, 97, B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24), B200SD_F8(32), B200SD_F8(40), B200SD_F8(48), B200SD_F8(56), B200SD_F8(64), B200SD_F8(72), B200SD_F8(80), B200SD_F8(88))
B200SD_WGMMA_SS_BOTH(256,
                     "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                     "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                     "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                     "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
                     "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
                     "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
                     "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
                     "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127",
                     130, 128, 129, B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24), B200SD_F8(32), B200SD_F8(40), B200SD_F8(48), B200SD_F8(56), B200SD_F8(64), B200SD_F8(72), B200SD_F8(80), B200SD_F8(88), B200SD_F8(96), B200SD_F8(104), B200SD_F8(112), B200SD_F8(120))
#undef B200SD_WGMMA_SS_BOTH
#undef B200SD_WGMMA_SS

// D[64 x N] (+)= A[64 x 32] * B[N x 32]^T with signed int8 operands (K-major, smem) and int32 accumulators: the same
// 32-byte k step and the same accumulator layout as wgmma_ss<N> (IGMMA in SASS).
template <int N>
__device__ __forceinline__ void wgmma_ss_s8(int32_t* d, uint64_t da, uint64_t db, uint32_t acc);
#define B200SD_I8(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), "+r"(d[i + 6]), "+r"(d[i + 7])
#define B200SD_WGMMA_S8(N, REGS, IP, IA, IB, ...)                                                                    \
    template <>                                                                                                      \
    __device__ __forceinline__ void wgmma_ss_s8<N>(int32_t* d, uint64_t da, uint64_t db, uint32_t acc) {             \
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IP ", 0;\n\t"                                          \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k32.s32.s8.s8 {" REGS "}, %" #IA ", %" #IB ", p;\n\t}\n"  \
                     : __VA_ARGS__                                                                                   \
                     : "l"(da), "l"(db), "r"(acc)                                                                    \
                     : "memory");                                                                                    \
    }
#define B200SD_R16 "%0, %1, %2, %3, %4, %5, %6, %7"
#define B200SD_R32 B200SD_R16 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define B200SD_R64 B200SD_R32 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define B200SD_R96 B200SD_R64 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define B200SD_R128 B200SD_R96 ", %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define B200SD_R160 B200SD_R128 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
#define B200SD_R192 B200SD_R160 ", %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define B200SD_R256 B200SD_R192 ", %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, " \
    "%111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
B200SD_WGMMA_S8(16, B200SD_R16, 10, 8, 9, B200SD_I8(0))
B200SD_WGMMA_S8(32, B200SD_R32, 18, 16, 17, B200SD_I8(0), B200SD_I8(8))
B200SD_WGMMA_S8(64, B200SD_R64, 34, 32, 33, B200SD_I8(0), B200SD_I8(8), B200SD_I8(16), B200SD_I8(24))
B200SD_WGMMA_S8(96, B200SD_R96, 50, 48, 49, B200SD_I8(0), B200SD_I8(8), B200SD_I8(16), B200SD_I8(24), B200SD_I8(32),
                B200SD_I8(40))
B200SD_WGMMA_S8(128, B200SD_R128, 66, 64, 65, B200SD_I8(0), B200SD_I8(8), B200SD_I8(16), B200SD_I8(24), B200SD_I8(32),
                B200SD_I8(40), B200SD_I8(48), B200SD_I8(56))
B200SD_WGMMA_S8(160, B200SD_R160, 82, 80, 81, B200SD_I8(0), B200SD_I8(8), B200SD_I8(16), B200SD_I8(24), B200SD_I8(32),
                B200SD_I8(40), B200SD_I8(48), B200SD_I8(56), B200SD_I8(64), B200SD_I8(72))
B200SD_WGMMA_S8(192, B200SD_R192, 98, 96, 97, B200SD_I8(0), B200SD_I8(8), B200SD_I8(16), B200SD_I8(24), B200SD_I8(32),
                B200SD_I8(40), B200SD_I8(48), B200SD_I8(56), B200SD_I8(64), B200SD_I8(72), B200SD_I8(80), B200SD_I8(88))
B200SD_WGMMA_S8(256, B200SD_R256, 130, 128, 129, B200SD_I8(0), B200SD_I8(8), B200SD_I8(16), B200SD_I8(24), B200SD_I8(32),
                B200SD_I8(40), B200SD_I8(48), B200SD_I8(56), B200SD_I8(64), B200SD_I8(72), B200SD_I8(80), B200SD_I8(88),
                B200SD_I8(96), B200SD_I8(104), B200SD_I8(112), B200SD_I8(120))
#undef B200SD_R256
#undef B200SD_R192
#undef B200SD_R160
#undef B200SD_R128
#undef B200SD_R96
#undef B200SD_R64
#undef B200SD_R32
#undef B200SD_R16
#undef B200SD_WGMMA_S8
#undef B200SD_I8
template <int R>
__device__ __forceinline__ void wgmma_fence_regs_s32(int32_t* d) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// A from registers (fp16 pairs in the accumulator layout of a 64 x 16 tile), B [16 x 64] from smem, MN-major
__device__ __forceinline__ void wgmma_m64n64_rs_tb(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n"
        : B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc)
        : "memory");
}
// the same for B [16 x N], N = 64 / 128 / 192 (one, two or three 64-wide MN chunks, LBO apart)
template <int N>
__device__ __forceinline__ void wgmma_rs_tb(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t acc);
template <>
__device__ __forceinline__ void wgmma_rs_tb<64>(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    wgmma_m64n64_rs_tb(d, a, db, acc);
}
template <>
__device__ __forceinline__ void wgmma_rs_tb<128>(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 1;\n\t}\n"
        : B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24), B200SD_F8(32), B200SD_F8(40), B200SD_F8(48), B200SD_F8(56)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc)
        : "memory");
}
template <>
__device__ __forceinline__ void wgmma_rs_tb<192>(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %101, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, "
        "{%96, %97, %98, %99}, %100, p, 1, 1, 1;\n\t}\n"
        : B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24), B200SD_F8(32), B200SD_F8(40), B200SD_F8(48), B200SD_F8(56),
          B200SD_F8(64), B200SD_F8(72), B200SD_F8(80), B200SD_F8(88)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc)
        : "memory");
}
#undef B200SD_F8

// D[64 x bn] (+)= A[64 x 16] * B[bn x 16]^T as 64 / 32 / 16-column pieces for a RUNTIME width (bn: multiple of 16,
// <= 2 R; the halo kernels).  The pieces' accumulators are consecutive in `d`, so d keeps the layout of one 64 x bn
// accumulator.  The accumulators are written by predicated asm, so ptxas serialises the wgmma pipeline (each wgmma
// waits for the previous one); the GEMM kernel issues one wgmma_ss<kBN> per k16 step instead.
template <int R>
__device__ __forceinline__ void wgmma_rows64(float (&d)[R], int bn, uint64_t da, uint64_t db, uint32_t acc) {
#pragma unroll
    for (int c = 0; c + 64 <= 2 * R; c += 64)
        if (c + 64 <= bn) wgmma_ss<64>(d + c / 2, da, db + (c * 128 >> 4), acc);
    const int c32 = bn & ~63;
#pragma unroll
    for (int c = 0; c + 32 <= 2 * R; c += 64)
        if (c == c32 && (bn & 32)) wgmma_ss<32>(d + c / 2, da, db + (c * 128 >> 4), acc);
    const int c16 = bn & ~31;
#pragma unroll
    for (int c = 0; c + 16 <= 2 * R; c += 32)
        if (c == c16 && (bn & 16)) wgmma_ss<16>(d + c / 2, da, db + (c * 128 >> 4), acc);
}

// ---- wgmma shared-memory matrix descriptors -------------------------------------------------------------
// SWIZZLE_128B (layout type 1 in bits 62-63).
//   K-major tile  : rows of 128 B (64 fp16 along K), 8-row swizzle atoms 1024 B apart (SBO=1024),
//                   LBO unused (single atom along K).  +32 B (desc + 2) per K=16 step.
//   MN-major tile : rows of 128 B (64 fp16 along MN) indexed by k; 8-k atoms 1024 B apart (SBO=1024);
//                   LBO = byte distance between successive 64-wide MN chunks.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t sbo_bytes, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= static_cast<uint64_t>(1) << 62;  // SWIZZLE_128B
    return d;
}

// 2^x, single MUFU op, denormal results flushed to zero (softmax probabilities)
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// exact-erf GELU (unet.py:617 F.gelu default).  erf via Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, far below
// the fp16 output rounding): 1 MUFU.RCP + 1 MUFU.EX2 + ~10 FMA instead of libdevice erff's ~40 instructions --
// the GEGLU epilogue evaluates 128 of these per thread per tile and was the bottleneck of those GEMMs.
__device__ __forceinline__ float erf_as(float x) {
    const float ax = fabsf(x);
    float t;  // 1 / (1 + p |x|): MUFU.RCP (1 ulp) -- __frcp_rn would add an IEEE fix-up sequence
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, ax, 1.0f)));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    poly *= t;
    const float e = ex2_approx(-ax * ax * 1.4426950408889634f);
    const float r = fmaf(-poly, e, 1.0f);
    return copysignf(r, x);
}
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erf_as(x * 0.70710678118654752f)); }

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// The 16-bit activation types: fp16 everywhere, bf16 (fp32's exponent range) for the VAEs whose activations exceed
// fp16's 65504.  Conversions in the form the fp16 kernels were written in, so their fp16 code is unchanged.
// W8A8 activation quantization of eight fp32 values: q = clamp(rint(y * inv_scale), -127, 127), packed little-endian
__device__ __forceinline__ uint2 quantize8_s8(const float (&f)[8], float inv_scale) {
    uint32_t w[2] = {0u, 0u};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int q = min(127, max(-127, __float2int_rn(f[e] * inv_scale)));
        w[e >> 2] |= (static_cast<uint32_t>(q) & 0xffu) << (8 * (e & 3));
    }
    return make_uint2(w[0], w[1]);
}

template <typename T>
struct Elem16;
template <>
struct Elem16<__half> {
    using T2 = __half2;
    static __device__ __forceinline__ float2 to_float2(T2 v) { return __half22float2(v); }
    static __device__ __forceinline__ float to_float(__half v) { return __half2float(v); }
    static __device__ __forceinline__ __half from_float(float v) { return __float2half_rn(v); }
    static __device__ __forceinline__ uint32_t pack2(float a, float b) { return pack_half2(a, b); }
};
template <>
struct Elem16<__nv_bfloat16> {
    using T2 = __nv_bfloat162;
    static __device__ __forceinline__ float2 to_float2(T2 v) { return __bfloat1622float2(v); }
    static __device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ __nv_bfloat16 from_float(float v) { return __float2bfloat16_rn(v); }
    static __device__ __forceinline__ uint32_t pack2(float a, float b) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
};
#endif  // __CUDACC__

}  // namespace b200sd
