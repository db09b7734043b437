// b200sd -- shared device/host helpers for the sm_90a kernels (inline PTX wrappers for
// mbarrier, TMA, wgmma; host-side tensor-map encoding; error plumbing).
#pragma once

#include <cuda.h>
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
// bytes for dims 1..rank-1.  Returns 0 on success.
int encode_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides);

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
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define B200SD_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// D[64 x N] (+)= A[64 x 16] (smem, K-major) * B[N x 16]^T (smem, K-major unless trans_b); fp16 in, fp32 accumulate.
// Accumulator layout (thread t of the warpgroup): d[4 j + e] = (row 16 (t / 32) + (t % 32) / 4 + 8 (e / 2),
// column 8 j + 2 (t % 4) + e % 2).
template <int kTransB = 0>
__device__ __forceinline__ void wgmma_m64n64_ss(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, %35;\n\t}\n"
        : B200SD_F8(0), B200SD_F8(8), B200SD_F8(16), B200SD_F8(24)
        : "l"(da), "l"(db), "r"(acc), "n"(kTransB)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n32_ss(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
        : B200SD_F8(0), B200SD_F8(8)
        : "l"(da), "l"(db), "r"(acc)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n16_ss(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
        : B200SD_F8(0)
        : "l"(da), "l"(db), "r"(acc)
        : "memory");
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
#undef B200SD_F8

// D[64 x bn] (+)= A[64 x 16] * B[bn x 16]^T as 64 / 32 / 16-column pieces (bn: multiple of 16, <= 2 R).  The pieces'
// accumulators are consecutive in `d`, so d keeps the layout of one 64 x bn accumulator.  Every index is a compile-time
// constant: d stays in registers.
template <int R>
__device__ __forceinline__ void wgmma_rows64(float (&d)[R], int bn, uint64_t da, uint64_t db, uint32_t acc) {
#pragma unroll
    for (int c = 0; c + 64 <= 2 * R; c += 64)
        if (c + 64 <= bn) wgmma_m64n64_ss(d + c / 2, da, db + (c * 128 >> 4), acc);
    const int c32 = bn & ~63;
#pragma unroll
    for (int c = 0; c + 32 <= 2 * R; c += 64)
        if (c == c32 && (bn & 32)) wgmma_m64n32_ss(d + c / 2, da, db + (c * 128 >> 4), acc);
    const int c16 = bn & ~31;
#pragma unroll
    for (int c = 0; c + 16 <= 2 * R; c += 32)
        if (c == c16 && (bn & 16)) wgmma_m64n16_ss(d + c / 2, da, db + (c * 128 >> 4), acc);
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
#endif  // __CUDACC__

}  // namespace b200sd
