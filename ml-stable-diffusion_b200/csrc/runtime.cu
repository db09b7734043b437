// b200sd -- host runtime glue: error string, launch counter, device query, TMA tensor-map encoding.
#include "common.cuh"
#include "../../include/b200sd.h"

#include <atomic>
#include <mutex>
#include <stdarg.h>
#include <stdlib.h>

namespace b200sd {

static thread_local char g_error[1024] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }

static int g_pdl = -1;
static std::atomic<uint32_t> g_class_mask{0xFu};

bool launch_class_enabled(int cls) { return (g_class_mask.load(std::memory_order_relaxed) & static_cast<uint32_t>(cls)) != 0; }


bool pdl_enabled() {
    if (g_pdl < 0) {
        const char* e = getenv("B200SD_PDL");
        // on by default (B200SD_PDL=0 disables): every kernel executes griddepcontrol.wait before it touches global
        // memory and releases its dependents early, so the next kernel's prologue overlaps this one's tail
        g_pdl = (e != nullptr && e[0] == '0') ? 0 : 1;
    }
    return g_pdl == 1;
}

int num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    }
    return sms;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        // resolved through the runtime so the library has no link-time dependency on libcuda
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int encode_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, const uint32_t* elem_strides) {
    return encode_tmap(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base, rank, dims, strides_bytes, box, elem_strides);
}

int encode_tmap(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides, CUtensorMapSwizzle swizzle) {
    EncodeTiledFn fn = get_encode_fn();
    B200SD_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
    B200SD_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor map base %p is not 16-byte aligned", base);
    cuuint64_t gd[5], gs[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) {
        gd[i] = dims[i];
        bx[i] = box[i];
        es[i] = elem_strides[i];
        if (i + 1 < rank) {
            gs[i] = strides_bytes[i];
            B200SD_REQUIRE(gs[i] % 16 == 0, "tensor map stride %llu (dim %d) not a multiple of 16 bytes",
                           static_cast<unsigned long long>(gs[i]), i + 1);
        }
    }
    CUresult r = fn(map, dtype, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gd,
                    gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200SD_REQUIRE(r == CUDA_SUCCESS,
                   "cuTensorMapEncodeTiled failed (CUresult %d; rank %d dims %llu,%llu,%llu,%llu box %u,%u,%u,%u)",
                   static_cast<int>(r), rank, static_cast<unsigned long long>(gd[0]),
                   static_cast<unsigned long long>(rank > 1 ? gd[1] : 0),
                   static_cast<unsigned long long>(rank > 2 ? gd[2] : 0),
                   static_cast<unsigned long long>(rank > 3 ? gd[3] : 0), bx[0], rank > 1 ? bx[1] : 0,
                   rank > 2 ? bx[2] : 0, rank > 3 ? bx[3] : 0);
    return 0;
}

}  // namespace b200sd

extern "C" const char* b200sd_last_error(void) { return b200sd::g_error; }
extern "C" int b200sd_version(void) { return 1; }
extern "C" uint64_t b200sd_launch_count(void) { return b200sd::g_launches.load(); }
extern "C" void b200sd_set_pdl(int enabled) { b200sd::g_pdl = enabled ? 1 : 0; }
extern "C" void b200sd_set_launch_classes(uint32_t mask) { b200sd::g_class_mask.store(mask & 0xFu); }
