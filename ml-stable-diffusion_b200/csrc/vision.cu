// b200sd -- kernels of the Stable Diffusion safety checker's own stages: the CLIP image preprocessing (Pillow's
// BICUBIC resize in its 8-bit fixed-point form, centre crop, rescale, normalise), patch extraction for the patch
// embedding GEMM, concept scoring and the blacking out of flagged images.  The vision tower between them runs on the
// GEMM, LayerNorm and attention kernels.
#include "common.cuh"
#include "../../include/b200sd.h"

#include <algorithm>

namespace b200sd {

extern void count_launch(int n);

static inline int vision_grid(size_t n, int threads) {
    return static_cast<int>(std::min<size_t>((n + threads - 1) / threads, static_cast<size_t>(num_sms()) * 16));
}

// Pillow's clip8 (Resample.c): the accumulator holds 22 fractional bits, values outside [0, 255] saturate
__device__ __forceinline__ uint8_t clip8_fixed(int acc) {
    return static_cast<uint8_t>(min(max(acc >> 22, 0), 255));
}

struct ClipNorm {
    float mean[3];
    float std[3];
};

// ---- horizontal pass: u8 NHWC [n, h, w, 3] -> u8 [n, h, ow, 3] for the ow output columns the crop keeps ----------
// bounds [ow][2] = (first input column, taps), coeffs [ow][ksize]: the host's fixed-point BICUBIC table
__global__ void clip_resize_h_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ tmp, int n, int h, int w,
                                     const int32_t* __restrict__ bounds, const int32_t* __restrict__ coeffs, int ksize,
                                     int ow) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = static_cast<size_t>(n) * h * ow * 3;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int ch = static_cast<int>(i % 3);
        size_t r = i / 3;
        const int x = static_cast<int>(r % ow);
        r /= ow;  // b * h + y
        const int xmin = bounds[2 * x], taps = bounds[2 * x + 1];
        const uint8_t* src = in + (r * w + xmin) * 3 + ch;
        const int32_t* k = coeffs + static_cast<size_t>(x) * ksize;
        int acc = 1 << 21;
        for (int j = 0; j < taps; ++j) acc += static_cast<int>(src[3 * j]) * k[j];
        tmp[i] = clip8_fixed(acc);
    }
}

// ---- vertical pass + rescale + normalise: u8 [n, h, ow, 3] -> fp32 NCHW [n, 3, oh, ow] --------------------------
// v = float32(float64(u8) * (1 / 255)), then (v - mean) / std in fp32 with IEEE division (transformers' rescale and
// normalize on a float32 image)
__global__ void clip_resize_v_norm_kernel(const uint8_t* __restrict__ tmp, float* __restrict__ out, int n, int h,
                                          int ow, const int32_t* __restrict__ bounds,
                                          const int32_t* __restrict__ coeffs, int ksize, int oh, ClipNorm nm) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = static_cast<size_t>(n) * 3 * oh * ow;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(i % ow);
        size_t r = i / ow;
        const int y = static_cast<int>(r % oh);
        r /= oh;
        const int ch = static_cast<int>(r % 3);
        const size_t b = r / 3;
        const int ymin = bounds[2 * y], taps = bounds[2 * y + 1];
        const uint8_t* src = tmp + ((b * h + ymin) * ow + x) * 3 + ch;
        const int32_t* k = coeffs + static_cast<size_t>(y) * ksize;
        int acc = 1 << 21;
        for (int j = 0; j < taps; ++j) acc += static_cast<int>(src[static_cast<size_t>(j) * ow * 3]) * k[j];
        const float v = __double2float_rn(static_cast<double>(clip8_fixed(acc)) * (1.0 / 255.0));
        // select, not index: a dynamically indexed parameter array would be copied to local memory
        const float mean = ch == 0 ? nm.mean[0] : (ch == 1 ? nm.mean[1] : nm.mean[2]);
        const float sd = ch == 0 ? nm.std[0] : (ch == 1 ? nm.std[1] : nm.std[2]);
        out[i] = __fdiv_rn(__fsub_rn(v, mean), sd);
    }
}

// ---- patch extraction: fp32 NCHW [n, c, g*p, g*p] -> fp16 [n * (1 + g*g), k_pad] ---------------------------------
// Row t of image b's 1 + g*g rows: t = 0 is the class token's row and stays zero, t = 1 + py*g + px holds patch
// (py, px) in (channel, ky, kx) order -- the order of the flattened [D, c, p, p] patch-embedding weight; columns past
// c*p*p are zero.  The patch-embedding GEMM then writes every token row, the class token's included.
__global__ void patchify_kernel(const float* __restrict__ px, __half* __restrict__ out, int n, int c, int p, int g,
                                int k_pad) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int rows_per_img = 1 + g * g, pp = p * p, img = g * p;
    const size_t total = static_cast<size_t>(n) * rows_per_img * k_pad;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int col = static_cast<int>(i % k_pad);
        const size_t row = i / k_pad;
        const int t = static_cast<int>(row % rows_per_img);
        const size_t b = row / rows_per_img;
        float v = 0.f;
        if (t > 0 && col < c * pp) {
            const int py = (t - 1) / g, pxi = (t - 1) % g;
            const int ch = col / pp, ky = (col % pp) / p, kx = col % p;
            v = px[((b * c + ch) * img + py * p + ky) * img + pxi * p + kx];
        }
        out[i] = __float2half_rn(v);
    }
}

// ---- concept scoring (the safety checker head): one CTA per image, one warp per concept row ---------------------
// cos = <x, c> / max(|x|, 1e-12) against the pre-normalised concept rows (F.normalize on both sides);
// special = any(cos_special - w_special + adjustment > 0); score_j = (cos_j - w_j) + (special ? 0.01 : 0);
// flag = any(score_j > 0).
constexpr int kMaxConcepts = 32;

__global__ void __launch_bounds__(kMaxConcepts * 32) safety_concepts_kernel(
    const float* __restrict__ emb, int dim, const float* __restrict__ concepts, const float* __restrict__ concept_w,
    int nc, const float* __restrict__ special, const float* __restrict__ special_w, int ns,
    const float* __restrict__ adjustment, float* __restrict__ scores, float* __restrict__ flags) {
    __shared__ float cos_s[kMaxConcepts];
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* x = emb + static_cast<size_t>(b) * dim;
    if (warp < nc + ns) {
        const float* row = warp < nc ? concepts + static_cast<size_t>(warp) * dim
                                     : special + static_cast<size_t>(warp - nc) * dim;
        float ss = 0.f, dot = 0.f;
        for (int k = lane; k < dim; k += 32) {
            const float xv = x[k];
            ss = fmaf(xv, xv, ss);
            dot = fmaf(xv, row[k], dot);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            ss += __shfl_xor_sync(0xffffffffu, ss, o);
            dot += __shfl_xor_sync(0xffffffffu, dot, o);
        }
        if (lane == 0) cos_s[warp] = __fdiv_rn(dot, fmaxf(sqrtf(ss), 1e-12f));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float adj = adjustment ? adjustment[0] : 0.f;
        bool care = false;
        for (int k = 0; k < ns; ++k) care |= (cos_s[nc + k] - special_w[k]) + adj > 0.f;
        const float lift = care ? 0.01f : 0.f;
        bool any = false;
        for (int j = 0; j < nc; ++j) {
            const float s = (cos_s[j] - concept_w[j]) + lift;
            scores[static_cast<size_t>(b) * nc + j] = s;
            any |= s > 0.f;
        }
        flags[b] = any ? 1.f : 0.f;
    }
}

// ---- zero every flagged image in place (fp32 and the optional u8 copy); others are not written ----------------
__global__ void filter_images_kernel(const float* __restrict__ flags, float* __restrict__ img, uint8_t* __restrict__ u8,
                                     int n, size_t per_image) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = static_cast<size_t>(n) * per_image;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        if (flags[i / per_image] != 0.f) {
            if (img) img[i] = 0.f;
            if (u8) u8[i] = 0;
        }
    }
}

}  // namespace b200sd

using namespace b200sd;

extern "C" int b200sd_clip_preprocess(const uint8_t* images, int32_t n, int32_t h, int32_t w, uint8_t* tmp,
                                      const int32_t* h_bounds, const int32_t* h_coeffs, int32_t h_ksize,
                                      const int32_t* v_bounds, const int32_t* v_coeffs, int32_t v_ksize,
                                      int32_t crop_h, int32_t crop_w, const float* mean, const float* std,
                                      float* out, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(images && tmp && h_bounds && h_coeffs && v_bounds && v_coeffs && mean && std && out,
                   "b200sd_clip_preprocess: null pointer");
    B200SD_REQUIRE(n > 0 && h > 0 && w > 0 && crop_h > 0 && crop_w > 0 && h_ksize > 0 && v_ksize > 0,
                   "b200sd_clip_preprocess: bad sizes (n=%d h=%d w=%d crop=%dx%d)", n, h, w, crop_h, crop_w);
    ClipNorm nm;
    for (int c = 0; c < 3; ++c) {
        nm.mean[c] = mean[c];
        nm.std[c] = std[c];
    }
    const size_t th = static_cast<size_t>(n) * h * crop_w * 3;
    B200SD_CHECK_CUDA(launch_kernel(clip_resize_h_kernel, dim3(vision_grid(th, 256)), dim3(256), 0, stream, images, tmp,
                                    n, h, w, h_bounds, h_coeffs, h_ksize, crop_w));
    B200SD_CHECK_CUDA(cudaGetLastError());
    const size_t tv = static_cast<size_t>(n) * 3 * crop_h * crop_w;
    B200SD_CHECK_CUDA(launch_kernel(clip_resize_v_norm_kernel, dim3(vision_grid(tv, 256)), dim3(256), 0, stream, tmp,
                                    out, n, h, crop_w, v_bounds, v_coeffs, v_ksize, crop_h, nm));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(2);
    return 0;
}

extern "C" int b200sd_patchify(const float* pixel_values, int32_t n, int32_t c, int32_t image_size, int32_t patch,
                               int32_t k_pad, void* out, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(pixel_values && out, "b200sd_patchify: null pointer");
    B200SD_REQUIRE(n > 0 && c > 0 && patch > 0 && image_size % patch == 0 && k_pad >= c * patch * patch,
                   "b200sd_patchify: bad sizes (image %d, patch %d, c %d, k_pad %d)", image_size, patch, c, k_pad);
    const int g = image_size / patch;
    const size_t total = static_cast<size_t>(n) * (1 + g * g) * k_pad;
    B200SD_CHECK_CUDA(launch_kernel(patchify_kernel, dim3(vision_grid(total, 256)), dim3(256), 0, stream, pixel_values,
                                    reinterpret_cast<__half*>(out), n, c, patch, g, k_pad));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_safety_concepts(const float* image_embeds, int32_t n, int32_t dim, const float* concepts,
                                      const float* concept_weights, int32_t n_concepts, const float* special,
                                      const float* special_weights, int32_t n_special, const float* adjustment,
                                      float* concept_scores, float* has_nsfw, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(image_embeds && concepts && concept_weights && concept_scores && has_nsfw &&
                       (n_special == 0 || (special && special_weights)),
                   "b200sd_safety_concepts: null pointer");
    B200SD_REQUIRE(n > 0 && dim > 0 && n_concepts > 0 && n_special >= 0 && n_concepts + n_special <= kMaxConcepts,
                   "b200sd_safety_concepts: bad sizes (n=%d dim=%d concepts=%d special=%d, at most %d rows)", n, dim,
                   n_concepts, n_special, kMaxConcepts);
    B200SD_CHECK_CUDA(launch_kernel(safety_concepts_kernel, dim3(n), dim3(kMaxConcepts * 32), 0, stream, image_embeds,
                                    dim, concepts, concept_weights, n_concepts, special, special_weights, n_special,
                                    adjustment, concept_scores, has_nsfw));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_filter_images(const float* has_nsfw, float* images, uint8_t* images_u8, int32_t n, int32_t h,
                                    int32_t w, int32_t c, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(has_nsfw && (images || images_u8), "b200sd_filter_images: null pointer");
    const size_t per = static_cast<size_t>(h) * w * c;
    B200SD_CHECK_CUDA(launch_kernel(filter_images_kernel, dim3(vision_grid(per * n, 256)), dim3(256), 0, stream,
                                    has_nsfw, images, images_u8, n, per));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}
