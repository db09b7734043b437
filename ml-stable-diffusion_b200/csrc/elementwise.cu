// b200sd -- layout conversion, small-M linear, timestep embedding, fused CFG + scheduler step and
// image post-processing kernels (HBM / latency bound; vectorised, coalesced, one launch each).
#include "common.cuh"
#include "../../include/b200sd.h"

#include <algorithm>
#include <cmath>

namespace b200sd {

extern void count_launch(int n);

static inline int grid_for(size_t n, int threads) {
    return static_cast<int>(std::min<size_t>((n + threads - 1) / threads, static_cast<size_t>(num_sms()) * 16));
}

// ---- NCHW -> NHWC fp16 / bf16 (pad channels) ------------------------------------------------
template <typename T, typename TO = __half>
__global__ void nchw_to_nhwc_kernel(const T* __restrict__ in, TO* __restrict__ out, int n, int c, int hw,
                                    int c_pad) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = static_cast<size_t>(n) * hw * c_pad;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int ch = static_cast<int>(i % c_pad);
        const size_t px = i / c_pad;
        const int p = static_cast<int>(px % hw);
        const int b = static_cast<int>(px / hw);
        float v = 0.f;
        if (ch < c) v = static_cast<float>(in[(static_cast<size_t>(b) * c + ch) * hw + p]);
        out[i] = Elem16<TO>::from_float(v);
    }
}

template <typename T>
__global__ void nhwc_to_nchw_f32_kernel(const T* __restrict__ in, float* __restrict__ out, int n, int c, int hw,
                                        int c_pad) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = static_cast<size_t>(n) * c * hw;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int p = static_cast<int>(i % hw);
        const size_t r = i / hw;
        const int ch = static_cast<int>(r % c);
        const int b = static_cast<int>(r / c);
        out[i] = static_cast<float>(in[(static_cast<size_t>(b) * hw + p) * c_pad + ch]);
    }
}

// ---- (B, D, 1, S) -> [B*S, D] fp16 (tiled transpose through shared memory) -------------------
template <typename T>
__global__ void ctx_to_tokens_kernel(const T* __restrict__ in, __half* __restrict__ out, int d, int s) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int d0 = blockIdx.y * 32, s0 = blockIdx.x * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int dd = d0 + r, ss = s0 + threadIdx.x;
        if (dd < d && ss < s) tile[r][threadIdx.x] = static_cast<float>(in[(static_cast<size_t>(b) * d + dd) * s + ss]);
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int ss = s0 + r, dd = d0 + threadIdx.x;
        if (dd < d && ss < s) out[(static_cast<size_t>(b) * s + ss) * d + dd] = __float2half_rn(tile[threadIdx.x][r]);
    }
}

// ---- CLIP text embeddings: out[b*s + t, :] = token_embedding[ids[b, t]] + position_embedding[t] -----------
// ids arrive as float32 (the reference feeds input_ids as floats, pipeline.py:173); out-of-range ids clamp.
__global__ void embed_tokens_kernel(const float* __restrict__ ids, const uint4* __restrict__ tok,
                                    const uint4* __restrict__ pos, uint4* __restrict__ out, int rows, int s, int vecs,
                                    int vocab) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = static_cast<size_t>(rows) * vecs;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int r = static_cast<int>(i / vecs), v = static_cast<int>(i - static_cast<size_t>(r) * vecs);
        const int id = min(max(__float2int_rn(ids[r]), 0), vocab - 1);
        uint4 a = tok[static_cast<size_t>(id) * vecs + v];
        const uint4 b = pos[static_cast<size_t>(r % s) * vecs + v];
        __half2* ah = reinterpret_cast<__half2*>(&a);
        const __half2* bh = reinterpret_cast<const __half2*>(&b);
#pragma unroll
        for (int q = 0; q < 4; ++q) ah[q] = __hadd2(ah[q], bh[q]);
        out[i] = a;
    }
}

// ---- nearest x2 upsample, NHWC fp16, 16-byte vectors ------------------------------------------
__global__ void upsample2x_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int n, int h, int w,
                                  int vecs) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = static_cast<size_t>(n) * (2 * h) * (2 * w) * vecs;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int v = static_cast<int>(i % vecs);
        size_t r = i / vecs;
        const int ox = static_cast<int>(r % (2 * w));
        r /= (2 * w);
        const int oy = static_cast<int>(r % (2 * h));
        const int b = static_cast<int>(r / (2 * h));
        out[i] = in[((static_cast<size_t>(b) * h + (oy >> 1)) * w + (ox >> 1)) * vecs + v];
    }
}

// nearest x2 upsample of an fp16 NHWC tensor into the int8 operand of the W8A8 convolution: each source vector of eight
// channels is quantized once (q = clamp(rint(x * inv_scale), -127, 127)) and written to its four output pixels
__global__ void upsample2x_s8_kernel(const uint4* __restrict__ in, uint2* __restrict__ out, int n, int h, int w, int vecs,
                                     float inv_scale) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = static_cast<size_t>(n) * h * w * vecs;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int v = static_cast<int>(i % vecs);
        size_t r = i / vecs;
        const int x = static_cast<int>(r % w);
        r /= w;
        const int y = static_cast<int>(r % h);
        const int b = static_cast<int>(r / h);
        const uint4 raw = in[i];
        const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
        float f[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 t = __half22float2(h2[q]);
            f[2 * q] = t.x;
            f[2 * q + 1] = t.y;
        }
        const uint2 pk = quantize8_s8(f, inv_scale);
        const size_t o = ((static_cast<size_t>(b) * 2 * h + 2 * y) * (2 * w) + 2 * x) * vecs + v;
        out[o] = pk;
        out[o + vecs] = pk;
        out[o + static_cast<size_t>(2 * w) * vecs] = pk;
        out[o + static_cast<size_t>(2 * w) * vecs + vecs] = pk;
    }
}

// max |x| of an fp16 tensor folded into *slot: a non-negative float orders like its bit pattern, so atomicMax on the
// bits gives the same result in any order (W8A8 calibration)
__global__ void absmax_f16_kernel(const __half2* __restrict__ x, size_t n2, unsigned int* __restrict__ slot) {
    pdl_trigger();
    pdl_wait();
    float m = 0.f;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n2;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const float2 f = __half22float2(x[i]);
        m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(slot, __float_as_uint(m));
}

__global__ void add_kernel(const __half2* __restrict__ a, const __half2* __restrict__ b, __half2* __restrict__ out,
                           size_t n2) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n2;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const float2 x = __half22float2(a[i]), y = __half22float2(b[i]);
        out[i] = __floats2half2_rn(x.x + y.x, x.y + y.y);
    }
}

// ---- ControlNet residual injection: out = skip + sum_k scales[k] * res[k] ------------------------------------------
// diffusers' fp16 operation order (ControlNetModel's conditioning_scale, MultiControlNetModel's sum, the UNet's add):
// t = fp16(s_0 r_0), t = fp16(t + fp16(s_k r_k)) for each following net, out = fp16(skip + t).  Each product and sum
// is computed in fp32 and rounded to fp16, as torch does for an fp16 tensor op.  At s = 1 the product is exact, so one
// net gives fp16(skip + r_0) and two give fp16(skip + fp16(r_0 + r_1)): b200sd_add's bits.  The scales are read from
// device memory, so a captured graph sees new values on replay.  skip == nullptr: out = t.
struct ControlResiduals {
    const __half* r[B200SD_MAX_CONTROLNETS];
};

__device__ __forceinline__ float control_inject_one(const __half* skip, const ControlResiduals& res, const float* s,
                                                    int n_res, size_t i) {
    float t = __half2float(__float2half_rn(s[0] * __half2float(res.r[0][i])));
    for (int k = 1; k < n_res; ++k)
        t = __half2float(__float2half_rn(t + __half2float(__float2half_rn(s[k] * __half2float(res.r[k][i])))));
    if (skip) t = __half2float(__float2half_rn(__half2float(skip[i]) + t));
    return t;
}

// vec: every pointer is 16-byte aligned, so numel / 8 groups of eight go through 16-byte loads and stores; the tail
// (and everything when vec is 0) is done one element per thread
__global__ void control_inject_kernel(const __half* skip, ControlResiduals res, const float* __restrict__ scales,
                                      int n_res, __half* out, size_t numel, int vec) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    float s[B200SD_MAX_CONTROLNETS];
#pragma unroll
    for (int k = 0; k < B200SD_MAX_CONTROLNETS; ++k) s[k] = k < n_res ? scales[k] : 0.f;
    const size_t n8 = vec ? numel / 8 : 0;
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t step = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t v = tid; v < n8; v += step) {
        float t[8];
        {
            const uint4 a = reinterpret_cast<const uint4*>(res.r[0])[v];
            const __half* h = reinterpret_cast<const __half*>(&a);
#pragma unroll
            for (int j = 0; j < 8; ++j) t[j] = __half2float(__float2half_rn(s[0] * __half2float(h[j])));
        }
        for (int k = 1; k < n_res; ++k) {
            const uint4 a = reinterpret_cast<const uint4*>(res.r[k])[v];
            const __half* h = reinterpret_cast<const __half*>(&a);
#pragma unroll
            for (int j = 0; j < 8; ++j)
                t[j] = __half2float(__float2half_rn(t[j] + __half2float(__float2half_rn(s[k] * __half2float(h[j])))));
        }
        if (skip) {
            const uint4 a = reinterpret_cast<const uint4*>(skip)[v];
            const __half* h = reinterpret_cast<const __half*>(&a);
#pragma unroll
            for (int j = 0; j < 8; ++j) t[j] = __half2float(h[j]) + t[j];
        }
        uint4 o;
        __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
        for (int j = 0; j < 8; ++j) oh[j] = __float2half_rn(t[j]);
        reinterpret_cast<uint4*>(out)[v] = o;
    }
    for (size_t i = n8 * 8 + tid; i < numel; i += step) out[i] = __float2half_rn(control_inject_one(skip, res, s, n_res, i));
}

// ---- small-M linear: one warp per output column, all M rows at once (M <= 8) -------------------
// The (optionally SiLU-activated) input rows are staged in shared memory ONCE per block -- every column warp used to
// re-read and re-activate them (the 20 800-column time-embedding projection was MUFU-bound on 20 800 redundant SiLU
// passes) -- and a warp requests four weight vectors per lane before the first one is consumed.
template <int kM>
__global__ void __launch_bounds__(256) linear_small_kernel(const float* __restrict__ x, const __half* __restrict__ w,
                                                           const float* __restrict__ bias,
                                                           const float* __restrict__ add, float* __restrict__ out,
                                                           int m, int n, int k, int act_in, int act_out) {
    extern __shared__ __align__(16) float xs[];  // [kM][k]
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    for (int i = threadIdx.x; i < kM * k; i += blockDim.x) {
        const int r = i / k;
        float v = r < m ? x[i] : 0.f;
        if (act_in) v = silu_f(v);
        xs[i] = v;
    }
    __syncthreads();
    const int col = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (col >= n) return;
    const __half* wr = w + static_cast<size_t>(col) * k;
    float acc[kM];
#pragma unroll
    for (int r = 0; r < kM; ++r) acc[r] = 0.f;
    constexpr int kInFlight = 4;
    for (int kb = lane * 8; kb < k; kb += 32 * 8 * kInFlight) {
        uint4 raw[kInFlight];
#pragma unroll
        for (int i = 0; i < kInFlight; ++i) {
            const int kk = kb + i * 256;
            raw[i] = kk < k ? __ldg(reinterpret_cast<const uint4*>(wr + kk)) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int i = 0; i < kInFlight; ++i) {
            const int kk = kb + i * 256;
            if (kk >= k) break;
            const __half2* h2 = reinterpret_cast<const __half2*>(&raw[i]);
            float wf[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 t = __half22float2(h2[q]);
                wf[2 * q] = t.x;
                wf[2 * q + 1] = t.y;
            }
#pragma unroll
            for (int r = 0; r < kM; ++r) {
                const float4 x0 = *reinterpret_cast<const float4*>(xs + r * k + kk);
                const float4 x1 = *reinterpret_cast<const float4*>(xs + r * k + kk + 4);
                acc[r] += x0.x * wf[0] + x0.y * wf[1] + x0.z * wf[2] + x0.w * wf[3] + x1.x * wf[4] + x1.y * wf[5] + x1.z * wf[6] +
                          x1.w * wf[7];
            }
        }
    }
#pragma unroll
    for (int r = 0; r < kM; ++r) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
    }
    if (lane == 0) {
        const float b = (bias ? bias[col] : 0.f) + (add ? add[col] : 0.f);
        for (int r = 0; r < m && r < kM; ++r) {
            float v = acc[r] + b;
            if (act_out) v = silu_f(v);
            out[static_cast<size_t>(r) * n + col] = v;
        }
    }
}

// ---- sinusoidal timestep embedding (unet.py:703-728) -------------------------------------------
__global__ void timestep_embedding_kernel(const float* __restrict__ t, float* __restrict__ out, int m, int dim,
                                          int flip, float freq_shift) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int half = dim / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m * half) return;
    const int r = i / half, j = i % half;
    const float freq = expf(-logf(10000.0f) * static_cast<float>(j) / (static_cast<float>(half) - freq_shift));
    const float ang = t[r] * freq;
    const float s = sinf(ang), c = cosf(ang);
    float* o = out + static_cast<size_t>(r) * dim;
    if (flip) {
        o[j] = c;
        o[half + j] = s;
    } else {
        o[j] = s;
        o[half + j] = c;
    }
}

// ---- fused CFG + scheduler step ------------------------------------------------------------------
// Standard normal number `idx` of noise draw `offset` under `key`: Philox-4x32-10 with counter (offset, 0, idx, 0), then
// Box-Muller on the first two words -- the rng.NvRandomSource stream (NvRandomSource.swift), so
// NvRandomSource(key) at that offset reproduces it on the host.  The transform runs in double, like the host twin.
__device__ __forceinline__ float philox_normal(uint32_t key, uint32_t offset, uint32_t idx) {
    uint32_t c0 = offset, c1 = 0u, c2 = idx, c3 = 0u, k0 = key, k1 = 0u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(c0, 0xD2511F53u), lo0 = c0 * 0xD2511F53u;
        const uint32_t hi1 = __umulhi(c2, 0xCD9E8D57u), lo1 = c2 * 0xCD9E8D57u;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    const double u = static_cast<double>(c0) * (1.0 / 4294967296.0) + (1.0 / 8589934592.0);
    // sin(v), v = c1 * pi / 2^31 + pi / 2^32, as sinpi of the exact v / pi (no large-argument reduction)
    const double v_over_pi = static_cast<double>(c1) * (1.0 / 2147483648.0) + (1.0 / 4294967296.0);
    return static_cast<float>(sqrt(-2.0 * log(u)) * sinpi(v_over_pi));
}

// One thread per latent element (n*c*h*w, NCHW fp32).  See include/b200sd.h for the algebra.  kNoise (ancestral
// samplers): x_prev += noise_scale * z with z = philox_normal(*philox_key, philox_offset, i); the kNoise = false
// instantiation never reads noise_scale / philox_key / philox_offset.  kBlend (inpainting): after the update and the
// noise, x_prev = m x_prev + (1 - m)(a x0_img + b z); history pushes and `denoised` keep their pre-blend values.  The
// kBlend = false instantiations never read `blend` (appended last, so the other parameters keep their offsets).
// kGuided = false (guidance-free): noise_pred holds one prediction per image, [n, ...], used as eps' directly (no
// k.guidance), and only the first n rows of unet_in are written.  The body is shared by two kernel templates so the
// guided kernels keep their names and their code.
template <bool kNoise, bool kBlend, bool kGuided>
__device__ __forceinline__ void step_body(const float* __restrict__ noise_pred, float* __restrict__ latents,
                                          float* __restrict__ hist, float* __restrict__ denoised,
                                          __half* __restrict__ unet_in, int c_pad, int n, int c, int hw,
                                          const b200sd_step_coeffs& k, float noise_scale,
                                          const uint32_t* __restrict__ philox_key, uint32_t philox_offset,
                                          const b200sd_blend_args& blend) {
    const int numel = n * c * hw;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= numel) return;
    int ni = i;  // index of this element inside one CFG half of noise_pred
    if (k.noise_pred_nhwc) {  // the UNet's conv_out output as it leaves the epilogue: [2n | n, h*w, c]
        const int p = i % hw;
        const int ch = (i / hw) % c;
        const int b = i / (hw * c);
        ni = (b * hw + p) * c + ch;
    }
    float eps;
    if constexpr (kGuided) {
        const float eu = noise_pred[ni];
        const float ec = noise_pred[numel + ni];
        eps = eu + k.guidance * (ec - eu);
    } else {
        eps = noise_pred[ni];
    }
    const float x = latents[i];
    float xp = k.cx * x + k.ce * eps;
    float x0 = k.x0_cx * x + k.x0_ce * eps;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j < k.n_hist) {
            const float hv = hist[static_cast<size_t>(j) * numel + i];
            xp += k.ch[j] * hv;
            x0 += k.x0_ch[j] * hv;
        }
    }
    if (k.push_eps_slot >= 0) hist[static_cast<size_t>(k.push_eps_slot) * numel + i] = eps;
    if (k.push_x0_slot >= 0) hist[static_cast<size_t>(k.push_x0_slot) * numel + i] = x0;
    if (k.push_x_slot >= 0) hist[static_cast<size_t>(k.push_x_slot) * numel + i] = x;
    if constexpr (kNoise) xp += noise_scale * philox_normal(*philox_key, philox_offset, static_cast<uint32_t>(i));
    if constexpr (kBlend) {
        // the latent mask is per pixel [n, h*w], shared by the channels
        const float m = __ldg(blend.mask + (i / (hw * c)) * hw + i % hw);
        const float keep = blend.a * __ldg(blend.image_latents + i) + blend.b * __ldg(blend.noise + i);
        xp = m * xp + (1.f - m) * keep;
    }
    if (denoised) denoised[i] = x0;
    latents[i] = xp;
    if (unet_in) {
        // NCHW index -> NHWC, duplicated for the (uncond, cond) batch halves
        const int p = i % hw;
        const int ch = (i / hw) % c;
        const int b = i / (hw * c);
        const __half hv = __float2half_rn(xp);
        unet_in[(static_cast<size_t>(b) * hw + p) * c_pad + ch] = hv;
        if constexpr (kGuided) unet_in[(static_cast<size_t>(n + b) * hw + p) * c_pad + ch] = hv;
    }
}

template <bool kNoise, bool kBlend>
__global__ void cfg_step_kernel(const float* __restrict__ noise_pred, float* __restrict__ latents,
                                float* __restrict__ hist, float* __restrict__ denoised, __half* __restrict__ unet_in,
                                int c_pad, int n, int c, int hw, b200sd_step_coeffs k, float noise_scale,
                                const uint32_t* __restrict__ philox_key, uint32_t philox_offset,
                                b200sd_blend_args blend) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    step_body<kNoise, kBlend, true>(noise_pred, latents, hist, denoised, unet_in, c_pad, n, c, hw, k, noise_scale,
                                    philox_key, philox_offset, blend);
}

template <bool kNoise, bool kBlend>
__global__ void guidance_free_step_kernel(const float* __restrict__ noise_pred, float* __restrict__ latents,
                                          float* __restrict__ hist, float* __restrict__ denoised,
                                          __half* __restrict__ unet_in, int c_pad, int n, int c, int hw,
                                          b200sd_step_coeffs k, float noise_scale,
                                          const uint32_t* __restrict__ philox_key, uint32_t philox_offset,
                                          b200sd_blend_args blend) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    step_body<kNoise, kBlend, false>(noise_pred, latents, hist, denoised, unet_in, c_pad, n, c, hw, k, noise_scale,
                                     philox_key, philox_offset, blend);
}

// ---- image post-process: clip(x/2+0.5, 0, 1), NHWC(c_pad) -> NHWC(c) fp32 and/or u8 -------------
template <typename T>
__global__ void image_post_kernel(const T* __restrict__ in, int c_pad, float* __restrict__ of, uint8_t* __restrict__ ou,
                                  size_t pixels, int c) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t total = pixels * c;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t px = i / c;
        const int ch = static_cast<int>(i % c);
        float v = static_cast<float>(in[px * c_pad + ch]) * 0.5f + 0.5f;
        v = fminf(fmaxf(v, 0.f), 1.f);
        if (of) of[i] = v;
        if (ou) ou[i] = static_cast<uint8_t>(__float2int_rn(v * 255.f));
    }
}


// ---- latent prep for the VAE decoder: z/scaling -> post_quant_conv (1x1, <= 8 channels) -> NHWC fp16 / bf16 ----
template <typename TO>
__global__ void latent_prep_kernel(const float* __restrict__ z, const float* __restrict__ w /* [c, c] */,
                                   const float* __restrict__ b, float inv_scale, TO* __restrict__ out, int n, int c,
                                   int hw, int c_pad) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * hw) return;
    const int p = i % hw, img = i / hw;
    float v[8];
#pragma unroll
    for (int ci = 0; ci < 8; ++ci) v[ci] = ci < c ? z[(static_cast<size_t>(img) * c + ci) * hw + p] * inv_scale : 0.f;
    for (int co = 0; co < c_pad; ++co) {
        float acc = 0.f;
        if (co < c) {
            acc = b ? b[co] : 0.f;
            for (int ci = 0; ci < c; ++ci) acc += w[co * c + ci] * v[ci];
        }
        out[static_cast<size_t>(i) * c_pad + co] = Elem16<TO>::from_float(acc);
    }
}

}  // namespace b200sd

using namespace b200sd;

// TO: the output type (fp16 for b200sd_nchw_to_nhwc, bf16 for b200sd_nchw_to_nhwc_bf16)
template <typename TO>
static int nchw_to_nhwc(const void* in, int32_t in_f32, void* out, int32_t n, int32_t c, int32_t h, int32_t w,
                        int32_t c_pad, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(in && out && c_pad >= c, "b200sd_nchw_to_nhwc: bad arguments");
    const size_t total = static_cast<size_t>(n) * h * w * c_pad;
    if (in_f32)
        B200SD_CHECK_CUDA(launch_kernel(nchw_to_nhwc_kernel<float, TO>, dim3(grid_for(total, 256)), dim3(256), 0, stream, reinterpret_cast<const float*>(in),
                                                                             reinterpret_cast<TO*>(out), n, c,
                                                                             h * w, c_pad));
    else
        B200SD_CHECK_CUDA(launch_kernel(nchw_to_nhwc_kernel<__half, TO>, dim3(grid_for(total, 256)), dim3(256), 0, stream, reinterpret_cast<const __half*>(in),
                                                                              reinterpret_cast<TO*>(out), n, c,
                                                                              h * w, c_pad));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_nchw_to_nhwc(const void* in, int32_t in_f32, void* out, int32_t n, int32_t c, int32_t h,
                                   int32_t w, int32_t c_pad, void* stream) {
    return nchw_to_nhwc<__half>(in, in_f32, out, n, c, h, w, c_pad, stream);
}
extern "C" int b200sd_nchw_to_nhwc_bf16(const void* in, int32_t in_f32, void* out, int32_t n, int32_t c, int32_t h,
                                        int32_t w, int32_t c_pad, void* stream) {
    return nchw_to_nhwc<__nv_bfloat16>(in, in_f32, out, n, c, h, w, c_pad, stream);
}

extern "C" int b200sd_nhwc_to_nchw_f32(const void* in, int32_t in_f32, float* out, int32_t n, int32_t c, int32_t h,
                                       int32_t w, int32_t c_pad, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(in && out && c_pad >= c, "b200sd_nhwc_to_nchw_f32: bad arguments");
    const size_t total = static_cast<size_t>(n) * c * h * w;
    if (in_f32)
        B200SD_CHECK_CUDA(launch_kernel(nhwc_to_nchw_f32_kernel<float>, dim3(grid_for(total, 256)), dim3(256), 0, stream, reinterpret_cast<const float*>(in),
                                                                                 out, n, c, h * w, c_pad));
    else
        B200SD_CHECK_CUDA(launch_kernel(nhwc_to_nchw_f32_kernel<__half>, dim3(grid_for(total, 256)), dim3(256), 0, stream, reinterpret_cast<const __half*>(in),
                                                                                  out, n, c, h * w, c_pad));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_ctx_to_tokens(const void* in, int32_t in_f32, void* out, int32_t b, int32_t d, int32_t s,
                                    void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(in && out, "b200sd_ctx_to_tokens: null pointer");
    dim3 grid((s + 31) / 32, (d + 31) / 32, b), block(32, 8);
    if (in_f32)
        B200SD_CHECK_CUDA(launch_kernel(ctx_to_tokens_kernel<float>, dim3(grid), dim3(block), 0, stream, reinterpret_cast<const float*>(in),
                                                                reinterpret_cast<__half*>(out), d, s));
    else
        B200SD_CHECK_CUDA(launch_kernel(ctx_to_tokens_kernel<__half>, dim3(grid), dim3(block), 0, stream, reinterpret_cast<const __half*>(in),
                                                                 reinterpret_cast<__half*>(out), d, s));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_embed_tokens(const float* ids, const void* token_embedding, const void* position_embedding,
                                   void* out, int32_t batch, int32_t s, int32_t d, int32_t vocab, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(ids && token_embedding && position_embedding && out && d % 8 == 0 && vocab > 0,
                   "b200sd_embed_tokens: bad arguments (d=%d must be a multiple of 8)", d);
    const size_t total = static_cast<size_t>(batch) * s * (d / 8);
    B200SD_CHECK_CUDA(launch_kernel(embed_tokens_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, ids,
                                    reinterpret_cast<const uint4*>(token_embedding),
                                    reinterpret_cast<const uint4*>(position_embedding), reinterpret_cast<uint4*>(out),
                                    batch * s, s, d / 8, vocab));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

// nearest x2 upsample: a 16-byte copy per vector, so it serves fp16 and bf16 tensors alike
extern "C" int b200sd_upsample2x(const void* in, void* out, int32_t n, int32_t h, int32_t w, int32_t c,
                                 void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(in && out && c % 8 == 0, "b200sd_upsample2x: c=%d must be a multiple of 8", c);
    const size_t total = static_cast<size_t>(n) * 4 * h * w * (c / 8);
    B200SD_CHECK_CUDA(launch_kernel(upsample2x_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, reinterpret_cast<const uint4*>(in),
                                                                reinterpret_cast<uint4*>(out), n, h, w, c / 8));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_upsample2x_s8(const void* in, void* out, int32_t n, int32_t h, int32_t w, int32_t c, float inv_scale,
                                    void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(in && out && c % 8 == 0, "b200sd_upsample2x_s8: c=%d must be a multiple of 8", c);
    B200SD_REQUIRE(std::isfinite(inv_scale) && inv_scale > 0.f, "b200sd_upsample2x_s8: inv_scale=%g must be positive and finite",
                   static_cast<double>(inv_scale));
    const size_t total = static_cast<size_t>(n) * h * w * (c / 8);
    B200SD_CHECK_CUDA(launch_kernel(upsample2x_s8_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream,
                                    reinterpret_cast<const uint4*>(in), reinterpret_cast<uint2*>(out), n, h, w, c / 8, inv_scale));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_absmax_f16(const void* x, size_t numel, float* slot, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(x && slot && numel % 2 == 0, "b200sd_absmax_f16: bad arguments (numel=%zu must be even)", numel);
    B200SD_CHECK_CUDA(launch_kernel(absmax_f16_kernel, dim3(std::min(grid_for(numel / 2, 256), 1024)), dim3(256), 0,
                                    stream, reinterpret_cast<const __half2*>(x), numel / 2,
                                    reinterpret_cast<unsigned int*>(slot)));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_add(const void* a, const void* b, void* out, size_t numel, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(a && b && out && numel % 2 == 0, "b200sd_add: bad arguments");
    B200SD_CHECK_CUDA(launch_kernel(add_kernel, dim3(grid_for(numel / 2, 256)), dim3(256), 0, stream, reinterpret_cast<const __half2*>(a),
                                                             reinterpret_cast<const __half2*>(b),
                                                             reinterpret_cast<__half2*>(out), numel / 2));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_control_inject(const void* skip, const void* const* res, const float* scales, int32_t n_res,
                                     void* out, size_t numel, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(res && scales && out && numel > 0, "b200sd_control_inject: null pointer or empty tensor");
    B200SD_REQUIRE(n_res >= 1 && n_res <= B200SD_MAX_CONTROLNETS, "b200sd_control_inject: n_res=%d must be in [1, %d]",
                   n_res, B200SD_MAX_CONTROLNETS);
    ControlResiduals r{};
    bool aligned = reinterpret_cast<uintptr_t>(out) % 16 == 0 && reinterpret_cast<uintptr_t>(skip) % 16 == 0;
    for (int k = 0; k < n_res; ++k) {
        B200SD_REQUIRE(res[k], "b200sd_control_inject: res[%d] is null", k);
        r.r[k] = static_cast<const __half*>(res[k]);
        aligned = aligned && reinterpret_cast<uintptr_t>(res[k]) % 16 == 0;
    }
    const size_t work = aligned ? numel / 8 + numel % 8 : numel;
    B200SD_CHECK_CUDA(launch_kernel(control_inject_kernel, dim3(grid_for(work, 256)), dim3(256), 0, stream,
                                    static_cast<const __half*>(skip), r, scales, static_cast<int>(n_res),
                                    static_cast<__half*>(out), numel, static_cast<int>(aligned)));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_linear_small(const float* x, const void* wgt, const float* bias, const float* add, float* out,
                                   int32_t m, int32_t n, int32_t k, int32_t act_in, int32_t act_out, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(x && wgt && out, "b200sd_linear_small: null pointer");
    B200SD_REQUIRE(m >= 1 && m <= 32 && k % 8 == 0, "b200sd_linear_small: need 1 <= m <= 32 and k %% 8 == 0 (m=%d k=%d)",
                   m, k);
    const int blocks = (n + 7) / 8;
    const __half* w = reinterpret_cast<const __half*>(wgt);
    for (int r0 = 0; r0 < m; r0 += 8) {
        const int mm = std::min(8, m - r0);
        const float* xr = x + static_cast<size_t>(r0) * k;
        float* orow = out + static_cast<size_t>(r0) * n;
        const size_t smem = static_cast<size_t>(mm <= 2 ? 2 : 8) * k * sizeof(float);
        B200SD_REQUIRE(smem <= 160 * 1024, "b200sd_linear_small: k = %d too large for the staged input rows", k);
        static bool attr = false;
        if (!attr) {
            B200SD_CHECK_CUDA(cudaFuncSetAttribute(linear_small_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
            B200SD_CHECK_CUDA(cudaFuncSetAttribute(linear_small_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
            attr = true;
        }
        if (mm <= 2)
            B200SD_CHECK_CUDA(launch_kernel(linear_small_kernel<2>, dim3(blocks), dim3(256), smem, stream, xr, w, bias, add, orow, mm, n, k, act_in, act_out));
        else
            B200SD_CHECK_CUDA(launch_kernel(linear_small_kernel<8>, dim3(blocks), dim3(256), smem, stream, xr, w, bias, add, orow, mm, n, k, act_in, act_out));
        B200SD_CHECK_CUDA(cudaGetLastError());
        count_launch(1);
    }
    return 0;
}

extern "C" int b200sd_timestep_embedding(const float* timesteps, float* out, int32_t m, int32_t dim,
                                         int32_t flip_sin_to_cos, float freq_shift, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(timesteps && out && dim % 2 == 0, "b200sd_timestep_embedding: bad arguments");
    const int total = m * (dim / 2);
    B200SD_CHECK_CUDA(launch_kernel(timestep_embedding_kernel, dim3((total + 127) / 128), dim3(128), 0, stream, timesteps, out, m, dim, flip_sin_to_cos,
                                                                      freq_shift));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_cfg_scheduler_step(const float* noise_pred, float* latents, float* hist, float* denoised,
                                         void* unet_in, int32_t c_pad, int32_t n, int32_t c, int32_t h, int32_t w,
                                         const b200sd_step_coeffs* coeffs, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(noise_pred && latents && coeffs, "b200sd_cfg_scheduler_step: null pointer");
    B200SD_REQUIRE(coeffs->n_hist >= 0 && coeffs->n_hist <= 4 && (coeffs->n_hist == 0 || hist),
                   "b200sd_cfg_scheduler_step: bad history arguments");
    B200SD_REQUIRE(coeffs->push_eps_slot < 4 && coeffs->push_x0_slot < 4 && coeffs->push_x_slot < 4 &&
                       (hist || (coeffs->push_eps_slot < 0 && coeffs->push_x0_slot < 0 && coeffs->push_x_slot < 0)),
                   "b200sd_cfg_scheduler_step: bad history ring slot");
    const int numel = n * c * h * w;
    B200SD_CHECK_CUDA(launch_kernel(cfg_step_kernel<false, false>, dim3((numel + 255) / 256), dim3(256), 0, stream, noise_pred, latents, hist, denoised,
                                                             reinterpret_cast<__half*>(unet_in), c_pad, n, c, h * w,
                                                             *coeffs, 0.f, static_cast<const uint32_t*>(nullptr), 0u,
                                                             b200sd_blend_args{}));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_cfg_scheduler_step_noised(const float* noise_pred, float* latents, float* hist, float* denoised,
                                                void* unet_in, int32_t c_pad, int32_t n, int32_t c, int32_t h,
                                                int32_t w, const b200sd_step_coeffs* coeffs, float noise_scale,
                                                const uint32_t* philox_key, uint32_t philox_offset, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(noise_pred && latents && coeffs && philox_key, "b200sd_cfg_scheduler_step_noised: null pointer");
    B200SD_REQUIRE(coeffs->n_hist >= 0 && coeffs->n_hist <= 4 && (coeffs->n_hist == 0 || hist),
                   "b200sd_cfg_scheduler_step_noised: bad history arguments");
    B200SD_REQUIRE(coeffs->push_eps_slot < 4 && coeffs->push_x0_slot < 4 && coeffs->push_x_slot < 4 &&
                       (hist || (coeffs->push_eps_slot < 0 && coeffs->push_x0_slot < 0 && coeffs->push_x_slot < 0)),
                   "b200sd_cfg_scheduler_step_noised: bad history ring slot");
    const int numel = n * c * h * w;
    B200SD_CHECK_CUDA(launch_kernel(cfg_step_kernel<true, false>, dim3((numel + 255) / 256), dim3(256), 0, stream, noise_pred,
                                    latents, hist, denoised, reinterpret_cast<__half*>(unet_in), c_pad, n, c, h * w,
                                    *coeffs, noise_scale, philox_key, philox_offset, b200sd_blend_args{}));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_cfg_scheduler_step_blend(const float* noise_pred, float* latents, float* hist, float* denoised,
                                               void* unet_in, int32_t c_pad, int32_t n, int32_t c, int32_t h,
                                               int32_t w, const b200sd_step_coeffs* coeffs, float noise_scale,
                                               const uint32_t* philox_key, uint32_t philox_offset,
                                               const b200sd_blend_args* blend, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(noise_pred && latents && coeffs && blend, "b200sd_cfg_scheduler_step_blend: null pointer");
    B200SD_REQUIRE(blend->mask && blend->image_latents && blend->noise,
                   "b200sd_cfg_scheduler_step_blend: null blend buffer");
    B200SD_REQUIRE(coeffs->n_hist >= 0 && coeffs->n_hist <= 4 && (coeffs->n_hist == 0 || hist),
                   "b200sd_cfg_scheduler_step_blend: bad history arguments");
    B200SD_REQUIRE(coeffs->push_eps_slot < 4 && coeffs->push_x0_slot < 4 && coeffs->push_x_slot < 4 &&
                       (hist || (coeffs->push_eps_slot < 0 && coeffs->push_x0_slot < 0 && coeffs->push_x_slot < 0)),
                   "b200sd_cfg_scheduler_step_blend: bad history ring slot");
    B200SD_REQUIRE(!unet_in || c_pad >= c, "b200sd_cfg_scheduler_step_blend: c_pad < c");
    const int numel = n * c * h * w;
    const dim3 grid((numel + 255) / 256);
    if (philox_key)
        B200SD_CHECK_CUDA(launch_kernel(cfg_step_kernel<true, true>, grid, dim3(256), 0, stream, noise_pred, latents,
                                        hist, denoised, reinterpret_cast<__half*>(unet_in), c_pad, n, c, h * w,
                                        *coeffs, noise_scale, philox_key, philox_offset, *blend));
    else
        B200SD_CHECK_CUDA(launch_kernel(cfg_step_kernel<false, true>, grid, dim3(256), 0, stream, noise_pred, latents,
                                        hist, denoised, reinterpret_cast<__half*>(unet_in), c_pad, n, c, h * w,
                                        *coeffs, 0.f, static_cast<const uint32_t*>(nullptr), 0u, *blend));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_scheduler_step_guidance_free(const float* noise_pred, float* latents, float* hist,
                                                  float* denoised, void* unet_in, int32_t c_pad, int32_t n, int32_t c,
                                                  int32_t h, int32_t w, const b200sd_step_coeffs* coeffs,
                                                  float noise_scale, const uint32_t* philox_key,
                                                  uint32_t philox_offset, const b200sd_blend_args* blend,
                                                  void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(noise_pred && latents && coeffs, "b200sd_scheduler_step_guidance_free: null pointer");
    B200SD_REQUIRE(!blend || (blend->mask && blend->image_latents && blend->noise),
                   "b200sd_scheduler_step_guidance_free: null blend buffer");
    B200SD_REQUIRE(coeffs->n_hist >= 0 && coeffs->n_hist <= 4 && (coeffs->n_hist == 0 || hist),
                   "b200sd_scheduler_step_guidance_free: bad history arguments");
    B200SD_REQUIRE(coeffs->push_eps_slot < 4 && coeffs->push_x0_slot < 4 && coeffs->push_x_slot < 4 &&
                       (hist || (coeffs->push_eps_slot < 0 && coeffs->push_x0_slot < 0 && coeffs->push_x_slot < 0)),
                   "b200sd_scheduler_step_guidance_free: bad history ring slot");
    B200SD_REQUIRE(!unet_in || c_pad >= c, "b200sd_scheduler_step_guidance_free: c_pad < c");
    const int numel = n * c * h * w;
    auto* kern = philox_key ? (blend ? guidance_free_step_kernel<true, true> : guidance_free_step_kernel<true, false>)
                            : (blend ? guidance_free_step_kernel<false, true> : guidance_free_step_kernel<false, false>);
    B200SD_CHECK_CUDA(launch_kernel(kern, dim3((numel + 255) / 256), dim3(256), 0, stream, noise_pred, latents, hist,
                                    denoised, reinterpret_cast<__half*>(unet_in), c_pad, n, c, h * w, *coeffs,
                                    philox_key ? noise_scale : 0.f, philox_key, philox_key ? philox_offset : 0u,
                                    blend ? *blend : b200sd_blend_args{}));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_image_postprocess(const void* in, int32_t in_f32, int32_t c_pad, float* out_f32,
                                        uint8_t* out_u8, int32_t n, int32_t h, int32_t w, int32_t c, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(in && (out_f32 || out_u8), "b200sd_image_postprocess: null pointer");
    const size_t pixels = static_cast<size_t>(n) * h * w;
    if (in_f32)
        B200SD_CHECK_CUDA(launch_kernel(image_post_kernel<float>, dim3(grid_for(pixels * c, 256)), dim3(256), 0, stream, reinterpret_cast<const float*>(in),
                                                                                c_pad, out_f32, out_u8, pixels, c));
    else
        B200SD_CHECK_CUDA(launch_kernel(image_post_kernel<__half>, dim3(grid_for(pixels * c, 256)), dim3(256), 0, stream, reinterpret_cast<const __half*>(in),
                                                                                 c_pad, out_f32, out_u8, pixels, c));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

template <typename TO>
static int latent_prep(const float* z, const float* w, const float* b, float inv_scale, void* out, int32_t n, int32_t c,
                       int32_t h, int32_t wd, int32_t c_pad, void* stream_) {
    if (!b200sd::launch_class_enabled(8)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(z && w && out && c >= 1 && c <= 8 && c_pad >= c, "b200sd_latent_prep: bad arguments");
    const int total = n * h * wd;
    B200SD_CHECK_CUDA(launch_kernel(latent_prep_kernel<TO>, dim3((total + 255) / 256), dim3(256), 0, stream, z, w, b, inv_scale, reinterpret_cast<TO*>(out), n,
                                                               c, h * wd, c_pad));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_latent_prep(const float* z, const float* w, const float* b, float inv_scale, void* out,
                                  int32_t n, int32_t c, int32_t h, int32_t wd, int32_t c_pad, void* stream) {
    return latent_prep<__half>(z, w, b, inv_scale, out, n, c, h, wd, c_pad, stream);
}
extern "C" int b200sd_latent_prep_bf16(const float* z, const float* w, const float* b, float inv_scale, void* out,
                                       int32_t n, int32_t c, int32_t h, int32_t wd, int32_t c_pad, void* stream) {
    return latent_prep<__nv_bfloat16>(z, w, b, inv_scale, out, n, c, h, wd, c_pad, stream);
}
