// b200sd -- GroupNorm (+SiLU, + channel concat of two sources) and LayerNorm for sm_90a.
// HBM/L2-bound elementwise + reduction kernels: 16-byte vectorised, coalesced along channels.
//
// GroupNorm replaces torch.nn.GroupNorm in the reference (unet.py:430,448,528,966; eps 1e-5 in
// ResnetBlock2D / conv_norm_out, 1e-6 in SpatialTransformer and the VAE decoder) together with the
// SiLU that follows it (unet.py:472-473,480-481,1044-1045).  LayerNorm replaces LayerNormANE
// (layer_norm.py:51-80).
#include "common.cuh"
#include "../../include/b200sd.h"

#include <algorithm>
#include <cooperative_groups.h>
#include <stdlib.h>

namespace b200sd {

extern void count_launch(int n);

static constexpr int kGnMaxImages = 1024;

__device__ __forceinline__ void load8(const __half* src, float (&f)[8]) {
    const uint4 raw = *reinterpret_cast<const uint4*>(src);
    const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 t = __half22float2(h2[q]);
        f[2 * q] = t.x;
        f[2 * q + 1] = t.y;
    }
}

// ---- GroupNorm pass 1: deterministic statistics ------------------------------------------------
// grid = (chunks, n_img), block = vecs * R threads (vecs = C/8 16-byte vectors per pixel, R pixel rows
// in flight) so thread t always owns vector column t % vecs: per-channel (sum, sumsq) accumulate in
// registers over the chunk's pixels with perfectly coalesced 16 B loads; a fixed-order shared-memory
// tree folds rows -> channels -> groups (no atomics: bitwise reproducible).  The last block of each
// image (ticket counter) merges the chunk partials in chunk order with Chan's formula and writes the
// final (mean, rstd) per group.
__global__ void __launch_bounds__(416) gn_stats_kernel(const __half* __restrict__ x0, const __half* __restrict__ x1,
                                                       int c0, int c1, int hw, int groups, int chunks, int rows,
                                                       float eps, float* __restrict__ partial /* [n][chunks][g][2] */,
                                                       float* __restrict__ final_stats /* [n][g][2] */,
                                                       unsigned int* __restrict__ tickets /* [n] */) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int C = c0 + c1;
    const int cpg = C / groups;
    const int vecs = C / 8;
    const int n = blockIdx.y, chunk = blockIdx.x;
    const int px_per_chunk = (hw + chunks - 1) / chunks;
    const int px0 = chunk * px_per_chunk;
    const int px1 = min(hw, px0 + px_per_chunk);
    const int v = threadIdx.x % vecs;
    const int r = threadIdx.x / vecs;
    const int ch = v * 8;

    extern __shared__ float sm[];  // [rows][C][2] then [C][2] then [groups][2]
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    const bool from0 = ch < c0;
    const __half* base = from0 ? x0 + static_cast<size_t>(n) * hw * c0 + ch
                               : x1 + static_cast<size_t>(n) * hw * c1 + (ch - c0);
    const int cs = from0 ? c0 : c1;
    const bool active = r < rows;  // the block is padded to whole warps; padding threads only help reduce
#pragma unroll 4
    for (int px = px0 + r; active && px < px1; px += rows) {
        float f[8];
        load8(base + static_cast<size_t>(px) * cs, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            s[e] += f[e];
            q[e] += f[e] * f[e];
        }
    }
    if (active) {
        float* row_buf = sm + (static_cast<size_t>(r) * C + ch) * 2;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            row_buf[2 * e] = s[e];
            row_buf[2 * e + 1] = q[e];
        }
    }
    __syncthreads();
    // rows -> channel totals (thread c < C), fixed order
    float* ch_buf = sm + static_cast<size_t>(rows) * C * 2;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int rr = 0; rr < rows; ++rr) {
            a += sm[(static_cast<size_t>(rr) * C + c) * 2];
            b += sm[(static_cast<size_t>(rr) * C + c) * 2 + 1];
        }
        ch_buf[2 * c] = a;
        ch_buf[2 * c + 1] = b;
    }
    __syncthreads();
    const float cnt = static_cast<float>(max(0, px1 - px0) * cpg);
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
            a += ch_buf[2 * c];
            b += ch_buf[2 * c + 1];
        }
        const float mean = cnt > 0.f ? a / cnt : 0.f;
        float* o = partial + ((static_cast<size_t>(n) * chunks + chunk) * groups + g) * 2;
        o[0] = mean;
        o[1] = cnt > 0.f ? fmaxf(b - a * mean, 0.f) : 0.f;
    }
    // ---- last block of this image finalises ----
    __shared__ unsigned int s_ticket;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_ticket = atomicAdd(&tickets[n], 1u);
    __syncthreads();
    if (s_ticket != static_cast<unsigned int>(chunks - 1)) return;
    __threadfence();
    // one warp per group; lanes stride over the chunks (fixed assignment), then a fixed butterfly of Chan
    // merges: deterministic and ~log-depth instead of a serial walk over all chunks
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
    for (int g = wrp; g < groups; g += nwarps) {
        float tot = 0.f, mean = 0.f, m2 = 0.f;
        // up to 4 chunk partials per lane (chunks <= 128): issue all loads first, then merge in fixed order
        float cbv[4], mbv[4], m2v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int k = lane + 32 * q;
            cbv[q] = 0.f, mbv[q] = 0.f, m2v[q] = 0.f;
            if (k < chunks) {
                const int p0 = k * px_per_chunk;
                const int p1 = min(hw, p0 + px_per_chunk);
                cbv[q] = static_cast<float>(max(0, p1 - p0) * cpg);
                const float* pp = partial + ((static_cast<size_t>(n) * chunks + k) * groups + g) * 2;
                mbv[q] = __ldcg(pp);
                m2v[q] = __ldcg(pp + 1);
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (cbv[q] > 0.f) {
                const float nt = tot + cbv[q];
                const float delta = mbv[q] - mean;
                mean += delta * (cbv[q] / nt);
                m2 += m2v[q] + delta * delta * (tot * cbv[q] / nt);
                tot = nt;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float tot_b = __shfl_xor_sync(0xffffffffu, tot, o);
            const float mean_b = __shfl_xor_sync(0xffffffffu, mean, o);
            const float m2_b = __shfl_xor_sync(0xffffffffu, m2, o);
            // symmetric merge so both partners compute the identical result
            const float nt = tot + tot_b;
            if (nt > 0.f) {
                const float lo_t = (lane & o) ? tot_b : tot, hi_t = (lane & o) ? tot : tot_b;
                const float lo_m = (lane & o) ? mean_b : mean, hi_m = (lane & o) ? mean : mean_b;
                const float lo_2 = (lane & o) ? m2_b : m2, hi_2 = (lane & o) ? m2 : m2_b;
                const float delta = hi_m - lo_m;
                mean = lo_m + delta * (hi_t / nt);
                m2 = lo_2 + hi_2 + delta * delta * (lo_t * hi_t / nt);
                tot = nt;
            }
        }
        if (lane == 0) {
            final_stats[(static_cast<size_t>(n) * groups + g) * 2] = mean;
            final_stats[(static_cast<size_t>(n) * groups + g) * 2 + 1] = rsqrtf(m2 / tot + eps);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) tickets[n] = 0;  // self-reset for the next launch
}

// ---- GroupNorm pass 2: normalise, affine, optional SiLU (and concat of the two sources) ------------
__global__ void __launch_bounds__(256) gn_apply_kernel(const __half* __restrict__ x0, const __half* __restrict__ x1,
                                                       int c0, int c1, int hw, int groups,
                                                       const float* __restrict__ final_stats,
                                                       const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, int silu,
                                                       __half* __restrict__ out, int px_per_block) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int C = c0 + c1;
    const int cpg = C / groups;
    const int vecs = C / 8;
    const int n = blockIdx.y;
    extern __shared__ float sm[];  // scale[C], shift[C]
    float* s_scale = sm;
    float* s_shift = sm + C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c / cpg;
        const float mean = final_stats[(static_cast<size_t>(n) * groups + g) * 2];
        const float rstd = final_stats[(static_cast<size_t>(n) * groups + g) * 2 + 1];
        const float sc = gamma[c] * rstd;
        s_scale[c] = sc;
        s_shift[c] = beta[c] - mean * sc;
    }
    __syncthreads();
    const int px0 = blockIdx.x * px_per_block;
    const int px1 = min(hw, px0 + px_per_block);
    const int total = (px1 - px0) * vecs;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const int px = px0 + i / vecs;
        const int ch = (i % vecs) * 8;
        const __half* src = (ch < c0) ? x0 + (static_cast<size_t>(n) * hw + px) * c0 + ch
                                      : x1 + (static_cast<size_t>(n) * hw + px) * c1 + (ch - c0);
        float f[8];
        load8(src, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float y = f[e] * s_scale[ch + e] + s_shift[ch + e];
            f[e] = silu ? silu_f(y) : y;
        }
        uint4 pk;
        pk.x = pack_half2(f[0], f[1]);
        pk.y = pack_half2(f[2], f[3]);
        pk.z = pack_half2(f[4], f[5]);
        pk.w = pack_half2(f[6], f[7]);
        *reinterpret_cast<uint4*>(out + (static_cast<size_t>(n) * hw + px) * C + ch) = pk;
    }
}

// ---- GroupNorm apply from producer-side statistics -----------------------------------------------------------------
// The statistics pass is gone: the kernel that produced the tensor left per-channel (sum, sum of squares) behind
// (staged GEMM epilogue, b200sd_gemm_args.cs_chan).  grid = (pixel blocks, n_img); every block folds the channel sums
// of its image into group statistics (warp per group, fixed order), builds the per-channel scale / shift table in
// shared memory and normalises (+SiLU, + concat of two sources) its pixel range: one read and one write of the tensor.
__global__ void __launch_bounds__(256) gn_apply_chan_kernel(const __half* __restrict__ x0, const __half* __restrict__ x1,
                                                            int c0, int c1, int hw, int groups, float eps,
                                                            const float* __restrict__ chan0, const float* __restrict__ chan1,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            int silu, __half* __restrict__ out, int px_per_block) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int C = c0 + c1;
    const int cpg = C / groups;
    const int vecs = C / 8;
    const int n = blockIdx.y;
    extern __shared__ float sm[];  // scale[C], shift[C], stat[groups][2]
    float* s_scale = sm;
    float* s_shift = sm + C;
    float* s_stat = sm + 2 * C;
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const float inv_cnt = 1.0f / (static_cast<float>(cpg) * static_cast<float>(hw));
    for (int g = wrp; g < groups; g += 8) {
        float s = 0.f, q = 0.f;
        for (int c = g * cpg + lane; c < (g + 1) * cpg; c += 32) {
            const float2 v = (c < c0) ? *reinterpret_cast<const float2*>(chan0 + (static_cast<size_t>(n) * c0 + c) * 2)
                                      : *reinterpret_cast<const float2*>(chan1 + (static_cast<size_t>(n) * c1 + c - c0) * 2);
            s += v.x, q += v.y;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, o);
            q += __shfl_xor_sync(0xffffffffu, q, o);
        }
        if (lane == 0) {
            const float mean = s * inv_cnt;
            s_stat[2 * g] = mean;
            s_stat[2 * g + 1] = rsqrtf(fmaxf(q * inv_cnt - mean * mean, 0.f) + eps);
        }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c / cpg;
        const float sc = gamma[c] * s_stat[2 * g + 1];
        s_scale[c] = sc;
        s_shift[c] = beta[c] - s_stat[2 * g] * sc;
    }
    __syncthreads();
    const int px0 = blockIdx.x * px_per_block;
    const int px1 = min(hw, px0 + px_per_block);
    const int total = (px1 - px0) * vecs;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const int px = px0 + i / vecs;
        const int ch = (i % vecs) * 8;
        const __half* src = (ch < c0) ? x0 + (static_cast<size_t>(n) * hw + px) * c0 + ch
                                      : x1 + (static_cast<size_t>(n) * hw + px) * c1 + (ch - c0);
        float f[8];
        load8(src, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float y = f[e] * s_scale[ch + e] + s_shift[ch + e];
            f[e] = silu ? silu_f(y) : y;
        }
        uint4 pk;
        pk.x = pack_half2(f[0], f[1]);
        pk.y = pack_half2(f[2], f[3]);
        pk.z = pack_half2(f[4], f[5]);
        pk.w = pack_half2(f[6], f[7]);
        *reinterpret_cast<uint4*>(out + (static_cast<size_t>(n) * hw + px) * C + ch) = pk;
    }
}

// ---- GroupNorm on thread-block clusters (the default path) ---------------------------------------
// grid = (cs, C / chunk, n_img) with cluster dims (cs, 1, 1): one cluster per (image, channel chunk), where a
// chunk is a whole number of groups and of 16-byte vectors.  The cs CTAs of a cluster split the image's
// pixels; each keeps its [pixels x chunk] slab in shared memory, so the tensor is read from L2/HBM exactly
// once.  Statistics are one pass (sum and sum of squares in fp32, see below) and are exchanged ONCE between the CTAs
// through distributed shared memory in rank order -- no global barrier, no partial buffers, no atomics (bitwise
// reproducible).  Thread t owns vector column t % vpr for all its pixels, so per-channel
// partial sums live in registers and fold rows -> channels -> groups in a fixed order.
template <int kRowsInFlight>
__global__ void gn_cluster_kernel(const __half* __restrict__ x0, const __half* __restrict__ x1, int c0, int c1, int hw,
                                  int groups, int chunk_ch, int rows_per_cta, float eps,
                                  const float* __restrict__ gamma, const float* __restrict__ beta, int silu,
                                  __half* __restrict__ out) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const int cs = gridDim.x, rank = blockIdx.x;
    const int C = c0 + c1, cpg = C / groups;
    const int vpr = chunk_ch >> 3;
    const int ng = chunk_ch / cpg;
    const int ch0 = blockIdx.y * chunk_ch;
    const int n = blockIdx.z;
    const int TY = blockDim.x / vpr;
    const int cv = threadIdx.x % vpr, ty = threadIdx.x / vpr;
    const bool active = ty < TY;
    const int px0 = rank * rows_per_cta, px1 = min(hw, px0 + rows_per_cta);
    const int ch = ch0 + cv * 8;
    const bool from0 = ch < c0;
    const int ld = from0 ? c0 : c1;
    const __half* src = from0 ? x0 + static_cast<size_t>(n) * hw * c0 + ch : x1 + static_cast<size_t>(n) * hw * c1 + (ch - c0);

    extern __shared__ __align__(16) uint8_t csm[];
    uint4* slab = reinterpret_cast<uint4*>(csm);                                   // [rows_per_cta][vpr]
    float* red = reinterpret_cast<float*>(slab + static_cast<size_t>(rows_per_cta) * vpr);  // [TY][2][chunk_ch]
    float* chsum = red + 2 * TY * chunk_ch;                                        // [2][chunk_ch]
    float* xchg = chsum + 2 * chunk_ch;                                            // [2][ng]  (read by the peers)
    float* stat = xchg + 2 * ng;                                                   // [2][ng]  mean, rstd
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();

    // ---- one pass: global -> shared slab, per-channel (sum, sum of squares) in registers; ONE exchange through
    // distributed shared memory yields mean and variance of every group (fp32 sums over <= a few 10^4 elements:
    // E[x^2] - mean^2 keeps > 4 significant digits for |mean| / sigma up to ~30, far beyond these activations) ----
    float acc[8], acq[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = acq[e] = 0.f;
    if (active) {
        // eight rows per thread are requested before the first one is consumed (the compiler keeps only two loads in
        // flight across the shared-memory stores of a plainly unrolled loop: ncu showed every row's first use stalling)
        // (kRowsInFlight = 2 for the small maps: a thread has one or two rows there and the 32 extra registers would cost a
        // resident CTA per SM)
        for (int pxb = px0 + ty; pxb < px1; pxb += TY * kRowsInFlight) {
            uint4 raw[kRowsInFlight];
#pragma unroll
            for (int i = 0; i < kRowsInFlight; ++i) {
                const int px = pxb + i * TY;
                raw[i] = px < px1 ? __ldg(reinterpret_cast<const uint4*>(src + static_cast<size_t>(px) * ld)) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int i = 0; i < kRowsInFlight; ++i) {
                const int px = pxb + i * TY;
                if (px < px1) {
                    slab[(px - px0) * vpr + cv] = raw[i];
                    const __half2* h2 = reinterpret_cast<const __half2*>(&raw[i]);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float2 t = __half22float2(h2[q]);
                        acc[2 * q] += t.x;
                        acc[2 * q + 1] += t.y;
                        acq[2 * q] = fmaf(t.x, t.x, acq[2 * q]);
                        acq[2 * q + 1] = fmaf(t.y, t.y, acq[2 * q + 1]);
                    }
                }
            }
        }
    }
    // rows -> channels -> groups in a fixed order (red holds [TY][2][chunk_ch]), then across the cluster in rank order
    if (active) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            red[(ty * 2) * chunk_ch + cv * 8 + e] = acc[e];
            red[(ty * 2 + 1) * chunk_ch + cv * 8 + e] = acq[e];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * chunk_ch; i += blockDim.x) {
        const int which = i / chunk_ch, c = i - which * chunk_ch;
        float a = 0.f;
        for (int r = 0; r < TY; ++r) a += red[(r * 2 + which) * chunk_ch + c];
        chsum[which * chunk_ch + c] = a;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * ng; i += blockDim.x) {
        const int which = i / ng, g = i - which * ng;
        float a = 0.f;
        for (int c = 0; c < cpg; ++c) a += chsum[which * chunk_ch + g * cpg + c];
        xchg[which * ng + g] = a;
    }
    cluster.sync();
    const float inv_cnt = 1.0f / (static_cast<float>(hw) * static_cast<float>(cpg));
    for (int g = threadIdx.x; g < ng; g += blockDim.x) {
        float s = 0.f, q = 0.f;
        for (int r = 0; r < cs; ++r) {
            s += *cluster.map_shared_rank(&xchg[g], r);
            q += *cluster.map_shared_rank(&xchg[ng + g], r);
        }
        const float mean = s * inv_cnt;
        stat[g] = mean;
        stat[ng + g] = rsqrtf(fmaxf(q * inv_cnt - mean * mean, 0.f) + eps);
    }
    float mean8[8];
    cluster.barrier_arrive();  // done reading the peers' shared memory; matched by the wait before exit
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 8; ++e) mean8[e] = active ? stat[(cv * 8 + e) / cpg] : 0.f;
    // ---- apply: y = (x - mean) * rstd * gamma + beta (+ SiLU), slab -> global ----
    if (active) {
        float sc8[8], sh8[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int g = (cv * 8 + e) / cpg;
            sc8[e] = stat[ng + g] * gamma[ch + e];
            sh8[e] = fmaf(-mean8[e], sc8[e], beta[ch + e]);
        }
        __half* dst = out + static_cast<size_t>(n) * hw * C + ch;
#pragma unroll 2
        for (int px = px0 + ty; px < px1; px += TY) {
            const uint4 raw = slab[(px - px0) * vpr + cv];
            const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
            float f[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 t = __half22float2(h2[q]);
                f[2 * q] = t.x;
                f[2 * q + 1] = t.y;
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float y = fmaf(f[e], sc8[e], sh8[e]);
                f[e] = silu ? __fdividef(y, 1.0f + __expf(-y)) : y;
            }
            uint4 pk;
            pk.x = pack_half2(f[0], f[1]);
            pk.y = pack_half2(f[2], f[3]);
            pk.z = pack_half2(f[4], f[5]);
            pk.w = pack_half2(f[6], f[7]);
            *reinterpret_cast<uint4*>(dst + static_cast<size_t>(px) * C) = pk;
        }
    }
    cluster.barrier_wait();
}

static int gn_chunks(int hw, int n_img) {
    // enough blocks to keep many loads in flight (the data is a few MB, L2 resident), at most 128 so the
    // finalising warps read <= 4 partials per lane
    (void)n_img;
    return std::max(1, std::min(128, hw / 16));
}

static unsigned int* gn_tickets() {
    static unsigned int* t = nullptr;
    if (!t) {
        if (cudaMalloc(&t, kGnMaxImages * sizeof(unsigned int)) != cudaSuccess) return nullptr;
        cudaMemset(t, 0, kGnMaxImages * sizeof(unsigned int));
    }
    return t;
}

// ---- LayerNorm over channels of [rows, c]; one warp per row, two-pass in registers -----------
template <int kVecsPerLane>
__global__ void __launch_bounds__(256) layer_norm_kernel(const __half* __restrict__ x, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, __half* __restrict__ out,
                                                         int rows, int c, float eps) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const int vecs = c / 8;
    const __half* src = x + static_cast<size_t>(warp) * c;
    float f[kVecsPerLane][8];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < kVecsPerLane; ++k) {
        const int v = lane + 32 * k;
        if (v < vecs) {
            const uint4 raw = *reinterpret_cast<const uint4*>(src + v * 8);
            const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 t = __half22float2(h2[q]);
                f[k][2 * q] = t.x;
                f[k][2 * q + 1] = t.y;
                s += t.x + t.y;
            }
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) f[k][e] = 0.f;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / c;
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < kVecsPerLane; ++k) {
        const int v = lane + 32 * k;
        if (v < vecs) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float d = f[k][e] - mean;
                sq += d * d;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq / c + eps);
    __half* dst = out + static_cast<size_t>(warp) * c;
#pragma unroll
    for (int k = 0; k < kVecsPerLane; ++k) {
        const int v = lane + 32 * k;
        if (v < vecs) {
            float y[8];
            const float4 g0 = *reinterpret_cast<const float4*>(gamma + v * 8);
            const float4 g1 = *reinterpret_cast<const float4*>(gamma + v * 8 + 4);
            const float4 b0 = *reinterpret_cast<const float4*>(beta + v * 8);
            const float4 b1 = *reinterpret_cast<const float4*>(beta + v * 8 + 4);
            const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) y[e] = (f[k][e] - mean) * rstd * gg[e] + bb[e];
            uint4 pk;
            pk.x = pack_half2(y[0], y[1]);
            pk.y = pack_half2(y[2], y[3]);
            pk.z = pack_half2(y[4], y[5]);
            pk.w = pack_half2(y[6], y[7]);
            *reinterpret_cast<uint4*>(dst + v * 8) = pk;
        }
    }
}


// ---- row softmax: fp32 scores [rows, cols] -> fp16 probabilities (VAE mid-block attention, d=512) ----
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ in, __half* __restrict__ out,
                                                           int cols, float scale_log2) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const size_t row = blockIdx.x;
    const float* src = in + row * cols;
    __half* dst = out + row * cols;
    __shared__ float red[8];
    float m = -INFINITY;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, src[c] * scale_log2);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = red[0];
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    __syncthreads();
    float s = 0.f;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) s += exp2f(src[c] * scale_log2 - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0.f;
    for (int i = 0; i < 8; ++i) s += red[i];
    const float inv = 1.0f / s;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) dst[c] = __float2half_rn(exp2f(src[c] * scale_log2 - m) * inv);
}

}  // namespace b200sd

using namespace b200sd;

extern "C" size_t b200sd_group_norm_workspace_bytes(int32_t n_img, int32_t hw, int32_t c, int32_t groups) {
    (void)c;
    // chunk partials + final (mean, rstd)
    const size_t two_kernel = static_cast<size_t>(n_img) * gn_chunks(hw, n_img) * groups * 2 +
                              static_cast<size_t>(n_img) * groups * 2;
    return two_kernel * sizeof(float);
}

extern "C" int b200sd_group_norm(const void* x0, const void* x1, int32_t c0, int32_t c1, int32_t n_img, int32_t hw,
                                 int32_t groups, float eps, const float* gamma, const float* beta, int32_t silu,
                                 void* out, float* stats_ws, size_t stats_ws_bytes, void* stream_) {
    if (!b200sd::launch_class_enabled(4)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int C = c0 + c1;
    B200SD_REQUIRE(x0 && out && gamma && beta && stats_ws, "b200sd_group_norm: null pointer");
    B200SD_REQUIRE(c0 > 0 && c0 % 8 == 0 && c1 >= 0 && c1 % 8 == 0 && (c1 == 0 || x1),
                   "b200sd_group_norm: channels must be multiples of 8 (c0=%d c1=%d)", c0, c1);
    B200SD_REQUIRE(groups > 0 && C % groups == 0, "b200sd_group_norm: %d channels not divisible by %d groups", C,
                   groups);
    B200SD_REQUIRE(n_img <= kGnMaxImages, "b200sd_group_norm: at most %d images per call", kGnMaxImages);
    B200SD_REQUIRE(stats_ws_bytes >= b200sd_group_norm_workspace_bytes(n_img, hw, C, groups),
                   "b200sd_group_norm: workspace too small");
    unsigned int* tickets = gn_tickets();
    B200SD_REQUIRE(tickets != nullptr, "b200sd_group_norm: could not allocate ticket counters");
    const int vecs = C / 8;
    B200SD_REQUIRE(vecs <= 384, "b200sd_group_norm: too many channels (%d)", C);
    // ---- cluster path: one cluster of <= 8 CTAs per (image, channel chunk), slab in shared memory ----
    {
        static int mode = -1;  // B200SD_GN_CLUSTER=0 disables
        if (mode < 0) {
            const char* e = getenv("B200SD_GN_CLUSTER");
            mode = (e && e[0] == '0') ? 0 : 1;
        }
        const int cpg = C / groups;
        int chunk = cpg;
        while (chunk % 8 != 0) chunk += cpg;                       // lcm(cpg, 8)
        while (chunk < 32 && C % (2 * chunk) == 0) chunk *= 2;     // at least 64-byte pieces per pixel
        const int vpr = chunk / 8;
        const long clusters = static_cast<long>(C / chunk) * n_img;
        int cs = 8;
        while (cs > 1 && (hw / cs < 32 || clusters * cs > 4L * num_sms())) cs >>= 1;
        const int rows_per_cta = (hw + cs - 1) / cs;
        // B200SD_GN_THREADS (tuning aid): 512 threads for slabs of >= 256 rows
        static int big_threads = -1;
        if (big_threads < 0) {
            const char* e = getenv("B200SD_GN_THREADS");
            big_threads = (e && atoi(e) == 512) ? 512 : 256;
        }
        const int threads = rows_per_cta >= 256 ? big_threads : 256;
        const int TY = threads / std::max(1, vpr);
        const size_t csmem = static_cast<size_t>(rows_per_cta) * vpr * 16 +
                             (2 * static_cast<size_t>(TY) * chunk + 2 * chunk + 4 * (chunk / cpg)) * sizeof(float);
        if (mode == 1 && vpr <= 64 && C % chunk == 0 && csmem <= 200 * 1024 && n_img <= 65535 && C / chunk <= 65535) {
            const int deep = (rows_per_cta + TY - 1) / TY >= 3 ? 1 : 0;
            auto kern = deep ? gn_cluster_kernel<8> : gn_cluster_kernel<2>;
            static bool attr[2] = {false, false};
            if (!attr[deep]) {
                B200SD_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
                attr[deep] = true;
            }
            cudaLaunchConfig_t cfg;
            memset(&cfg, 0, sizeof(cfg));
            cfg.gridDim = dim3(cs, C / chunk, n_img);
            cfg.blockDim = dim3(threads);
            cfg.dynamicSmemBytes = csmem;
            cfg.stream = stream;
            cudaLaunchAttribute at[2];
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = cs;
            at[0].val.clusterDim.y = 1;
            at[0].val.clusterDim.z = 1;
            cfg.attrs = at;
            cfg.numAttrs = 1;
            if (pdl_enabled()) {
                at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
                at[1].val.programmaticStreamSerializationAllowed = 1;
                cfg.numAttrs = 2;
            }
            B200SD_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, reinterpret_cast<const __half*>(x0),
                                                 reinterpret_cast<const __half*>(x1), static_cast<int>(c0),
                                                 static_cast<int>(c1), static_cast<int>(hw), static_cast<int>(groups), chunk,
                                                 rows_per_cta, eps, gamma, beta, static_cast<int>(silu),
                                                 reinterpret_cast<__half*>(out)));
            B200SD_CHECK_CUDA(cudaGetLastError());
            count_launch(1);
            return 0;
        }
    }
    // ---- fallback (slab larger than shared memory, e.g. the VAE decoder's 512x512 maps): statistics + apply ----
    const int chunks = gn_chunks(hw, n_img);
    const int rows = std::max(1, std::min(256 / vecs, (hw + chunks - 1) / chunks));
    const int threads = (vecs * rows + 31) / 32 * 32;
    float* partial = stats_ws;
    float* final_stats = stats_ws + static_cast<size_t>(n_img) * chunks * groups * 2;
    const size_t smem1 = (static_cast<size_t>(rows) * C * 2 + static_cast<size_t>(C) * 2) * sizeof(float);
    static size_t smem1_max = 48 * 1024;
    if (smem1 > smem1_max) {
        B200SD_CHECK_CUDA(cudaFuncSetAttribute(gn_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem1)));
        smem1_max = smem1;
    }
    B200SD_CHECK_CUDA(launch_kernel(gn_stats_kernel, dim3(dim3(chunks, n_img)), dim3(threads), smem1, stream, 
        reinterpret_cast<const __half*>(x0), reinterpret_cast<const __half*>(x1), c0, c1, hw, groups, chunks, rows, eps,
        partial, final_stats, tickets));
    B200SD_CHECK_CUDA(cudaGetLastError());
    const int want_blocks = std::max(1, (num_sms() * 4) / std::max(1, n_img));
    const int px_per_block = std::max(1, (hw + want_blocks - 1) / want_blocks);
    const int blocks = (hw + px_per_block - 1) / px_per_block;
    const size_t smem2 = 2 * static_cast<size_t>(C) * sizeof(float);
    B200SD_CHECK_CUDA(launch_kernel(gn_apply_kernel, dim3(dim3(blocks, n_img)), dim3(256), smem2, stream, 
        reinterpret_cast<const __half*>(x0), reinterpret_cast<const __half*>(x1), c0, c1, hw, groups, final_stats,
        gamma, beta, silu, reinterpret_cast<__half*>(out), px_per_block));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(2);
    return 0;
}

extern "C" int b200sd_group_norm_apply(const void* x0, const void* x1, int32_t c0, int32_t c1, int32_t n_img, int32_t hw,
                                       int32_t groups, float eps, const float* chan0, const float* chan1,
                                       const float* gamma, const float* beta, int32_t silu, void* out, void* stream_) {
    if (!b200sd::launch_class_enabled(4)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int C = c0 + c1;
    B200SD_REQUIRE(x0 && out && gamma && beta && chan0 && (c1 == 0 || (x1 && chan1)), "b200sd_group_norm_apply: null pointer");
    B200SD_REQUIRE(c0 > 0 && c0 % 8 == 0 && c1 >= 0 && c1 % 8 == 0 && groups > 0 && C % groups == 0 && n_img <= 65535,
                   "b200sd_group_norm_apply: bad channel / group counts (c0=%d c1=%d groups=%d)", c0, c1, groups);
    const int want_blocks = std::max(1, (num_sms() * 2) / std::max(1, n_img));
    const int px_per_block = std::max(1, (hw + want_blocks - 1) / want_blocks);
    const int blocks = (hw + px_per_block - 1) / px_per_block;
    const size_t smem = (2 * static_cast<size_t>(C) + 2 * groups) * sizeof(float);
    B200SD_REQUIRE(smem <= 48 * 1024, "b200sd_group_norm_apply: too many channels (%d)", C);
    B200SD_CHECK_CUDA(launch_kernel(gn_apply_chan_kernel, dim3(blocks, n_img), dim3(256), smem, stream,
                                    reinterpret_cast<const __half*>(x0), reinterpret_cast<const __half*>(x1), c0, c1, hw, groups, eps,
                                    chan0, chan1, gamma, beta, silu, reinterpret_cast<__half*>(out), px_per_block));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_layer_norm(const void* x, const float* gamma, const float* beta, void* out, int32_t rows,
                                 int32_t c, float eps, void* stream_) {
    if (!b200sd::launch_class_enabled(4)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(x && gamma && beta && out, "b200sd_layer_norm: null pointer");
    B200SD_REQUIRE(c % 8 == 0 && c > 0 && c <= 2048, "b200sd_layer_norm: c=%d must be a multiple of 8, <= 2048", c);
    const int vecs = c / 8;
    const int per_lane = (vecs + 31) / 32;
    const int blocks = (rows + 7) / 8;
    const __half* xi = reinterpret_cast<const __half*>(x);
    __half* xo = reinterpret_cast<__half*>(out);
    if (per_lane <= 2)
        B200SD_CHECK_CUDA(launch_kernel(layer_norm_kernel<2>, dim3(blocks), dim3(256), 0, stream, xi, gamma, beta, xo, rows, c, eps));
    else if (per_lane <= 5)
        B200SD_CHECK_CUDA(launch_kernel(layer_norm_kernel<5>, dim3(blocks), dim3(256), 0, stream, xi, gamma, beta, xo, rows, c, eps));
    else
        B200SD_CHECK_CUDA(launch_kernel(layer_norm_kernel<8>, dim3(blocks), dim3(256), 0, stream, xi, gamma, beta, xo, rows, c, eps));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_softmax_rows(const float* in, void* out, int32_t rows, int32_t cols, float scale,
                                   void* stream_) {
    if (!b200sd::launch_class_enabled(4)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(in && out && rows > 0 && cols > 0, "b200sd_softmax_rows: bad arguments");
    B200SD_CHECK_CUDA(launch_kernel(softmax_rows_kernel, dim3(rows), dim3(256), 0, stream, in, reinterpret_cast<__half*>(out), cols,
                                                  scale * 1.4426950408889634f));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}
