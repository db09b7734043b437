// b200sd -- wgmma GEMM / im2col-free implicit-GEMM 3x3 convolution for sm_90a.
//
// One persistent, warp-specialised kernel, compiled per tile width kBN:
//   warps 8..11 producer warpgroup: warp 8 issues TMA (cp.async.bulk.tensor 2D/4D boxes, SWIZZLE_128B, mbarrier tx);
//               the warpgroup gives its registers to the consumers (setmaxnreg)
//   warps 0..7  two consumer warpgroups: wgmma m64nNk16 (fp16 operands from shared memory, fp32 accumulators in
//               registers; warpgroup w owns tile rows [64 w, 64 w + 64)), then the epilogue: the accumulators are parked
//               in shared memory over the drained stages and read back row-wise (bias / time-embedding / GEGLU /
//               residual; fp16|fp32 stores or fp32 split-K partials)
//
// Replaces every nn.Conv2d of the reference UNet / VAE decoder (reference
// python_coreml_stable_diffusion/unet.py:74-84, 435-464, 499-507, 533-551, 601-617, 853, 970).
// The 3x3 convolution never materialises im2col: k-block (tap, 64-channel chunk) is one TMA box
// of the NHWC activation shifted by the tap offset; TMA's out-of-bounds zero fill is the padding.
#include "common.cuh"
#include "../../include/b200sd.h"

#include <algorithm>
#include <cmath>
#include <stdlib.h>
#include <type_traits>

namespace b200sd {

static constexpr int kBM = 128;
static constexpr int kBK = 64;
static constexpr int kAStage = kBM * kBK * 2;  // 16 KiB
// GEMM kernel: warps 0..7 are two consumer warpgroups (wgmma + epilogue), warps 8..11 the producer warpgroup (warp 8,
// lane 0 issues TMA).  The producer warpgroup hands most of its registers to the consumers (setmaxnreg), so a 64 x 256
// fp32 accumulator tile (128 registers per thread) fits: 128 x kProducerRegs + 256 x kConsumerRegs <= 65536.
static constexpr int kGemmThreads = 384;
static constexpr int kProducerRegs = 40;
static constexpr int kConsumerRegs = 232;
static constexpr int kHaloThreads = 288;  // halo kernels: warps 0..7 consumers, warp 8 producer
static constexpr int kEpiThreads = 256;
static constexpr int kProducerWarp = 8;
static constexpr int kMaxStages = 8;
static constexpr int kHaloMaxStages = 24;  // weight ring of the halo kernel (narrow tiles need many stages in flight)
static constexpr int kSmemBudget = 220 * 1024;
static constexpr int kEpiFixed = 2 * 256 * 4 + 256 * 4 + 64;  // bias vectors, LayerNorm fold vector, flags + image ids

// Shared-memory budget of one GEMM CTA.  B200SD_SMEM_KB (read per call: tuning scripts flip it) caps the pipeline
// depth.  The register file holds one GEMM CTA per SM, so a smaller budget only shortens the pipeline.
static int smem_budget() {
    const char* e = getenv("B200SD_SMEM_KB");
    if (e && e[0]) {
        const int kb = atoi(e);
        if (kb >= 48 && kb <= 220) return kb * 1024;
    }
    return kSmemBudget;
}

struct __align__(64) GemmParams {
    CUtensorMap tmA0, tmA1, tmB;
    CUtensorMap tmA2, tmA3;  // mode 1: centre-tap-only sources (the ResNet shortcut folded into conv2 as extra k-blocks)
    int kc2, kc3;            // their 64-channel chunk counts; k-blocks [taps * kc, taps * kc + kc2 + kc3)
    int mode, M, N, n_store;  // n_store: columns written per row (N or N/2 for GEGLU)
    int C0, Kpt, kc0, kc, taps;
    int kb_total, kb_per_split, splits;
    int m_tiles, n_tiles, block_n, stages;
    int n_img, Hout, Wout, stride, bw_log2, bh_log2, tiles_w, tiles_h;
    int bias_rows, bias_stride, geglu, out_f32;
    int act;         // 0 none, 1 SiLU after bias (generic variant only)
    int cluster;     // split-K on a thread-block cluster: the `splits` CTAs of a tile reduce it through DSMEM
    int pad_lo;      // conv: zero padding before the first row / column (1 = symmetric pad 1; 0 = pad only after: the
                     // VAE encoder's F.pad(x, (0, 1, 0, 1)) + stride-2 conv)
    int wgt_tiled;   // B operand pre-tiled: tile (n_tile, kb) starts at row (n_tile * kb_total + kb) * block_n
    int bias_mode;   // 0 none, 1 staged in smem (<= 2 vectors per tile), 2 read from global per chunk
    int res_smem;    // 1: residual tile prefetched into smem with cp.async
    void* out;
    const float* bias;
    const __half* residual;
    float* partial;
    // ---- mode 2 (halo-reuse 3x3 convolution): the image is walked in padded-linear order q = y * (W + 1) + x ----
    int H, W, Wp, tiles_per_img, patch_rows, patch_bytes, upsample;
    int inv_wp;                // ceil(2^20 / Wp): i / Wp == (i * inv_wp) >> 20 for the patch indices used here
    int win, tw, th, tiles_x;  // mode 2 windowed tiling (wide images): tiles of th rows x tw columns, pitch Wp = tw + halo
    int desc_bo;            // 1: row-shifted A descriptors carry (address >> 7) & 7 in the matrix-base-offset field
    int tma_patch, patch_tx;  // plain convolution: the producer warp loads each patch with ONE 4-D TMA box of patch_tx bytes
    const __half* a0;       // raw NHWC sources (loader warps read them with plain loads)
    const __half* a1;
    int C1;
    // ---- GroupNorm (+SiLU) applied to the A operand by the loader warps (mode 2) ----
    const float* gn_chan0;  // [n_img][C0][2] per-channel (sum, sum of squares) of a0, produced by a0's producer
    const float* gn_chan1;
    const float* gn_gamma;  // [C0 + C1]
    const float* gn_beta;
    int gn_groups, gn_silu, gn_hw;  // gn_hw: pixels per image the sums run over
    float gn_eps;
    // ---- statistics side outputs of the staged epilogue ----
    float* cs_partial;         // [n_img][cs_slots][N][2] per-tile column sums
    float* cs_chan;            // [n_img][N][2] per-channel sums over the image (written by the last CTA to arrive)
    unsigned int* cs_tickets;  // [n_img][n_tiles], zero-initialised, self-resetting
    int cs_slots, cs_hw;       // partial slots per image; output rows (pixels) per image
    float* rs_out;             // [n_tiles][M][2] per-row (sum, sum of squares) over this tile's columns
    // ---- LayerNorm folded into this GEMM: out = rstd_r * (acc - mu_r * wg) + bias', statistics from the producer ----
    const float* ln_stat;      // [ln_parts][M][2]
    const float* ln_wg;        // [N] sum_k W'[j, k]
    int ln_parts, ln_k;
    float ln_eps;
    int staged;                // staged epilogue (fp16 tile in shared memory, coalesced row-wise stores)
    int stage_dedicated;       // the staging tile has its own shared memory (persistent CTAs with several tiles)
    long long* dbg;            // optional timeline of CTA 0 (clock64 at fixed points; tools/halo_timeline.py)
    const float* col_scale;    // int8 convolution: [N] s_a * s_w[n], applied to the int32 accumulators
    // ---- palettized B operand (b200sd_gemm_lut): tmB maps the packed n-bit indices [N][kb_total * 8 * nbits bytes];
    // the producer warpgroup decodes each k-block through the row segment's palette into the fp16 B stage ----
    const __half* lut;         // [3][256] palettes of output rows [0, seg_end0), [seg_end0, seg_end1), [seg_end1, N)
    const float* kscale;       // [kb_total * 64] per-k scale (LayerNorm fold) or null
    int nbits, pk_box, pk_slots, seg_end0, seg_end1;
    float out_inv_scale;       // int8 output (kOutS8): q = clamp(rint(y * out_inv_scale), -127, 127)
};

struct TileCoord {
    int m_tile, n_tile, split;
    int n0, h0, w0;  // conv: output-space origin of the 128-pixel box
    // mode 2: output row r of the tile is patch pixel c0 + r; patch pixel i is image pixel (ya + i / P, xa + i % P);
    // rows whose pixel falls outside [ylo, yhi) x [xlo, xhi) are junk (pad columns, tile tail)
    int ya, xa, c0, xlo, xhi, ylo, yhi;
};

__device__ __forceinline__ TileCoord decode_work(const GemmParams& p, int work) {
    TileCoord t;
    if (p.cluster) {  // the CTAs of a cluster (consecutive blockIdx.x) are the k-splits of one tile
        t.split = work % p.splits;
        const int r = work / p.splits;
        t.m_tile = r % p.m_tiles;
        t.n_tile = r / p.m_tiles;
    } else {
        t.m_tile = work % p.m_tiles;
        const int r = work / p.m_tiles;
        t.n_tile = r % p.n_tiles;
        t.split = r / p.n_tiles;
    }
    t.n0 = t.h0 = t.w0 = 0;
    if (p.mode == 2) {
        t.n0 = t.m_tile / p.tiles_per_img;
        const int tt = t.m_tile - t.n0 * p.tiles_per_img;
        const int halo = p.taps == 9 ? 1 : 0;
        if (p.win) {  // a th x tw window of the image; the patch adds the halo ring, pitch Wp = tw + 2 * halo
            const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
            const int y0 = ty * p.th, x0 = tx * p.tw;
            t.w0 = tt;
            t.ya = y0 - halo, t.xa = x0 - halo, t.c0 = halo * (p.Wp + 1);
            t.xlo = x0, t.xhi = min(x0 + p.tw, p.W), t.ylo = y0, t.yhi = min(y0 + p.th, p.H);
        } else {      // 128 consecutive positions of the padded-linear walk q = y * (W + 1) + x (pad column x == W)
            const int q0 = tt * kBM;
            const int y0 = q0 / p.Wp;
            t.w0 = tt;
            t.ya = y0 - halo, t.xa = 0, t.c0 = (q0 - y0 * p.Wp) + halo * p.Wp;
            t.xlo = 0, t.xhi = p.W, t.ylo = 0, t.yhi = p.H;
        }
    }
    if (p.mode == 1) {
        int tw = t.m_tile % p.tiles_w;
        int r2 = t.m_tile / p.tiles_w;
        int th = r2 % p.tiles_h;
        int tn = r2 / p.tiles_h;
        t.w0 = tw << p.bw_log2;
        t.h0 = th << p.bh_log2;
        t.n0 = tn << (7 - p.bw_log2 - p.bh_log2);
    }
    return t;
}

// k-block range of one split: even floor/ceil distribution on clusters (every split non-empty), fixed stride otherwise
__device__ __forceinline__ void split_range(const GemmParams& p, int split, int& kb0, int& kb1) {
    if (p.cluster) {
        kb0 = split * p.kb_total / p.splits;
        kb1 = (split + 1) * p.kb_total / p.splits;
    } else {
        kb0 = split * p.kb_per_split;
        kb1 = min(kb0 + p.kb_per_split, p.kb_total);
    }
}

// Applies the epilogue to 16 consecutive accumulator columns of one output row and stores them.
// `bias` / `res` are already resolved to this row and column (shared or global memory); null = absent.
// kGeneric = false: compile-time variant for the hot shapes (N % 16 == 0, 16-byte aligned rows): straight-line
// vector code only, which keeps the kernel small enough for the instruction cache of these microsecond kernels.
// T: the 16-bit type of the residual and of a 16-bit output (fp16, or bf16 for the overflow-prone VAEs).
// kOutS8: the output is int8, q = clamp(rint(y * p.out_inv_scale), -127, 127) of the fp32 y after bias / GEGLU /
// residual (the operand of an int8 consumer); regular variants only (!kGeneric, no partials, no row statistics).
template <typename T, bool kGeneric, bool kGeglu, bool kOutF32, bool kPartial, bool kOutS8 = false>
__device__ __forceinline__ void epilogue_store16(const GemmParams& p, float (&acc)[16], int out_row, int col0,
                                                 int split, const float* bias, const T* res, float2& rowacc) {
    using E = Elem16<T>;
    const bool partial = kGeneric ? (p.partial != nullptr) : kPartial;
    const bool geglu = kGeneric ? (p.geglu != 0) : kGeglu;
    const bool out_f32 = kGeneric ? (p.out_f32 != 0) : kOutF32;
    if (partial) {
        float* dst = p.partial + (static_cast<size_t>(split) * p.M + out_row) * p.N + col0;
        if (!kGeneric || (col0 + 16 <= p.N && (p.N & 3) == 0)) {
#pragma unroll
            for (int j = 0; j < 16; j += 4)
                *reinterpret_cast<float4*>(dst + j) = make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (col0 + j < p.N) dst[j] = acc[j];
        }
        return;
    }
    if (bias != nullptr) {
        if (!kGeneric || (col0 + 16 <= p.N && (p.N & 3) == 0)) {
#pragma unroll
            for (int j = 0; j < 16; j += 4) {
                const float4 bv = *reinterpret_cast<const float4*>(bias + j);
                acc[j] += bv.x, acc[j + 1] += bv.y, acc[j + 2] += bv.z, acc[j + 3] += bv.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (col0 + j < p.N) acc[j] += bias[j];
        }
    }
    if (kGeneric && p.act != 0) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            if (p.act == 1) acc[j] = silu_f(acc[j]);
            else if (p.act == 2) acc[j] = gelu_erf_f(acc[j]);                              // OpenCLIP MLP ("gelu")
            else acc[j] = __fdividef(acc[j], 1.0f + __expf(-1.702f * acc[j]));             // CLIP "quick_gelu"
        }
    }
    int ocol0 = col0;
    const int nvals = geglu ? 8 : 16;
    if (geglu) {
        // interleaved columns: even = value, odd = gate  (unet.py:616-617: a * gelu(g))
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = acc[2 * j] * gelu_erf_f(acc[2 * j + 1]);
        ocol0 = col0 >> 1;
    }
    const int ld = p.n_store;
    const size_t off = static_cast<size_t>(out_row) * ld + ocol0;
    const bool vec_ok = !kGeneric || ((ocol0 + nvals <= ld) && ((ld & 7) == 0));
    if (res != nullptr) {
        if (vec_ok) {
#pragma unroll
            for (int j = 0; j < 16; j += 8) {
                if (j < nvals) {
                    const uint4 rv = *reinterpret_cast<const uint4*>(res + j);
                    const typename E::T2* h2 = reinterpret_cast<const typename E::T2*>(&rv);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float2 f = E::to_float2(h2[q]);
                        acc[j + 2 * q] += f.x;
                        acc[j + 2 * q + 1] += f.y;
                    }
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (j < nvals && ocol0 + j < ld) acc[j] += E::to_float(res[j]);
        }
    }
    if constexpr (kOutS8) {
        static_assert(!kGeneric && !kPartial && !kOutF32, "int8 output: regular epilogue variants only");
        int8_t* o = reinterpret_cast<int8_t*>(p.out) + off;
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = acc[e];
        const uint2 lo = quantize8_s8(f, p.out_inv_scale);
        if (nvals == 8) {
            *reinterpret_cast<uint2*>(o) = lo;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = acc[8 + e];
            const uint2 hi = quantize8_s8(f, p.out_inv_scale);
            *reinterpret_cast<uint4*>(o) = make_uint4(lo.x, lo.y, hi.x, hi.y);
        }
        return;
    }
    if (out_f32) {
        float* o = reinterpret_cast<float*>(p.out) + off;
        if (vec_ok) {
#pragma unroll
            for (int j = 0; j < 16; j += 4)
                if (j < nvals)
                    *reinterpret_cast<float4*>(o + j) = make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (j < nvals && ocol0 + j < ld) o[j] = acc[j];
        }
    } else {
        T* o = reinterpret_cast<T*>(p.out) + off;
        if (vec_ok) {
#pragma unroll
            for (int j = 0; j < 16; j += 8) {
                if (j < nvals) {
                    uint4 pk;
                    pk.x = E::pack2(acc[j], acc[j + 1]);
                    pk.y = E::pack2(acc[j + 2], acc[j + 3]);
                    pk.z = E::pack2(acc[j + 4], acc[j + 5]);
                    pk.w = E::pack2(acc[j + 6], acc[j + 7]);
                    *reinterpret_cast<uint4*>(o + j) = pk;
                    if (p.rs_out != nullptr) {  // per-row sums of the ROUNDED outputs for the consumer's LayerNorm
                        const typename E::T2* h2 = reinterpret_cast<const typename E::T2*>(&pk);
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const float2 f = E::to_float2(h2[q]);
                            rowacc.x += f.x + f.y;
                            rowacc.y = fmaf(f.x, f.x, fmaf(f.y, f.y, rowacc.y));
                        }
                    }
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (j < nvals && ocol0 + j < ld) o[j] = E::from_float(acc[j]);
        }
    }
}

// tile-local row -> (global output row, in-bounds)
__device__ __forceinline__ bool tile_row(const GemmParams& p, const TileCoord& t, int row, int& out_row) {
    if (p.mode == 0) {
        out_row = t.m_tile * kBM + row;
        return out_row < p.M;
    }
    if (p.mode == 2) {  // patch pixel -> image pixel; pad columns and the tile tail are junk rows
        const int pi = t.c0 + row;
        const int r = (pi * p.inv_wp) >> 20;
        const int y = t.ya + r, x = t.xa + (pi - r * p.Wp);
        out_row = (t.n0 * p.H + y) * p.W + x;
        return x >= t.xlo && x < t.xhi && y >= t.ylo && y < t.yhi;
    }
    const int dw = row & ((1 << p.bw_log2) - 1);
    const int dh = (row >> p.bw_log2) & ((1 << p.bh_log2) - 1);
    const int dn = row >> (p.bw_log2 + p.bh_log2);
    const int on = t.n0 + dn, oy = t.h0 + dh, ox = t.w0 + dw;
    out_row = (on * p.Hout + oy) * p.Wout + ox;
    return (on < p.n_img) && (oy < p.Hout) && (ox < p.Wout);
}

__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// ---- thread-block cluster primitives (distributed shared memory) ----
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t local_addr, uint32_t cta_rank) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(cta_rank));
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "r"(ra)
                 : "memory");
    return v;
}


// (kept inline: an out-of-line copy would read the kernel parameters through a generic pointer -- LD.E instead of the
// constant bank -- which measured 2.5x slower for the whole epilogue)
__device__ __forceinline__ bool tile_row_nl(const GemmParams& p, const TileCoord& t, int row, int& out_row) {
    return tile_row(p, t, row, out_row);
}

// image a tile row belongs to (statistics are per image); -1 for rows outside the problem
__device__ __forceinline__ int row_image(const GemmParams& p, const TileCoord& t, int row) {
    int out_row;
    if (!tile_row_nl(p, t, row, out_row)) {
        if (p.mode != 2) return -1;
        return t.n0;  // a junk row of a mode-2 tile still belongs to the tile's image
    }
    if (p.mode == 2) return t.n0;
    return out_row / p.cs_hw;
}

// LayerNorm folded into the GEMM (layer_norm.py:66-78 applied to the A operand): the weights were multiplied by gamma
// at pack time, so out = rstd_r * (acc - mu_r * wg_j) + bias'_j with the row statistics summed from the producer's
// per-tile partials.  Returns (rstd, -mu * rstd).
__device__ __forceinline__ float2 ln_row_coeffs(const GemmParams& p, int out_row, bool valid) {
    if (p.ln_parts == 0 || !valid) return make_float2(1.f, 0.f);
    float s = 0.f, q = 0.f;
    for (int part = 0; part < p.ln_parts; ++part) {
        const float2 v = *reinterpret_cast<const float2*>(p.ln_stat + (static_cast<size_t>(part) * p.M + out_row) * 2);
        s += v.x, q += v.y;
    }
    const float inv = 1.0f / static_cast<float>(p.ln_k);
    const float mu = s * inv;
    const float rstd = rsqrtf(fmaxf(q * inv - mu * mu, 0.f) + p.ln_eps);
    return make_float2(rstd, -mu * rstd);
}

// lane <-> (row slot, 16-byte column vector) mapping of the staged epilogue's store pass: L lanes walk one tile row
struct StagedMap {
    int L, rpi, lr, lcv, nit;
    bool col_ok;
};
__device__ __forceinline__ StagedMap staged_map(const GemmParams& p, const TileCoord& t, int lane) {
    StagedMap m;
    const int vpr = p.block_n >> 3;
    m.L = 8;
    while (m.L < vpr) m.L <<= 1;
    m.rpi = 32 / m.L;
    m.lr = lane / m.L;
    m.lcv = lane - m.lr * m.L;
    m.nit = 16 / m.rpi;
    m.col_ok = m.lcv < vpr && (t.n_tile * p.block_n + m.lcv * 8) < p.N;
    return m;
}

// Residual vectors of four consecutive store-pass iterations of this warp (zeros where there is nothing to add).
__device__ __forceinline__ void staged_load_residual(const GemmParams& p, const TileCoord& t, const StagedMap& m, int ew,
                                                     int it0, uint4 (&res)[4]) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        res[q] = make_uint4(0, 0, 0, 0);
        const int it = it0 + q;
        if (p.residual != nullptr && it < m.nit && m.col_ok) {
            int orow;
            if (tile_row_nl(p, t, ew * 16 + it * m.rpi + m.lr, orow))
                res[q] = *reinterpret_cast<const uint4*>(p.residual + static_cast<size_t>(orow) * p.N + t.n_tile * p.block_n + m.lcv * 8);
        }
    }
}

// ---- staged epilogue (fp16 outputs) ------------------------------------------------------------------------------
// Phase A (stage_accumulators): each consumer thread converts its accumulator fragment ((+LN fold) + bias -> fp16) into
//          the staging tile in shared memory [128][block_n + 8].
// Phase B: warp w owns rows [16 w, 16 w + 16); its lanes walk a row as 16-byte vectors, so the residual read and the
//          output store are contiguous row segments; the same pass accumulates the per-channel (column) sums that the
//          consumer's GroupNorm needs and the per-row sums its LayerNorm needs, from the ROUNDED outputs.  Residual
//          vectors are requested four iterations ahead (the first four before the main loop).
// Phase C: column sums: lanes -> warps (shared memory, fixed order) -> one partial per (image, tile); the last CTA to
//          arrive for an (image, n_tile) adds the partials of all tiles in slot order: deterministic, no float atomics.
// Kept compact on purpose (runtime loops, small unroll factors): these kernels execute every instruction once per
// CTA, so code size is instruction-fetch time.  Inlined: the parameters must come from the constant bank and the
// shared-memory pointers must keep their address space (an out-of-line version used generic LD.E / ST.E for both).
__device__ __forceinline__ void staged_epilogue(const GemmParams& p, const TileCoord& t, __half* tile_s, float* scratch,
                                             unsigned int* flag_s, int ew, int lane, uint4 (&res)[4]) {
    const int bn = p.block_n;
    const int ldt = bn + 8;
    const int ncol0 = t.n_tile * bn;
    epi_bar_sync();  // phase A of every thread is in the staging tile
    // ---------------- phase B ----------------
    const StagedMap m = staged_map(p, t, lane);
    const bool want_stats = p.cs_partial != nullptr || p.rs_out != nullptr;
    float cs[8], cq[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) cs[e] = cq[e] = 0.f;
#pragma unroll 1
    for (int it0 = 0; it0 < m.nit; it0 += 4) {
        uint4 nxt[4];
        staged_load_residual(p, t, m, ew, it0 + 4, nxt);  // lands while this group is processed
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int it = it0 + q;
            if (it >= m.nit) break;
            const int r = ew * 16 + it * m.rpi + m.lr;
            int orow;
            const bool rv = tile_row_nl(p, t, r, orow);
            float rsum = 0.f, rsq = 0.f;
            if (rv && m.col_ok) {
                const uint4 raw = *reinterpret_cast<const uint4*>(tile_s + r * ldt + m.lcv * 8);
                const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
                const __half2* r2 = reinterpret_cast<const __half2*>(&res[q]);
                uint4 pk;
                __half2* o2 = reinterpret_cast<__half2*>(&pk);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2 f = __half22float2(h2[k]), g = __half22float2(r2[k]);
                    o2[k] = __floats2half2_rn(f.x + g.x, f.y + g.y);
                }
                *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.out) + static_cast<size_t>(orow) * p.N + ncol0 + m.lcv * 8) = pk;
                if (want_stats) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {  // statistics of what the consumer will read: the rounded values
                        const float2 f = __half22float2(o2[k]);
                        cs[2 * k] += f.x, cs[2 * k + 1] += f.y;
                        cq[2 * k] = fmaf(f.x, f.x, cq[2 * k]), cq[2 * k + 1] = fmaf(f.y, f.y, cq[2 * k + 1]);
                        rsum += f.x + f.y;
                        rsq = fmaf(f.x, f.x, fmaf(f.y, f.y, rsq));
                    }
                }
            }
            if (p.rs_out != nullptr) {
                for (int o = 1; o < m.L; o <<= 1) {
                    rsum += __shfl_xor_sync(0xffffffffu, rsum, o);
                    rsq += __shfl_xor_sync(0xffffffffu, rsq, o);
                }
                if (rv && m.lcv == 0)
                    *reinterpret_cast<float2*>(p.rs_out + (static_cast<size_t>(t.n_tile) * p.M + orow) * 2) = make_float2(rsum, rsq);
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) res[q] = nxt[q];
    }
    if (p.cs_partial == nullptr) return;
    // ---------------- phase C ----------------
    for (int o = m.L; o < 32; o <<= 1) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            cs[e] += __shfl_xor_sync(0xffffffffu, cs[e], o);
            cq[e] += __shfl_xor_sync(0xffffffffu, cq[e], o);
        }
    }
    if (m.lr == 0 && m.lcv < (bn >> 3)) {
        float2* dst = reinterpret_cast<float2*>(scratch) + ew * bn + m.lcv * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) dst[e] = make_float2(cs[e], cq[e]);
    }
    // the image of each of the tile's eight 16-row groups (uniform inside a group by construction, see the launcher)
    int* img_s = reinterpret_cast<int*>(flag_s) + 8;
    if (lane == 0) img_s[ew] = row_image(p, t, ew * 16);
    epi_bar_sync();
    const int tid_e = ew * 32 + lane;
    int slot = 0;
    if (p.mode == 2) slot = t.w0;
    else if (p.mode == 0) slot = p.cs_hw >= kBM ? (t.m_tile % (p.cs_hw / kBM)) : 0;
    else slot = (p.cs_slots > 1) ? ((t.h0 >> p.bh_log2) * p.tiles_w + (t.w0 >> p.bw_log2)) : 0;
    const float2* sc2 = reinterpret_cast<const float2*>(scratch);
    for (int col = tid_e; col < bn; col += kEpiThreads) {
        if (ncol0 + col >= p.N) continue;
        int w = 0;
        while (w < 8) {
            const int img = img_s[w];
            float a = 0.f, b = 0.f;
            int w2 = w;
            while (w2 < 8 && img_s[w2] == img) {
                a += sc2[w2 * bn + col].x, b += sc2[w2 * bn + col].y;
                ++w2;
            }
            if (img >= 0)
                *reinterpret_cast<float2*>(p.cs_partial + ((static_cast<size_t>(img) * p.cs_slots + slot) * p.N + ncol0 + col) * 2) =
                    make_float2(a, b);
            w = w2;
        }
    }
    epi_bar_sync();  // every thread's partial is written (CTA scope) ...
    if (tid_e == 0) {
        __threadfence();  // ... and published at GPU scope by the thread that takes the tickets (cumulative fence)
        int w = 0;
        while (w < 8) {
            const int img = img_s[w];
            int w2 = w;
            while (w2 < 8 && img_s[w2] == img) ++w2;
            unsigned int last = 0;
            if (img >= 0) {
                const unsigned int old = atomicAdd(&p.cs_tickets[img * p.n_tiles + t.n_tile], 1u);
                last = (old == static_cast<unsigned int>(p.cs_slots - 1)) ? 1u : 0u;
                if (last) p.cs_tickets[img * p.n_tiles + t.n_tile] = 0;  // self-reset for the next launch
            }
            flag_s[w] = last;  // indexed by the group's first warp
            w = w2;
        }
    }
    epi_bar_sync();
    {
        int w = 0;
        while (w < 8) {
            const int img = img_s[w];
            int w2 = w;
            while (w2 < 8 && img_s[w2] == img) ++w2;
            if (flag_s[w] != 0) {
                __threadfence();
                for (int col = tid_e; col < bn; col += kEpiThreads) {
                    if (ncol0 + col >= p.N) continue;
                    float a = 0.f, b = 0.f;
                    for (int sl = 0; sl < p.cs_slots; ++sl) {
                        const float2 v = __ldcg(reinterpret_cast<const float2*>(
                            p.cs_partial + ((static_cast<size_t>(img) * p.cs_slots + sl) * p.N + ncol0 + col) * 2));
                        a += v.x, b += v.y;
                    }
                    *reinterpret_cast<float2*>(p.cs_chan + (static_cast<size_t>(img) * p.N + ncol0 + col) * 2) = make_float2(a, b);
                }
            }
            w = w2;
        }
    }
}

// Main loop of one tile on a consumer warpgroup: rows [64 wg, 64 wg + 64) of the tile, all kBN columns, over the
// k-blocks [kb0, kb1) of the ring.  A stage is released (one arrival per warpgroup) once the wgmma that read it retired;
// one k-block stays in flight behind the one being issued.  One unconditional m64nkBNk16 per k16 step: ptxas only
// pipelines wgmma whose accumulator registers no predicated instruction writes.
template <typename T, int kBN>
__device__ __forceinline__ void gemm_mainloop(const GemmParams& p, float (&acc)[kBN / 2], const uint8_t* smem_a,
                                              const uint8_t* smem_b, uint64_t* full_bar,
                                              uint64_t* empty_bar, int kb0, int kb1, int& stage, uint32_t& phase,
                                              int wg, bool leader) {
    constexpr int b_stage = kBN * kBK * 2;
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t adesc = make_smem_desc_sw128(smem_u32(smem_a + stage * kAStage + wg * (kAStage / 2)), 1024, 0);
        const uint64_t bdesc = make_smem_desc_sw128(smem_u32(smem_b + stage * b_stage), 1024, 0);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)
            wgmma_ss<kBN, T>(acc, adesc + 2 * k, bdesc + 2 * k, (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
        }
    }
    wgmma_wait<0>();
    wgmma_fence_regs<kBN / 2>(acc);
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
}

// gemm_mainloop for int8 operands: a 128-byte k-block is 128 channels, four m64nkBNk32 steps, int32 accumulators.
template <int kBN>
__device__ __forceinline__ void gemm_mainloop_s8(const GemmParams& p, int32_t (&acc)[kBN / 2], const uint8_t* smem_a,
                                                 const uint8_t* smem_b, uint64_t* full_bar, uint64_t* empty_bar, int kb0,
                                                 int kb1, int& stage, uint32_t& phase, int wg, bool leader) {
    constexpr int b_stage = kBN * kBK * 2;
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t adesc = make_smem_desc_sw128(smem_u32(smem_a + stage * kAStage + wg * (kAStage / 2)), 1024, 0);
        const uint64_t bdesc = make_smem_desc_sw128(smem_u32(smem_b + stage * b_stage), 1024, 0);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
            wgmma_ss_s8<kBN>(acc, adesc + 2 * k, bdesc + 2 * k, (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
        }
    }
    wgmma_wait<0>();
    wgmma_fence_regs_s32<kBN / 2>(acc);
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
}

// Accumulator fragment of a consumer thread -> fp32 tile in shared memory, row-major with row stride `ld` floats
// (the layout the row-wise epilogue and the cluster split-K reduction read).
template <int R>
__device__ __forceinline__ void park_accumulators(const float (&acc)[R], int bn, float* dst, int ld, int r0, int lane) {
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
        if (8 * j < bn) {
            *reinterpret_cast<float2*>(dst + r0 * ld + 8 * j + cq) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(dst + (r0 + 8) * ld + 8 * j + cq) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
    }
}

// Phase A of the staged epilogue straight from the accumulator fragment: (+LayerNorm fold) + bias -> fp16 staging tile
// [128][block_n + 8].  `bias0` / `bias1`: bias vectors of rows r0 and r0 + 8 (null = none).
template <int R>
__device__ __forceinline__ void stage_accumulators(const GemmParams& p, const TileCoord& t, const float (&acc)[R],
                                                   __half* tile_s, const float* bias0, const float* bias1,
                                                   const float* wg_s, int r0, int lane) {
    const int bn = p.block_n;
    const int ldt = bn + 8;
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        int out_row;
        const bool valid = tile_row(p, t, r, out_row);
        const float2 lc = ln_row_coeffs(p, out_row, valid);
        const bool ln = p.ln_parts != 0;
        const float* bias = h ? bias1 : bias0;
#pragma unroll
        for (int j = 0; j < R / 4; ++j) {
            if (8 * j < bn) {
                const int c = 8 * j + cq;
                float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
                if (ln) x0 = fmaf(x0, lc.x, lc.y * wg_s[c]), x1 = fmaf(x1, lc.x, lc.y * wg_s[c + 1]);
                if (bias != nullptr) x0 += bias[c], x1 += bias[c + 1];
                *reinterpret_cast<uint32_t*>(tile_s + r * ldt + c) = pack_half2(x0, x1);
            }
        }
    }
}

__device__ __forceinline__ void acc_ld32(const float* src, uint32_t (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
        const float4 f = *reinterpret_cast<const float4*>(src + j);
        v[j] = __float_as_uint(f.x), v[j + 1] = __float_as_uint(f.y), v[j + 2] = __float_as_uint(f.z), v[j + 3] = __float_as_uint(f.w);
    }
}
__device__ __forceinline__ void acc_ld16(const float* src, uint32_t (&v)[16]) {
#pragma unroll
    for (int j = 0; j < 16; j += 4) {
        const float4 f = *reinterpret_cast<const float4*>(src + j);
        v[j] = __float_as_uint(f.x), v[j + 1] = __float_as_uint(f.y), v[j + 2] = __float_as_uint(f.z), v[j + 3] = __float_as_uint(f.w);
    }
}

// Split-K reduction inside a thread-block cluster, run by the 256 consumer threads of every CTA: each CTA has parked its
// fp32 tile in shared memory; CTA `rank` sums its 1/splits slice of the tile over all peers through DSMEM in rank order
// (deterministic), applies bias / residual / conversion and stores it.  No workspace round trip, no second launch.
__device__ __forceinline__ void cluster_splitk_reduce(const GemmParams& p, const uint8_t* smem, int tid) {
    const TileCoord t = decode_work(p, blockIdx.x);
    const int ncol0 = t.n_tile * p.block_n;
    const int ldred = p.block_n + 4;
    const int q4 = p.block_n >> 2;
    const int total4 = kBM * q4;
    const int lo = static_cast<int>(static_cast<long long>(total4) * t.split / p.splits);
    const int hi = static_cast<int>(static_cast<long long>(total4) * (t.split + 1) / p.splits);
    const uint32_t red_base = smem_u32(smem);
    for (int idx = lo + tid; idx < hi; idx += kEpiThreads) {
        const int r = idx / q4, c4 = idx - r * q4;
        const int col = ncol0 + c4 * 4;
        int orow;
        if (!tile_row(p, t, r, orow) || col >= p.N) continue;
        const uint32_t la = red_base + static_cast<uint32_t>(r * ldred + c4 * 4) * 4u;
        float4 a4 = ld_dsmem_f4(la, 0);
        for (int sp = 1; sp < p.splits; ++sp) {
            const float4 v = ld_dsmem_f4(la, sp);
            a4.x += v.x, a4.y += v.y, a4.z += v.z, a4.w += v.w;
        }
        if (p.bias != nullptr) {
            const float4 b = *reinterpret_cast<const float4*>(
                p.bias + (p.bias_rows > 0 ? (orow / p.bias_rows) * p.bias_stride : 0) + col);
            a4.x += b.x, a4.y += b.y, a4.z += b.z, a4.w += b.w;
        }
        const size_t off = static_cast<size_t>(orow) * p.N + col;
        if (p.residual != nullptr) {
            const uint2 rr = *reinterpret_cast<const uint2*>(p.residual + off);
            const float2 q0 = __half22float2(*reinterpret_cast<const __half2*>(&rr.x));
            const float2 q1 = __half22float2(*reinterpret_cast<const __half2*>(&rr.y));
            a4.x += q0.x, a4.y += q0.y, a4.z += q1.x, a4.w += q1.y;
        }
        if (p.out_f32) {
            *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + off) = a4;
        } else {
            uint2 pk;
            pk.x = pack_half2(a4.x, a4.y);
            pk.y = pack_half2(a4.z, a4.w);
            *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(p.out) + off) = pk;
        }
    }
}

// T: operand / 16-bit output type (__half; __nv_bfloat16 for the generic, plain and fp32-output variants only).
// kBN: tile width (columns); p.block_n == kBN.  Each consumer thread holds kBN / 2 fp32 accumulators.
// kS8: int8 operands (k-block = 128 channels, int32 accumulators scaled by p.col_scale into the fp32 ones before the
// epilogue); T is then the type of the residual and the output.
// Palettized B operand: shared memory after the B stages holds `pk_slots` packed-index slots of kBN * pk_box bytes, then
// the three palettes ([3][256] fp16) and the slots' full / empty barriers.  Narrow slots (1 / 2 bits) may outnumber the
// pipeline stages: a wide tile parks its accumulators over stages and slots together.
static constexpr int kMaxPkSlots = 32;
static constexpr int kLutSmem = 3 * 256 * 2 + 2 * kMaxPkSlots * 8;
static constexpr int kLutDecodeThreads = 96;  // producer warps 9..11 decode; warp 8 keeps issuing TMA

// Little-endian bit stream of one 8-index chunk (nbits bytes at a 2-byte aligned offset for 6 bits, nbits-aligned
// otherwise; 1 bit: one byte).
__device__ __forceinline__ uint64_t lut_chunk_bits(const uint8_t* src, int nbits) {
    switch (nbits) {
        case 1: return *src;
        case 2: return *reinterpret_cast<const uint16_t*>(src);
        case 4: return *reinterpret_cast<const uint32_t*>(src);
        case 6: {
            const uint16_t* s = reinterpret_cast<const uint16_t*>(src);
            return static_cast<uint64_t>(s[0]) | (static_cast<uint64_t>(s[1]) << 16) | (static_cast<uint64_t>(s[2]) << 32);
        }
        default: return *reinterpret_cast<const uint64_t*>(src);
    }
}

// Decodes k-block kb of the tile at output row n0 from a packed slot into a B stage, in the SWIZZLE_128B layout a TMA
// load of the fp16 tile writes (16-byte chunk c of row r at chunk c ^ (r & 7)).  Rows >= N decode to zero.
template <int kBN>
__device__ __forceinline__ void lut_decode_stage(const GemmParams& p, const uint8_t* pk, uint8_t* dst, const __half* lut_s,
                                                 int n0, int kb, int dt) {
    const int boff = p.nbits == 1 ? (kb & 1) * 8 : 0;  // 1 bit: the 16-byte box holds k-blocks (kb & ~1, kb | 1)
    const uint32_t mask = (1u << p.nbits) - 1u;
    for (int u = dt; u < kBN * 8; u += kLutDecodeThreads) {
        const int r = u >> 3, c = u & 7;
        const int row = n0 + r;
        uint32_t w[4] = {0u, 0u, 0u, 0u};
        if (row < p.N) {
            const uint64_t bits = lut_chunk_bits(pk + r * p.pk_box + boff + c * p.nbits, p.nbits);
            const __half* lut = lut_s + ((row >= p.seg_end0) + (row >= p.seg_end1)) * 256;
            __half h[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) h[i] = lut[static_cast<uint32_t>(bits >> (i * p.nbits)) & mask];
            if (p.kscale != nullptr) {
                const float4* ks = reinterpret_cast<const float4*>(p.kscale + kb * kBK + c * 8);
                const float4 s0 = __ldg(ks), s1 = __ldg(ks + 1);
                const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i) h[i] = __float2half_rn(__half2float(h[i]) * s[i]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
                w[i] = static_cast<uint32_t>(__half_as_ushort(h[2 * i])) | (static_cast<uint32_t>(__half_as_ushort(h[2 * i + 1])) << 16);
        }
        *reinterpret_cast<uint4*>(dst + r * 128 + ((c ^ (r & 7)) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

template <typename T, bool kGeneric, bool kGeglu, bool kOutF32, bool kPartial, bool kStaged, int kBN, bool kS8, bool kLut = false,
          bool kOutS8 = false>
__device__ __forceinline__ void gemm_kernel_body(const GemmParams& p) {
    constexpr int kChunk = kS8 ? 2 * kBK : kBK;  // channels per k-block (128 bytes either way)
    // 1024-byte aligned by declaration (SWIZZLE_128B atoms): keeping the base a plain shared-memory symbol -- not an
    // integer-rounded pointer -- lets the compiler emit LDS / STS for everything derived from it; rounding through
    // uintptr_t turned every shared access of the loader and the epilogues into generic LD.E / ST.E
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw;
    if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();
    constexpr int b_stage = kBN * kBK * 2;
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + p.stages * kAStage;
    // palettized B: packed slots, palettes and slot barriers between the B stages and the barriers of the pipeline
    const int pk_stage = kLut ? kBN * p.pk_box : 0;
    uint8_t* smem_pk = smem_b + p.stages * b_stage;
    __half* lut_s = reinterpret_cast<__half*>(smem_pk + (kLut ? p.pk_slots * pk_stage : 0));
    uint64_t* pk_full = reinterpret_cast<uint64_t*>(lut_s + 3 * 256);
    uint64_t* pk_empty = pk_full + kMaxPkSlots;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(kLut ? reinterpret_cast<uint8_t*>(lut_s) + kLutSmem : smem_pk);
    uint64_t* empty_bar = full_bar + kMaxStages;
    uint64_t* acc_free = empty_bar + kMaxStages;                     // the pipeline memory is free for the next tile
    float* bias_s = reinterpret_cast<float*>(acc_free + 4);           // [2][block_n] (16 B aligned)
    float* wg_s = bias_s + 2 * 256;                                   // [block_n] LayerNorm fold vector
    unsigned int* flag_s = reinterpret_cast<unsigned int*>(wg_s + 256);  // [8]
    __half* res_s = reinterpret_cast<__half*>(flag_s + 16);           // [128][block_n + 8] residual / staging tile
    const int ldr = p.block_n + 8;
    // fp32 accumulator tile [128][block_n + 4] over the drained pipeline stages (the producer waits on acc_free before it
    // loads the next tile); the row stride keeps the 32 rows a warp reads on distinct banks
    float* acc_s = reinterpret_cast<float*>(smem);
    const int lda = p.block_n + 4;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == kProducerWarp && lane == 0) {
        prefetch_tmap(&p.tmA0);
        prefetch_tmap(&p.tmA1);
        prefetch_tmap(&p.tmB);
        for (int s = 0; s < p.stages; ++s) {
            // palettized B: the A load's arrival plus one per decoding thread (each fences its stores to the async proxy)
            mbar_init(&full_bar[s], kLut ? 1 + kLutDecodeThreads : 1);
            mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
        }
        if constexpr (kLut) {
            for (int s = 0; s < p.pk_slots; ++s) {
                mbar_init(&pk_full[s], 1);
                mbar_init(&pk_empty[s], kLutDecodeThreads);
            }
        }
        mbar_init(acc_free, 1);
        fence_barrier_init();
    }
    __syncthreads();
    // PDL: everything above overlapped the previous kernel's tail.  Each role executes griddepcontrol.wait itself,
    // right before its first access to memory the previous kernels may still be producing: the TMA producer first
    // prefetches the (constant) weight tiles of its first pipeline stages, so the HBM latency of the weights hides
    // behind the previous kernel's tail; the next kernel in the stream may be scheduled as soon as every CTA of this
    // grid is resident.
    pdl_trigger();

    const int total_work = p.m_tiles * p.n_tiles * p.splits;
    const int work0 = blockIdx.x;
    const int work_step = gridDim.x;

    if (warp >= kProducerWarp) {
        // ------------------------- producer warpgroup: warp 8, lane 0 issues TMA -------------------------
        setmaxnreg_dec<kProducerRegs>();
        if (warp == kProducerWarp && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            const uint32_t tx_bytes = kAStage + (kLut ? 0 : b_stage);
            int ps = 0;  // palettized B: packed slot and its phase
            uint32_t pph = 0;
            auto load_pk = [&](const TileCoord& t, int kb) {  // the packed indices of k-block kb into slot ps
                mbar_expect_tx(&pk_full[ps], pk_stage);
                const int x = p.nbits == 1 ? (kb >> 1) * 16 : kb * 8 * p.nbits;
                tma_load_2d(smem_pk + ps * pk_stage, &p.tmB, &pk_full[ps], x, t.n_tile * kBN, kEvictLast);
                if (++ps == p.pk_slots) {
                    ps = 0;
                    pph ^= 1;
                }
            };
            auto load_b = [&](const TileCoord& t, int kb, int st) {
                const int tap = kb / p.kc;
                const int j = kb - tap * p.kc;
                const bool src1 = j >= p.kc0;
                const int c = (src1 ? (j - p.kc0) : j) * kChunk;
                const int wk = tap * p.Kpt + (src1 ? p.C0 : 0) + c;
                void* dst_b = smem_b + st * b_stage;
                const int brow = p.wgt_tiled ? (t.n_tile * p.kb_total + kb) * p.block_n : t.n_tile * p.block_n;
                tma_load_2d(dst_b, &p.tmB, &full_bar[st], p.wgt_tiled ? 0 : wk, brow, p.wgt_tiled ? kEvictFirst : kEvictLast);
            };
            auto load_a = [&](const TileCoord& t, int kb, int st) {
                int tap = kb / p.kc;
                int j = kb - tap * p.kc;
                const CUtensorMap* tmA;
                int c;
                if (tap >= p.taps) {  // shortcut region: a 1x1 convolution = the centre tap over its own sources
                    j = kb - p.taps * p.kc;
                    const bool src3 = j >= p.kc2;
                    c = (src3 ? (j - p.kc2) : j) * kBK;
                    tmA = src3 ? &p.tmA3 : &p.tmA2;
                    tap = 4;
                } else {
                    const bool src1 = j >= p.kc0;
                    c = (src1 ? (j - p.kc0) : j) * kChunk;
                    tmA = src1 ? &p.tmA1 : &p.tmA0;
                }
                void* dst_a = smem_a + st * kAStage;
                const int r = tap / 3, s3 = tap - 3 * r;
                if (p.mode == 0) tma_load_2d(dst_a, tmA, &full_bar[st], c, t.m_tile * kBM, kEvictNormal);
                else tma_load_4d(dst_a, tmA, &full_bar[st], c, t.w0 * p.stride + s3 - p.pad_lo,
                                 t.h0 * p.stride + r - p.pad_lo, t.n0, kEvictNormal);
            };
            // ---- weight prefetch ahead of the grid dependency (constant weights only: pre-tiled B operands) ----
            int npre = 0;
            if ((kLut || p.wgt_tiled) && work0 < total_work) {
                const TileCoord t = decode_work(p, work0);
                int kb0, kb1;
                split_range(p, t.split, kb0, kb1);
                npre = min(kLut ? min(p.stages, p.pk_slots) : p.stages, kb1 - kb0);
                for (int i = 0; i < npre; ++i) {
                    if constexpr (kLut) {
                        load_pk(t, kb0 + i);  // stages and slots are all free before the first tile
                    } else {
                        mbar_expect_tx(&full_bar[i], tx_bytes);
                        load_b(t, kb0 + i, i);
                    }
                }
            }
            pdl_wait();
            int it = 0;  // k-blocks issued so far by this CTA
            int iter = 0;
            for (int work = work0; work < total_work; work += work_step, ++iter) {
                const TileCoord t = decode_work(p, work);
                int kb0, kb1;
                split_range(p, t.split, kb0, kb1);
                if (iter > 0) mbar_wait(acc_free, (iter - 1) & 1);  // the previous tile's epilogue left the stages
                for (int kb = kb0; kb < kb1; ++kb, ++it) {
                    if constexpr (kLut) {
                        // the packed slot is loaded only once the B stage it decodes into is free, so a decoder that
                        // sees the slot full may write the stage
                        if (it >= npre) mbar_wait(&empty_bar[stage], phase ^ 1);
                        mbar_expect_tx(&full_bar[stage], tx_bytes);
                        load_a(t, kb, stage);
                        if (it >= npre) {
                            mbar_wait(&pk_empty[ps], pph ^ 1);
                            load_pk(t, kb);
                        }
                    } else if (it >= npre) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        mbar_expect_tx(&full_bar[stage], tx_bytes);
                        load_a(t, kb, stage);
                        load_b(t, kb, stage);
                    } else {
                        load_a(t, kb, stage);  // its weights are already in flight
                    }
                    if (++stage == p.stages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        } else if (kLut && warp > kProducerWarp) {
            // ---- palettized B: warps 9..11 decode each packed slot into its B stage (constant operands only: no
            // griddepcontrol.wait needed) ----
            const int dt = threadIdx.x - (kProducerWarp + 1) * 32;
            for (int i = dt; i < 3 * 256; i += kLutDecodeThreads) lut_s[i] = p.lut[i];
            asm volatile("bar.sync 2, %0;" ::"n"(kLutDecodeThreads) : "memory");
            int stage = 0, ps = 0;
            uint32_t pph = 0;
            for (int work = work0; work < total_work; work += work_step) {
                const TileCoord t = decode_work(p, work);
                int kb0, kb1;
                split_range(p, t.split, kb0, kb1);
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&pk_full[ps], pph);
                    lut_decode_stage<kBN>(p, smem_pk + ps * pk_stage, smem_b + stage * b_stage, lut_s, t.n_tile * kBN, kb, dt);
                    fence_proxy_async_smem();  // the generic-proxy stores become visible to wgmma
                    mbar_arrive(&full_bar[stage]);
                    mbar_arrive(&pk_empty[ps]);
                    if (++stage == p.stages) stage = 0;
                    if (++ps == p.pk_slots) {
                        ps = 0;
                        pph ^= 1;
                    }
                }
            }
        }
        if (kPartial && p.cluster) {  // the consumers' two cluster barriers around the split-K reduction
            __syncwarp();
            cluster_sync_all();
            cluster_sync_all();
        }
    } else {
        // ------------------------- consumers: wgmma main loop, then the epilogue -------------------------
        setmaxnreg_inc<kConsumerRegs>();
        const int wg = warp >> 2;          // rows [64 wg, 64 wg + 64) of the tile in the main loop
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // accumulator rows r0, r0 + 8 of this thread
        const int half = warp >> 2;        // epilogue: which of the two warps of a 32-row group; it takes every other chunk
        const int row = (warp & 3) * 32 + lane;  // epilogue: the tile row this thread owns
        const int tid_e = threadIdx.x;     // 0..255
        const bool leader = (threadIdx.x & 127) == 0;
        float acc[kBN / 2];
        int stage = 0;
        uint32_t phase = 0;
        pdl_wait();  // bias / residual / output buffers belong to the stream order
        for (int work = work0; work < total_work; work += work_step) {
            const TileCoord t = decode_work(p, work);
            const int ncol0 = t.n_tile * p.block_n;
            int out_row;
            const bool valid = tile_row(p, t, row, out_row);
            int kb0, kb1;
            split_range(p, t.split, kb0, kb1);
            // ---- operand prefetch ahead of the main loop: bias -> smem, residual -> smem (cp.async) ----
            int bias_sel = 0, img0 = 0;
            if (p.bias_mode == 1) {
                int row0;
                tile_row(p, t, 0, row0);
                img0 = p.bias_rows > 0 ? row0 / p.bias_rows : 0;
                const int nvec = p.bias_rows > 0 ? (p.M + p.bias_rows - 1) / p.bias_rows : 1;
                for (int c = tid_e; c < 2 * p.block_n; c += kEpiThreads) {
                    const int which = c >= p.block_n ? 1 : 0;
                    const int cc = c - which * p.block_n;
                    const int col = ncol0 + cc;
                    float v = 0.f;
                    if (col < p.N && img0 + which < nvec && (which == 0 || p.bias_rows > 0))
                        v = p.bias[static_cast<size_t>(img0 + which) * p.bias_stride + col];
                    bias_s[which * p.block_n + cc] = v;
                }
                if (p.bias_rows > 0 && valid) bias_sel = min(1, max(0, out_row / p.bias_rows - img0));
            }
            if constexpr (kS8) {  // the int8 convolution has no LayerNorm fold: its column scales take that vector
                for (int c = tid_e; c < p.block_n; c += kEpiThreads) wg_s[c] = (ncol0 + c < p.N) ? p.col_scale[ncol0 + c] : 0.f;
            } else if (p.ln_parts != 0) {
                for (int c = tid_e; c < p.block_n; c += kEpiThreads) wg_s[c] = (ncol0 + c < p.N) ? p.ln_wg[ncol0 + c] : 0.f;
            }
            uint4 res_pre[4];
            if (kStaged) staged_load_residual(p, t, staged_map(p, t, lane), warp, 0, res_pre);
            if (p.res_smem) {
                const int vpr = p.block_n >> 3;  // 16-byte vectors per tile row
                for (int i = tid_e; i < kBM * vpr; i += kEpiThreads) {
                    const int r = i / vpr, cv = i - r * vpr;
                    int orow;
                    if (tile_row(p, t, r, orow) && ncol0 + cv * 8 < p.N)
                        cp_async16(res_s + r * ldr + cv * 8, p.residual + static_cast<size_t>(orow) * p.n_store + ncol0 + cv * 8);
                }
            }
            const int bias_base = (p.bias_mode == 2 && p.bias_rows > 0 && valid) ? (out_row / p.bias_rows) * p.bias_stride : 0;

            if constexpr (kS8) {
                int32_t iacc[kBN / 2];
                gemm_mainloop_s8<kBN>(p, iacc, smem_a, smem_b, full_bar, empty_bar, kb0, kb1, stage, phase, wg, leader);
                epi_bar_sync();  // the column scales are in wg_s
                const int cq = 2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < kBN / 8; ++j) {
                    const float s0 = wg_s[8 * j + cq], s1 = wg_s[8 * j + cq + 1];
                    acc[4 * j] = static_cast<float>(iacc[4 * j]) * s0;
                    acc[4 * j + 1] = static_cast<float>(iacc[4 * j + 1]) * s1;
                    acc[4 * j + 2] = static_cast<float>(iacc[4 * j + 2]) * s0;
                    acc[4 * j + 3] = static_cast<float>(iacc[4 * j + 3]) * s1;
                }
            } else {
                gemm_mainloop<T, kBN>(p, acc, smem_a, smem_b, full_bar, empty_bar, kb0, kb1, stage, phase, wg, leader);
            }

            if (p.res_smem) cp_async_wait_all();
            epi_bar_sync();  // every wgmma of the tile retired: the stages may be overwritten; staged operands visible
            if (kStaged) {
                // staging tile: over the drained pipeline stages when this CTA has no further tile, else dedicated
                __half* tile_s = p.stage_dedicated ? res_s : reinterpret_cast<__half*>(smem);
                float* scratch = reinterpret_cast<float*>(tile_s + kBM * (p.block_n + 8));
                const float* b0 = nullptr;
                const float* b1 = nullptr;
                if (p.bias_mode == 1) {
                    int o0, o1;
                    const bool v0 = tile_row(p, t, r0, o0), v1 = tile_row(p, t, r0 + 8, o1);
                    const int s0 = (p.bias_rows > 0 && v0) ? min(1, max(0, o0 / p.bias_rows - img0)) : 0;
                    const int s1 = (p.bias_rows > 0 && v1) ? min(1, max(0, o1 / p.bias_rows - img0)) : 0;
                    b0 = bias_s + s0 * p.block_n, b1 = bias_s + s1 * p.block_n;
                }
                stage_accumulators(p, t, acc, tile_s, b0, b1, wg_s, r0, lane);
                staged_epilogue(p, t, tile_s, scratch, flag_s, warp, lane, res_pre);
            } else {
                park_accumulators(acc, kBN, acc_s, lda, r0, lane);
                epi_bar_sync();
                if (!(kPartial && p.cluster)) {  // cluster split-K: the parked tile is what the peers reduce
                    const float* arow = acc_s + row * lda;
                    const float2 lnc = ln_row_coeffs(p, out_row, valid);
                    float2 rowacc = make_float2(0.f, 0.f);
                    auto process16 = [&](float (&a16)[16], int c) {  // c: column offset inside the tile
                        if (p.ln_parts != 0) {
#pragma unroll
                            for (int j = 0; j < 16; ++j) a16[j] = fmaf(a16[j], lnc.x, lnc.y * wg_s[c + j]);
                        }
                        const float* bptr = nullptr;
                        if (p.bias_mode == 1) bptr = bias_s + bias_sel * p.block_n + c;
                        else if (kGeneric && p.bias_mode == 2) bptr = p.bias + bias_base + ncol0 + c;
                        const T* rptr = nullptr;
                        if (p.res_smem) rptr = reinterpret_cast<const T*>(res_s + row * ldr + c);
                        else if (kGeneric && p.residual != nullptr)
                            rptr = reinterpret_cast<const T*>(p.residual + static_cast<size_t>(out_row) * p.n_store +
                                                              ((ncol0 + c) >> (p.geglu ? 1 : 0)));
                        epilogue_store16<T, kGeneric, kGeglu, kOutF32, kPartial, kOutS8>(p, a16, out_row, ncol0 + c, t.split, bptr, rptr,
                                                                                          rowacc);
                    };
                    auto process32 = [&](const uint32_t (&v)[32], int c) {
                        if (!valid) return;
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            if (ncol0 + c + 16 * hh < p.N) {
                                float a16[16];
#pragma unroll
                                for (int j = 0; j < 16; ++j) a16[j] = __uint_as_float(v[16 * hh + j]);
                                process16(a16, c + 16 * hh);
                            }
                        }
                    };
                    if (!kGeneric || (p.block_n & 31) == 0) {
                        // this warp's 32-column chunks: half, half+2, ...
                        for (int c = 32 * half; c < p.block_n; c += 64) {
                            uint32_t va[32];
                            acc_ld32(arow + c, va);
                            process32(va, c);
                        }
                    } else if (kGeneric) {
                        for (int c = 16 * half; c < p.block_n; c += 32) {
                            uint32_t v[16];
                            acc_ld16(arow + c, v);
                            if (valid && ncol0 + c < p.N) {
                                float a16[16];
#pragma unroll
                                for (int j = 0; j < 16; ++j) a16[j] = __uint_as_float(v[j]);
                                process16(a16, c);
                            }
                        }
                    }
                    if (!kPartial && p.rs_out != nullptr && valid)  // one partial per (n_tile, column half): 2 * n_tiles parts
                        *reinterpret_cast<float2*>(p.rs_out + (static_cast<size_t>(t.n_tile * 2 + half) * p.M + out_row) * 2) = rowacc;
                }
            }
            // generic-proxy accesses of the staging / accumulator tiles are ordered before the producer's next TMA writes
            fence_proxy_async_smem();
            epi_bar_sync();  // everyone is done with the accumulator / staging tiles and the staged bias / residual
            if (threadIdx.x == 0) mbar_arrive(acc_free);
        }
        if (kPartial && p.cluster) {  // every CTA of the cluster has parked its tile (one tile per CTA)
            cluster_sync_all();
            cluster_splitk_reduce(p, smem, threadIdx.x);
            cluster_sync_all();  // nobody leaves (or frees its shared memory) while a peer may still read it
        }
    }
}

template <typename T, bool kGeneric, bool kGeglu, bool kOutF32, bool kPartial, bool kStaged, int kBN>
__global__ void __launch_bounds__(kGemmThreads, 1) wgmma_gemm_kernel(const __grid_constant__ GemmParams p) {
    // the shared body executes pdl_wait() before its first access to global memory
    gemm_kernel_body<T, kGeneric, kGeglu, kOutF32, kPartial, kStaged, kBN, false>(p);
}

// Palettized weights (b200sd_gemm_lut): the fp16 kernel with a B operand decoded from n-bit palette indices.  Variants:
// generic, plain, split-K and GEGLU epilogues (nbits is a runtime switch of the decoder).
template <bool kGeneric, bool kGeglu, bool kPartial, int kBN>
__global__ void __launch_bounds__(kGemmThreads, 1) wgmma_gemm_lut_kernel(const __grid_constant__ GemmParams p) {
    // the shared body executes pdl_wait() before its first access to global memory
    gemm_kernel_body<__half, kGeneric, kGeglu, false, kPartial, false, kBN, false, true>(p);
}

// W8A8 3x3 convolution (b200sd_gemm_s8): int8 NHWC activations and pre-tiled int8 weights on IGMMA, fp16 residual and
// output.  Variants: generic, plain and split-K epilogues.
template <bool kGeneric, bool kPartial, int kBN>
__global__ void __launch_bounds__(kGemmThreads, 1) igmma_conv_kernel(const __grid_constant__ GemmParams p) {
    // the shared body executes pdl_wait() before its first access to global memory
    gemm_kernel_body<__half, kGeneric, false, false, kPartial, false, kBN, true>(p);
}

// W8A8 linear GEMM (b200sd_gemm_s8_linear), the epilogues only its launches use: GEGLU (fp16 or int8 output) and a
// plain int8 output.  Its generic, plain and split-K launches run igmma_conv_kernel, whose body branches on p.mode.
template <bool kGeglu, bool kOutS8, int kBN>
__global__ void __launch_bounds__(kGemmThreads, 1) igmma_linear_kernel(const __grid_constant__ GemmParams p) {
    // the shared body executes pdl_wait() before its first access to global memory
    gemm_kernel_body<__half, false, kGeglu, false, false, false, kBN, true, false, kOutS8>(p);
}

// fp16 linear GEMM whose output is the int8 operand of a W8A8 consumer (b200sd_gemm with out_s8_inv_scale > 0):
// plain and GEGLU epilogues.
template <bool kGeglu, int kBN>
__global__ void __launch_bounds__(kGemmThreads, 1) wgmma_gemm_s8out_kernel(const __grid_constant__ GemmParams p) {
    // the shared body executes pdl_wait() before its first access to global memory
    gemm_kernel_body<__half, false, kGeglu, false, false, false, kBN, false, false, true>(p);
}


// Tile widths the GEMM kernel is compiled for; plan_gemm chooses among exactly these (widest first).
static constexpr int kGemmWidths[] = {256, 192, 160, 128, 96, 64, 32, 16};
static constexpr int kNumGemmWidths = sizeof(kGemmWidths) / sizeof(kGemmWidths[0]);
static int gemm_width_index(int bn) {
    for (int i = 0; i < kNumGemmWidths; ++i)
        if (kGemmWidths[i] == bn) return i;
    return -1;
}
using KernelFn = void (*)(GemmParams);
// The instantiation for one width.  bf16 (the VAEs that overflow fp16) is compiled for the generic variant at every
// width and for the plain / fp32-output variants at the widths >= 32 (plan_gemm sends width 16 to the generic one):
// 8 + 7 + 7 = 22 kernels; the fp16 variants keep all eight widths.
template <typename T, bool kGeneric, bool kGeglu, bool kOutF32, bool kPartial, bool kStaged, int kBN>
static constexpr KernelFn gemm_fn() {
    if constexpr (kBN == 16 && !kGeneric && !std::is_same<T, __half>::value) return nullptr;
    else return wgmma_gemm_kernel<T, kGeneric, kGeglu, kOutF32, kPartial, kStaged, kBN>;
}
template <typename T, bool kGeneric, bool kGeglu, bool kOutF32, bool kPartial, bool kStaged>
static KernelFn gemm_kernel(int width_index) {
#define B200SD_GEMM_FN(bn) gemm_fn<T, kGeneric, kGeglu, kOutF32, kPartial, kStaged, bn>()
    static const KernelFn fns[kNumGemmWidths] = {B200SD_GEMM_FN(256), B200SD_GEMM_FN(192), B200SD_GEMM_FN(160),
                                                 B200SD_GEMM_FN(128), B200SD_GEMM_FN(96),  B200SD_GEMM_FN(64),
                                                 B200SD_GEMM_FN(32),  B200SD_GEMM_FN(16)};
#undef B200SD_GEMM_FN
    return fns[width_index];
}
template <bool kGeneric, bool kPartial, int kBN>
static constexpr KernelFn s8_fn() {
    if constexpr (kBN == 16 && !kGeneric) return nullptr;  // the regular variants need block_n % 32 == 0
    else return igmma_conv_kernel<kGeneric, kPartial, kBN>;
}
template <bool kGeneric, bool kPartial>
static KernelFn s8_kernel(int width_index) {
#define B200SD_S8_FN(bn) s8_fn<kGeneric, kPartial, bn>()
    static const KernelFn fns[kNumGemmWidths] = {B200SD_S8_FN(256), B200SD_S8_FN(192), B200SD_S8_FN(160),
                                                 B200SD_S8_FN(128), B200SD_S8_FN(96),  B200SD_S8_FN(64),
                                                 B200SD_S8_FN(32),  B200SD_S8_FN(16)};
#undef B200SD_S8_FN
    return fns[width_index];
}
// the int8-output and int8 GEGLU epilogues are regular variants only: widths >= 32
template <bool kS8, bool kGeglu, bool kOutS8, int kBN>
static constexpr KernelFn s8io_fn() {
    if constexpr (kBN == 16) return nullptr;
    else if constexpr (kS8) return igmma_linear_kernel<kGeglu, kOutS8, kBN>;
    else return wgmma_gemm_s8out_kernel<kGeglu, kBN>;
}
template <bool kS8, bool kGeglu, bool kOutS8>
static KernelFn s8io_kernel(int width_index) {
#define B200SD_S8IO_FN(bn) s8io_fn<kS8, kGeglu, kOutS8, bn>()
    static const KernelFn fns[kNumGemmWidths] = {B200SD_S8IO_FN(256), B200SD_S8IO_FN(192), B200SD_S8IO_FN(160),
                                                 B200SD_S8IO_FN(128), B200SD_S8IO_FN(96),  B200SD_S8IO_FN(64),
                                                 B200SD_S8IO_FN(32),  B200SD_S8IO_FN(16)};
#undef B200SD_S8IO_FN
    return fns[width_index];
}

template <bool kGeneric, bool kGeglu, bool kPartial, int kBN>
static constexpr KernelFn lut_fn() {
    if constexpr (kBN == 16 && !kGeneric) return nullptr;  // the regular variants need block_n % 32 == 0
    else return wgmma_gemm_lut_kernel<kGeneric, kGeglu, kPartial, kBN>;
}
template <bool kGeneric, bool kGeglu, bool kPartial>
static KernelFn lut_kernel(int width_index) {
#define B200SD_LUT_FN(bn) lut_fn<kGeneric, kGeglu, kPartial, bn>()
    static const KernelFn fns[kNumGemmWidths] = {B200SD_LUT_FN(256), B200SD_LUT_FN(192), B200SD_LUT_FN(160),
                                                 B200SD_LUT_FN(128), B200SD_LUT_FN(96),  B200SD_LUT_FN(64),
                                                 B200SD_LUT_FN(32),  B200SD_LUT_FN(16)};
#undef B200SD_LUT_FN
    return fns[width_index];
}

// =====================================================================================================================
// Halo-reuse 3x3 convolution (mode 2) with GroupNorm-apply + SiLU fused into the operand path
// (reference unet.py:470-489: norm1 -> nonlinearity -> conv1, norm2 -> nonlinearity -> conv2; :1044-1046 conv_norm_out).
//
// The image is walked in padded-linear order q = y * (W + 1) + x (one shared zero column between image rows), so the
// input of output position q for tap (dy, dx) is position q + dy * (W + 1) + dx: every tap of a 128-position tile is
// the SAME shared-memory patch read from a row-shifted start address.  Per 64-channel chunk:
//   warps 0..7  (two consumer warpgroups) issue 9 x 4 wgmma per warpgroup whose A descriptors start at
//               patch + (s_tap + 64 wg) * 128 bytes, and between the taps load the NEXT chunk's (rows + 2) x (W + 1)
//               pixel patch with plain 16-byte loads, apply x * sc[n, c] + sh[n, c] (GroupNorm with the statistics its
//               producer left behind) and SiLU in registers, and store it in the 128-byte-swizzled K-major layout the
//               tensor core reads (zero rows for the padding / pad column) into the other patch buffer;
//   warp 8      streams the nine [block_n x 64] weight tiles of the chunk with TMA.
// One activation byte enters shared memory once per chunk instead of nine times, is normalised once, and the
// standalone GroupNorm launch (and its round trip through L2) disappears.  Warps 0..7 then run the epilogue.
// =====================================================================================================================
__device__ __forceinline__ float silu_fast(float y) {
    // y * sigmoid(y) with sigmoid(y) = 0.5 * tanh(0.5 y) + 0.5: one MUFU op per element (the patch transform is MUFU
    // bound otherwise: ex2 + rcp); tanh.approx has 2^-11 relative error, half an fp16 ulp of the stored result
    float th;
    asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(0.5f * y));
    const float hy = 0.5f * y;
    return fmaf(hy, th, hy);
}

__device__ __forceinline__ void dbg_mark(const GemmParams& p, int slot) {
    if (p.dbg != nullptr && blockIdx.x == 0) p.dbg[slot] = clock64();
}

__device__ __forceinline__ void ldr_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// kKind 0: loader warps + staged epilogue (GroupNorm / upsample on the patch, column statistics);  1: loader warps + tiny
// fp32 epilogue (conv_out);  2: plain convolution -- the producer warp fetches each patch with one TMA box (hardware zero
// fill for the padding ring and the pad column) and the consumer warps use the register epilogue of the GEMM kernel.
// kR: accumulator registers per consumer thread (block_n / 2): the loader kinds hold the patch vectors in registers too.
template <int kKind, int kR>
__global__ void __launch_bounds__(kHaloThreads, 1) halo_conv_kernel(const __grid_constant__ GemmParams p) {
    constexpr bool kFp32Direct = kKind == 1;
    constexpr bool kTmaPatch = kKind == 2;
    // 1024-byte aligned by declaration (SWIZZLE_128B atoms): keeping the base a plain shared-memory symbol -- not an
    // integer-rounded pointer -- lets the compiler emit LDS / STS for everything derived from it; rounding through
    // uintptr_t turned every shared access of the loader and the epilogues into generic LD.E / ST.E
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw;
    if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();
    const int b_stage = p.block_n * (kBK * 2);
    uint8_t* patch = smem;                                  // [2][patch_bytes]
    uint8_t* smem_b = smem + 2 * p.patch_bytes;             // [stages][block_n * 128]
    uint64_t* full_b = reinterpret_cast<uint64_t*>(smem_b + p.stages * b_stage);
    uint64_t* empty_b = full_b + kHaloMaxStages;
    uint64_t* full_a = empty_b + kHaloMaxStages;            // [2]
    uint64_t* empty_a = full_a + 2;                         // [2]
    uint64_t* acc_free = empty_a + 2;                       // the patch / weight memory is free for the next tile
    float* bias_s = reinterpret_cast<float*>(acc_free + 4);               // [256]
    unsigned int* flag_s = reinterpret_cast<unsigned int*>(bias_s + 256);   // [8]
    float2* stat_s = reinterpret_cast<float2*>(flag_s + 16);              // [64] (mean, rstd) per group
    float2* scsh = stat_s + 64;                                           // [C0 + C1] (scale, shift) per channel
    const int Cin = p.C0 + p.C1;
    __half* stage_tile = reinterpret_cast<__half*>(scsh + ((Cin + 7) & ~7));  // dedicated staging tile (if any)
    float* acc_s = reinterpret_cast<float*>(smem);          // fp32 accumulator tile over the drained patches / stages
    const int lda = p.block_n + 4;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (warp == kProducerWarp && lane == 0) {
        prefetch_tmap(&p.tmB);
        if (kTmaPatch) {
            prefetch_tmap(&p.tmA0);
            prefetch_tmap(&p.tmA1);
        }
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(&full_b[s], 1);
            mbar_init(&empty_b[s], 2);
        }
        for (int s = 0; s < 2; ++s) {
            mbar_init(&full_a[s], 1);
            mbar_init(&empty_a[s], 2);
        }
        mbar_init(acc_free, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_trigger();

    const int total_work = p.m_tiles * p.n_tiles;
    const int work0 = blockIdx.x, work_step = gridDim.x;
    const int kc = p.kc;

    if (warp == kProducerWarp) {
        // ------------------------------- weight producer (TMA; constant data: no grid dependency) -------------------
        if (lane == 0) {
            int it = 0, iter = 0;
            // kTmaPatch: this thread also fetches the activation patches, one chunk ahead of the weight tiles that use
            // them (two patch buffers): the next patch of the tile is requested as soon as its buffer is free, checked
            // without blocking between weight tiles so the weight ring never drains behind a patch wait
            int ci = 0, pai = 0, pwork = work0, pj = 0;
            auto issue_patch = [&](bool blocking) -> bool {
                const int pa = pai & 1;
                const uint32_t ph = ((pai >> 1) & 1) ^ 1;
                if (blocking) mbar_wait(&empty_a[pa], ph);
                else if (!mbar_try_wait(&empty_a[pa], ph)) return false;
                const TileCoord pt = decode_work(p, pwork);
                const bool src1 = pj >= p.kc0;
                mbar_expect_tx(&full_a[pa], static_cast<uint32_t>(p.patch_tx));
                tma_load_4d(patch + pa * p.patch_bytes + 1024, src1 ? &p.tmA1 : &p.tmA0, &full_a[pa],
                            (src1 ? pj - p.kc0 : pj) * kBK, pt.xa, pt.ya, pt.n0, kEvictNormal);
                ++pai;
                if (++pj == kc) pj = 0, pwork += work_step;
                return true;
            };
            if (kTmaPatch) pdl_wait();  // the activations are the previous kernel's output
            for (int work = work0; work < total_work; work += work_step, ++iter) {
                const TileCoord t = decode_work(p, work);
                if (iter > 0) mbar_wait(acc_free, (iter - 1) & 1);  // the previous tile's epilogue left the buffers
                for (int j = 0; j < kc; ++j, ++ci) {
                    if (kTmaPatch && pai == ci) issue_patch(true);
                    for (int tap = 0; tap < p.taps; ++tap, ++it) {
                        if (kTmaPatch && pai == ci + 1 && pwork == work) issue_patch(false);
                        const int st = it % p.stages;
                        const uint32_t ph = (it / p.stages) & 1;
                        mbar_wait(&empty_b[st], ph ^ 1);
                        mbar_expect_tx(&full_b[st], b_stage);
                        tma_load_2d(smem_b + st * b_stage, &p.tmB, &full_b[st], 0,
                                    (t.n_tile * p.kb_total + j * p.taps + tap) * p.block_n, kEvictFirst);
                    }
                }
            }
        }
    } else if (warp < kProducerWarp) {
        // --------------------- consumers: patch loader / transform, wgmma, epilogue ---------------------
        const int ltid = threadIdx.x;
        const int ew = warp;
        const int wg = warp >> 2;
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // accumulator rows r0, r0 + 8 of this thread
        const int row = (warp & 3) * 32 + lane;                   // epilogue: the tile row this thread owns
        const bool leader = (threadIdx.x & 127) == 0;
        const bool gn = p.gn_gamma != nullptr;
        const bool ups = p.upsample != 0;
        const int Hs = ups ? (p.H >> 1) : p.H, Ws = ups ? (p.W >> 1) : p.W;
        float acc[kR];
        if (ltid == 0) dbg_mark(p, 0);
        pdl_wait();
        if (ltid == 0) dbg_mark(p, 1);
        int cur_img = -1, ait = 0, it = 0;
        for (int work = work0; work < total_work; work += work_step) {
            const TileCoord t = decode_work(p, work);
            const int img = t.n0;
            const int ya = t.ya, xa = t.xa;
            const int ncol0 = t.n_tile * p.block_n;
            if (p.bias != nullptr) {
                const float* bsrc = p.bias + (p.bias_rows > 0 ? static_cast<size_t>(img) * p.bias_stride : 0);
                for (int c = ltid; c < p.block_n; c += kEpiThreads) bias_s[c] = (ncol0 + c < p.N) ? bsrc[ncol0 + c] : 0.f;
            }
            if (ltid < 16) {  // "pixel -1" of both patches: the zero pad column that precedes the patch
                const int which = ltid >> 3;
                *reinterpret_cast<uint4*>(patch + which * p.patch_bytes + 7 * 128 + (ltid & 7) * 16) = make_uint4(0, 0, 0, 0);
            }
            // ---- operand patches (loader kinds): one per 64-channel chunk ----
            // Thread t always handles vector (t & 7) of the patch pixels t / 8, t / 8 + 32, ...: pixel offsets and
            // shared-memory destinations are computed once per tile, the eight (scale, shift) pairs once per chunk, and
            // the raw vectors of chunk j + 1 are requested while chunk j is being normalised (one register set: a slot is
            // refilled as soon as its vector has been consumed), so the L2 latency hides behind the transform.
            constexpr int NBMAX = kTmaPatch ? 1 : 12;
            const int nvec = p.patch_rows * p.Wp * 8;
            const int nb = (nvec + kEpiThreads - 1) / kEpiThreads;
            const int jj = ltid & 7;
            int soff[NBMAX], doff[NBMAX];
            uint4 regs[NBMAX];
            auto chunk_src = [&](int j, int& csrc) -> const __half* {
                const bool src1 = j >= p.kc0;
                const int cbase = (src1 ? j - p.kc0 : j) * kBK + jj * 8;
                csrc = src1 ? p.C1 : p.C0;
                if (cbase >= csrc) return nullptr;  // ragged last chunk: channels beyond the source are zeros
                return (src1 ? p.a1 : p.a0) + static_cast<size_t>(img) * Hs * Ws * csrc + cbase;
            };
            // per-chunk state of the transform of chunk `tj`
            float4 cf[4];
            bool chan_ok = false;
            int csrc_nxt = 0;
            const __half* nsrc = nullptr;
            auto transform_begin = [&](int tj) {
                const bool src1 = tj >= p.kc0;
                int csrc_cur;
                chan_ok = chunk_src(tj, csrc_cur) != nullptr;
                nsrc = (tj + 1 < kc) ? chunk_src(tj + 1, csrc_nxt) : nullptr;
                if (gn) {
                    const float2* tab = scsh + (src1 ? p.C0 : 0) + (src1 ? tj - p.kc0 : tj) * kBK + jj * 8;
#pragma unroll
                    for (int q = 0; q < 4; ++q) cf[q] = chan_ok ? *reinterpret_cast<const float4*>(tab + 2 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
            };
            // the vectors i with i % nslices == slice of chunk `tj` into patch buffer `pa`
            auto transform_slice = [&](int pa, int slice, int nslices) {
                uint8_t* pbase = patch + pa * p.patch_bytes + 1024;
#pragma unroll
                for (int i = 0; i < NBMAX; ++i) {
                    if (doff[i] < 0 || i % nslices != slice) continue;
                    uint4 val = regs[i];
                    const bool live = soff[i] >= 0;
                    regs[i] = make_uint4(0, 0, 0, 0);
                    if (nsrc != nullptr && live)
                        regs[i] = __ldg(reinterpret_cast<const uint4*>(nsrc + static_cast<size_t>(soff[i]) * csrc_nxt));
                    if (gn && live && chan_ok) {
                        __half2* h2 = reinterpret_cast<__half2*>(&val);
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const float2 f = __half22float2(h2[q]);
                            float a = fmaf(f.x, cf[q].x, cf[q].y), b = fmaf(f.y, cf[q].z, cf[q].w);
                            if (p.gn_silu) a = silu_fast(a), b = silu_fast(b);
                            h2[q] = __floats2half2_rn(a, b);
                        }
                    }
                    *reinterpret_cast<uint4*>(pbase + doff[i]) = val;
                }
            };
            if (!kTmaPatch) {
#pragma unroll
                for (int i = 0; i < NBMAX; ++i) {
                    const int v = ltid + kEpiThreads * i;
                    const int pi = v >> 3;
                    const int prow = (pi * p.inv_wp) >> 20;
                    const int yy = ya + prow, xx = xa + (pi - prow * p.Wp);
                    const bool in_patch = i < nb && v < nvec;
                    const bool ok = in_patch && yy >= 0 && yy < p.H && xx >= 0 && xx < p.W;
                    const int ys = ups ? (yy >> 1) : yy, xs = ups ? (xx >> 1) : xx;
                    soff[i] = ok ? (ys * Ws + xs) : -1;
                    doff[i] = in_patch ? pi * 128 + ((jj ^ (pi & 7)) << 4) : -1;
                }
                {
                    int csrc;
                    const __half* src = chunk_src(0, csrc);
#pragma unroll
                    for (int i = 0; i < NBMAX; ++i) {
                        regs[i] = make_uint4(0, 0, 0, 0);
                        if (src != nullptr && soff[i] >= 0)
                            regs[i] = __ldg(reinterpret_cast<const uint4*>(src + static_cast<size_t>(soff[i]) * csrc));
                    }
                }
                if (ltid == 0) dbg_mark(p, 2);
                // (the first chunk's vectors are already in flight while the coefficient table is built)
                if (gn && img != cur_img) {
                    // ---- GroupNorm coefficients of this image: group statistics from the producers' per-channel sums ----
                    const int cpg = Cin / p.gn_groups;
                    const float inv_cnt = 1.0f / (static_cast<float>(cpg) * static_cast<float>(p.gn_hw));
                    ldr_bar_sync();  // previous tile's readers of the table are done
                    // eight lanes per group, all groups of a round in flight at once (one L2 round trip for <= 32 groups)
                    for (int g = ltid >> 3; g < p.gn_groups; g += kEpiThreads >> 3) {
                        float s = 0.f, q = 0.f;
                        for (int c = g * cpg + (ltid & 7); c < (g + 1) * cpg; c += 8) {
                            const float2 v = (c < p.C0)
                                ? __ldg(reinterpret_cast<const float2*>(p.gn_chan0 + (static_cast<size_t>(img) * p.C0 + c) * 2))
                                : __ldg(reinterpret_cast<const float2*>(p.gn_chan1 + (static_cast<size_t>(img) * p.C1 + c - p.C0) * 2));
                            s += v.x, q += v.y;
                        }
#pragma unroll
                        for (int o = 4; o > 0; o >>= 1) {
                            s += __shfl_xor_sync(0xffffffffu, s, o);
                            q += __shfl_xor_sync(0xffffffffu, q, o);
                        }
                        if ((ltid & 7) == 0) {
                            const float mean = s * inv_cnt;
                            stat_s[g] = make_float2(mean, rsqrtf(fmaxf(q * inv_cnt - mean * mean, 0.f) + p.gn_eps));
                        }
                    }
                    ldr_bar_sync();
                    for (int c = ltid; c < Cin; c += kEpiThreads) {
                        const float2 st = stat_s[c / cpg];
                        const float sc = p.gn_gamma[c] * st.y;
                        scsh[c] = make_float2(sc, fmaf(-st.x, sc, p.gn_beta[c]));
                    }
                    ldr_bar_sync();
                    cur_img = img;
                }
                if (ltid == 0) dbg_mark(p, 8);
                transform_begin(0);
                transform_slice(ait & 1, 0, 1);
            }
            fence_proxy_async_smem();  // generic-proxy writes (patch, pad column) -> visible to the tensor core
            epi_bar_sync();
            if (ltid == 0) {
                if (!kTmaPatch) dbg_mark(p, 9);  // loader: chunk 0 stored
                dbg_mark(p, 3);
            }
            // ---- main loop: chunks x taps; the loader kinds transform chunk j + 1 between the taps of chunk j ----
            for (int j = 0; j < kc; ++j, ++ait) {
                const int pa = ait & 1;
                if (kTmaPatch) mbar_wait(&full_a[pa], (ait >> 1) & 1);
                const bool more = !kTmaPatch && j + 1 < kc;
                if (ltid == 0 && j < 24) dbg_mark(p, 64 + 2 * j);
                if (more) {
                    if (ltid == 0 && j < 23) dbg_mark(p, 10 + 2 * j);  // loader: chunk j + 1 begins
                    transform_begin(j + 1);
                }
                const uint32_t pbase = smem_u32(patch + pa * p.patch_bytes) + 1024;
                int prev = -1;
                for (int tap = 0; tap < p.taps; ++tap, ++it) {
                    const int st = it % p.stages;
                    mbar_wait(&full_b[st], (it / p.stages) & 1);
                    const int dy = p.taps == 9 ? tap / 3 - 1 : 0, dx = p.taps == 9 ? tap - (tap / 3) * 3 - 1 : 0;
                    // patch pixel of this warpgroup's first output position for this tap (>= -1)
                    const int srow = t.c0 + dy * p.Wp + dx + 64 * wg;
                    const uint32_t a_addr = pbase + srow * 128;
                    // start address shifted by whole 128-byte rows inside the 1024-byte swizzle atom (the patch was
                    // written in the absolute-address swizzle pattern of a 1024-byte aligned buffer)
                    const uint64_t adesc = make_smem_desc_sw128(a_addr, 1024, 0) |
                                           (static_cast<uint64_t>(p.desc_bo ? ((a_addr >> 7) & 7) : 0) << 49);
                    const uint64_t bdesc = make_smem_desc_sw128(smem_u32(smem_b + st * b_stage), 1024, 0);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < kBK / 16; ++k)
                        wgmma_rows64(acc, p.block_n, adesc + 2 * k, bdesc + 2 * k, (j > 0 || tap > 0 || k > 0) ? 1u : 0u);
                    wgmma_commit();
                    if (more) transform_slice(pa ^ 1, tap, p.taps);
                    wgmma_wait<1>();
                    if (prev >= 0 && leader) mbar_arrive(&empty_b[prev]);
                    prev = st;
                }
                wgmma_wait<0>();
                wgmma_fence_regs<kR>(acc);
                if (ltid == 0 && j < 24) dbg_mark(p, 65 + 2 * j);
                if (leader) {
                    mbar_arrive(&empty_b[prev]);
                    if (kTmaPatch) mbar_arrive(&empty_a[pa]);
                }
                if (more) {
                    fence_proxy_async_smem();
                    epi_bar_sync();  // chunk j + 1 is in its buffer; both warpgroups are done reading chunk j's
                    if (ltid == 0 && j < 23) dbg_mark(p, 11 + 2 * j);  // loader: chunk j + 1 stored
                }
            }
            // ---- epilogue ----
            int out_row;
            const bool valid = tile_row(p, t, row, out_row);
            uint4 res_pre[4];
            if (kKind == 0) staged_load_residual(p, t, staged_map(p, t, lane), ew, 0, res_pre);
            epi_bar_sync();  // every wgmma of the tile retired: patches and stages may be overwritten
            if (ltid == 0) dbg_mark(p, 4);
            if (kKind == 0) {
                __half* tile_s = p.stage_dedicated ? stage_tile : reinterpret_cast<__half*>(smem);
                float* scratch = reinterpret_cast<float*>(tile_s + kBM * (p.block_n + 8));
                const float* bias = p.bias != nullptr ? bias_s : nullptr;
                stage_accumulators(p, t, acc, tile_s, bias, bias, bias_s, r0, lane);
                staged_epilogue(p, t, tile_s, scratch, flag_s, ew, lane, res_pre);
            } else {
                park_accumulators(acc, p.block_n, acc_s, lda, r0, lane);
                epi_bar_sync();
                const float* arow = acc_s + row * lda;
                if (kFp32Direct) {
                    // tiny output width (conv_out: 4 channels, fp32): one thread per output pixel
                    if (ew < 4) {
                        uint32_t v[16];
                        acc_ld16(arow, v);
                        if (valid) {
                            for (int c = 0; c < 16 && ncol0 + c < p.N; ++c) {
                                const float x = __uint_as_float(v[c]) + (p.bias != nullptr ? bias_s[c] : 0.f);
                                if (p.out_f32) reinterpret_cast<float*>(p.out)[static_cast<size_t>(out_row) * p.N + ncol0 + c] = x;
                                else reinterpret_cast<__half*>(p.out)[static_cast<size_t>(out_row) * p.N + ncol0 + c] = __float2half_rn(x);
                            }
                        }
                    }
                } else {
                    // register epilogue: this warp's 32-column chunks (two warps per 32-row group)
                    const int half = ew >> 2;
                    float2 rowacc = make_float2(0.f, 0.f);
                    for (int c = 32 * half; c < p.block_n && valid; c += 64) {
                        uint32_t v[32];
                        acc_ld32(arow + c, v);
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            const int cc = c + 16 * hh;
                            if (ncol0 + cc < p.N) {
                                float a16[16];
#pragma unroll
                                for (int q = 0; q < 16; ++q) a16[q] = __uint_as_float(v[16 * hh + q]);
                                const float* bptr = p.bias != nullptr ? bias_s + cc : nullptr;
                                const __half* rptr = p.residual != nullptr
                                    ? p.residual + static_cast<size_t>(out_row) * p.n_store + ncol0 + cc : nullptr;
                                epilogue_store16<__half, true, false, false, false>(p, a16, out_row, ncol0 + cc, 0, bptr, rptr, rowacc);
                            }
                        }
                    }
                }
            }
            // generic-proxy accesses of the staging / accumulator tiles are ordered before the producer's next TMA writes
            fence_proxy_async_smem();
            epi_bar_sync();  // staging buffers (and the patch / weight memory under them) are free again
            if (ltid == 0) {
                dbg_mark(p, 5);
                mbar_arrive(acc_free);
            }
        }
    }
}

// Sums split-K partials and applies the same epilogue (bias, residual); no GEGLU.
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int splits, int M, int N,
                                     const float* __restrict__ bias, int bias_rows, int bias_stride,
                                     const __half* __restrict__ residual, void* __restrict__ out, int out_f32) {
    pdl_wait();
    const size_t total4 = static_cast<size_t>(M) * N / 4;
    const size_t stride = static_cast<size_t>(M) * N;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total4;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t e = i * 4;
        float4 acc = *reinterpret_cast<const float4*>(partial + e);
        for (int s = 1; s < splits; ++s) {
            const float4 v = *reinterpret_cast<const float4*>(partial + s * stride + e);
            acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
        }
        const int row = static_cast<int>(e / N);
        const int col = static_cast<int>(e - static_cast<size_t>(row) * N);
        if (bias != nullptr) {
            const float* b = bias + (bias_rows > 0 ? (row / bias_rows) * bias_stride : 0) + col;
            acc.x += b[0], acc.y += b[1], acc.z += b[2], acc.w += b[3];
        }
        if (residual != nullptr) {
            const __half2* r = reinterpret_cast<const __half2*>(residual + e);
            const float2 r0 = __half22float2(r[0]), r1 = __half22float2(r[1]);
            acc.x += r0.x, acc.y += r0.y, acc.z += r1.x, acc.w += r1.y;
        }
        if (out_f32) {
            *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + e) = acc;
        } else {
            uint2 pk;
            pk.x = pack_half2(acc.x, acc.y);
            pk.y = pack_half2(acc.z, acc.w);
            *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out) + e) = pk;
        }
    }
}

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
struct GemmPlan {
    int M, N, Kpt, taps, kc0, kc1, kb_total;
    int m_tiles, n_tiles, block_n, splits, kb_per_split, stages;
    int Hout, Wout, bw, bh, bn_img, tiles_w, tiles_h, tiles_n;
    int bias_mode, res_smem, epi_smem;
    int cluster;  // split-K reduced inside a thread-block cluster of `splits` CTAs (DSMEM) instead of a second kernel
    int halo;     // mode 2: halo-reuse convolution
    int Wp, tiles_per_img, patch_rows, patch_bytes;
    int win, tw, th, tiles_x;
    int staged, stage_dedicated;
    int tma_patch;
    int cs_slots;  // statistics slots per image this tiling produces (0: column statistics not available)
    int smem_bytes;
    int variant;    // GEMM kernel: one of GemmVariant (-1 for the halo convolution)
    int pk_box, pk_slots;  // palettized B: bytes per tile row of a packed slot, slots in the ring (0: fp16 B operand)
    int halo_kind;  // halo convolution: 0 loader warps + staged epilogue, 1 fp32 / narrow epilogue, 2 TMA patches (-1: GEMM)
};

// Epilogue instantiations of wgmma_gemm_kernel, each compiled for every width of kGemmWidths (plan_gemm sends width 16
// to the generic one: the others need block_n % 32 == 0)
enum GemmVariant {
    kVariantGeneric = 0, kVariantSplitK = 1, kVariantGeglu = 2, kVariantF32 = 3, kVariantPlain = 4, kVariantStaged = 5,
    kVariantS8Out = 6, kVariantGegluS8Out = 7  // int8 output: wgmma_gemm_s8out_kernel / igmma_linear_kernel
};

static bool cluster_splitk_enabled() {
    // B200SD_CLUSTER_SPLITK=0: always take the workspace + reduce-kernel path (read per call: tuning scripts flip it)
    const char* e = getenv("B200SD_CLUSTER_SPLITK");
    return !(e && e[0] == '0');
}

static int ilog2(int v) {
    int l = 0;
    while ((1 << l) < v) ++l;
    return l;
}

static bool staged_enabled() {
    // B200SD_STAGED=1: residual-only GEMMs also take the staged epilogue (default: the register epilogue with the
    // residual tile prefetched into shared memory during the main loop; column statistics always need the staged one)
    const char* e = getenv("B200SD_STAGED");
    return e && e[0] == '1';
}

static bool desc_base_offset_enabled() {
    // how row-shifted SWIZZLE_128B descriptors are formed: 0 (default) = the start address alone (the hardware applies
    // the swizzle to absolute address bits; the halo tests pass on H100 only this way), 1 = also the matrix-base-offset
    // field; read per call
    const char* e = getenv("B200SD_DESC_BO");
    return e && e[0] == '1';
}

// Tiling of the halo-reuse convolution (mode 2).
static int plan_halo(const b200sd_gemm_args& a, GemmPlan& pl) {
    B200SD_REQUIRE((a.mode == 0 || a.stride == 1) && !a.pad_after_only, "b200sd_gemm: halo needs a stride-1 pad-1 convolution");
    B200SD_REQUIRE(!a.geglu && a.act == 0 && a.split_k <= 1, "b200sd_gemm: halo kernel: no GEGLU / activation / split-K");
    B200SD_REQUIRE(a.wgt_tiled && a.block_n > 0, "b200sd_gemm: halo kernel needs chunk-major pre-tiled weights (explicit block_n)");
    B200SD_REQUIRE(a.n_img > 0 && a.h > 0 && a.w > 0, "b200sd_gemm: bad image geometry for the halo kernel");
    B200SD_REQUIRE(!a.upsample2x || (a.h % 2 == 0 && a.w % 2 == 0 && a.c1 == 0 && a.gn_groups == 0),
                   "b200sd_gemm: upsample2x needs even output size, one source, no GroupNorm");
    pl.halo = 1;
    pl.tma_patch = a.halo == 2 ? 1 : 0;
    B200SD_REQUIRE(!pl.tma_patch || (a.gn_groups == 0 && !a.upsample2x && a.cs_partial == nullptr && !a.out_f32 &&
                                     a.block_n % 32 == 0 && a.c0 % 8 == 0 && a.c1 % 8 == 0),
                   "b200sd_gemm: halo = 2 (TMA patches) is the plain convolution: no GroupNorm / upsample / statistics / fp32 output");
    pl.bw = pl.bh = pl.bn_img = pl.tiles_w = pl.tiles_h = pl.tiles_n = 1;
    pl.Hout = a.h, pl.Wout = a.w;
    pl.M = a.n_img * a.h * a.w;
    const bool conv = a.mode == 1;  // mode 0 + halo: a 1x1 convolution over an image (one tap, no halo ring)
    const int halo = conv ? 1 : 0;
    pl.win = 0, pl.tw = pl.th = pl.tiles_x = 0;
    if (a.w + 1 <= 80) {
        // narrow images: padded-linear walk, full-width patches
        pl.Wp = a.w + 1;
        pl.tiles_per_img = (a.h * pl.Wp + kBM - 1) / kBM;
        const int span = (kBM - 1 + pl.Wp - 1) / pl.Wp + 1;  // image rows a 128-position tile can touch
        pl.patch_rows = span + 2 * halo;
    } else {
        // wide images: th x tw windows with th * (tw + 2 halo) <= 128 positions; pick the shape that wastes least
        double best = -1.0;
        for (int th = 1; th <= 8; th *= 2) {
            const int pitch = kBM / th, tw = pitch - 2 * halo;
            const int tx = (a.w + tw - 1) / tw, ty = (a.h + th - 1) / th;
            const double eff = static_cast<double>(a.w) * a.h / (static_cast<double>(tx) * ty * kBM);
            if (eff > best) best = eff, pl.th = th, pl.tw = tw, pl.tiles_x = tx, pl.tiles_per_img = tx * ty;
        }
        pl.win = 1;
        pl.Wp = pl.tw + 2 * halo;
        pl.patch_rows = pl.th + 2 * halo;
    }
    pl.m_tiles = a.n_img * pl.tiles_per_img;
    const int rows_needed = std::max(pl.patch_rows * pl.Wp, (2 * halo + 1) * pl.Wp + kBM) + 8 + 1;
    pl.patch_bytes = ((rows_needed + 7) / 8) * 1024;
    B200SD_REQUIRE(pl.tma_patch || pl.patch_rows * pl.Wp * 8 <= 12 * kEpiThreads, "b200sd_gemm: image too wide for the halo kernel's patch (w=%d)", a.w);
    B200SD_REQUIRE(!pl.tma_patch || (pl.Wp <= 256 && pl.patch_rows <= 256), "b200sd_gemm: patch exceeds a TMA box (w=%d)", a.w);
    pl.block_n = a.block_n;
    B200SD_REQUIRE(pl.block_n == 16 || (pl.block_n % 32 == 0 && pl.block_n <= 256), "b200sd_gemm: halo block_n %d", pl.block_n);
    pl.n_tiles = (a.n + pl.block_n - 1) / pl.block_n;
    pl.splits = 1, pl.kb_per_split = pl.kb_total, pl.cluster = 0;
    pl.bias_mode = a.bias != nullptr ? 1 : 0;
    pl.res_smem = 0;
    const bool fp32_direct = a.out_f32 || pl.block_n == 16;
    B200SD_REQUIRE(!fp32_direct || (pl.block_n == 16 && a.residual == nullptr && a.cs_partial == nullptr),
                   "b200sd_gemm: halo fp32 / narrow output needs block_n 16, no residual, no statistics");
    pl.staged = (fp32_direct || pl.tma_patch) ? 0 : 1;
    // the loader kinds keep twelve patch vectors per thread in registers beside the accumulators
    B200SD_REQUIRE(pl.tma_patch || pl.block_n <= 128, "b200sd_gemm: halo block_n %d > 128 needs halo = 2", pl.block_n);
    // the epilogue tiles live over the drained patches / weight stages (the producer waits for them between tiles)
    pl.stage_dedicated = 0;
    const int cin = a.c0 + a.c1;
    const int fixed = 2 * pl.patch_bytes + (2 * kHaloMaxStages + 8) * 8 + 16 + 256 * 4 + 64 + 64 * 8 + ((cin + 7) & ~7) * 8 +
                      (pl.stage_dedicated ? kBM * (pl.block_n + 8) * 2 + 8 * pl.block_n * 8 : 0) + 1024;
    const int b_stage = pl.block_n * kBK * 2;
    pl.stages = std::min(kHaloMaxStages, (227 * 1024 - fixed) / b_stage);
    B200SD_REQUIRE(pl.stages >= 3, "b200sd_gemm: halo kernel does not fit shared memory (w=%d c=%d block_n=%d)", a.w, cin, pl.block_n);
    pl.smem_bytes = fixed + pl.stages * b_stage;
    const int over = 2 * pl.patch_bytes + pl.stages * b_stage;
    B200SD_REQUIRE(over >= (pl.staged ? kBM * (pl.block_n + 8) * 2 + 8 * pl.block_n * 8 : kBM * (pl.block_n + 4) * 4),
                   "b200sd_gemm: halo epilogue tile does not fit over the pipeline memory (block_n=%d)", pl.block_n);
    pl.epi_smem = 0;
    pl.cs_slots = pl.tiles_per_img;
    pl.variant = -1;
    pl.halo_kind = pl.tma_patch ? 2 : (pl.staged == 0 ? 1 : 0);
    return 0;
}

// block_n the halo kernel would like for these arguments (smallest one-wave tile wins: the kernel is bound by
// shared-memory bandwidth, reads (128 + bn) + writes (patch share + bn) rows of 32 bytes per MMA of bn / 2 cycles)
static int halo_pick_block_n(const b200sd_gemm_args& a) {
    if (a.n <= 16) return 16;
    const int wp = a.w + 1;
    long m_tiles = static_cast<long>(a.n_img) * ((a.h * wp + kBM - 1) / kBM);
    if (wp > 80) m_tiles = static_cast<long>(a.n_img) * ((static_cast<long>(a.h) * a.w + 101) / 102);  // windows: ~80 % useful rows
    double best = 1e30;
    int best_bn = 128;
    for (int bn = a.halo == 2 ? 256 : 128; bn >= 32; bn -= 32) {
        const int nt = (a.n + bn - 1) / bn;
        if (nt * bn > a.n + a.n / 4 + 31) continue;
        const double waves = std::ceil(static_cast<double>(m_tiles * nt) / num_sms());
        const double t = waves * ((41.0 + bn / 2.0) * (a.mode == 1 ? 36.0 : 4.0) * ((a.c0 + a.c1 + 63) / 64) + 4000.0) + 2.0 * nt;
        if (t < best) best = t, best_bn = bn;
    }
    return best_bn;
}

// bf16: the operands, the residual and a 16-bit output are bf16 (b200sd_gemm_bf16).  That path serves the VAEs whose
// activations overflow fp16: modes 0 / 1, stride 1 / 2, pad_after_only, bias, residual, fp32 output and tiled weights,
// on the generic, plain and fp32-output epilogues.  Everything else is rejected by name, and the plan never takes
// split-K (workspace or cluster) or the staged epilogue, whatever the environment switches say.
// s8: the W8A8 convolution (b200sd_gemm_s8): int8 activations and weights, k-blocks of 128 channels.  It serves the
// stride-1 pad-1 3x3 convolution of one source with a bias vector or per-image bias rows, an fp16 residual, fp16 output
// and split-K; everything else is rejected by name.
// s8_linear: the W8A8 linear GEMM (b200sd_gemm_s8_linear, s8 set too): mode 0, one int8 source [m, c0], bias, fp16
// residual, GEGLU, row statistics, fp16 or int8 output, split-K (fp16 output); everything else is rejected by name.
// out_s8_inv_scale > 0 (fp16 or int8 operands): int8 output of a linear GEMM on the plain or GEGLU epilogue, no split-K.
static int plan_gemm(const b200sd_gemm_args& a, GemmPlan& pl, bool bf16 = false, bool s8 = false, bool s8_linear = false) {
    if (s8_linear) {
        B200SD_REQUIRE(a.mode == 0, "b200sd_gemm_s8_linear: mode=%d is not supported (the linear GEMM, mode 0)", a.mode);
        B200SD_REQUIRE(!a.a1 && a.c1 == 0, "b200sd_gemm_s8_linear: a1 (second source) is not supported");
        B200SD_REQUIRE(!a.a2 && !a.a3 && a.c2 == 0 && a.c3 == 0, "b200sd_gemm_s8_linear: a2 / a3 (folded shortcut) are not supported");
        B200SD_REQUIRE(!a.pad_after_only, "b200sd_gemm_s8_linear: pad_after_only is not supported");
        B200SD_REQUIRE(a.act == 0, "b200sd_gemm_s8_linear: act=%d is not supported", a.act);
        B200SD_REQUIRE(!a.out_f32, "b200sd_gemm_s8_linear: out_f32 is not supported (fp16 or int8 output)");
        B200SD_REQUIRE(a.bias_rows == 0, "b200sd_gemm_s8_linear: bias_rows is not supported (one bias vector)");
        B200SD_REQUIRE(!a.halo, "b200sd_gemm_s8_linear: halo is not supported");
        B200SD_REQUIRE(!a.upsample2x, "b200sd_gemm_s8_linear: upsample2x is not supported");
        B200SD_REQUIRE(a.gn_groups == 0 && !a.gn_chan0 && !a.gn_chan1 && !a.gn_gamma && !a.gn_beta,
                       "b200sd_gemm_s8_linear: gn_* (fused GroupNorm) is not supported");
        B200SD_REQUIRE(!a.cs_partial && !a.cs_chan && !a.cs_tickets, "b200sd_gemm_s8_linear: cs_* (column statistics) are not supported");
        B200SD_REQUIRE(a.ln_parts == 0 && !a.ln_stat && !a.ln_wg, "b200sd_gemm_s8_linear: ln_* (LayerNorm fold) is not supported");
        B200SD_REQUIRE(a.c0 > 0 && a.c0 % 16 == 0, "b200sd_gemm_s8_linear: c0=%d must be a positive multiple of 16 (TMA row stride)", a.c0);
    } else if (s8) {
        B200SD_REQUIRE(a.mode == 1, "b200sd_gemm_s8: mode=%d is not supported (the 3x3 convolution, mode 1)", a.mode);
        B200SD_REQUIRE(a.stride == 1, "b200sd_gemm_s8: stride=%d is not supported (1)", a.stride);
        B200SD_REQUIRE(!a.pad_after_only, "b200sd_gemm_s8: pad_after_only is not supported");
        B200SD_REQUIRE(!a.a1 && a.c1 == 0, "b200sd_gemm_s8: a1 (second source) is not supported");
        B200SD_REQUIRE(!a.a2 && !a.a3 && a.c2 == 0 && a.c3 == 0, "b200sd_gemm_s8: a2 / a3 (folded shortcut) are not supported");
        B200SD_REQUIRE(!a.geglu, "b200sd_gemm_s8: geglu is not supported");
        B200SD_REQUIRE(a.act == 0, "b200sd_gemm_s8: act=%d is not supported", a.act);
        B200SD_REQUIRE(!a.out_f32, "b200sd_gemm_s8: out_f32 is not supported (fp16 output)");
        B200SD_REQUIRE(!a.halo, "b200sd_gemm_s8: halo is not supported");
        B200SD_REQUIRE(!a.upsample2x, "b200sd_gemm_s8: upsample2x is not supported");
        B200SD_REQUIRE(a.gn_groups == 0 && !a.gn_chan0 && !a.gn_chan1 && !a.gn_gamma && !a.gn_beta,
                       "b200sd_gemm_s8: gn_* (fused GroupNorm) is not supported");
        B200SD_REQUIRE(!a.cs_partial && !a.cs_chan && !a.cs_tickets, "b200sd_gemm_s8: cs_* (column statistics) are not supported");
        B200SD_REQUIRE(!a.rs_out, "b200sd_gemm_s8: rs_out (row statistics) is not supported");
        B200SD_REQUIRE(a.ln_parts == 0 && !a.ln_stat && !a.ln_wg, "b200sd_gemm_s8: ln_* (LayerNorm fold) is not supported");
        B200SD_REQUIRE(a.c0 > 0 && a.c0 % 16 == 0, "b200sd_gemm_s8: c0=%d must be a positive multiple of 16 (TMA row stride)", a.c0);
    }
    B200SD_REQUIRE(a.mode == 0 || a.mode == 1, "b200sd_gemm: bad mode %d", a.mode);
    if (bf16) {
        B200SD_REQUIRE(!a.geglu, "b200sd_gemm_bf16: geglu is not supported in bf16");
        B200SD_REQUIRE(a.split_k <= 1, "b200sd_gemm_bf16: split_k=%d is not supported in bf16 (0 or 1)", a.split_k);
        B200SD_REQUIRE(!a.halo && !a.upsample2x, "b200sd_gemm_bf16: halo / upsample2x are not supported in bf16");
        B200SD_REQUIRE(a.gn_groups == 0 && !a.gn_chan0 && !a.gn_chan1 && !a.gn_gamma && !a.gn_beta,
                       "b200sd_gemm_bf16: gn_* (fused GroupNorm) is not supported in bf16");
        B200SD_REQUIRE(!a.cs_partial && !a.cs_chan && !a.cs_tickets && !a.rs_out,
                       "b200sd_gemm_bf16: cs_* / rs_out (statistics outputs) are not supported in bf16");
        B200SD_REQUIRE(a.ln_parts == 0 && !a.ln_stat && !a.ln_wg, "b200sd_gemm_bf16: ln_* (LayerNorm fold) is not supported in bf16");
        B200SD_REQUIRE(!a.a2 && !a.a3 && a.c2 == 0 && a.c3 == 0,
                       "b200sd_gemm_bf16: a2 / a3 (folded shortcut) are not supported in bf16");
        B200SD_REQUIRE(a.act == 0, "b200sd_gemm_bf16: act=%d is not supported in bf16", a.act);
    }
    B200SD_REQUIRE(!a.pad_after_only || (a.mode == 1 && a.stride == 2), "b200sd_gemm: pad_after_only is for stride-2 convolutions");
    B200SD_REQUIRE(a.c0 > 0 && a.c0 % 8 == 0 && a.c1 >= 0 && a.c1 % 8 == 0,
                   "b200sd_gemm: channel counts must be positive multiples of 8 (c0=%d c1=%d)", a.c0, a.c1);
    B200SD_REQUIRE(a.n > 0, "b200sd_gemm: n=%d", a.n);
    pl.N = a.n;
    pl.Kpt = a.c0 + a.c1;
    const int chunk = s8 ? 2 * kBK : kBK;  // channels per 128-byte k-block
    pl.kc0 = (a.c0 + chunk - 1) / chunk;
    pl.kc1 = (a.c1 + chunk - 1) / chunk;
    pl.taps = a.mode == 1 ? 9 : 1;
    pl.kb_total = pl.taps * (pl.kc0 + pl.kc1) + (a.c2 + kBK - 1) / kBK + (a.c3 + kBK - 1) / kBK;
    B200SD_REQUIRE((a.c2 == 0 && a.c3 == 0) || (a.mode == 1 && a.stride == 1 && !a.halo && a.c2 > 0 && a.c2 % 8 == 0 && a.c3 % 8 == 0),
                   "b200sd_gemm: shortcut sources (a2 / a3) need a stride-1 3x3 convolution and channel counts that are multiples of 8");
    pl.halo = 0, pl.Wp = 0, pl.tiles_per_img = 0, pl.patch_rows = 0, pl.patch_bytes = 0;
    pl.staged = 0, pl.stage_dedicated = 0, pl.cs_slots = 0, pl.smem_bytes = 0;
    const bool want_stats = a.cs_partial != nullptr || a.rs_out != nullptr;
    B200SD_REQUIRE(!want_stats || (!a.geglu && !a.out_f32 && a.act == 0 && a.n % 8 == 0 && a.split_k <= 1),
                   "b200sd_gemm: statistics outputs need a plain fp16 epilogue without split-K");
    B200SD_REQUIRE(a.ln_parts == 0 || (a.mode == 0 && a.ln_stat && a.ln_wg && a.split_k <= 1),
                   "b200sd_gemm: LayerNorm fold needs mode 0, statistics, the fold vector and no split-K");
    const bool out_s8 = a.out_s8_inv_scale != 0.f;
    B200SD_REQUIRE(!out_s8 || (std::isfinite(a.out_s8_inv_scale) && a.out_s8_inv_scale > 0.f),
                   "b200sd_gemm: out_s8_inv_scale=%g must be positive and finite", static_cast<double>(a.out_s8_inv_scale));
    B200SD_REQUIRE(!out_s8 || (!bf16 && a.mode == 0 && !a.halo && !a.out_f32 && !want_stats && a.act == 0 && a.split_k <= 1 &&
                               a.n % 32 == 0),
                   "b200sd_gemm: out_s8_inv_scale (int8 output) needs an fp16 / int8 linear GEMM (mode 0) without halo, out_f32, "
                   "cs_* / rs_out, act or split-K, n a multiple of 32");
    if (a.halo) return plan_halo(a, pl);
    if (a.mode == 0) {
        B200SD_REQUIRE(a.m > 0, "b200sd_gemm: m=%d", a.m);
        pl.M = a.m;
        pl.m_tiles = (a.m + kBM - 1) / kBM;
        pl.Hout = pl.Wout = pl.bw = pl.bh = pl.bn_img = pl.tiles_w = pl.tiles_h = pl.tiles_n = 1;
    } else {
        B200SD_REQUIRE(a.stride == 1 || a.stride == 2, "b200sd_gemm: stride %d", a.stride);
        B200SD_REQUIRE(a.n_img > 0 && a.h > 0 && a.w > 0, "b200sd_gemm: bad image geometry");
        B200SD_REQUIRE(a.stride == 1 || (a.h % 2 == 0 && a.w % 2 == 0), "b200sd_gemm: stride-2 needs even h, w");
        pl.Hout = a.h / a.stride;
        pl.Wout = a.w / a.stride;
        pl.M = a.n_img * pl.Hout * pl.Wout;
        // pick the 128-pixel box (bn_img x bh x bw, powers of two) with the least padding
        long best = -1;
        for (int bw = 128; bw >= 1; bw >>= 1) {
            if (bw * a.stride > 256) continue;
            for (int bh = 128 / bw; bh >= 1; bh >>= 1) {
                if (bh * a.stride > 256) continue;
                const int bn = 128 / (bw * bh);
                const int tw = (pl.Wout + bw - 1) / bw, th = (pl.Hout + bh - 1) / bh, tn = (a.n_img + bn - 1) / bn;
                const long tiles = static_cast<long>(tw) * th * tn;
                // prefer fewer tiles, then wider rows
                const long score = tiles * 1024 - bw;
                if (best < 0 || score < best) {
                    best = score;
                    pl.bw = bw, pl.bh = bh, pl.bn_img = bn, pl.tiles_w = tw, pl.tiles_h = th, pl.tiles_n = tn;
                }
            }
        }
        pl.m_tiles = pl.tiles_w * pl.tiles_h * pl.tiles_n;
    }
    if (a.geglu) B200SD_REQUIRE(a.n % 16 == 0, "b200sd_gemm: GEGLU needs n %% 16 == 0");
    // ---- tile shape / split-K selection by a small cost model (cycles per SM).  The constants were fitted to B200 runs;
    // checked on an H100 (400 W) with tools/bench_gemm_shapes.py over the 28 SD-2.1 shapes it times: the plans this model
    // picks take 1080 us in total against 1058 us for the fastest candidate of every shape (2 %, about the run-to-run
    // spread of a single shape), so they were kept.  The largest misses: conv 2560->1280 at 8x8 (1.3x) and linear
    // 1280->1280 at M = 512 (1.25x). ----
    const int sms = num_sms();
    const bool can_split = !bf16 && !a.geglu && a.n % 4 == 0 && a.act == 0 && !want_stats && a.ln_parts == 0 && !out_s8;
    auto epi_cycles = [&](int bn) { return 400.0 + (bn / 32.0) * (a.geglu ? 520.0 : 230.0); };
    auto kb_cycles = [&](int bn) { return std::max(2.0 * bn, (kAStage + 128.0 * bn) / 38.0); };
    double best_t = 1e30;
    int best_bn = 0, best_s = 1, best_cluster = 0;
    static const int kSplits[] = {1, 2, 3, 4, 6, 8, 12, 16, 24, 32};
    const bool can_cluster = can_split && cluster_splitk_enabled() && a.n % 16 == 0;
    for (int bn : kGemmWidths) {
        if (a.block_n > 0 && bn != a.block_n) continue;
        const int nt = (a.n + bn - 1) / bn;
        if (a.block_n == 0 && bn > 16 && nt * bn > a.n + a.n / 4 + 15) continue;  // > 25 % padding
        if ((want_stats || out_s8) && bn % 32 != 0) continue;
        const int stages_bn = std::min(kMaxStages, (smem_budget() - kEpiFixed) / (kAStage + bn * kBK * 2));
        for (int sp : kSplits) {
            if (a.split_k > 0 && sp != a.split_k) continue;
            if (sp > 1 && (!can_split || sp * 2 > pl.kb_total) && a.split_k == 0) continue;
            const int kb = (pl.kb_total + sp - 1) / sp;
            const int se = (pl.kb_total + kb - 1) / kb;
            const double main = kb * kb_cycles(bn);
            for (int cl = 0; cl < 2; ++cl) {
                double t;
                if (cl == 1) {
                    // cluster of sp CTAs per tile: portable sizes only, fp32 tile must fit over the pipeline stages
                    if (!can_cluster || (sp != 2 && sp != 4 && sp != 8) || bn % 32 != 0 || sp > pl.kb_total) continue;
                    if (512L * (bn + 4) > static_cast<long>(stages_bn) * (kAStage + bn * kBK * 2)) continue;
                    const long units = static_cast<long>(pl.m_tiles) * nt * sp;
                    // clusters need sp free SMs of one GPC: count ~10 % of the SMs as stranded
                    const double waves = std::ceil(static_cast<double>(units) / (sms - sms / 10));
                    const double epi = 1500.0 + (bn / 32.0) * 120.0 + 128.0 * bn * 4.0 / 17.0;  // registers->smem, 2 syncs, DSMEM
                    t = 5000.0 + waves * (main + epi);
                } else {
                    const long units = static_cast<long>(pl.m_tiles) * nt * se;
                    const double waves = std::ceil(static_cast<double>(units) / sms);
                    t = 5000.0 + main + epi_cycles(bn) + (waves - 1.0) * std::max(main, epi_cycles(bn));
                    if (se > 1) t += 6000.0 + static_cast<double>(se) * pl.M * a.n * 8.0 / 3000.0;
                }
                if (t < best_t) {
                    best_t = t;
                    best_bn = bn;
                    best_s = sp;
                    best_cluster = cl;
                }
            }
        }
    }
    if (best_bn == 0) {  // explicit overrides that the loops above did not enumerate
        best_bn = a.block_n > 0 ? a.block_n : 128;
        best_s = a.split_k > 0 ? a.split_k : 1;
    }
    B200SD_REQUIRE(gemm_width_index(best_bn) >= 0, "b200sd_gemm: block_n %d is not a compiled tile width", best_bn);
    pl.block_n = best_bn;
    pl.n_tiles = (a.n + pl.block_n - 1) / pl.block_n;
    int splits = std::max(1, std::min(best_s, pl.kb_total));
    pl.kb_per_split = (pl.kb_total + splits - 1) / splits;
    pl.splits = (pl.kb_total + pl.kb_per_split - 1) / pl.kb_per_split;
    pl.cluster = 0;
    if (best_cluster && splits > 1) {  // even distribution, exactly `splits` non-empty ranges (split_range())
        pl.cluster = 1;
        pl.splits = splits;
    }
    if (pl.splits > 1) {
        B200SD_REQUIRE(!a.geglu, "b200sd_gemm: split-K with GEGLU is not supported");
        B200SD_REQUIRE(a.n % 4 == 0, "b200sd_gemm: split-K needs n %% 4 == 0");
    }
    // ---- epilogue operand staging ----
    pl.bias_mode = 0;
    pl.res_smem = 0;
    if (pl.splits == 1) {
        if (a.bias != nullptr) {
            const bool two_vec_ok = a.bias_rows == 0 || a.bias_rows >= kBM ||
                                    (a.mode == 1 && a.bias_rows == pl.Hout * pl.Wout && pl.bn_img <= 2);
            pl.bias_mode = two_vec_ok ? 1 : 2;
        }
        if (a.residual != nullptr && !a.geglu && a.n % 8 == 0) pl.res_smem = 1;
    }
    // the compile-time epilogue variants (everything but kVariantGeneric) need these shapes and operands
    const bool regular_shape = (a.act == 0) && (a.n % 16 == 0) && ((a.geglu ? a.n / 2 : a.n) % 8 == 0) &&
                               (pl.block_n % 32 == 0) && pl.bias_mode != 2;
    const bool regular = regular_shape && (a.residual == nullptr || pl.res_smem);
    const int per_stage = kAStage + pl.block_n * kBK * 2;
    {
        // staged epilogue: fp16 tile in shared memory, row-contiguous residual reads / stores, statistics outputs
        const bool eligible = !bf16 && !s8 && !out_s8 && regular && pl.splits == 1 && !a.geglu && !a.out_f32 && a.n % 8 == 0;
        // column statistics need the staged epilogue; row statistics alone ride on the register epilogue (every thread
        // owns a row there), which keeps the residual tile prefetched in shared memory during the main loop
        pl.staged = (eligible && (a.cs_partial != nullptr || (a.residual != nullptr && staged_enabled()))) ? 1 : 0;
        B200SD_REQUIRE(a.cs_partial == nullptr || pl.staged, "b200sd_gemm: this shape cannot emit column statistics (n=%d block_n=%d)", a.n,
                       pl.block_n);
        B200SD_REQUIRE(a.rs_out == nullptr || pl.staged || (regular && !a.geglu && !a.out_f32 && pl.splits == 1),
                       "b200sd_gemm: this shape cannot emit row statistics (n=%d block_n=%d)", a.n, pl.block_n);
        if (pl.staged) pl.res_smem = 0;
        // the staging tile lives over the drained pipeline stages (the producer waits for it between tiles)
        pl.stage_dedicated = 0;
        if (a.cs_partial != nullptr) {
            // every 16-row group of a tile must lie inside one image, and the tiles of an image must be countable
            int slots = 0;
            if (a.mode == 0) {
                if (a.cs_hw >= kBM && a.cs_hw % kBM == 0) slots = a.cs_hw / kBM;
                else if (a.cs_hw >= 16 && kBM % a.cs_hw == 0) slots = 1;
            } else {
                if (pl.bn_img == 1) slots = pl.tiles_w * pl.tiles_h;
                else if (pl.bn_img <= 8 && pl.tiles_w * pl.tiles_h == 1) slots = 1;
            }
            B200SD_REQUIRE(slots > 0, "b200sd_gemm: column statistics are not available for this geometry (rows per image %d)", a.cs_hw);
            pl.cs_slots = slots;
        }
    }
    pl.epi_smem = kEpiFixed + (pl.res_smem ? kBM * (pl.block_n + 8) * 2 : 0) +
                  (pl.stage_dedicated ? kBM * (pl.block_n + 8) * 2 + 8 * pl.block_n * 8 : 0);
    pl.stages = std::max(2, std::min(kMaxStages, (smem_budget() - pl.epi_smem) / per_stage));
    // the fp32 accumulator tile (or the fp16 staging tile) is parked over the drained stages
    const int park = pl.staged ? kBM * (pl.block_n + 8) * 2 + 8 * pl.block_n * 8 : kBM * (pl.block_n + 4) * 4;
    while (pl.stages * per_stage < park && pl.stages < kMaxStages) ++pl.stages;
    B200SD_REQUIRE(pl.stages * per_stage >= park, "b200sd_gemm: epilogue tile does not fit over the stages (block_n=%d)", pl.block_n);
    pl.smem_bytes = pl.stages * per_stage + (2 * kMaxStages + 4) * 8 + 16 + pl.epi_smem + 1024;
    // compile-time epilogue variants for the hot shapes; anything irregular takes the generic kernel (split-K and the
    // staged epilogue read the residual row-contiguously, so they need no residual tile in shared memory)
    const bool regular_epi = regular || (regular_shape && a.residual != nullptr && (pl.splits > 1 || pl.staged));
    B200SD_REQUIRE(!out_s8 || regular, "b200sd_gemm: out_s8_inv_scale (int8 output) needs the regular epilogue (n=%d block_n=%d)",
                   a.n, pl.block_n);
    if (out_s8) pl.variant = a.geglu ? kVariantGegluS8Out : kVariantS8Out;
    else if (!regular_epi) pl.variant = kVariantGeneric;
    else if (pl.staged) pl.variant = kVariantStaged;
    else if (pl.splits > 1) pl.variant = kVariantSplitK;
    else if (a.geglu) pl.variant = kVariantGeglu;
    else if (a.out_f32) pl.variant = kVariantF32;
    else pl.variant = kVariantPlain;
    pl.halo_kind = -1;
    return 0;
}

static size_t plan_workspace(const GemmPlan& pl) {
    return (pl.splits > 1 && !pl.cluster) ? static_cast<size_t>(pl.splits) * pl.M * pl.N * sizeof(float) : 0;
}

// Palettized B operand (b200sd_gemm_lut): the fp16 plan of the same arguments -- tile width, split-K and k order, so
// the launch is bit-identical to b200sd_gemm on the decoded weights -- with a pipeline depth that makes room for the
// packed-index slots.  The accumulator tile is parked over the A / B stages and the slots (contiguous, all drained
// at the end of a tile).
static int plan_lut(const b200sd_gemm_args& a, const b200sd_lut_args& l, GemmPlan& pl) {
    B200SD_REQUIRE(l.nbits == 1 || l.nbits == 2 || l.nbits == 4 || l.nbits == 6 || l.nbits == 8,
                   "b200sd_gemm_lut: nbits=%d is not supported (1, 2, 4, 6 or 8)", l.nbits);
    B200SD_REQUIRE(!a.wgt_tiled, "b200sd_gemm_lut: wgt_tiled is not supported (the packed indices are the B operand)");
    B200SD_REQUIRE(!a.halo && !a.upsample2x && a.gn_groups == 0, "b200sd_gemm_lut: halo / upsample2x / gn_* are not supported");
    B200SD_REQUIRE(!a.cs_partial && !a.cs_chan && !a.cs_tickets, "b200sd_gemm_lut: cs_* (column statistics) are not supported");
    B200SD_REQUIRE(!a.a2 && !a.a3 && a.c2 == 0 && a.c3 == 0, "b200sd_gemm_lut: a2 / a3 (folded shortcut) are not supported");
    B200SD_REQUIRE(!a.out_f32, "b200sd_gemm_lut: out_f32 is not supported");
    B200SD_REQUIRE(a.out_s8_inv_scale == 0.f, "b200sd_gemm_lut: out_s8_inv_scale (int8 output) is not supported");
    // whole 64-channel k-blocks per source: k-block kb holds weight columns [64 kb, 64 kb + 64), no padding positions
    B200SD_REQUIRE(a.c0 % kBK == 0 && a.c1 % kBK == 0, "b200sd_gemm_lut: c0=%d / c1=%d must be multiples of 64", a.c0, a.c1);
    B200SD_REQUIRE(l.packed && l.lut, "b200sd_gemm_lut: packed / lut is null");
    B200SD_REQUIRE((reinterpret_cast<uintptr_t>(l.kscale) & 15) == 0, "b200sd_gemm_lut: kscale %p is not 16-byte aligned",
                   static_cast<const void*>(l.kscale));
    B200SD_REQUIRE(0 <= l.seg_end0 && l.seg_end0 <= l.seg_end1, "b200sd_gemm_lut: bad row segments (%d, %d)", l.seg_end0, l.seg_end1);
    if (int rc = plan_gemm(a, pl)) return rc;
    B200SD_REQUIRE(!pl.staged, "b200sd_gemm_lut: the staged epilogue is not supported");
    const long row_min = (pl.kb_total * 8L * l.nbits + 15) / 16 * 16;
    B200SD_REQUIRE(l.row_bytes % 16 == 0 && l.row_bytes >= row_min, "b200sd_gemm_lut: row_bytes=%d (need a multiple of 16 >= %ld)",
                   l.row_bytes, row_min);
    pl.pk_box = std::max(16, 8 * l.nbits);  // TMA boxes are at least 16 bytes wide: at 1 bit one box holds two k-blocks
    const int per_stage = kAStage + pl.block_n * kBK * 2;
    const int pk_stage = pl.block_n * pl.pk_box;
    const int fixed = pl.smem_bytes - pl.stages * per_stage + kLutSmem;
    const int limit = std::min(227 * 1024, std::max(smem_budget(), pl.smem_bytes));
    const int park = kBM * (pl.block_n + 4) * 4;
    int best_s = 0, best_k = 0;
    for (int s = pl.stages; s >= 2; --s) {
        const int k = std::min(kMaxPkSlots, (limit - fixed - s * per_stage) / pk_stage);
        if (k < 2 || s * per_stage + k * pk_stage < park) continue;
        if (std::min(s, k) > std::min(best_s, best_k)) best_s = s, best_k = k;
    }
    B200SD_REQUIRE(best_s > 0, "b200sd_gemm_lut: the pipeline does not fit in shared memory (block_n=%d nbits=%d)", pl.block_n, l.nbits);
    pl.stages = best_s;
    pl.pk_slots = best_k;
    pl.smem_bytes = fixed + best_s * per_stage + best_k * pk_stage;
    return 0;
}

extern void count_launch(int n);

static int launch_gemm(const b200sd_gemm_args& a, cudaStream_t stream, bool bf16, const float* col_scale = nullptr,
                       const b200sd_lut_args* lut = nullptr, bool s8_linear = false) {
    const bool s8 = col_scale != nullptr;
    const char* s8_name = s8_linear ? "b200sd_gemm_s8_linear" : "b200sd_gemm_s8";
    GemmPlan pl;
    if (lut) {
        if (int rc = plan_lut(a, *lut, pl)) return rc;
    } else if (int rc = plan_gemm(a, pl, bf16, s8, s8_linear)) {
        return rc;
    }
    B200SD_REQUIRE(a.a0 && (a.wgt || lut) && a.out, "b200sd_gemm: null pointer");
    B200SD_REQUIRE(!s8 || a.wgt_tiled, "%s: the weights must be pre-tiled (wgt_tiled = 1, explicit block_n)", s8_name);
    B200SD_REQUIRE(a.c1 == 0 || a.a1, "b200sd_gemm: a1 is null but c1 > 0");
    const size_t ws = plan_workspace(pl);
    B200SD_REQUIRE(ws == 0 || (a.workspace && a.workspace_bytes >= ws),
                   "b200sd_gemm: split-K needs %zu workspace bytes, got %zu", ws, a.workspace_bytes);

    GemmParams p;
    memset(&p, 0, sizeof(p));
    // ---- tensor maps ----
    const uint32_t es1[4] = {1, 1, 1, 1};
    if (pl.halo) {
        // activations are read by the loader warps with plain loads (only the weights go through TMA) unless this is the
        // plain convolution, whose patches are 4-D boxes {64 channels, patch pitch, patch rows, 1 image}; positions outside
        // the image (the padding ring, the pad column of the padded-linear walk) are zero-filled by the hardware
        if (pl.tma_patch) {
            const uint32_t box[4] = {kBK, static_cast<uint32_t>(pl.Wp), static_cast<uint32_t>(pl.patch_rows), 1};
            for (int src = 0; src < 2; ++src) {
                const int c = src == 0 ? a.c0 : a.c1;
                if (c == 0) {
                    p.tmA1 = p.tmA0;
                    continue;
                }
                const uint64_t dims[4] = {static_cast<uint64_t>(c), static_cast<uint64_t>(a.w),
                                          static_cast<uint64_t>(a.h), static_cast<uint64_t>(a.n_img)};
                const uint64_t str[3] = {static_cast<uint64_t>(c) * 2, static_cast<uint64_t>(c) * 2 * a.w,
                                         static_cast<uint64_t>(c) * 2 * a.w * a.h};
                if (int rc = encode_tmap_f16(src == 0 ? &p.tmA0 : &p.tmA1, src == 0 ? a.a0 : a.a1, 4, dims, str, box, es1))
                    return rc;
            }
        }
    } else if (s8 && a.mode == 0) {
        // int8 [m, c0] source: a box is 128 channels (128 bytes, one swizzle row) of 128 rows, the channel tail is zero filled
        const uint32_t box[2] = {2 * kBK, kBM};
        const uint64_t dims[2] = {static_cast<uint64_t>(a.c0), static_cast<uint64_t>(a.m)};
        const uint64_t str[1] = {static_cast<uint64_t>(a.c0)};
        if (int rc = encode_tmap(&p.tmA0, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.a0, 2, dims, str, box, es1)) return rc;
        p.tmA1 = p.tmA2 = p.tmA3 = p.tmA0;
    } else if (a.mode == 0) {
        const uint32_t box[2] = {kBK, kBM};
        {
            const uint64_t dims[2] = {static_cast<uint64_t>(a.c0), static_cast<uint64_t>(a.m)};
            const uint64_t str[1] = {static_cast<uint64_t>(a.c0) * 2};
            if (int rc = encode_tmap_f16(&p.tmA0, a.a0, 2, dims, str, box, es1)) return rc;
        }
        if (a.c1 > 0) {
            const uint64_t dims[2] = {static_cast<uint64_t>(a.c1), static_cast<uint64_t>(a.m)};
            const uint64_t str[1] = {static_cast<uint64_t>(a.c1) * 2};
            if (int rc = encode_tmap_f16(&p.tmA1, a.a1, 2, dims, str, box, es1)) return rc;
        } else {
            p.tmA1 = p.tmA0;
        }
    } else if (s8) {
        // int8 NHWC source: a box is 128 channels (128 bytes, one swizzle row), the channel tail is zero filled
        const uint32_t box[4] = {2 * kBK, static_cast<uint32_t>(pl.bw), static_cast<uint32_t>(pl.bh),
                                 static_cast<uint32_t>(pl.bn_img)};
        const uint64_t c = static_cast<uint64_t>(a.c0);
        const uint64_t dims[4] = {c, static_cast<uint64_t>(a.w), static_cast<uint64_t>(a.h), static_cast<uint64_t>(a.n_img)};
        const uint64_t str[3] = {c, c * a.w, c * a.w * a.h};
        if (int rc = encode_tmap(&p.tmA0, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.a0, 4, dims, str, box, es1)) return rc;
        p.tmA1 = p.tmA2 = p.tmA3 = p.tmA0;
    } else {
        const uint32_t st = static_cast<uint32_t>(a.stride);
        const uint32_t box[4] = {kBK, static_cast<uint32_t>(pl.bw) * st, static_cast<uint32_t>(pl.bh) * st,
                                 static_cast<uint32_t>(pl.bn_img)};
        const uint32_t es[4] = {1, st, st, 1};
        CUtensorMap* maps[4] = {&p.tmA0, &p.tmA1, &p.tmA2, &p.tmA3};
        const void* ptrs[4] = {a.a0, a.a1, a.a2, a.a3};
        const int chans[4] = {a.c0, a.c1, a.c2, a.c3};
        for (int src = 0; src < 4; ++src) {
            const int c = chans[src];
            if (c == 0) {
                *maps[src] = p.tmA0;
                continue;
            }
            B200SD_REQUIRE(ptrs[src] != nullptr, "b200sd_gemm: source %d has %d channels but a null pointer", src, c);
            const uint64_t dims[4] = {static_cast<uint64_t>(c), static_cast<uint64_t>(a.w),
                                      static_cast<uint64_t>(a.h), static_cast<uint64_t>(a.n_img)};
            const uint64_t str[3] = {static_cast<uint64_t>(c) * 2, static_cast<uint64_t>(c) * 2 * a.w,
                                     static_cast<uint64_t>(c) * 2 * a.w * a.h};
            if (int rc = encode_tmap_f16(maps[src], ptrs[src], 4, dims, str, box, es)) return rc;
        }
    }
    if (lut) {
        // packed indices [N][row_bytes], one box = pk_box bytes of block_n rows (rows >= N are zero filled)
        const uint64_t dims[2] = {static_cast<uint64_t>(lut->row_bytes), static_cast<uint64_t>(a.n)};
        const uint64_t str[1] = {static_cast<uint64_t>(lut->row_bytes)};
        const uint32_t box[2] = {static_cast<uint32_t>(pl.pk_box), static_cast<uint32_t>(pl.block_n)};
        if (int rc = encode_tmap(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_UINT8, lut->packed, 2, dims, str, box, es1,
                                 CU_TENSOR_MAP_SWIZZLE_NONE))
            return rc;
        p.lut = reinterpret_cast<const __half*>(lut->lut);
        p.kscale = lut->kscale;
        p.nbits = lut->nbits, p.pk_box = pl.pk_box, p.pk_slots = pl.pk_slots;
        p.seg_end0 = lut->seg_end0, p.seg_end1 = lut->seg_end1;
    } else if (s8) {
        B200SD_REQUIRE(a.block_n == pl.block_n, "%s: tiled weights need an explicit block_n", s8_name);
        const uint64_t rows = static_cast<uint64_t>(pl.n_tiles) * pl.kb_total * pl.block_n;
        const uint64_t dims[2] = {2 * kBK, rows};
        const uint64_t str[1] = {2 * kBK};
        const uint32_t box[2] = {2 * kBK, static_cast<uint32_t>(pl.block_n)};
        if (int rc = encode_tmap(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_UINT8, a.wgt, 2, dims, str, box, es1)) return rc;
    } else if (a.wgt_tiled) {
        B200SD_REQUIRE(a.block_n == pl.block_n, "b200sd_gemm: tiled weights need an explicit block_n");
        const uint64_t rows = static_cast<uint64_t>(pl.n_tiles) * pl.kb_total * pl.block_n;
        const uint64_t dims[2] = {kBK, rows};
        const uint64_t str[1] = {kBK * 2};
        const uint32_t box[2] = {kBK, static_cast<uint32_t>(pl.block_n)};
        if (int rc = encode_tmap_f16(&p.tmB, a.wgt, 2, dims, str, box, es1)) return rc;
    } else {
        const uint64_t ktot = static_cast<uint64_t>(pl.taps) * pl.Kpt;
        const uint64_t dims[2] = {ktot, static_cast<uint64_t>(a.n)};
        const uint64_t str[1] = {ktot * 2};
        const uint32_t box[2] = {kBK, static_cast<uint32_t>(pl.block_n)};
        if (int rc = encode_tmap_f16(&p.tmB, a.wgt, 2, dims, str, box, es1)) return rc;
    }
    p.mode = pl.halo ? 2 : a.mode;
    p.M = pl.M;
    p.N = a.n;
    p.n_store = a.geglu ? a.n / 2 : a.n;
    p.C0 = a.c0;
    p.Kpt = pl.Kpt;
    p.kc0 = pl.kc0;
    p.kc = pl.kc0 + pl.kc1;
    p.kc2 = (a.c2 + kBK - 1) / kBK, p.kc3 = (a.c3 + kBK - 1) / kBK;
    p.taps = pl.taps;
    p.kb_total = pl.kb_total;
    p.kb_per_split = pl.kb_per_split;
    p.splits = pl.splits;
    p.m_tiles = pl.m_tiles;
    p.n_tiles = pl.n_tiles;
    p.block_n = pl.block_n;
    p.stages = pl.stages;
    p.n_img = a.n_img;
    p.Hout = pl.Hout;
    p.Wout = pl.Wout;
    p.stride = a.mode == 1 ? a.stride : 1;
    p.bw_log2 = ilog2(pl.bw);
    p.bh_log2 = ilog2(pl.bh);
    p.tiles_w = pl.tiles_w;
    p.tiles_h = pl.tiles_h;
    p.bias_rows = a.bias_rows;
    p.bias_stride = a.bias_stride > 0 ? a.bias_stride : a.n;
    p.geglu = a.geglu;
    p.out_f32 = a.out_f32;
    p.act = a.act;
    p.pad_lo = a.pad_after_only ? 0 : 1;
    p.wgt_tiled = a.wgt_tiled;
    p.bias_mode = pl.bias_mode;
    p.res_smem = pl.res_smem;
    p.out = a.out;
    p.bias = a.bias;
    p.residual = reinterpret_cast<const __half*>(a.residual);
    p.partial = (pl.splits > 1 && !pl.cluster) ? a.workspace : nullptr;
    p.cluster = pl.cluster;
    p.H = a.h, p.W = a.w, p.Wp = pl.Wp, p.tiles_per_img = pl.tiles_per_img;
    p.win = pl.win, p.tw = pl.tw, p.th = pl.th, p.tiles_x = pl.tiles_x;
    p.inv_wp = pl.Wp > 0 ? (1 << 20) / pl.Wp + 1 : 0;
    p.patch_rows = pl.patch_rows, p.patch_bytes = pl.patch_bytes;
    p.upsample = a.upsample2x, p.desc_bo = desc_base_offset_enabled() ? 1 : 0;
    p.tma_patch = pl.tma_patch, p.patch_tx = pl.patch_rows * pl.Wp * kBK * 2;
    p.a0 = reinterpret_cast<const __half*>(a.a0), p.a1 = reinterpret_cast<const __half*>(a.a1), p.C1 = a.c1;
    if (pl.halo && a.gn_groups > 0) {
        B200SD_REQUIRE(a.gn_chan0 && a.gn_gamma && a.gn_beta && (a.c1 == 0 || a.gn_chan1) && a.gn_groups <= 64 &&
                           (a.c0 + a.c1) % a.gn_groups == 0,
                       "b200sd_gemm: bad fused GroupNorm arguments");
        p.gn_chan0 = a.gn_chan0, p.gn_chan1 = a.gn_chan1, p.gn_gamma = a.gn_gamma, p.gn_beta = a.gn_beta;
        p.gn_groups = a.gn_groups, p.gn_silu = a.gn_silu, p.gn_eps = a.gn_eps, p.gn_hw = a.h * a.w;
    }
    p.cs_partial = a.cs_partial, p.cs_chan = a.cs_chan, p.cs_tickets = a.cs_tickets;
    p.cs_slots = pl.cs_slots;
    p.cs_hw = a.mode == 0 ? a.cs_hw : pl.Hout * pl.Wout;
    if (p.cs_hw <= 0) p.cs_hw = 1;
    B200SD_REQUIRE(a.cs_partial == nullptr || (a.cs_chan && a.cs_tickets), "b200sd_gemm: statistics outputs need cs_chan and cs_tickets");
    p.rs_out = a.rs_out;
    p.ln_stat = a.ln_stat, p.ln_wg = a.ln_wg, p.ln_parts = a.ln_parts, p.ln_eps = a.ln_eps, p.ln_k = a.c0 + a.c1;
    p.staged = pl.staged, p.stage_dedicated = pl.stage_dedicated;
    {
        const char* e = getenv("B200SD_DBG_PTR");  // tools/halo_timeline.py: device address of a 128-slot int64 buffer
        p.dbg = (e && e[0]) ? reinterpret_cast<long long*>(strtoull(e, nullptr, 0)) : nullptr;
    }
    if (pl.halo) {
        using HaloFn = void (*)(GemmParams);
        const int kind = pl.halo_kind;
        const bool wide = pl.block_n > 128;  // (only the TMA-patch kind takes tiles wider than 128 columns)
        HaloFn hfn = kind == 2 ? (wide ? halo_conv_kernel<2, 128> : halo_conv_kernel<2, 64>)
                               : (kind == 1 ? halo_conv_kernel<1, 8> : halo_conv_kernel<0, 64>);
        const int hslot = kind == 2 && wide ? 3 : kind;
        static bool hattr[4] = {false, false, false, false};
        if (!hattr[hslot]) {
            B200SD_CHECK_CUDA(cudaFuncSetAttribute(hfn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            hattr[hslot] = true;
        }
        const int units = pl.m_tiles * pl.n_tiles;
        B200SD_CHECK_CUDA(launch_kernel(hfn, dim3(std::min(units, num_sms())), dim3(kHaloThreads), pl.smem_bytes, stream, p));
        B200SD_CHECK_CUDA(cudaGetLastError());
        count_launch(1);
        return 0;
    }

    const int smem_bytes = pl.smem_bytes;
    const int total = pl.m_tiles * pl.n_tiles * pl.splits;
    const int grid = std::min(total, num_sms());
    B200SD_REQUIRE(a.act == 0 || (a.act >= 1 && a.act <= 3 && pl.splits == 1 && !a.geglu), "b200sd_gemm: act=%d unsupported here", a.act);
    const int wi = gemm_width_index(pl.block_n);
    const int variant = pl.variant;
    KernelFn fn = nullptr;
    p.col_scale = col_scale;
    p.out_inv_scale = a.out_s8_inv_scale;
    if (lut) {
        switch (variant) {
            case kVariantGeneric: fn = lut_kernel<true, false, false>(wi); break;
            case kVariantSplitK: fn = lut_kernel<false, false, true>(wi); break;
            case kVariantGeglu: fn = lut_kernel<false, true, false>(wi); break;
            case kVariantPlain: fn = lut_kernel<false, false, false>(wi); break;
            default: break;
        }
    } else if (s8) {  // plan_gemm gives the int8 convolution the first three variants only
        switch (variant) {
            case kVariantGeneric: fn = s8_kernel<true, false>(wi); break;
            case kVariantSplitK: fn = s8_kernel<false, true>(wi); break;
            case kVariantPlain: fn = s8_kernel<false, false>(wi); break;
            case kVariantGeglu: fn = s8io_kernel<true, true, false>(wi); break;
            case kVariantS8Out: fn = s8io_kernel<true, false, true>(wi); break;
            case kVariantGegluS8Out: fn = s8io_kernel<true, true, true>(wi); break;
            default: break;
        }
    } else if (bf16) {  // plan_gemm gives bf16 only these three variants
        switch (variant) {
            case kVariantGeneric: fn = gemm_kernel<__nv_bfloat16, true, false, false, false, false>(wi); break;
            case kVariantF32: fn = gemm_kernel<__nv_bfloat16, false, false, true, false, false>(wi); break;
            case kVariantPlain: fn = gemm_kernel<__nv_bfloat16, false, false, false, false, false>(wi); break;
            default: break;
        }
    } else {
        switch (variant) {
            case kVariantGeneric: fn = gemm_kernel<__half, true, false, false, false, false>(wi); break;
            case kVariantStaged: fn = gemm_kernel<__half, false, false, false, false, true>(wi); break;
            case kVariantSplitK: fn = gemm_kernel<__half, false, false, false, true, false>(wi); break;
            case kVariantGeglu: fn = gemm_kernel<__half, false, true, false, false, false>(wi); break;
            case kVariantF32: fn = gemm_kernel<__half, false, false, true, false, false>(wi); break;
            case kVariantS8Out: fn = s8io_kernel<false, false, true>(wi); break;
            case kVariantGegluS8Out: fn = s8io_kernel<false, true, true>(wi); break;
            default: fn = gemm_kernel<__half, false, false, false, false, false>(wi); break;
        }
    }
    B200SD_REQUIRE(fn != nullptr, "b200sd_gemm: no %s kernel for variant %d at block_n %d",
                   lut ? "palettized" : (s8 ? "int8" : (bf16 ? "bf16" : "fp16")),
                   variant, pl.block_n);
    if (pl.splits > 1 && !pl.cluster) {
        // the separate reduce kernel applies bias / residual; the partial writer must not
        p.bias = nullptr;
        p.residual = nullptr;
    }
    static bool attr_set[4][8][kNumGemmWidths] = {};
    const int dt = lut ? 3 : (s8 ? 2 : (bf16 ? 1 : 0));
    if (!attr_set[dt][variant][wi]) {
        B200SD_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set[dt][variant][wi] = true;
    }
    if (pl.cluster) {
        B200SD_REQUIRE(variant == 1, "b200sd_gemm: cluster split-K needs the regular epilogue variant");
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        // split-K: one (tile, split) per CTA, the splits of a tile are one cluster
        cfg.gridDim = dim3(total);
        cfg.blockDim = dim3(kGemmThreads);
        cfg.dynamicSmemBytes = smem_bytes;
        cfg.stream = stream;
        cudaLaunchAttribute at[2];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = pl.splits;
        at[0].val.clusterDim.y = 1;
        at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        if (pdl_enabled()) {
            at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            at[1].val.programmaticStreamSerializationAllowed = 1;
            cfg.numAttrs = 2;
        }
        B200SD_CHECK_CUDA(cudaLaunchKernelEx(&cfg, fn, p));
        B200SD_CHECK_CUDA(cudaGetLastError());
        count_launch(1);
        return 0;
    }
    B200SD_CHECK_CUDA(launch_kernel(fn, dim3(grid), dim3(kGemmThreads), smem_bytes, stream, p));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    if (pl.splits > 1) {
        const size_t total4 = static_cast<size_t>(pl.M) * a.n / 4;
        const int rgrid = static_cast<int>(std::min<size_t>((total4 + 255) / 256, static_cast<size_t>(num_sms()) * 8));
        B200SD_CHECK_CUDA(launch_kernel(splitk_reduce_kernel, dim3(rgrid), dim3(256), 0, stream, a.workspace, pl.splits, pl.M, a.n, a.bias, a.bias_rows,
                                                        a.bias_stride > 0 ? a.bias_stride : a.n,
                                                        reinterpret_cast<const __half*>(a.residual), a.out, a.out_f32));
        B200SD_CHECK_CUDA(cudaGetLastError());
        count_launch(1);
    }
    return 0;
}

}  // namespace b200sd

static int gemm_entry(const b200sd_gemm_args* args, void* stream, bool bf16, const float* col_scale = nullptr,
                      bool s8_linear = false) {
    if (!b200sd::launch_class_enabled(1)) return 0;  // bench.py's per-class timing graphs
    if (!args) {
        b200sd::set_error(s8_linear ? "b200sd_gemm_s8_linear: args is null"
                                    : (col_scale ? "b200sd_gemm_s8: args is null"
                                                 : (bf16 ? "b200sd_gemm_bf16: args is null" : "b200sd_gemm: args is null")));
        return 2;
    }
    return b200sd::launch_gemm(*args, static_cast<cudaStream_t>(stream), bf16, col_scale, nullptr, s8_linear);
}

extern "C" int b200sd_gemm(const b200sd_gemm_args* args, void* stream) { return gemm_entry(args, stream, false); }
extern "C" int b200sd_gemm_bf16(const b200sd_gemm_args* args, void* stream) { return gemm_entry(args, stream, true); }
extern "C" int b200sd_gemm_s8(const b200sd_gemm_args* args, const float* col_scale, void* stream) {
    if (!col_scale) {
        b200sd::set_error("b200sd_gemm_s8: col_scale is null");
        return 2;
    }
    return gemm_entry(args, stream, false, col_scale);
}
extern "C" int b200sd_gemm_s8_linear(const b200sd_gemm_args* args, const float* col_scale, void* stream) {
    if (!col_scale) {
        b200sd::set_error("b200sd_gemm_s8_linear: col_scale is null");
        return 2;
    }
    return gemm_entry(args, stream, false, col_scale, true);
}

extern "C" int b200sd_gemm_lut(const b200sd_gemm_args* args, const b200sd_lut_args* lut, void* stream) {
    if (!b200sd::launch_class_enabled(1)) return 0;  // bench.py's per-class timing graphs
    if (!args || !lut) {
        b200sd::set_error("b200sd_gemm_lut: args or lut is null");
        return 2;
    }
    return b200sd::launch_gemm(*args, static_cast<cudaStream_t>(stream), false, nullptr, lut);
}

extern "C" int b200sd_gemm_describe_plan_lut(const b200sd_gemm_args* args, const b200sd_lut_args* lut, char* buf, size_t buf_size) {
    if (!args || !lut || !buf || buf_size == 0) return 2;
    b200sd::GemmPlan pl;
    if (int rc = b200sd::plan_lut(*args, *lut, pl)) return rc;
    snprintf(buf, buf_size, "M=%d N=%d kb_total=%d m_tiles=%d n_tiles=%d block_n=%d splits=%d kb_per_split=%d stages=%d "
             "pk_slots=%d pk_box=%d cluster=%d variant=%d smem=%d",
             pl.M, pl.N, pl.kb_total, pl.m_tiles, pl.n_tiles, pl.block_n, pl.splits, pl.kb_per_split, pl.stages,
             pl.pk_slots, pl.pk_box, pl.cluster, pl.variant, pl.smem_bytes);
    return 0;
}

extern "C" int b200sd_gemm_plan(const b200sd_gemm_args* args, int32_t* out4) {
    if (!args || !out4) return 2;
    b200sd::GemmPlan pl;
    if (int rc = b200sd::plan_gemm(*args, pl)) return rc;
    out4[0] = pl.block_n, out4[1] = pl.splits, out4[2] = pl.kb_total, out4[3] = pl.n_tiles;
    return 0;
}

// Planning query before the weights are tiled: a halo call plans for chunk-major tiled weights of the requested (or the
// preferred) width.
static int plan_query(const b200sd_gemm_args* args, b200sd::GemmPlan& pl, bool bf16, bool s8 = false, bool s8_linear = false) {
    b200sd_gemm_args a = *args;
    if (a.halo && !bf16 && !s8) {
        if (a.block_n == 0) a.block_n = b200sd::halo_pick_block_n(a);
        a.wgt_tiled = 1;
    }
    return b200sd::plan_gemm(a, pl, bf16, s8, s8_linear);
}

static int plan_ex(const b200sd_gemm_args* args, int32_t* out8, bool bf16, bool s8 = false, bool s8_linear = false) {
    if (!args || !out8) return 2;
    b200sd::GemmPlan pl;
    if (int rc = plan_query(args, pl, bf16, s8, s8_linear)) return rc;
    out8[0] = pl.block_n, out8[1] = pl.splits, out8[2] = pl.kb_total, out8[3] = pl.n_tiles;
    out8[4] = pl.cs_slots, out8[5] = pl.staged, out8[6] = pl.stages, out8[7] = pl.m_tiles;
    return 0;
}

extern "C" int b200sd_gemm_plan_ex(const b200sd_gemm_args* args, int32_t* out8) { return plan_ex(args, out8, false); }
extern "C" int b200sd_gemm_plan_ex_bf16(const b200sd_gemm_args* args, int32_t* out8) { return plan_ex(args, out8, true); }
extern "C" int b200sd_gemm_plan_ex_s8(const b200sd_gemm_args* args, int32_t* out8) { return plan_ex(args, out8, false, true); }
extern "C" int b200sd_gemm_plan_ex_s8_linear(const b200sd_gemm_args* args, int32_t* out8) {
    return plan_ex(args, out8, false, true, true);
}

static int describe_plan(const b200sd_gemm_args* args, char* buf, size_t buf_size, bool bf16, bool s8 = false,
                         bool s8_linear = false) {
    if (!args || !buf || buf_size == 0) return 2;
    b200sd::GemmPlan pl;
    if (int rc = plan_query(args, pl, bf16, s8, s8_linear)) return rc;
    // variant: GemmVariant of the GEMM kernel (-1: halo convolution); halo_kind / halo_wide: which halo_conv_kernel
    // instantiation runs (-1 / 0 for the GEMM kernel); win: the halo walk over th x tw windows instead of image rows
    snprintf(buf, buf_size,
             "M=%d N=%d kb_total=%d m_tiles=%d n_tiles=%d block_n=%d splits=%d kb_per_split=%d stages=%d "
             "box=%dx%dx%d bias_mode=%d res_smem=%d epi_smem=%d cluster=%d staged=%d variant=%d halo_kind=%d halo_wide=%d win=%d",
             pl.M, pl.N, pl.kb_total, pl.m_tiles, pl.n_tiles, pl.block_n, pl.splits, pl.kb_per_split, pl.stages,
             pl.bn_img, pl.bh, pl.bw, pl.bias_mode, pl.res_smem, pl.epi_smem, pl.cluster, pl.staged, pl.variant, pl.halo_kind,
             pl.halo && pl.block_n > 128 ? 1 : 0, pl.halo ? pl.win : 0);
    return 0;
}

extern "C" int b200sd_gemm_describe_plan(const b200sd_gemm_args* args, char* buf, size_t buf_size) {
    return describe_plan(args, buf, buf_size, false);
}
extern "C" int b200sd_gemm_describe_plan_bf16(const b200sd_gemm_args* args, char* buf, size_t buf_size) {
    return describe_plan(args, buf, buf_size, true);
}
extern "C" int b200sd_gemm_describe_plan_s8(const b200sd_gemm_args* args, char* buf, size_t buf_size) {
    return describe_plan(args, buf, buf_size, false, true);
}
extern "C" int b200sd_gemm_describe_plan_s8_linear(const b200sd_gemm_args* args, char* buf, size_t buf_size) {
    return describe_plan(args, buf, buf_size, false, true, true);
}

extern "C" size_t b200sd_gemm_workspace_bytes(const b200sd_gemm_args* args) {
    if (!args) return 0;
    b200sd::GemmPlan pl;
    if (b200sd::plan_gemm(*args, pl)) return 0;
    return b200sd::plan_workspace(pl);
}

extern "C" size_t b200sd_gemm_workspace_bytes_s8(const b200sd_gemm_args* args) {
    if (!args) return 0;
    b200sd::GemmPlan pl;
    if (b200sd::plan_gemm(*args, pl, false, true)) return 0;
    return b200sd::plan_workspace(pl);
}

extern "C" size_t b200sd_gemm_workspace_bytes_s8_linear(const b200sd_gemm_args* args) {
    if (!args) return 0;
    b200sd::GemmPlan pl;
    if (b200sd::plan_gemm(*args, pl, false, true, true)) return 0;
    return b200sd::plan_workspace(pl);
}
