// b200sd -- flash-style attention for sm_90a: S = Q K^T and O += P V on wgmma tensor cores (fp32 accumulators in
// registers), Q/K/V tiles staged by TMA (SWIZZLE_128B), online softmax (exp2 domain) in registers, P handed to the
// tensor core straight from registers (wgmma with A in registers).
//
// Replaces attention.original / split_einsum / split_einsum_v2 of the reference
// (python_coreml_stable_diffusion/attention.py:24-168, dispatched by Einsum unet.py:45-59): the
// three variants are one function, softmax(q^T k / sqrt(d) + mask) v per (batch, head); the
// (B, heads, Sq, Sk) score tensor the reference materialises (671 MB at S=4096) never leaves the SM.
//
// CTA = 128 queries x 1 head; warps 0..7 are two consumer warpgroups (64 query rows each), warp 8 the TMA producer.
// The K/V ring holds two 128-key tiles; each warpgroup walks them in 64-key halves: S_h = Q K_h^T, softmax, O += P_h V_h.
// While one warpgroup is in its exponentials the other one keeps the tensor core busy.
#include "common.cuh"
#include "../../include/b200sd.h"

namespace b200sd {

extern void count_launch(int n);

static constexpr int kQ = 128;   // queries per CTA
static constexpr int kKV = 128;  // keys per K/V tile (one TMA load)
static constexpr int kHalf = 64;  // keys per pipeline step
static constexpr int kD = 64;    // head dim
static constexpr int kAttnThreads = 288;
static constexpr int kProducerWarp = 8;
static constexpr int kTileBytes = 128 * 64 * 2;  // 16 KiB: one [128 x 64] fp16 tile
static constexpr int kKvStages = 2;

struct __align__(64) AttnParams {
    CUtensorMap tmQ, tmK, tmV;
    __half* out;
    const float* mask;  // [batch, sk] additive or null
    int sq, sk, ldo;
    int causal;  // 1: key j is visible to query i only if j <= i (CLIP text encoder)
    float scale_log2;  // scale * log2(e)
    // work decomposition: query tile t -> (q tile t % q_tiles, head (t / q_tiles) % heads, image t / (q_tiles * heads)).
    // streamk == 0: grid = tiles, one CTA per query tile.  streamk == 1: the tiles x n_kv (query tile, K/V tile) units are
    // cut into gridDim.x equal contiguous ranges, so a CTA works on the tail of one query tile and the head of the next;
    // pieces of a split tile go through `ws` and the last piece to finish merges them in slot order.
    int q_tiles, heads, n_kv, streamk;
    long long total_units;
    float* ws;      // [gridDim.x][2] partials of kPartialFloats floats
    int* counters;  // [tiles], zero between launches
};

// one partial: O [64 d][128 rows] fp32 (column-major so consecutive rows are contiguous), then m_ref[128], l[128]
static constexpr int kPartialFloats = (kD + 2) * kQ;
static constexpr size_t kCounterBytes = 64 * 1024;

// smem layout (1024-aligned): Q | K[2] | V[2] | barriers
static constexpr int kSmemQ = 0;
static constexpr int kSmemK = kSmemQ + kTileBytes;
static constexpr int kSmemV = kSmemK + kKvStages * kTileBytes;
static constexpr int kSmemBar = kSmemV + kKvStages * kTileBytes;
static constexpr int kAttnSmemBytes = kSmemBar + 128;

__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// A CTA's share of the work: query tile `tile`, K/V tiles [k0, k1) of it.
struct AttnSegment {
    int tile, k0, k1;
};

// first unit of slot s / the slot that owns unit u, for the floor partition u0(s) = s * total / slots
__device__ __forceinline__ long long slot_begin(const AttnParams& p, long long s) { return s * p.total_units / gridDim.x; }
__device__ __forceinline__ int slot_of(const AttnParams& p, long long u) {
    return static_cast<int>(((u + 1) * gridDim.x - 1) / p.total_units);
}

// Walks this CTA's segments in order.  Returns false when the range is exhausted.
struct SegmentWalk {
    long long u, u1;
    __device__ __forceinline__ void init(const AttnParams& p) {
        if (p.streamk) {
            u = slot_begin(p, blockIdx.x), u1 = slot_begin(p, blockIdx.x + 1);
        } else {
            u = static_cast<long long>(blockIdx.x) * p.n_kv, u1 = u + p.n_kv;
        }
    }
    __device__ __forceinline__ bool next(const AttnParams& p, AttnSegment& sg) {
        if (u >= u1) return false;
        sg.tile = static_cast<int>(u / p.n_kv);
        sg.k0 = static_cast<int>(u - static_cast<long long>(sg.tile) * p.n_kv);
        sg.k1 = static_cast<int>(min(static_cast<long long>(p.n_kv), sg.k0 + (u1 - u)));
        u += sg.k1 - sg.k0;
        return true;
    }
};

// number of 64-key halves a segment visits (the last K/V tile may be ragged; causal tiles stop at the diagonal)
__device__ __forceinline__ int segment_halves(const AttnParams& p, const AttnSegment& sg, int q0) {
    const int sk_eff = p.causal ? min(p.sk, q0 + kQ) : p.sk;
    const int n_half = (sk_eff + kHalf - 1) / kHalf;
    return min(2 * sg.k1, n_half) - 2 * sg.k0;
}

__global__ void __launch_bounds__(kAttnThreads, 1) attention_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kSmemBar);
    uint64_t* q_full = bars + 0;
    uint64_t* kv_full = bars + 1;   // [2]
    uint64_t* kv_empty = bars + 3;  // [2]
    uint64_t* q_empty = bars + 5;   // every S MMA of the segment retired: Q may be overwritten
    int* last_flag = reinterpret_cast<int*>(bars + 6);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        // SWIZZLE_128B tiles need a 1024-byte aligned base; a misaligned launch (never observed: the kernel has no
        // static shared memory) fails loudly instead
        if ((smem_u32(smem) & 1023u) != 0) __trap();
        prefetch_tmap(&p.tmQ);
        prefetch_tmap(&p.tmK);
        prefetch_tmap(&p.tmV);
        mbar_init(q_full, 1);
        mbar_init(q_empty, 2);
        for (int s = 0; s < kKvStages; ++s) {
            mbar_init(&kv_full[s], 1);
            mbar_init(&kv_empty[s], 2);  // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();     // PDL: the prologue above overlapped the previous kernel's tail

    // Both roles walk the same segment list.  The K/V tile counter jg runs ACROSS segments (smem stage jg % 2).
    SegmentWalk walk;
    walk.init(p);
    AttnSegment sg;

    if (warp == kProducerWarp) {
        if (lane == 0) {
            int seg = 0, jg = 0;
            while (walk.next(p, sg)) {
                const int qt = sg.tile % p.q_tiles, head = (sg.tile / p.q_tiles) % p.heads, batch = sg.tile / (p.q_tiles * p.heads);
                const int nh = segment_halves(p, sg, qt * kQ);
                if (seg > 0) mbar_wait(q_empty, (seg - 1) & 1);
                mbar_expect_tx(q_full, kTileBytes);
                tma_load_3d(smem + kSmemQ, &p.tmQ, q_full, head * kD, qt * kQ, batch, kEvictFirst);
                for (int jl = 0; jl < (nh + 1) / 2; ++jl, ++jg) {
                    const int st = jg % kKvStages;
                    const uint32_t ph = (jg / kKvStages) & 1;
                    mbar_wait(&kv_empty[st], ph ^ 1);
                    mbar_expect_tx(&kv_full[st], 2 * kTileBytes);
                    tma_load_3d(smem + kSmemK + st * kTileBytes, &p.tmK, &kv_full[st], head * kD, (sg.k0 + jl) * kKV, batch,
                                kEvictLast);
                    tma_load_3d(smem + kSmemV + st * kTileBytes, &p.tmV, &kv_full[st], head * kD, (sg.k0 + jl) * kKV, batch,
                                kEvictLast);
                }
                ++seg;
            }
        }
    } else if (warp < kProducerWarp) {
        // ---------------- consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile ----------------
        // Accumulator layout (m64n64): this thread holds rows lr and lr + 8 (lr = 16 (warp % 4) + lane / 4 inside the
        // warpgroup's 64), columns 8 j + 2 (lane % 4) + {0, 1}, j = 0..7: s[4 j + {0, 1}] row lr, s[4 j + {2, 3}] row lr + 8.
        // A row is spread over the four lanes of a quad: row maxima / sums reduce with two shuffles.
        const int wg = warp >> 2;
        const int lr = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // tile-local row of s[.. 0, 1]; lr + 8 for s[.. 2, 3]
        const int cq = 2 * (lane & 3);
        const bool leader = (threadIdx.x & 127) == 0;
        const float sl2 = p.scale_log2;
        const uint32_t q_addr = smem_u32(smem + kSmemQ) + wg * 64 * 128;
        int seg = 0, jg0 = 0;
        while (walk.next(p, sg)) {
            const int qt = sg.tile % p.q_tiles, head = (sg.tile / p.q_tiles) % p.heads, batch = sg.tile / (p.q_tiles * p.heads);
            const int q0 = qt * kQ;
            const int nh = segment_halves(p, sg, q0);
            const float* mask_row = p.mask ? p.mask + static_cast<size_t>(batch) * p.sk : nullptr;
            float o[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) o[i] = 0.f;
            float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
            mbar_wait(q_full, seg & 1);
            for (int hl = 0; hl < nh; ++hl) {
                const int jg = jg0 + (hl >> 1), st = jg % kKvStages, hi = hl & 1;
                if (hi == 0) mbar_wait(&kv_full[st], (jg / kKvStages) & 1);
                // ---- S = Q K_h^T ----
                float s[32];
                const uint64_t qdesc = make_smem_desc_sw128(q_addr, 1024, 0);
                const uint64_t kdesc = make_smem_desc_sw128(smem_u32(smem + kSmemK + st * kTileBytes) + hi * (kHalf * 128), 1024, 0);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kD / 16; ++k) wgmma_m64n64_ss(s, qdesc + 2 * k, kdesc + 2 * k, k > 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs<32>(s);
                if (hl == nh - 1 && leader) mbar_arrive(q_empty);  // the segment's last read of Q retired
                // ---- online softmax (log2 domain) ----
                const int h = 2 * sg.k0 + hl;                     // this half's position among the keys
                const int kvalid = min(kHalf, p.sk - h * kHalf);  // >= 1
                // causal: a half whose last key is <= the tile's first query is fully visible to every row
                const bool diag = p.causal && (h * kHalf + kHalf - 1 > q0);
                const bool general = mask_row != nullptr || kvalid < kHalf || diag;
#pragma unroll
                for (int e = 0; e < 32; ++e) {
                    float v = s[e] * sl2;
                    if (general) {
                        const int key = 8 * (e >> 2) + cq + (e & 1);
                        const int qi = q0 + lr + 8 * ((e >> 1) & 1);
                        const bool vis = key < kvalid && (!diag || h * kHalf + key <= qi);
                        if (mask_row != nullptr && vis) v += mask_row[h * kHalf + key] * 1.4426950408889634f;
                        if (!vis) v = -INFINITY;
                    }
                    s[e] = v;
                }
                float m_use[2];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    float mx = -INFINITY;
#pragma unroll
                    for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * r], s[4 * j + 2 * r + 1]));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    const float m_new = fmaxf(m_run[r], mx);
                    m_use[r] = m_new == -INFINITY ? 0.f : m_new;  // a row with nothing visible yet
                    const float factor = ex2_approx(m_run[r] - m_use[r]);
                    m_run[r] = m_new;
                    l_run[r] *= factor;
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[4 * j + 2 * r] *= factor, o[4 * j + 2 * r + 1] *= factor;
                }
                uint32_t pa[4][4];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float p0 = ex2_approx(s[4 * j] - m_use[0]), p1 = ex2_approx(s[4 * j + 1] - m_use[0]);
                    const float p2 = ex2_approx(s[4 * j + 2] - m_use[1]), p3 = ex2_approx(s[4 * j + 3] - m_use[1]);
                    l_run[0] += p0 + p1;
                    l_run[1] += p2 + p3;
                    // A fragment of keys [16 kk, 16 kk + 16): {row lr, keys 0..7}, {lr + 8, 0..7}, {lr, 8..15}, {lr + 8, 8..15}
                    pa[j >> 1][2 * (j & 1)] = pack_half2(p0, p1);
                    pa[j >> 1][2 * (j & 1) + 1] = pack_half2(p2, p3);
                }
                // ---- O += P V_h: B = 64 rows of the V tile [keys][d] = MN-major, 16 keys = 2048 B per step ----
                const uint32_t v_addr = smem_u32(smem + kSmemV + st * kTileBytes) + hi * (kHalf * 128);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < kHalf / 16; ++kk)
                    wgmma_m64n64_rs_tb(o, pa[kk], make_smem_desc_sw128(v_addr + kk * 2048, 1024, kKV * 128), 1u);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs<32>(o);
                if ((hi == 1 || hl == nh - 1) && leader) mbar_arrive(&kv_empty[st]);  // last half of this K/V tile
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
                l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
            }
            ++seg, jg0 += (nh + 1) / 2;
            if (sg.k0 == 0 && sg.k1 == p.n_kv) {
                // whole query tile in this CTA: normalise and store
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int qi = q0 + lr + 8 * r;
                    if (qi >= p.sq) continue;
                    const float inv_l = 1.0f / l_run[r];
                    __half* dst = p.out + (static_cast<size_t>(batch) * p.sq + qi) * p.ldo + head * kD;
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        *reinterpret_cast<uint32_t*>(dst + 8 * j + cq) = pack_half2(o[4 * j + 2 * r] * inv_l, o[4 * j + 2 * r + 1] * inv_l);
                }
            } else {
                // ---- a piece of a split tile: park (O, m_ref, l) in the workspace; the piece that finishes last merges
                // ALL pieces (its own included) in slot order, so the result does not depend on who was last ----
                const long long t0 = static_cast<long long>(sg.tile) * p.n_kv;
                const int first = slot_of(p, t0), last = slot_of(p, t0 + p.n_kv - 1);
                float* mine = p.ws + (static_cast<size_t>(blockIdx.x) * 2 + (sg.k0 > 0 ? 1 : 0)) * kPartialFloats;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int row = lr + 8 * r;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        __stcg(mine + (8 * j + cq) * kQ + row, o[4 * j + 2 * r]);
                        __stcg(mine + (8 * j + cq + 1) * kQ + row, o[4 * j + 2 * r + 1]);
                    }
                    if ((lane & 3) == 0) {
                        __stcg(mine + kD * kQ + row, m_run[r]);
                        __stcg(mine + (kD + 1) * kQ + row, l_run[r]);
                    }
                }
                __threadfence();
                named_bar_sync(1, 256);
                if (threadIdx.x == 0) {
                    const int old = atomicAdd(p.counters + sg.tile, 1);
                    const int is_last = old == last - first;
                    if (is_last) p.counters[sg.tile] = 0;  // every piece has checked in: ready for the next launch
                    *last_flag = is_last;
                }
                named_bar_sync(1, 256);
                if (*last_flag) {
                    __threadfence();
                    // merge: thread t takes row t % 128, head-dim columns [32 (t / 128), + 32)
                    const int row = threadIdx.x & 127;
                    const int cbase = 32 * (threadIdx.x >> 7);
                    const bool store = q0 + row < p.sq;
                    __half* dst = p.out + (static_cast<size_t>(batch) * p.sq + (store ? q0 + row : 0)) * p.ldo + head * kD;
                    float m = -INFINITY;
                    for (int s2 = first; s2 <= last; ++s2) {
                        const float* part = p.ws + (static_cast<size_t>(s2) * 2 + (slot_begin(p, s2) > t0 ? 1 : 0)) * kPartialFloats;
                        m = fmaxf(m, __ldcg(part + kD * kQ + row));
                    }
                    float l = 0.f;
                    for (int s2 = first; s2 <= last; ++s2) {
                        const float* part = p.ws + (static_cast<size_t>(s2) * 2 + (slot_begin(p, s2) > t0 ? 1 : 0)) * kPartialFloats;
                        l += __ldcg(part + (kD + 1) * kQ + row) * ex2_approx(__ldcg(part + kD * kQ + row) - m);
                    }
                    const float inv_l = 1.0f / l;
#pragma unroll 1
                    for (int c = cbase; c < cbase + 32; c += 16) {
                        float acc[16];
#pragma unroll
                        for (int i = 0; i < 16; ++i) acc[i] = 0.f;
                        for (int s2 = first; s2 <= last; ++s2) {
                            const float* part =
                                p.ws + (static_cast<size_t>(s2) * 2 + (slot_begin(p, s2) > t0 ? 1 : 0)) * kPartialFloats;
                            const float f = ex2_approx(__ldcg(part + kD * kQ + row) - m);
#pragma unroll
                            for (int i = 0; i < 16; ++i) acc[i] = fmaf(__ldcg(part + (c + i) * kQ + row), f, acc[i]);
                        }
                        if (store) {
#pragma unroll
                            for (int i = 0; i < 16; i += 8) {
                                uint4 val;
                                val.x = pack_half2(acc[i] * inv_l, acc[i + 1] * inv_l);
                                val.y = pack_half2(acc[i + 2] * inv_l, acc[i + 3] * inv_l);
                                val.z = pack_half2(acc[i + 4] * inv_l, acc[i + 5] * inv_l);
                                val.w = pack_half2(acc[i + 6] * inv_l, acc[i + 7] * inv_l);
                                *reinterpret_cast<uint4*>(dst + c + i) = val;
                            }
                        }
                    }
                }
                named_bar_sync(1, 256);  // last_flag is rewritten by the next segment
            }
        }
    }
}

}  // namespace b200sd

using namespace b200sd;

// Stream-K pays when whole-tile scheduling leaves a badly filled last wave (320 tiles on 132 CTA slots at S = 4096) or
// too few tiles to fill the GPU; cost model in K/V-tile units with ~2 units of fixed cost per segment.  One CTA per SM.
static int attention_slots(int tiles, int n_kv, int causal, bool have_ws) {
    const int slots = num_sms();
    if (!have_ws || causal || n_kv < 8 || static_cast<size_t>(tiles) * 4 > kCounterBytes) return 0;
    {
        const char* e = getenv("B200SD_ATTN_STREAMK");
        if (e && e[0] == '0') return 0;
    }
    const double cost_tiles = static_cast<double>((tiles + slots - 1) / slots) * (n_kv + 2);
    const double per_slot = static_cast<double>(tiles) * n_kv / slots;
    const double cost_streamk = per_slot + 2 * 2 + 1.5;
    if (per_slot < 0.5 * n_kv || cost_streamk > 0.9 * cost_tiles) return 0;
    return slots;
}

extern "C" size_t b200sd_attention_workspace_bytes(void) {
    return kCounterBytes + static_cast<size_t>(num_sms()) * 2 * kPartialFloats * sizeof(float);
}

extern "C" int b200sd_attention_ws(const void* q, const void* k, const void* v, void* out, const float* mask,
                                   int32_t batch, int32_t heads, int32_t sq, int32_t sk, int32_t d, int32_t ldq,
                                   int32_t ldk, int32_t ldv, int32_t ldo, float scale, int32_t impl, void* workspace,
                                   size_t workspace_bytes, void* stream_) {
    if (!b200sd::launch_class_enabled(2)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(q && k && v && out, "b200sd_attention: null pointer");
    B200SD_REQUIRE(d == kD, "b200sd_attention: head dim %d not supported by this kernel (needs 64)", d);
    B200SD_REQUIRE(impl >= 0 && (impl & 0xff) <= 2 && (impl & ~0x1ff) == 0, "b200sd_attention: unknown attention implementation %d", impl);
    B200SD_REQUIRE(batch > 0 && heads > 0 && sq > 0 && sk > 0, "b200sd_attention: bad sizes");
    B200SD_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
                   "b200sd_attention: leading dimensions must be multiples of 8");
    AttnParams p;
    memset(&p, 0, sizeof(p));
    const uint32_t es[3] = {1, 1, 1};
    const uint32_t box[3] = {kD, 128, 1};
    const void* ptrs[3] = {q, k, v};
    const int lds[3] = {ldq, ldk, ldv};
    const int seqs[3] = {sq, sk, sk};
    CUtensorMap* maps[3] = {&p.tmQ, &p.tmK, &p.tmV};
    for (int i = 0; i < 3; ++i) {
        const uint64_t dims[3] = {static_cast<uint64_t>(heads) * kD, static_cast<uint64_t>(seqs[i]),
                                  static_cast<uint64_t>(batch)};
        const uint64_t str[2] = {static_cast<uint64_t>(lds[i]) * 2, static_cast<uint64_t>(lds[i]) * 2 * seqs[i]};
        if (int rc = encode_tmap_f16(maps[i], ptrs[i], 3, dims, str, box, es)) return rc;
    }
    p.out = reinterpret_cast<__half*>(out);
    p.mask = mask;
    p.sq = sq;
    p.sk = sk;
    p.ldo = ldo;
    p.causal = (impl & 0x100) ? 1 : 0;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.q_tiles = (sq + kQ - 1) / kQ;
    p.heads = heads;
    p.n_kv = (sk + kKV - 1) / kKV;
    const int tiles = p.q_tiles * heads * batch;
    p.total_units = static_cast<long long>(tiles) * p.n_kv;
    const bool have_ws = workspace != nullptr && workspace_bytes >= b200sd_attention_workspace_bytes();
    const int slots = attention_slots(tiles, p.n_kv, p.causal, have_ws);
    p.streamk = slots > 0 ? 1 : 0;
    if (p.streamk) {
        p.counters = reinterpret_cast<int*>(workspace);
        p.ws = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + kCounterBytes);
    }
    static bool attr_set = false;
    if (!attr_set) {
        B200SD_CHECK_CUDA(
            cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmemBytes));
        attr_set = true;
    }
    dim3 grid(p.streamk ? slots : tiles, 1, 1);
    B200SD_CHECK_CUDA(launch_kernel(attention_kernel, dim3(grid), dim3(kAttnThreads), kAttnSmemBytes, stream, p));
    B200SD_CHECK_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
}

extern "C" int b200sd_attention(const void* q, const void* k, const void* v, void* out, const float* mask,
                                int32_t batch, int32_t heads, int32_t sq, int32_t sk, int32_t d, int32_t ldq,
                                int32_t ldk, int32_t ldv, int32_t ldo, float scale, int32_t impl, void* stream_) {
    return b200sd_attention_ws(q, k, v, out, mask, batch, heads, sq, sk, d, ldq, ldk, ldv, ldo, scale, impl, nullptr, 0,
                               stream_);
}
