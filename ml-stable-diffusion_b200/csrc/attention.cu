// b200sd -- flash-style attention for sm_90a: S = Q K^T and O += P V on wgmma tensor cores (fp32 accumulators in
// registers), Q/K/V tiles staged by TMA (SWIZZLE_128B), online softmax (exp2 domain) in registers, P handed to the
// tensor core straight from registers (wgmma with A in registers).
//
// Replaces attention.original / split_einsum / split_einsum_v2 of the reference
// (python_coreml_stable_diffusion/attention.py:24-168, dispatched by Einsum unet.py:45-59): the
// three variants are one function, softmax(q^T k / sqrt(d) + mask) v per (batch, head); the
// (B, heads, Sq, Sk) score tensor the reference materialises (671 MB at S=4096) never leaves the SM.
//
// CTA = 128 queries x 1 head; warps 0..7 are two consumer warpgroups (64 query rows each), warps 8..11 the producer
// warpgroup (warp 8, lane 0 issues TMA; the warpgroup hands most of its registers to the consumers).  K and V tiles of
// KV keys sit in a kKvStages-deep ring with separate full / empty barriers.  Each consumer step j issues S_j = Q K_j^T
// and, behind it, O += P_{j-1} V_{j-1}; the exponentials of S_j run while that PV product is still on the tensor core.
// The two warpgroups issue independently: with the softmax already under the PV product, making them take turns
// (named-barrier ping-pong) measured 2-3 % slower at S = 4096.
//
// Head dims: 64 (SD 2.x, SDXL, CLIP) runs `attention_kernel`; 40, 80 and 160 (SD 1.x: 8 heads of 320 / 640 / 1280
// channels) run `attn_hd_kernel<D>`, the same body.  A row of a tile is ceil(D / 64) 128-byte swizzle atoms, each
// loaded as its own 64-column TMA box; TMA zero-fills the columns >= D, so S takes ceil(D / 16) exact k16 steps and the
// PV product runs 64 / 128 / 192 wide, of which only the D real columns are stored.  D = 160 steps 64 keys at a time:
// three stages of 128 keys would not fit in shared memory.
#include "common.cuh"
#include "../../include/b200sd.h"

namespace b200sd {

extern void count_launch(int n);

static constexpr int kQ = 128;   // queries per CTA
static constexpr int kAttnThreads = 384;
static constexpr int kProducerWarp = 8;
// 128 x kAttnProducerRegs + 256 x kAttnConsumerRegs <= 65536
static constexpr int kAttnProducerRegs = 24;
static constexpr int kAttnConsumerRegs = 240;
static constexpr int kKvStages = 3;
static constexpr int kMergeBar = 1;  // named barrier of the consumers' stream-K merge
static constexpr size_t kCounterBytes = 64 * 1024;

// keys per K/V tile (one TMA load) = keys per pipeline step
template <int D>
struct AttnKeys {
    static constexpr int value = D > 128 ? 64 : 128;
};

// Tile geometry of head dim D with KV keys per step.  smem layout (1024-aligned): Q | K[kKvStages] | V[kKvStages] |
// barriers; a tile is kAtoms column blocks of [rows x 64] fp16 (rows x 128 B), one after the other.
template <int D, int KV>
struct AttnShape {
    static constexpr int kAtoms = (D + 63) / 64;
    static constexpr int kDP = 64 * kAtoms;  // padded head dim: N of the PV product
    static constexpr int kQBytes = kAtoms * kQ * 128;
    static constexpr int kKvBytes = kAtoms * KV * 128;  // one K or V stage
    static constexpr int kSmemQ = 0;
    static constexpr int kSmemK = kSmemQ + kQBytes;
    static constexpr int kSmemV = kSmemK + kKvStages * kKvBytes;
    static constexpr int kSmemBar = kSmemV + kKvStages * kKvBytes;
    static constexpr int kSmemBytes = kSmemBar + 128;
    // one stream-K partial: O [D][128 rows] fp32 (column-major so consecutive rows are contiguous), then m_ref[128], l[128]
    static constexpr int kPartialFloats = (D + 2) * kQ;
    static_assert(kSmemBytes <= 227 * 1024, "attention tiles exceed shared memory");
};

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

// number of K/V tiles a segment visits (>= 1; causal tiles stop at the diagonal)
template <int KV>
__device__ __forceinline__ int segment_steps(const AttnParams& p, const AttnSegment& sg, int q0) {
    const int sk_eff = p.causal ? min(p.sk, q0 + kQ) : p.sk;
    return min(sg.k1, (sk_eff + KV - 1) / KV) - sg.k0;
}

// TMA load of `rows` rows of one head.  D = 64 uses a 3-D map {heads * 64, seq, batch} (a head is one whole box); the
// other head dims a 4-D map {D, heads, seq, batch} and one box {64, 1, rows, 1} per 64-column atom.
template <int D, int KV>
__device__ __forceinline__ void attn_load_rows(uint8_t* dst, const CUtensorMap* map, uint64_t* bar, int head, int row,
                                               int batch, int rows, uint64_t hint) {
    if constexpr (D == 64) {
        tma_load_3d(dst, map, bar, head * D, row, batch, hint);
    } else {
#pragma unroll
        for (int a = 0; a < AttnShape<D, KV>::kAtoms; ++a) tma_load_4d(dst + a * rows * 128, map, bar, 64 * a, head, row, batch, hint);
    }
}

// shared-memory barriers of the pipeline (after the tiles)
struct AttnBars {
    uint64_t *q_full, *q_empty, *k_full, *k_empty, *v_full, *v_empty;
    int* last_flag;
    __device__ __forceinline__ explicit AttnBars(uint8_t* base) {
        uint64_t* bars = reinterpret_cast<uint64_t*>(base);
        q_full = bars + 0;
        q_empty = bars + 1;             // every S MMA of the segment retired: Q may be overwritten
        k_full = bars + 2;              // [kKvStages]
        k_empty = k_full + kKvStages;   // [kKvStages] released once S_j retired
        v_full = k_empty + kKvStages;   // [kKvStages]
        v_empty = v_full + kKvStages;   // [kKvStages] released once P_j V_j retired
        last_flag = reinterpret_cast<int*>(v_empty + kKvStages);
    }
};

// Barrier initialisation and tensor-map prefetch: touches no global memory, so it runs before the kernel's pdl_wait()
// and overlaps the previous kernel's tail.
template <int D, int KV>
__device__ __forceinline__ void attention_prologue(const AttnParams& p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const AttnBars b(smem + AttnShape<D, KV>::kSmemBar);
    if (threadIdx.x == 0) {
        // SWIZZLE_128B tiles need a 1024-byte aligned base; a misaligned launch (never observed: the kernel has no
        // static shared memory) fails loudly instead
        if ((smem_u32(smem) & 1023u) != 0) __trap();
        prefetch_tmap(&p.tmQ);
        prefetch_tmap(&p.tmK);
        prefetch_tmap(&p.tmV);
        mbar_init(b.q_full, 1);
        mbar_init(b.q_empty, 2);
        for (int s = 0; s < kKvStages; ++s) {
            mbar_init(&b.k_full[s], 1);
            mbar_init(&b.v_full[s], 1);
            mbar_init(&b.k_empty[s], 2);  // one arrival per consumer warpgroup
            mbar_init(&b.v_empty[s], 2);
        }
        fence_barrier_init();
    }
    __syncthreads();
}

// Producer and consumer roles; runs after the kernel's pdl_wait().
template <int D, int KV>
__device__ __forceinline__ void attention_body(const AttnParams& p) {
    using Sh = AttnShape<D, KV>;
    constexpr int kNS = KV / 2;        // scores per thread per step
    constexpr int kNO = Sh::kDP / 2;   // O accumulators per thread
    extern __shared__ __align__(1024) uint8_t smem[];
    const AttnBars b(smem + Sh::kSmemBar);
    uint64_t* const q_full = b.q_full;
    uint64_t* const q_empty = b.q_empty;
    uint64_t* const k_full = b.k_full;
    uint64_t* const k_empty = b.k_empty;
    uint64_t* const v_full = b.v_full;
    uint64_t* const v_empty = b.v_empty;
    int* const last_flag = b.last_flag;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // Both roles walk the same segment list.  The K/V tile counter jg runs ACROSS segments (smem stage jg % kKvStages).
    SegmentWalk walk;
    walk.init(p);
    AttnSegment sg;

    if (warp >= kProducerWarp) {
        setmaxnreg_dec<kAttnProducerRegs>();
        if (warp == kProducerWarp && lane == 0) {
            int seg = 0, jg = 0;
            while (walk.next(p, sg)) {
                const int qt = sg.tile % p.q_tiles, head = (sg.tile / p.q_tiles) % p.heads, batch = sg.tile / (p.q_tiles * p.heads);
                const int ns = segment_steps<KV>(p, sg, qt * kQ);
                if (seg > 0) mbar_wait(q_empty, (seg - 1) & 1);
                mbar_expect_tx(q_full, Sh::kQBytes);
                attn_load_rows<D, KV>(smem + Sh::kSmemQ, &p.tmQ, q_full, head, qt * kQ, batch, kQ, kEvictFirst);
                for (int jl = 0; jl < ns; ++jl, ++jg) {
                    const int st = jg % kKvStages;
                    const uint32_t ph = (jg / kKvStages) & 1;
                    mbar_wait(&k_empty[st], ph ^ 1);
                    mbar_expect_tx(&k_full[st], Sh::kKvBytes);
                    attn_load_rows<D, KV>(smem + Sh::kSmemK + st * Sh::kKvBytes, &p.tmK, &k_full[st], head, (sg.k0 + jl) * KV,
                                          batch, KV, kEvictLast);
                    mbar_wait(&v_empty[st], ph ^ 1);
                    mbar_expect_tx(&v_full[st], Sh::kKvBytes);
                    attn_load_rows<D, KV>(smem + Sh::kSmemV + st * Sh::kKvBytes, &p.tmV, &v_full[st], head, (sg.k0 + jl) * KV,
                                          batch, KV, kEvictLast);
                }
                ++seg;
            }
        }
    } else {
        // ---------------- consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile ----------------
        setmaxnreg_inc<kAttnConsumerRegs>();
        // Accumulator layout (m64nN): this thread holds rows lr and lr + 8 (lr = 16 (warp % 4) + lane / 4 inside the
        // warpgroup's 64), columns 8 j + 2 (lane % 4) + {0, 1}: x[4 j + {0, 1}] row lr, x[4 j + {2, 3}] row lr + 8.
        // A row is spread over the four lanes of a quad: row maxima / sums reduce with two shuffles.
        const int wg = warp >> 2;
        const int lr = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // tile-local row of x[.. 0, 1]; lr + 8 for x[.. 2, 3]
        const int cq = 2 * (lane & 3);
        const bool leader = (threadIdx.x & 127) == 0;
        const float sl2 = p.scale_log2;
        const uint32_t q_addr = smem_u32(smem + Sh::kSmemQ) + wg * 64 * 128;
        const uint64_t qdesc = make_smem_desc_sw128(q_addr, 1024, 0);

        int seg = 0, jg0 = 0;
        while (walk.next(p, sg)) {
            const int qt = sg.tile % p.q_tiles, head = (sg.tile / p.q_tiles) % p.heads, batch = sg.tile / (p.q_tiles * p.heads);
            const int q0 = qt * kQ;
            const int ns = segment_steps<KV>(p, sg, q0);
            const float* mask_row = p.mask ? p.mask + static_cast<size_t>(batch) * p.sk : nullptr;
            float o[kNO];
#pragma unroll
            for (int i = 0; i < kNO; ++i) o[i] = 0.f;
            float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
            float s[kNS];            // S_j, then its probabilities (fp32)
            uint32_t pa[KV / 16][4];  // P_{j-1} as fp16 A fragments: pa[kk] covers keys [16 kk, 16 kk + 16)
            float factor[2];         // rescale of O for S_j's new row maxima, applied once P_{j-1} V_{j-1} retired

            // k16 step k reads columns [16 k, 16 k + 16): 32 B into atom k / 4 (descriptor units of 16 B)
            auto issue_s = [&](int st) {
                const uint64_t kdesc = make_smem_desc_sw128(smem_u32(smem + Sh::kSmemK + st * Sh::kKvBytes), 1024, 0);
#pragma unroll
                for (int k = 0; k < (D + 15) / 16; ++k)
                    wgmma_ss<KV>(s, qdesc + (k / 4) * (kQ * 128 / 16) + 2 * (k % 4), kdesc + (k / 4) * (KV * 128 / 16) + 2 * (k % 4),
                                 k > 0 ? 1u : 0u);
                wgmma_commit();
            };
            // B = the V tile [keys][d] = MN-major, 16 keys = 2048 B per k16 step, 64-column atoms KV * 128 B apart
            auto issue_pv = [&](int st) {
                const uint32_t v_addr = smem_u32(smem + Sh::kSmemV + st * Sh::kKvBytes);
#pragma unroll
                for (int kk = 0; kk < KV / 16; ++kk)
                    wgmma_rs_tb<Sh::kDP>(o, pa[kk], make_smem_desc_sw128(v_addr + kk * 2048, 1024, KV * 128), 1u);
                wgmma_commit();
            };
            // online softmax (log2 domain) of S_j in place; touches neither o nor pa (P_{j-1} V_{j-1} may be in flight).
            // The fast path leaves raw scores in s and folds the scale into the exponent's FFMA; the general path stores
            // scaled scores (mask added, invisible keys at -inf).  Called as `if (general) softmax(j, true); else
            // softmax(j, false);` so that each variant is a block of its own: ptxas hoists a wgmma wait to the top of
            // the basic block it sits in, and a wait<0> in the same block as the exponentials would run them after the
            // PV product instead of under it.
            auto softmax = [&](int j, bool general) {
                const int h = sg.k0 + j;                    // this K/V tile's position among the keys
                const int kvalid = min(KV, p.sk - h * KV);  // >= 1
                // causal: a tile whose last key is <= the tile's first query is fully visible to every row
                const bool diag = p.causal && (h * KV + KV - 1 > q0);
                const float sc = general ? 1.f : sl2;
                if (general) {
#pragma unroll
                    for (int e = 0; e < kNS; ++e) {
                        const int key = 8 * (e >> 2) + cq + (e & 1);
                        const int qi = q0 + lr + 8 * ((e >> 1) & 1);
                        const bool vis = key < kvalid && (!diag || h * KV + key <= qi);
                        float v = s[e] * sl2;
                        if (mask_row != nullptr && vis) v += mask_row[h * KV + key] * 1.4426950408889634f;
                        s[e] = vis ? v : -INFINITY;
                    }
                }
                // row maxima and sums as trees of KV / 16 partials: with two consumer warps per scheduler there is
                // little to hide a long dependency chain behind
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    float t[KV / 16];
#pragma unroll
                    for (int c = 0; c < KV / 16; ++c)
                        t[c] = fmaxf(fmaxf(s[8 * c + 2 * r], s[8 * c + 2 * r + 1]), fmaxf(s[8 * c + 4 + 2 * r], s[8 * c + 5 + 2 * r]));
#pragma unroll
                    for (int w = KV / 32; w >= 1; w >>= 1)
#pragma unroll
                        for (int c = 0; c < w; ++c) t[c] = fmaxf(t[c], t[c + w]);
                    float mx = t[0];
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    const float m_new = fmaxf(m_run[r], mx * sc);
                    const float m_use = m_new == -INFINITY ? 0.f : m_new;  // a row with nothing visible yet
                    factor[r] = ex2_approx(m_run[r] - m_use);
                    m_run[r] = m_new;
#pragma unroll
                    for (int c = 0; c < KV / 8; ++c) {
                        s[4 * c + 2 * r] = ex2_approx(fmaf(s[4 * c + 2 * r], sc, -m_use));
                        s[4 * c + 2 * r + 1] = ex2_approx(fmaf(s[4 * c + 2 * r + 1], sc, -m_use));
                    }
#pragma unroll
                    for (int c = 0; c < KV / 16; ++c) t[c] = (s[8 * c + 2 * r] + s[8 * c + 2 * r + 1]) + (s[8 * c + 4 + 2 * r] + s[8 * c + 5 + 2 * r]);
#pragma unroll
                    for (int w = KV / 32; w >= 1; w >>= 1)
#pragma unroll
                        for (int c = 0; c < w; ++c) t[c] += t[c + w];
                    l_run[r] = fmaf(l_run[r], factor[r], t[0]);
                }
            };
            auto is_general = [&](int j) {
                const int h = sg.k0 + j;
                return mask_row != nullptr || p.sk - h * KV < KV || (p.causal && h * KV + KV - 1 > q0);
            };
            // once P_{j-1} V_{j-1} retired: rescale O, and S_j's probabilities become the next A operand
            auto rescale_and_pack = [&]() {
#pragma unroll
                for (int c = 0; c < kNO / 4; ++c) {
                    o[4 * c] *= factor[0], o[4 * c + 1] *= factor[0];
                    o[4 * c + 2] *= factor[1], o[4 * c + 3] *= factor[1];
                }
                // A fragment of keys [16 kk, 16 kk + 16): {row lr, keys 0..7}, {lr + 8, 0..7}, {lr, 8..15}, {lr + 8, 8..15}
#pragma unroll
                for (int c = 0; c < KV / 8; ++c) {
                    pa[c >> 1][2 * (c & 1)] = pack_half2(s[4 * c], s[4 * c + 1]);
                    pa[c >> 1][2 * (c & 1) + 1] = pack_half2(s[4 * c + 2], s[4 * c + 3]);
                }
            };

            mbar_wait(q_full, seg & 1);
            // ---- step 0: S_0 alone ----
            {
                const int st = jg0 % kKvStages;
                mbar_wait(&k_full[st], (jg0 / kKvStages) & 1);
                wgmma_fence();
                issue_s(st);
                wgmma_wait<0>();
                wgmma_fence_regs<kNS>(s);
                if (leader) {
                    mbar_arrive(&k_empty[st]);
                    if (ns == 1) mbar_arrive(q_empty);  // the segment's last read of Q retired
                }
                if (is_general(0)) softmax(0, true);
                else softmax(0, false);
                rescale_and_pack();
            }
            // ---- steps 1..ns-1: S_j and P_{j-1} V_{j-1} in one burst; softmax(S_j) overlaps the PV product ----
            for (int j = 1; j < ns; ++j) {
                const int jg = jg0 + j, st = jg % kKvStages, sp = (jg - 1) % kKvStages;
                mbar_wait(&k_full[st], (jg / kKvStages) & 1);
                mbar_wait(&v_full[sp], ((jg - 1) / kKvStages) & 1);
                wgmma_fence();
                issue_s(st);
                issue_pv(sp);
                wgmma_wait<1>();  // S_j retired; P_{j-1} V_{j-1} may still run
                wgmma_fence_regs<kNS>(s);
                if (leader) {
                    mbar_arrive(&k_empty[st]);
                    if (j == ns - 1) mbar_arrive(q_empty);
                }
                if (is_general(j)) softmax(j, true);
                else softmax(j, false);
                wgmma_wait<0>();
                wgmma_fence_regs<kNO>(o);
                wgmma_fence_regs<kNS>(s);  // keeps the repacking of P behind the wait: P_{j-1} V_{j-1} reads pa
                if (leader) mbar_arrive(&v_empty[sp]);
                rescale_and_pack();
            }
            // ---- last PV ----
            {
                const int jg = jg0 + ns - 1, st = jg % kKvStages;
                mbar_wait(&v_full[st], (jg / kKvStages) & 1);
                wgmma_fence();
                issue_pv(st);
                wgmma_wait<0>();
                wgmma_fence_regs<kNO>(o);
                if (leader) mbar_arrive(&v_empty[st]);
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
                l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
            }
            ++seg, jg0 += ns;
            if (sg.k0 == 0 && sg.k1 == p.n_kv) {
                // whole query tile in this CTA: normalise and store the D real columns
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int qi = q0 + lr + 8 * r;
                    if (qi >= p.sq) continue;
                    const float inv_l = 1.0f / l_run[r];
                    __half* dst = p.out + (static_cast<size_t>(batch) * p.sq + qi) * p.ldo + head * D;
#pragma unroll
                    for (int j = 0; j < D / 8; ++j)
                        *reinterpret_cast<uint32_t*>(dst + 8 * j + cq) = pack_half2(o[4 * j + 2 * r] * inv_l, o[4 * j + 2 * r + 1] * inv_l);
                }
            } else {
                // ---- a piece of a split tile: park (O, m_ref, l) in the workspace; the piece that finishes last merges
                // ALL pieces (its own included) in slot order, so the result does not depend on who was last ----
                const long long t0 = static_cast<long long>(sg.tile) * p.n_kv;
                const int first = slot_of(p, t0), last = slot_of(p, t0 + p.n_kv - 1);
                float* mine = p.ws + (static_cast<size_t>(blockIdx.x) * 2 + (sg.k0 > 0 ? 1 : 0)) * Sh::kPartialFloats;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int row = lr + 8 * r;
#pragma unroll
                    for (int j = 0; j < D / 8; ++j) {
                        __stcg(mine + (8 * j + cq) * kQ + row, o[4 * j + 2 * r]);
                        __stcg(mine + (8 * j + cq + 1) * kQ + row, o[4 * j + 2 * r + 1]);
                    }
                    if ((lane & 3) == 0) {
                        __stcg(mine + D * kQ + row, m_run[r]);
                        __stcg(mine + (D + 1) * kQ + row, l_run[r]);
                    }
                }
                __threadfence();
                named_bar_sync(kMergeBar, 256);
                if (threadIdx.x == 0) {
                    const int old = atomicAdd(p.counters + sg.tile, 1);
                    const int is_last = old == last - first;
                    if (is_last) p.counters[sg.tile] = 0;  // every piece has checked in: ready for the next launch
                    *last_flag = is_last;
                }
                named_bar_sync(kMergeBar, 256);
                if (*last_flag) {
                    __threadfence();
                    // merge: thread t takes row t % 128 and, in passes of kC columns, head-dim columns [0, kHalf)
                    // (t < 128) or [kHalf, D)
                    constexpr int kC = D % 16 == 0 ? 16 : 8;
                    constexpr int kHalf = kC * ((D / kC + 1) / 2);
                    const int row = threadIdx.x & 127;
                    const int cbase = kHalf * (threadIdx.x >> 7);
                    const int cend = 2 * kHalf == D ? cbase + kHalf : min(D, cbase + kHalf);
                    const bool store = q0 + row < p.sq;
                    __half* dst = p.out + (static_cast<size_t>(batch) * p.sq + (store ? q0 + row : 0)) * p.ldo + head * D;
                    float m = -INFINITY;
                    for (int s2 = first; s2 <= last; ++s2) {
                        const float* part = p.ws + (static_cast<size_t>(s2) * 2 + (slot_begin(p, s2) > t0 ? 1 : 0)) * Sh::kPartialFloats;
                        m = fmaxf(m, __ldcg(part + D * kQ + row));
                    }
                    float l = 0.f;
                    for (int s2 = first; s2 <= last; ++s2) {
                        const float* part = p.ws + (static_cast<size_t>(s2) * 2 + (slot_begin(p, s2) > t0 ? 1 : 0)) * Sh::kPartialFloats;
                        l += __ldcg(part + (D + 1) * kQ + row) * ex2_approx(__ldcg(part + D * kQ + row) - m);
                    }
                    const float inv_l = 1.0f / l;
#pragma unroll 1
                    for (int c = cbase; c < cend; c += kC) {
                        float acc[kC];
#pragma unroll
                        for (int i = 0; i < kC; ++i) acc[i] = 0.f;
                        for (int s2 = first; s2 <= last; ++s2) {
                            const float* part =
                                p.ws + (static_cast<size_t>(s2) * 2 + (slot_begin(p, s2) > t0 ? 1 : 0)) * Sh::kPartialFloats;
                            const float f = ex2_approx(__ldcg(part + D * kQ + row) - m);
#pragma unroll
                            for (int i = 0; i < kC; ++i) acc[i] = fmaf(__ldcg(part + (c + i) * kQ + row), f, acc[i]);
                        }
                        if (store) {
#pragma unroll
                            for (int i = 0; i < kC; i += 8) {
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
                named_bar_sync(kMergeBar, 256);  // last_flag is rewritten by the next segment
            }
        }
    }
}

// head dim 64
__global__ void __launch_bounds__(kAttnThreads, 1) attention_kernel(const __grid_constant__ AttnParams p) {
    attention_prologue<64, 128>(p);
    pdl_trigger();
    pdl_wait();  // PDL: the prologue above overlapped the previous kernel's tail
    attention_body<64, 128>(p);
}

// head dims 40, 80, 160
template <int D>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_hd_kernel(const __grid_constant__ AttnParams p) {
    attention_prologue<D, AttnKeys<D>::value>(p);
    pdl_trigger();
    pdl_wait();  // PDL: the prologue above overlapped the previous kernel's tail
    attention_body<D, AttnKeys<D>::value>(p);
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

static bool attention_head_dim_supported(int d) { return d == 40 || d == 64 || d == 80 || d == 160; }

extern "C" size_t b200sd_attention_workspace_bytes_for(int32_t d) {
    if (!attention_head_dim_supported(d)) return 0;
    return kCounterBytes + static_cast<size_t>(num_sms()) * 2 * (d + 2) * kQ * sizeof(float);
}

extern "C" size_t b200sd_attention_workspace_bytes(void) { return b200sd_attention_workspace_bytes_for(64); }

// Sets the kernel's shared-memory limit on first use, then launches it.
template <int D, int KV>
static int attention_launch(void (*kernel)(AttnParams), int grid, cudaStream_t stream, const AttnParams& p) {
    constexpr int smem_bytes = AttnShape<D, KV>::kSmemBytes;
    static bool attr_set = false;
    if (!attr_set) {
        B200SD_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set = true;
    }
    B200SD_CHECK_CUDA(launch_kernel(kernel, dim3(grid), dim3(kAttnThreads), smem_bytes, stream, p));
    return 0;
}

extern "C" int b200sd_attention_ws(const void* q, const void* k, const void* v, void* out, const float* mask,
                                   int32_t batch, int32_t heads, int32_t sq, int32_t sk, int32_t d, int32_t ldq,
                                   int32_t ldk, int32_t ldv, int32_t ldo, float scale, int32_t impl, void* workspace,
                                   size_t workspace_bytes, void* stream_) {
    if (!b200sd::launch_class_enabled(2)) return 0;  // bench.py's per-class timing graphs
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    B200SD_REQUIRE(q && k && v && out, "b200sd_attention: null pointer");
    B200SD_REQUIRE(attention_head_dim_supported(d), "b200sd_attention: head dim %d not supported (40, 64, 80 or 160)", d);
    B200SD_REQUIRE(impl >= 0 && (impl & 0xff) <= 2 && (impl & ~0x1ff) == 0, "b200sd_attention: unknown attention implementation %d", impl);
    B200SD_REQUIRE(batch > 0 && heads > 0 && sq > 0 && sk > 0, "b200sd_attention: bad sizes");
    // the softmax takes row maxima of the unscaled scores and scales them afterwards: only valid for a positive scale
    B200SD_REQUIRE(scale > 0.f, "b200sd_attention: scale must be > 0 (got %g)", static_cast<double>(scale));
    B200SD_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
                   "b200sd_attention: leading dimensions must be multiples of 8");
    const int kv = d == 160 ? AttnKeys<160>::value : AttnKeys<64>::value;
    AttnParams p;
    memset(&p, 0, sizeof(p));
    const void* ptrs[3] = {q, k, v};
    const int lds[3] = {ldq, ldk, ldv};
    const int seqs[3] = {sq, sk, sk};
    CUtensorMap* maps[3] = {&p.tmQ, &p.tmK, &p.tmV};
    for (int i = 0; i < 3; ++i) {
        const uint64_t row_bytes = static_cast<uint64_t>(lds[i]) * 2;
        if (d == 64) {
            const uint32_t es[3] = {1, 1, 1};
            const uint32_t box[3] = {64, 128, 1};
            const uint64_t dims[3] = {static_cast<uint64_t>(heads) * 64, static_cast<uint64_t>(seqs[i]),
                                      static_cast<uint64_t>(batch)};
            const uint64_t str[2] = {row_bytes, row_bytes * seqs[i]};
            if (int rc = encode_tmap_f16(maps[i], ptrs[i], 3, dims, str, box, es)) return rc;
        } else {
            // {d, heads, seq, batch}: a 64-column box reaches past d and TMA fills those columns with zeros
            const uint32_t es[4] = {1, 1, 1, 1};
            const uint32_t box[4] = {64, 1, static_cast<uint32_t>(i == 0 ? kQ : kv), 1};
            const uint64_t dims[4] = {static_cast<uint64_t>(d), static_cast<uint64_t>(heads), static_cast<uint64_t>(seqs[i]),
                                      static_cast<uint64_t>(batch)};
            const uint64_t str[3] = {static_cast<uint64_t>(d) * 2, row_bytes, row_bytes * seqs[i]};
            if (int rc = encode_tmap_f16(maps[i], ptrs[i], 4, dims, str, box, es)) return rc;
        }
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
    p.n_kv = (sk + kv - 1) / kv;
    const int tiles = p.q_tiles * heads * batch;
    p.total_units = static_cast<long long>(tiles) * p.n_kv;
    const bool have_ws = workspace != nullptr && workspace_bytes >= b200sd_attention_workspace_bytes_for(d);
    const int slots = attention_slots(tiles, p.n_kv, p.causal, have_ws);
    p.streamk = slots > 0 ? 1 : 0;
    if (p.streamk) {
        p.counters = reinterpret_cast<int*>(workspace);
        p.ws = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + kCounterBytes);
    }
    const int grid = p.streamk ? slots : tiles;
    int rc = 0;
    switch (d) {
        case 64: rc = attention_launch<64, 128>(attention_kernel, grid, stream, p); break;
        case 40: rc = attention_launch<40, AttnKeys<40>::value>(attn_hd_kernel<40>, grid, stream, p); break;
        case 80: rc = attention_launch<80, AttnKeys<80>::value>(attn_hd_kernel<80>, grid, stream, p); break;
        default: rc = attention_launch<160, AttnKeys<160>::value>(attn_hd_kernel<160>, grid, stream, p); break;
    }
    if (rc) return rc;
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
