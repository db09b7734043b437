// b200sd -- model-level C-ABI: an opaque UNet handle that owns its packed weights, activation arena, statistics
// buffers and launch sequence (include/b200sd.h: b200sd_unet_create / _prepare_prompt / _forward / b200sd_destroy).
//
// What the reference's other front end binds per model is one "predict" (swift/StableDiffusion/pipeline/Unet.swift:90-144,
// python_coreml_stable_diffusion/coreml_model.py:118-120); this file is that granularity for a C / Swift host: weights
// in the reference's own parameter names and layouts (diffusers UNet2DConditionModel state dict, unet.py:121-146) go in
// once, device pointers go in per call.  The launch sequence is the fused graph of ml-stable-diffusion_b200/unet.py
// (GroupNorm + SiLU inside the halo convolution's operand path, LayerNorm folded into the consumer GEMM, statistics from
// the producers' epilogues) issued through the same entry points the Python host uses.
#include "common.cuh"
#include "../../include/b200sd.h"

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

namespace b200sd {
namespace {

#define MODEL_TRY(expr)                \
    do {                               \
        if (int _rc = (expr)) return _rc; \
    } while (0)

__global__ void add_f32_kernel(float* __restrict__ a, const float* __restrict__ b, int n) {
    pdl_trigger();  // no large shared memory here: dependents may start their prologue at once
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] += b[i];
}

struct HostTensor {
    std::vector<float> v;
    std::vector<int64_t> shape;
    int64_t numel() const {
        int64_t n = 1;
        for (auto s : shape) n *= s;
        return n;
    }
};

// one GEMM "B" operand: [n][taps * (c0 + c1)] fp16 on the host until its call site's tiling is known
struct Mat {
    int n = 0, k = 0;
    std::vector<__half> host;
    std::map<std::pair<int, int>, void*> tiled;  // (block_n, chunk_major) -> device copy
};

struct Act {  // NHWC fp16 activation + the per-channel sums its producer left behind (or null)
    __half* p = nullptr;
    int n = 0, h = 0, w = 0, c = 0;
    float* chan = nullptr;
    int rows() const { return n * h * w; }
};

struct RowStats {
    float* rows = nullptr;
    int parts = 0;
};

struct GnSpec {
    const float* chan0;
    const float* chan1;
    const float* gamma;
    const float* beta;
    int groups;
    float eps;
    int silu;
};

class UNet {
public:
    b200sd_unet_config cfg;
    int nb = 0, B = 0, H = 0, W = 0, S = 0, in_pad = 8, temb_total = 0, kv_total = 0;
    bool xl = false;
    cudaStream_t st = nullptr;
    std::unordered_map<std::string, HostTensor> hw;                 // host weights (released after the first forward)
    std::unordered_map<std::string, std::unique_ptr<Mat>> mats;     // GEMM operands
    std::unordered_map<std::string, float*> vecs;                   // fp32 device vectors
    std::unordered_map<std::string, __half*> small_w;               // untiled fp16 [n][k] (small-M linears)
    std::unordered_map<std::string, int> temb_off, kv_off;
    std::vector<void*> owned;                                       // every cudaMalloc of this handle
    // activation arena: per-tensor cudaMalloc during the first (sizing) forward, one bump arena afterwards
    bool bump = false;
    char* arena = nullptr;
    size_t arena_cap = 0, arena_off = 0, sized = 0;
    std::vector<void*> warm_allocs;
    float* scratch = nullptr;  // split-K / statistics partials
    size_t scratch_bytes = 0;
    unsigned int* tickets = nullptr;
    void* attn_ws = nullptr;                                        // b200sd_attention_ws workspace (zeroed once)
    size_t attn_ws_bytes = 0;
    __half* kv_all = nullptr;
    bool kv_ready = false;
    int attn_impl = 1;
    // GroupNorm fusion (B200SD_FUSED=1 at create time): GroupNorm + SiLU inside the halo convolution's operand path with
    // statistics from the producers' epilogues.  Default off, like the Python host (the one-launch cluster GroupNorm in
    // front of the 9-tap TMA convolution is the default path); LayerNorm is always folded into its consumer GEMM.
    bool fuse_gn = false;

    ~UNet() {
        for (void* p : warm_allocs) cudaFree(p);
        for (void* p : owned) cudaFree(p);
        if (arena) cudaFree(arena);
    }

    // ------------------------------------------------------------------ memory
    int dev_alloc(void** out, size_t bytes) {
        B200SD_CHECK_CUDA(cudaMalloc(out, std::max<size_t>(bytes, 16)));
        owned.push_back(*out);
        return 0;
    }
    int act_alloc(void** out, size_t bytes) {
        bytes = (bytes + 255) & ~size_t(255);
        if (bump) {
            B200SD_REQUIRE(arena_off + bytes <= arena_cap, "b200sd_unet: activation arena exhausted");
            *out = arena + arena_off;
            arena_off += bytes;
            return 0;
        }
        B200SD_CHECK_CUDA(cudaMalloc(out, bytes));
        warm_allocs.push_back(*out);
        sized += bytes;
        return 0;
    }
    int upload_f32(const std::string& name, const std::vector<float>& v) {
        void* d;
        MODEL_TRY(dev_alloc(&d, v.size() * 4));
        B200SD_CHECK_CUDA(cudaMemcpy(d, v.data(), v.size() * 4, cudaMemcpyHostToDevice));
        vecs[name] = static_cast<float*>(d);
        return 0;
    }

    // ------------------------------------------------------------------ weights
    const HostTensor* find(const std::string& k) const {
        auto it = hw.find(k);
        return it == hw.end() ? nullptr : &it->second;
    }
    int need(const std::string& k, const HostTensor** t) const {
        *t = find(k);
        B200SD_REQUIRE(*t != nullptr, "b200sd_unet_create: parameter %s missing", k.c_str());
        return 0;
    }
    // [Co, Ci, 3, 3] -> [Co][9][Ci_pad] (OHWI, k = (ky * 3 + kx) * C + c)
    int conv3(const std::string& key, Mat& m, int pad_in = 0) const {
        const HostTensor* t;
        MODEL_TRY(need(key + ".weight", &t));
        B200SD_REQUIRE(t->shape.size() == 4 && t->shape[2] == 3 && t->shape[3] == 3, "%s is not a 3x3 kernel", key.c_str());
        const int co = static_cast<int>(t->shape[0]), ci = static_cast<int>(t->shape[1]);
        const int cp = std::max(ci, pad_in);
        m.n = co, m.k = 9 * cp;
        m.host.assign(static_cast<size_t>(co) * 9 * cp, __float2half(0.f));
        for (int o = 0; o < co; ++o)
            for (int c = 0; c < ci; ++c)
                for (int tap = 0; tap < 9; ++tap)
                    m.host[(static_cast<size_t>(o) * 9 + tap) * cp + c] = __float2half(t->v[(static_cast<size_t>(o) * ci + c) * 9 + tap]);
        return 0;
    }
    int lin_f32(const std::string& key, std::vector<float>& out, int& n, int& k) const {
        const HostTensor* t;
        MODEL_TRY(need(key + ".weight", &t));
        B200SD_REQUIRE(t->shape.size() == 2 || (t->shape.size() == 4 && t->shape[2] == 1 && t->shape[3] == 1),
                       "%s is not a linear / 1x1 weight", key.c_str());
        n = static_cast<int>(t->shape[0]), k = static_cast<int>(t->shape[1]);
        out = t->v;
        return 0;
    }
    static void to_mat(const std::vector<float>& w, int n, int k, Mat& m) {
        m.n = n, m.k = k;
        m.host.resize(w.size());
        for (size_t i = 0; i < w.size(); ++i) m.host[i] = __float2half(w[i]);
    }
    int add_lin(const std::string& name, const std::string& key) {
        std::vector<float> w;
        int n, k;
        MODEL_TRY(lin_f32(key, w, n, k));
        auto m = std::make_unique<Mat>();
        to_mat(w, n, k, *m);
        mats[name] = std::move(m);
        return 0;
    }
    int add_bias(const std::string& name, const std::string& key) {
        const HostTensor* t = find(key + ".bias");
        if (t) MODEL_TRY(upload_f32(name, t->v));
        return 0;
    }
    int add_vec(const std::string& name, const std::string& key) {
        const HostTensor* t;
        MODEL_TRY(need(key, &t));
        return upload_f32(name, t->v);
    }
    int small(const std::string& name, const std::vector<float>& w) {
        std::vector<__half> h(w.size());
        for (size_t i = 0; i < w.size(); ++i) h[i] = __float2half(w[i]);
        void* d;
        MODEL_TRY(dev_alloc(&d, h.size() * 2));
        B200SD_CHECK_CUDA(cudaMemcpy(d, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
        small_w[name] = static_cast<__half*>(d);
        return 0;
    }

    std::vector<float> temb_w_all, temb_b_all;
    std::vector<__half> kv_w_all;
    int kv_k = 0;

    int pack_resnet(const std::string& p) {
        MODEL_TRY(add_vec(p + ".n1g", p + ".norm1.weight"));
        MODEL_TRY(add_vec(p + ".n1b", p + ".norm1.bias"));
        MODEL_TRY(add_vec(p + ".n2g", p + ".norm2.weight"));
        MODEL_TRY(add_vec(p + ".n2b", p + ".norm2.bias"));
        auto c1 = std::make_unique<Mat>();
        auto c2 = std::make_unique<Mat>();
        MODEL_TRY(conv3(p + ".conv1", *c1));
        MODEL_TRY(conv3(p + ".conv2", *c2));
        const int co = c1->n;
        mats[p + ".c1"] = std::move(c1);
        mats[p + ".c2"] = std::move(c2);
        MODEL_TRY(add_bias(p + ".c2b", p + ".conv2"));
        // time_emb_proj rows of all ResNets concatenated, conv1's bias folded in (unet.py:442, 476-478)
        std::vector<float> tw;
        int n, k;
        MODEL_TRY(lin_f32(p + ".time_emb_proj", tw, n, k));
        const HostTensor *tb, *cb;
        MODEL_TRY(need(p + ".time_emb_proj.bias", &tb));
        MODEL_TRY(need(p + ".conv1.bias", &cb));
        temb_off[p] = temb_total;
        temb_total += co;
        temb_w_all.insert(temb_w_all.end(), tw.begin(), tw.end());
        for (int i = 0; i < co; ++i) temb_b_all.push_back(tb->v[i] + cb->v[i]);
        if (find(p + ".conv_shortcut.weight")) {
            MODEL_TRY(add_lin(p + ".sc", p + ".conv_shortcut"));
            MODEL_TRY(add_bias(p + ".scb", p + ".conv_shortcut"));
            if (!fuse_gn) {
                // the shortcut folded into conv2 (like unet.py of this package): rows [conv2 (9 * Cout) | shortcut (Cin)],
                // one bias vector for both
                const Mat& c2 = *mats.at(p + ".c2");
                const Mat& sc = *mats.at(p + ".sc");
                auto m = std::make_unique<Mat>();
                m->n = c2.n, m->k = c2.k + sc.k;
                m->host.resize(static_cast<size_t>(m->n) * m->k);
                for (int r = 0; r < m->n; ++r) {
                    std::copy(c2.host.begin() + static_cast<size_t>(r) * c2.k, c2.host.begin() + static_cast<size_t>(r + 1) * c2.k,
                              m->host.begin() + static_cast<size_t>(r) * m->k);
                    std::copy(sc.host.begin() + static_cast<size_t>(r) * sc.k, sc.host.begin() + static_cast<size_t>(r + 1) * sc.k,
                              m->host.begin() + static_cast<size_t>(r) * m->k + c2.k);
                }
                mats[p + ".c2sc"] = std::move(m);
                const HostTensor *b2, *bs;
                MODEL_TRY(need(p + ".conv2.bias", &b2));
                MODEL_TRY(need(p + ".conv_shortcut.bias", &bs));
                std::vector<float> b(b2->v.size());
                for (size_t i = 0; i < b.size(); ++i) b[i] = b2->v[i] + bs->v[i];
                MODEL_TRY(upload_f32(p + ".c2scb", b));
            }
        }
        return 0;
    }

    // LayerNorm folded into the consumer: W' = gamma (.) W (fp16), wg = row sums of the ROUNDED W', bias' = W beta + bias
    int fold_ln(const std::string& name, const std::vector<float>& w, int n, int k, const std::vector<float>& gamma,
                const std::vector<float>& beta, const std::vector<float>* bias) {
        auto m = std::make_unique<Mat>();
        m->n = n, m->k = k;
        m->host.resize(w.size());
        std::vector<float> wg(n), wb(n);
        for (int r = 0; r < n; ++r) {
            float sg = 0.f, sb = 0.f;
            for (int c = 0; c < k; ++c) {
                const float wv = __half2float(__float2half(w[static_cast<size_t>(r) * k + c]));  // the packer's fp16 weight
                const __half f = __float2half(wv * gamma[c]);
                m->host[static_cast<size_t>(r) * k + c] = f;
                sg += __half2float(f);
                sb += wv * beta[c];
            }
            wg[r] = sg;
            wb[r] = sb + (bias ? (*bias)[r] : 0.f);
        }
        mats[name] = std::move(m);
        MODEL_TRY(upload_f32(name + ".wg", wg));
        MODEL_TRY(upload_f32(name + ".b", wb));
        return 0;
    }

    int pack_transformer(const std::string& p, int c, int depth) {
        MODEL_TRY(add_vec(p + ".ng", p + ".norm.weight"));
        MODEL_TRY(add_vec(p + ".nb", p + ".norm.bias"));
        MODEL_TRY(add_lin(p + ".pi", p + ".proj_in"));
        MODEL_TRY(add_bias(p + ".pib", p + ".proj_in"));
        MODEL_TRY(add_lin(p + ".po", p + ".proj_out"));
        MODEL_TRY(add_bias(p + ".pob", p + ".proj_out"));
        for (int d = 0; d < depth; ++d) {
            const std::string b = p + ".transformer_blocks." + std::to_string(d);
            const HostTensor *g1, *b1, *g2, *b2, *g3, *b3;
            MODEL_TRY(need(b + ".norm1.weight", &g1));
            MODEL_TRY(need(b + ".norm1.bias", &b1));
            MODEL_TRY(need(b + ".norm2.weight", &g2));
            MODEL_TRY(need(b + ".norm2.bias", &b2));
            MODEL_TRY(need(b + ".norm3.weight", &g3));
            MODEL_TRY(need(b + ".norm3.bias", &b3));
            std::vector<float> q, k, v, qkv;
            int n, kk;
            MODEL_TRY(lin_f32(b + ".attn1.to_q", q, n, kk));
            MODEL_TRY(lin_f32(b + ".attn1.to_k", k, n, kk));
            MODEL_TRY(lin_f32(b + ".attn1.to_v", v, n, kk));
            qkv = q;
            qkv.insert(qkv.end(), k.begin(), k.end());
            qkv.insert(qkv.end(), v.begin(), v.end());
            MODEL_TRY(fold_ln(b + ".qkv", qkv, 3 * c, c, g1->v, b1->v, nullptr));
            MODEL_TRY(add_lin(b + ".o1", b + ".attn1.to_out.0"));
            MODEL_TRY(add_bias(b + ".o1b", b + ".attn1.to_out.0"));
            std::vector<float> q2;
            MODEL_TRY(lin_f32(b + ".attn2.to_q", q2, n, kk));
            MODEL_TRY(fold_ln(b + ".q2", q2, c, c, g2->v, b2->v, nullptr));
            std::vector<float> ck, cv;
            int nk, dk;
            MODEL_TRY(lin_f32(b + ".attn2.to_k", ck, nk, dk));
            MODEL_TRY(lin_f32(b + ".attn2.to_v", cv, nk, dk));
            kv_k = dk;
            kv_off[b] = kv_total;
            kv_total += 2 * c;
            for (float f : ck) kv_w_all.push_back(__float2half(f));
            for (float f : cv) kv_w_all.push_back(__float2half(f));
            MODEL_TRY(add_lin(b + ".o2", b + ".attn2.to_out.0"));
            MODEL_TRY(add_bias(b + ".o2b", b + ".attn2.to_out.0"));
            // GEGLU projection with rows interleaved (value_i, gate_i) so the gate product is a GEMM epilogue
            std::vector<float> gw;
            int gn, gk;
            MODEL_TRY(lin_f32(b + ".ff.net.0.proj", gw, gn, gk));
            const HostTensor* gb;
            MODEL_TRY(need(b + ".ff.net.0.proj.bias", &gb));
            const int half = gn / 2;
            std::vector<float> gi(gw.size()), gbi(gn);
            for (int r = 0; r < half; ++r) {
                std::copy(gw.begin() + static_cast<size_t>(r) * gk, gw.begin() + static_cast<size_t>(r + 1) * gk,
                          gi.begin() + static_cast<size_t>(2 * r) * gk);
                std::copy(gw.begin() + static_cast<size_t>(half + r) * gk, gw.begin() + static_cast<size_t>(half + r + 1) * gk,
                          gi.begin() + static_cast<size_t>(2 * r + 1) * gk);
                gbi[2 * r] = gb->v[r], gbi[2 * r + 1] = gb->v[half + r];
            }
            MODEL_TRY(fold_ln(b + ".gg", gi, gn, gk, g3->v, b3->v, &gbi));
            MODEL_TRY(add_lin(b + ".f2", b + ".ff.net.2"));
            MODEL_TRY(add_bias(b + ".f2b", b + ".ff.net.2"));
        }
        return 0;
    }

    int pack() {
        nb = cfg.n_blocks;
        auto cin = std::make_unique<Mat>();
        MODEL_TRY(conv3("conv_in", *cin, in_pad));
        mats["conv_in"] = std::move(cin);
        MODEL_TRY(add_bias("conv_in.b", "conv_in"));
        for (const char* nm : {"time_embedding.linear_1", "time_embedding.linear_2"}) {
            std::vector<float> w;
            int n, k;
            MODEL_TRY(lin_f32(nm, w, n, k));
            MODEL_TRY(small(nm, w));
            MODEL_TRY(add_bias(std::string(nm) + ".b", nm));
        }
        if (xl)
            for (const char* nm : {"add_embedding.linear_1", "add_embedding.linear_2"}) {
                std::vector<float> w;
                int n, k;
                MODEL_TRY(lin_f32(nm, w, n, k));
                MODEL_TRY(small(nm, w));
                MODEL_TRY(add_bias(std::string(nm) + ".b", nm));
            }
        for (int i = 0; i < nb; ++i) {
            for (int j = 0; j < cfg.layers_per_block; ++j) {
                MODEL_TRY(pack_resnet("down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j)));
                if (cfg.down_cross_attn[i])
                    MODEL_TRY(pack_transformer("down_blocks." + std::to_string(i) + ".attentions." + std::to_string(j),
                                               cfg.block_out_channels[i], cfg.transformer_layers[i]));
            }
            if (i != nb - 1) {
                const std::string p = "down_blocks." + std::to_string(i) + ".downsamplers.0.conv";
                auto m = std::make_unique<Mat>();
                MODEL_TRY(conv3(p, *m));
                mats[p] = std::move(m);
                MODEL_TRY(add_bias(p + ".b", p));
            }
        }
        MODEL_TRY(pack_resnet("mid_block.resnets.0"));
        MODEL_TRY(pack_transformer("mid_block.attentions.0", cfg.block_out_channels[nb - 1], cfg.mid_transformer_layers));
        MODEL_TRY(pack_resnet("mid_block.resnets.1"));
        for (int i = 0; i < nb; ++i) {
            const int ri = nb - 1 - i;
            for (int j = 0; j < cfg.layers_per_block + 1; ++j) {
                MODEL_TRY(pack_resnet("up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j)));
                if (cfg.up_cross_attn[i])
                    MODEL_TRY(pack_transformer("up_blocks." + std::to_string(i) + ".attentions." + std::to_string(j),
                                               cfg.block_out_channels[ri], cfg.transformer_layers[ri]));
            }
            if (i != nb - 1) {
                const std::string p = "up_blocks." + std::to_string(i) + ".upsamplers.0.conv";
                auto m = std::make_unique<Mat>();
                MODEL_TRY(conv3(p, *m));
                mats[p] = std::move(m);
                MODEL_TRY(add_bias(p + ".b", p));
            }
        }
        MODEL_TRY(add_vec("out.g", "conv_norm_out.weight"));
        MODEL_TRY(add_vec("out.b", "conv_norm_out.bias"));
        auto co = std::make_unique<Mat>();
        MODEL_TRY(conv3("conv_out", *co));
        mats["conv_out"] = std::move(co);
        MODEL_TRY(add_bias("conv_out.b", "conv_out"));
        MODEL_TRY(small("temb_w", temb_w_all));
        MODEL_TRY(upload_f32("temb_b", temb_b_all));
        if (!kv_w_all.empty()) {
            auto m = std::make_unique<Mat>();
            m->n = kv_total, m->k = kv_k, m->host = kv_w_all;
            mats["kv"] = std::move(m);
        }
        return 0;
    }

    // ------------------------------------------------------------------ op wrappers (mirror ml-stable-diffusion_b200/lib.py)
    // weight tile of one call site: [n_tiles][k_blocks][bn][64], k-block order of the kernel's main loop
    int tiled(Mat& m, int c0, int c1, int taps, int bn, bool chunk_major, void** out, int c2 = 0, int c3 = 0) {
        const auto key = std::make_pair(bn, chunk_major ? 1 : 0);
        auto it = m.tiled.find(key);
        if (it != m.tiled.end()) {
            *out = it->second;
            return 0;
        }
        B200SD_REQUIRE(!m.host.empty(), "b200sd_unet: weight tiling requested after the host copy was released");
        const int kpt = c0 + c1, kc0 = (c0 + 63) / 64, kc1 = (c1 + 63) / 64, kc = kc0 + kc1;
        const int nt = (m.n + bn - 1) / bn;
        const int kc2 = (c2 + 63) / 64, kc3 = (c3 + 63) / 64, kbt = taps * kc + kc2 + kc3;  // (+ folded-shortcut k-blocks)
        const int ktot = taps * kpt + c2 + c3;
        B200SD_REQUIRE(ktot == m.k && (c2 + c3 == 0 || !chunk_major), "b200sd_unet: weight matrix / call site mismatch");
        std::vector<__half> t(static_cast<size_t>(nt) * kbt * bn * 64, __float2half(0.f));
        for (int tile = 0; tile < nt; ++tile)
            for (int tap = 0; tap < taps; ++tap)
                for (int j = 0; j < kc; ++j) {
                    const int lo = j < kc0 ? j * 64 : c0 + (j - kc0) * 64;
                    const int hi = std::min(lo + 64, j < kc0 ? c0 : kpt);
                    const int kb = chunk_major ? j * taps + tap : tap * kc + j;
                    for (int r = 0; r < bn; ++r) {
                        const int row = tile * bn + r;
                        if (row >= m.n) break;
                        const __half* src = m.host.data() + static_cast<size_t>(row) * ktot + static_cast<size_t>(tap) * kpt + lo;
                        __half* dst = t.data() + ((static_cast<size_t>(tile) * kbt + kb) * bn + r) * 64;
                        std::copy(src, src + (hi - lo), dst);
                    }
                }
        for (int tile = 0; tile < nt; ++tile)
            for (int j = 0; j < kc2 + kc3; ++j) {
                const int lo = j < kc2 ? j * 64 : c2 + (j - kc2) * 64;
                const int hi = std::min(lo + 64, j < kc2 ? c2 : c2 + c3);
                for (int r = 0; r < bn; ++r) {
                    const int row = tile * bn + r;
                    if (row >= m.n) break;
                    const __half* src = m.host.data() + static_cast<size_t>(row) * ktot + static_cast<size_t>(taps) * kpt + lo;
                    __half* dst = t.data() + ((static_cast<size_t>(tile) * kbt + taps * kc + j) * bn + r) * 64;
                    std::copy(src, src + (hi - lo), dst);
                }
            }
        void* d;
        MODEL_TRY(dev_alloc(&d, t.size() * 2));
        B200SD_CHECK_CUDA(cudaMemcpy(d, t.data(), t.size() * 2, cudaMemcpyHostToDevice));
        m.tiled[key] = d;
        *out = d;
        return 0;
    }

    int ensure_scratch(size_t bytes) {
        if (bytes <= scratch_bytes) return 0;
        void* d;
        MODEL_TRY(dev_alloc(&d, bytes));
        scratch = static_cast<float*>(d);
        scratch_bytes = bytes;
        return 0;
    }

    // out = epilogue(A * W^T): the common part of linear() / conv3x3() of lib.py (statistics, weight tiling, scratch)
    int gemm(b200sd_gemm_args a, Mat& w, int taps, int n_img_stats, bool want_cs, float** chan_out, RowStats* rs, int m_rows) {
        int32_t pl[8];
        want_cs = want_cs && fuse_gn;
        if (want_cs) {
            a.cs_partial = reinterpret_cast<float*>(16);
            if (b200sd_gemm_plan_ex(&a, pl) != 0) {  // this geometry cannot emit column statistics: consumer falls back
                want_cs = false;
                a.cs_partial = nullptr;
                a.cs_hw = 0;
            }
        }
        if (rs) a.rs_out = reinterpret_cast<float*>(16);
        MODEL_TRY(b200sd_gemm_plan_ex(&a, pl));
        const int bn = pl[0], n_tiles = pl[3], slots = pl[4];
        const int rs_parts = pl[5] ? n_tiles : 2 * n_tiles;  // register epilogue: one partial per column half of a tile
        if (want_cs) {
            void* c;
            MODEL_TRY(act_alloc(&c, static_cast<size_t>(n_img_stats) * a.n * 8));
            MODEL_TRY(ensure_scratch(static_cast<size_t>(n_img_stats) * slots * a.n * 8 + 64));
            a.cs_partial = scratch, a.cs_chan = static_cast<float*>(c), a.cs_tickets = tickets;
            if (chan_out) *chan_out = static_cast<float*>(c);
        } else if (chan_out) {
            *chan_out = nullptr;
        }
        if (rs) {
            void* r;
            MODEL_TRY(act_alloc(&r, static_cast<size_t>(rs_parts) * m_rows * 8));
            a.rs_out = static_cast<float*>(r);
            rs->rows = a.rs_out, rs->parts = rs_parts;
        }
        void* wt;
        MODEL_TRY(tiled(w, a.c0, a.c1, taps, bn, a.halo != 0, &wt, a.c2, a.c3));
        a.wgt = wt, a.block_n = bn, a.wgt_tiled = 1;
        const size_t ws = b200sd_gemm_workspace_bytes(&a);
        if (ws) {
            B200SD_REQUIRE(!want_cs, "b200sd_unet: split-K workspace and statistics in one call");
            MODEL_TRY(ensure_scratch(ws));
            a.workspace = scratch, a.workspace_bytes = scratch_bytes;
        }
        return b200sd_gemm(&a, st);
    }

    int linear(const __half* x, int m, int c0, Mat& w, const float* bias, const __half* residual, __half** out, const __half* x1 = nullptr,
               int c1 = 0, bool geglu = false, const RowStats* ln = nullptr, const float* ln_wg = nullptr, RowStats* rs = nullptr,
               float** chan = nullptr, int cs_hw = 0, void* out_override = nullptr) {
        b200sd_gemm_args a;
        memset(&a, 0, sizeof(a));
        a.mode = 0, a.m = m, a.n = w.n, a.c0 = c0, a.c1 = c1, a.stride = 1, a.geglu = geglu;
        a.a0 = x, a.a1 = x1, a.bias = bias, a.residual = residual;
        void* o = out_override;
        if (!o) MODEL_TRY(act_alloc(&o, static_cast<size_t>(m) * (geglu ? w.n / 2 : w.n) * 2));
        a.out = o;
        if (ln) a.ln_stat = ln->rows, a.ln_parts = ln->parts, a.ln_wg = ln_wg, a.ln_eps = 1e-5f;
        if (ln || rs || chan) a.split_k = 1;
        a.cs_hw = cs_hw;
        MODEL_TRY(gemm(a, w, 1, cs_hw ? m / cs_hw : 0, chan != nullptr && cs_hw > 0, chan, rs, m));
        *out = static_cast<__half*>(o);
        return 0;
    }

    int conv(const Act& x, const Act* x1, Mat& w, int cout, const float* bias, int bias_rows, int bias_stride, const __half* residual,
             bool halo, int taps, int stride, bool upsample, const GnSpec* gn, bool want_cs, RowStats* rs, bool out_f32, void* out_override,
             Act* out, const Act* sc0 = nullptr, const Act* sc1 = nullptr) {
        b200sd_gemm_args a;
        memset(&a, 0, sizeof(a));
        if (sc0) a.a2 = sc0->p, a.c2 = sc0->c;
        if (sc1) a.a3 = sc1->p, a.c3 = sc1->c;
        const int h = upsample ? 2 * x.h : x.h, wd = upsample ? 2 * x.w : x.w;
        const int ho = h / stride, wo = wd / stride;
        a.mode = taps == 9 ? 1 : 0, a.m = taps == 1 ? x.n * h * wd : 0, a.n = cout, a.c0 = x.c, a.c1 = x1 ? x1->c : 0;
        a.n_img = x.n, a.h = h, a.w = wd, a.stride = stride, a.out_f32 = out_f32;
        a.bias_rows = bias_rows, a.bias_stride = bias_stride;
        a.a0 = x.p, a.a1 = x1 ? x1->p : nullptr, a.bias = bias, a.residual = residual;
        a.halo = halo, a.upsample2x = upsample;
        if (gn) {
            a.gn_groups = gn->groups, a.gn_silu = gn->silu, a.gn_eps = gn->eps;
            a.gn_chan0 = gn->chan0, a.gn_chan1 = gn->chan1, a.gn_gamma = gn->gamma, a.gn_beta = gn->beta;
        }
        if (gn || want_cs || rs) a.split_k = 1;
        void* o = out_override;
        if (!o) MODEL_TRY(act_alloc(&o, static_cast<size_t>(x.n) * ho * wo * cout * (out_f32 ? 4 : 2)));
        a.out = o;
        a.cs_hw = ho * wo;
        float* chan = nullptr;
        MODEL_TRY(gemm(a, w, taps, x.n, want_cs, &chan, rs, x.n * ho * wo));
        out->p = static_cast<__half*>(o), out->n = x.n, out->h = ho, out->w = wo, out->c = cout, out->chan = chan;
        return 0;
    }

    int group_norm(const Act& x, const Act* x1, const float* gamma, const float* beta, float eps, int silu, Act* out) {
        const int c = x.c + (x1 ? x1->c : 0);
        void* o;
        MODEL_TRY(act_alloc(&o, static_cast<size_t>(x.rows()) * c * 2));
        const size_t ws = b200sd_group_norm_workspace_bytes(x.n, x.h * x.w, c, cfg.norm_num_groups);
        MODEL_TRY(ensure_scratch(ws + 64));
        MODEL_TRY(b200sd_group_norm(x.p, x1 ? x1->p : nullptr, x.c, x1 ? x1->c : 0, x.n, x.h * x.w, cfg.norm_num_groups, eps, gamma, beta,
                                    silu, o, scratch, scratch_bytes, st));
        *out = x;
        out->p = static_cast<__half*>(o), out->c = c, out->chan = nullptr;
        return 0;
    }

    // GroupNorm (+SiLU) -> conv: in the halo convolution's operand path when the producers left statistics behind
    int gn_conv(const Act& x, const Act* x1, const std::string& gkey, const std::string& bkey, float eps, int silu, Mat& w, int cout,
                const float* bias, int bias_rows, int bias_stride, const __half* residual, bool want_cs, bool out_f32, void* out_override,
                Act* out, const Act* sc0 = nullptr, const Act* sc1 = nullptr) {
        const float *gamma = vecs.at(gkey), *beta = vecs.at(bkey);
        if (!fuse_gn) {
            Act hn;
            MODEL_TRY(group_norm(x, x1, gamma, beta, eps, silu, &hn));
            return conv(hn, nullptr, w, cout, bias, bias_rows, bias_stride, residual, false, 9, 1, false, nullptr, false, nullptr, out_f32,
                        out_override, out, sc0, sc1);
        }
        if (x.chan && (!x1 || x1->chan)) {
            GnSpec g{x.chan, x1 ? x1->chan : nullptr, gamma, beta, cfg.norm_num_groups, eps, silu};
            return conv(x, x1, w, cout, bias, bias_rows, bias_stride, residual, true, 9, 1, false, &g, want_cs, nullptr, out_f32, out_override,
                        out);
        }
        Act hn;
        MODEL_TRY(group_norm(x, x1, gamma, beta, eps, silu, &hn));
        return conv(hn, nullptr, w, cout, bias, bias_rows, bias_stride, residual, true, 9, 1, false, nullptr, want_cs, nullptr, out_f32,
                    out_override, out);
    }

    const float* vec_or_null(const std::string& k) const {
        auto it = vecs.find(k);
        return it == vecs.end() ? nullptr : it->second;
    }

    int resnet(const std::string& p, const Act& x, const Act* x1, const float* temb, Act* out) {
        Mat& c1 = *mats.at(p + ".c1");
        Mat& c2 = *mats.at(p + ".c2");
        const int co = c1.n;
        Act h1;
        MODEL_TRY(gn_conv(x, x1, p + ".n1g", p + ".n1b", cfg.norm_eps, 1, c1, co, temb + temb_off.at(p), x.h * x.w, temb_total, nullptr, true,
                          false, nullptr, &h1));
        if (!fuse_gn && mats.count(p + ".c2sc"))  // conv2(h) + conv_shortcut(x ++ x1) as one launch
            return gn_conv(h1, nullptr, p + ".n2g", p + ".n2b", cfg.norm_eps, 1, *mats.at(p + ".c2sc"), co, vecs.at(p + ".c2scb"), 0, 0, nullptr,
                           false, false, nullptr, out, &x, x1);
        const __half* res = x.p;
        if (mats.count(p + ".sc")) {
            __half* r;
            MODEL_TRY(linear(x.p, x.rows(), x.c, *mats.at(p + ".sc"), vec_or_null(p + ".scb"), nullptr, &r, x1 ? x1->p : nullptr, x1 ? x1->c : 0));
            res = r;
        }
        return gn_conv(h1, nullptr, p + ".n2g", p + ".n2b", cfg.norm_eps, 1, c2, co, vec_or_null(p + ".c2b"), 0, 0, res, true, false, nullptr, out);
    }

    int attention(const __half* q, int ldq, const __half* k, const __half* v, int ldkv, int heads, int sq, int sk, __half** out, int c) {
        void* o;
        MODEL_TRY(act_alloc(&o, static_cast<size_t>(B) * sq * c * 2));
        const int d = c / heads;  // 64 (SD 2.x, SDXL) or 40 / 80 / 160 (SD 1.x)
        MODEL_TRY(b200sd_attention_ws(q, k, v, o, nullptr, B, heads, sq, sk, d, ldq, ldkv, ldkv, c, 1.0f / sqrtf(static_cast<float>(d)),
                                      attn_impl, attn_ws, attn_ws_bytes, st));
        *out = static_cast<__half*>(o);
        return 0;
    }

    int transformer(const std::string& p, const Act& x, int heads, int depth, Act* out) {
        const int c = x.c, m = x.rows(), s = x.h * x.w;
        RowStats rs;
        __half* tok;
        if (x.chan) {
            GnSpec g{x.chan, nullptr, vecs.at(p + ".ng"), vecs.at(p + ".nb"), 32, 1e-6f, 0};
            Act t;
            MODEL_TRY(conv(x, nullptr, *mats.at(p + ".pi"), c, vec_or_null(p + ".pib"), 0, 0, nullptr, true, 1, 1, false, &g, false, &rs, false,
                           nullptr, &t));
            tok = t.p;
        } else {
            Act hn;
            const int keep = cfg.norm_num_groups;
            cfg.norm_num_groups = 32;
            const int rc = group_norm(x, nullptr, vecs.at(p + ".ng"), vecs.at(p + ".nb"), 1e-6f, 0, &hn);
            cfg.norm_num_groups = keep;
            if (rc) return rc;
            MODEL_TRY(linear(hn.p, m, c, *mats.at(p + ".pi"), vec_or_null(p + ".pib"), nullptr, &tok, nullptr, 0, false, nullptr, nullptr, &rs));
        }
        for (int d = 0; d < depth; ++d) {
            const std::string b = p + ".transformer_blocks." + std::to_string(d);
            __half *qkv, *a, *q;
            MODEL_TRY(linear(tok, m, c, *mats.at(b + ".qkv"), vecs.at(b + ".qkv.b"), nullptr, &qkv, nullptr, 0, false, &rs, vecs.at(b + ".qkv.wg")));
            MODEL_TRY(attention(qkv, 3 * c, qkv + c, qkv + 2 * c, 3 * c, heads, s, s, &a, c));
            RowStats r1;
            MODEL_TRY(linear(a, m, c, *mats.at(b + ".o1"), vec_or_null(b + ".o1b"), tok, &tok, nullptr, 0, false, nullptr, nullptr, &r1));
            MODEL_TRY(linear(tok, m, c, *mats.at(b + ".q2"), vecs.at(b + ".q2.b"), nullptr, &q, nullptr, 0, false, &r1, vecs.at(b + ".q2.wg")));
            const int ko = kv_off.at(b);
            MODEL_TRY(attention(q, c, kv_all + ko, kv_all + ko + c, kv_total, heads, s, S, &a, c));
            RowStats r2;
            MODEL_TRY(linear(a, m, c, *mats.at(b + ".o2"), vec_or_null(b + ".o2b"), tok, &tok, nullptr, 0, false, nullptr, nullptr, &r2));
            __half* g;
            MODEL_TRY(linear(tok, m, c, *mats.at(b + ".gg"), vecs.at(b + ".gg.b"), nullptr, &g, nullptr, 0, true, &r2, vecs.at(b + ".gg.wg")));
            RowStats r3;
            MODEL_TRY(linear(g, m, 4 * c, *mats.at(b + ".f2"), vec_or_null(b + ".f2b"), tok, &tok, nullptr, 0, false, nullptr, nullptr,
                             d + 1 < depth ? &r3 : nullptr));
            rs = r3;
        }
        const bool ok = s % 128 == 0 || (s >= 16 && 128 % s == 0);  // geometries whose tiles map onto whole images
        __half* o;
        float* chan = nullptr;
        MODEL_TRY(linear(tok, m, c, *mats.at(p + ".po"), vec_or_null(p + ".pob"), x.p, &o, nullptr, 0, false, nullptr, nullptr, nullptr,
                         ok ? &chan : nullptr, ok ? s : 0));
        *out = x;
        out->p = o, out->chan = chan;
        return 0;
    }

    int linear_small(const float* x, const std::string& w, const float* bias, float** out, int m, int n, int k, int act_in, int act_out) {
        void* o;
        MODEL_TRY(act_alloc(&o, static_cast<size_t>(m) * n * 4));
        MODEL_TRY(b200sd_linear_small(x, small_w.at(w), bias, nullptr, static_cast<float*>(o), m, n, k, act_in, act_out, st));
        *out = static_cast<float*>(o);
        return 0;
    }

    // fp32 [B] timesteps (+ SDXL time_ids / text_embeds) -> per-image bias vectors of every ResNet block [B, sum Cout]
    int time_embedding(const float* timesteps, const float* time_ids, const float* text_embeds, float** temb) {
        const int c0 = cfg.block_out_channels[0], td = 4 * c0;
        void* te;
        MODEL_TRY(act_alloc(&te, static_cast<size_t>(B) * c0 * 4));
        MODEL_TRY(b200sd_timestep_embedding(timesteps, static_cast<float*>(te), B, c0, cfg.flip_sin_to_cos, cfg.freq_shift, st));
        float *e1, *emb;
        MODEL_TRY(linear_small(static_cast<float*>(te), "time_embedding.linear_1", vec_or_null("time_embedding.linear_1.b"), &e1, B, td, c0, 0, 1));
        MODEL_TRY(linear_small(e1, "time_embedding.linear_2", vec_or_null("time_embedding.linear_2.b"), &emb, B, td, td, 0, 0));
        if (xl) {
            B200SD_REQUIRE(time_ids && text_embeds, "b200sd_unet_forward: this UNet needs time_ids and text_embeds");
            const int nid = cfg.num_time_ids, ate = cfg.addition_time_embed_dim, pin = cfg.projection_class_embeddings_input_dim;
            const int pooled = pin - nid * ate;
            void *ids, *cat;
            MODEL_TRY(act_alloc(&ids, static_cast<size_t>(B) * nid * ate * 4));
            MODEL_TRY(act_alloc(&cat, static_cast<size_t>(B) * pin * 4));
            MODEL_TRY(b200sd_timestep_embedding(time_ids, static_cast<float*>(ids), B * nid, ate, cfg.flip_sin_to_cos, cfg.freq_shift, st));
            B200SD_CHECK_CUDA(cudaMemcpy2DAsync(cat, static_cast<size_t>(pin) * 4, text_embeds, static_cast<size_t>(pooled) * 4,
                                                static_cast<size_t>(pooled) * 4, B, cudaMemcpyDeviceToDevice, st));
            B200SD_CHECK_CUDA(cudaMemcpy2DAsync(static_cast<float*>(cat) + pooled, static_cast<size_t>(pin) * 4, ids,
                                                static_cast<size_t>(nid) * ate * 4, static_cast<size_t>(nid) * ate * 4, B,
                                                cudaMemcpyDeviceToDevice, st));
            float *a1, *aug;
            MODEL_TRY(linear_small(static_cast<float*>(cat), "add_embedding.linear_1", vec_or_null("add_embedding.linear_1.b"), &a1, B, td, pin, 0, 1));
            MODEL_TRY(linear_small(a1, "add_embedding.linear_2", vec_or_null("add_embedding.linear_2.b"), &aug, B, td, td, 0, 0));
            B200SD_CHECK_CUDA(launch_kernel(add_f32_kernel, dim3((B * td + 255) / 256), dim3(256), 0, st, emb, aug, B * td));
        }
        return linear_small(emb, "temb_w", vecs.at("temb_b"), temb, B, temb_total, td, 1, 0);
    }

    int prepare_prompt(const void* ctx) {
        if (!mats.count("kv")) return 0;
        void* tok;
        MODEL_TRY(act_alloc(&tok, static_cast<size_t>(B) * S * cfg.cross_attention_dim * 2));
        MODEL_TRY(b200sd_ctx_to_tokens(ctx, 0, tok, B, cfg.cross_attention_dim, S, st));
        __half* o;
        return linear(static_cast<__half*>(tok), B * S, cfg.cross_attention_dim, *mats.at("kv"), nullptr, nullptr, &o, nullptr, 0, false, nullptr,
                      nullptr, nullptr, nullptr, 0, kv_all);
    }

    int forward(const void* sample, int sample_f32, const float* timesteps, const void* ctx, const float* time_ids, const float* text_embeds,
                const void* const* residuals, float* noise_pred) {
        arena_off = 0;
        if (ctx) {
            MODEL_TRY(prepare_prompt(ctx));
            kv_ready = true;
        }
        B200SD_REQUIRE(kv_ready || !mats.count("kv"), "b200sd_unet_forward: no encoder_hidden_states given and b200sd_unet_prepare_prompt was not called");
        float* temb;
        MODEL_TRY(time_embedding(timesteps, time_ids, text_embeds, &temb));
        Act x0;
        void* xin;
        MODEL_TRY(act_alloc(&xin, static_cast<size_t>(B) * H * W * in_pad * 2));
        MODEL_TRY(b200sd_nchw_to_nhwc(sample, sample_f32, xin, B, cfg.in_channels, H, W, in_pad, st));
        x0.p = static_cast<__half*>(xin), x0.n = B, x0.h = H, x0.w = W, x0.c = in_pad;
        Act x;
        MODEL_TRY(conv(x0, nullptr, *mats.at("conv_in"), cfg.block_out_channels[0], vec_or_null("conv_in.b"), 0, 0, nullptr, false, 9, 1, false,
                       nullptr, true, nullptr, false, nullptr, &x));
        std::vector<Act> skips{x};
        for (int i = 0; i < nb; ++i) {
            for (int j = 0; j < cfg.layers_per_block; ++j) {
                Act y;
                MODEL_TRY(resnet("down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), x, nullptr, temb, &y));
                x = y;
                if (cfg.down_cross_attn[i]) {
                    MODEL_TRY(transformer("down_blocks." + std::to_string(i) + ".attentions." + std::to_string(j), x, cfg.attention_heads[i],
                                          cfg.transformer_layers[i], &y));
                    x = y;
                }
                skips.push_back(x);
            }
            if (i != nb - 1) {
                const std::string p = "down_blocks." + std::to_string(i) + ".downsamplers.0.conv";
                Act y;
                MODEL_TRY(conv(x, nullptr, *mats.at(p), x.c, vec_or_null(p + ".b"), 0, 0, nullptr, false, 9, 2, false, nullptr, true, nullptr, false,
                               nullptr, &y));
                x = y;
                skips.push_back(x);
            }
        }
        auto add_residual = [&](Act& t, const void* r_nchw) -> int {  // ControlNet injection (unet.py:1009-1022)
            void *rn, *o;
            MODEL_TRY(act_alloc(&rn, static_cast<size_t>(t.rows()) * t.c * 2));
            MODEL_TRY(b200sd_nchw_to_nhwc(r_nchw, 0, rn, t.n, t.c, t.h, t.w, t.c, st));
            MODEL_TRY(act_alloc(&o, static_cast<size_t>(t.rows()) * t.c * 2));
            MODEL_TRY(b200sd_add(t.p, rn, o, static_cast<size_t>(t.rows()) * t.c, st));
            t.p = static_cast<__half*>(o), t.chan = nullptr;  // the sum has no producer-side statistics
            return 0;
        };
        if (residuals)
            for (size_t i = 0; i < skips.size(); ++i) MODEL_TRY(add_residual(skips[i], residuals[i]));
        Act y;
        MODEL_TRY(resnet("mid_block.resnets.0", x, nullptr, temb, &y));
        x = y;
        MODEL_TRY(transformer("mid_block.attentions.0", x, cfg.attention_heads[nb - 1], cfg.mid_transformer_layers, &y));
        x = y;
        MODEL_TRY(resnet("mid_block.resnets.1", x, nullptr, temb, &y));
        x = y;
        if (residuals) MODEL_TRY(add_residual(x, residuals[skips.size()]));
        for (int i = 0; i < nb; ++i) {
            const int ri = nb - 1 - i;
            for (int j = 0; j < cfg.layers_per_block + 1; ++j) {
                Act sk = skips.back();
                skips.pop_back();
                MODEL_TRY(resnet("up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), x, &sk, temb, &y));
                x = y;
                if (cfg.up_cross_attn[i]) {
                    MODEL_TRY(transformer("up_blocks." + std::to_string(i) + ".attentions." + std::to_string(j), x, cfg.attention_heads[ri],
                                          cfg.transformer_layers[ri], &y));
                    x = y;
                }
            }
            if (i != nb - 1) {
                const std::string p = "up_blocks." + std::to_string(i) + ".upsamplers.0.conv";
                if (fuse_gn) {
                    MODEL_TRY(conv(x, nullptr, *mats.at(p), x.c, vec_or_null(p + ".b"), 0, 0, nullptr, true, 9, 1, true, nullptr, true, nullptr,
                                   false, nullptr, &y));
                } else {  // nearest x2 copy + 9-tap convolution
                    Act up = x;
                    void* u;
                    MODEL_TRY(act_alloc(&u, static_cast<size_t>(x.rows()) * 4 * x.c * 2));
                    MODEL_TRY(b200sd_upsample2x(x.p, u, x.n, x.h, x.w, x.c, st));
                    up.p = static_cast<__half*>(u), up.h = 2 * x.h, up.w = 2 * x.w, up.chan = nullptr;
                    MODEL_TRY(conv(up, nullptr, *mats.at(p), x.c, vec_or_null(p + ".b"), 0, 0, nullptr, false, 9, 1, false, nullptr, false, nullptr,
                                   false, nullptr, &y));
                }
                x = y;
            }
        }
        void* o_nhwc;
        MODEL_TRY(act_alloc(&o_nhwc, static_cast<size_t>(B) * H * W * cfg.out_channels * 4));
        MODEL_TRY(gn_conv(x, nullptr, "out.g", "out.b", cfg.norm_eps, 1, *mats.at("conv_out"), cfg.out_channels, vec_or_null("conv_out.b"), 0, 0,
                          nullptr, false, true, o_nhwc, &y));
        return b200sd_nhwc_to_nchw_f32(o_nhwc, 1, noise_pred, B, cfg.out_channels, H, W, cfg.out_channels, st);
    }

    // after the first (sizing) forward: one arena, host weight copies released
    int finalize() {
        B200SD_CHECK_CUDA(cudaStreamSynchronize(st));
        for (void* p : warm_allocs) cudaFree(p);
        warm_allocs.clear();
        arena_cap = sized + (1 << 20);
        B200SD_CHECK_CUDA(cudaMalloc(reinterpret_cast<void**>(&arena), arena_cap));
        bump = true;
        hw.clear();
        for (auto& kv : mats) {
            kv.second->host.clear();
            kv.second->host.shrink_to_fit();
        }
        temb_w_all.clear(), temb_b_all.clear(), kv_w_all.clear();
        return 0;
    }
};

}  // namespace
}  // namespace b200sd

struct b200sd_unet {
    b200sd::UNet impl;
};

extern "C" int b200sd_unet_create(const b200sd_unet_config* cfg, const b200sd_weight* weights, int32_t n_weights, void* stream,
                                  b200sd_unet** out) {
    using namespace b200sd;
    B200SD_REQUIRE(cfg && weights && out && n_weights > 0, "b200sd_unet_create: null argument");
    B200SD_REQUIRE(cfg->n_blocks >= 1 && cfg->n_blocks <= 8 && cfg->batch >= 1 && cfg->height >= 1 && cfg->width >= 1 && cfg->seq_len >= 1,
                   "b200sd_unet_create: bad geometry");
    {  // every down-sampler halves the map exactly (config.latent_multiple)
        const int mult = 1 << (cfg->n_blocks - 1);
        B200SD_REQUIRE(cfg->height % mult == 0 && cfg->width % mult == 0,
                       "b200sd_unet_create: latents of %dx%d cannot be halved %d times; height and width must be multiples of %d pixels "
                       "(%d latent pixels) for this model",
                       cfg->height, cfg->width, cfg->n_blocks - 1, 8 * mult, mult);
    }
    size_t attn_ws_bytes = 0;  // stream-K workspace for the largest head dim of the net
    for (int i = 0; i < cfg->n_blocks; ++i) {
        const int c = cfg->block_out_channels[i], heads = cfg->attention_heads[i];
        B200SD_REQUIRE(heads > 0 && c % heads == 0 && b200sd_attention_workspace_bytes_for(c / heads) > 0,
                       "b200sd_unet_create: block %d has head dim %d/%d; the attention kernel supports 40, 64, 80 and 160", i, c,
                       heads);
        attn_ws_bytes = std::max(attn_ws_bytes, b200sd_attention_workspace_bytes_for(c / heads));
    }
    auto h = std::make_unique<b200sd_unet>();
    UNet& u = h->impl;
    u.cfg = *cfg;
    if (u.cfg.num_time_ids <= 0) u.cfg.num_time_ids = 6;
    u.B = cfg->batch, u.H = cfg->height, u.W = cfg->width, u.S = cfg->seq_len;
    u.in_pad = std::max(8, (cfg->in_channels + 7) / 8 * 8);
    u.xl = cfg->addition_embed_text_time != 0;
    u.st = static_cast<cudaStream_t>(stream);
    {
        const char* e = getenv("B200SD_FUSED");
        u.fuse_gn = e && e[0] == '1';
    }
    for (int i = 0; i < n_weights; ++i) {
        const b200sd_weight& w = weights[i];
        B200SD_REQUIRE(w.name && w.data && w.ndim >= 1 && w.ndim <= 4 && (w.dtype == 0 || w.dtype == 1), "b200sd_unet_create: bad weight entry %d", i);
        HostTensor t;
        for (int d = 0; d < w.ndim; ++d) t.shape.push_back(w.shape[d]);
        const int64_t n = t.numel();
        t.v.resize(n);
        if (w.dtype == 1) {
            memcpy(t.v.data(), w.data, n * 4);
        } else {
            const __half* s = static_cast<const __half*>(w.data);
            for (int64_t e = 0; e < n; ++e) t.v[e] = __half2float(s[e]);
        }
        u.hw.emplace(w.name, std::move(t));
    }
    if (int rc = u.pack()) return rc;
    void* tk;
    if (int rc = u.dev_alloc(&tk, (1 << 16) * sizeof(unsigned int))) return rc;
    B200SD_CHECK_CUDA(cudaMemset(tk, 0, (1 << 16) * sizeof(unsigned int)));
    u.tickets = static_cast<unsigned int*>(tk);
    u.attn_ws_bytes = attn_ws_bytes;
    if (int rc = u.dev_alloc(&u.attn_ws, u.attn_ws_bytes)) return rc;
    B200SD_CHECK_CUDA(cudaMemset(u.attn_ws, 0, u.attn_ws_bytes));
    if (u.mats.count("kv")) {
        void* kv;
        if (int rc = u.dev_alloc(&kv, static_cast<size_t>(u.B) * u.S * u.kv_total * 2)) return rc;
        u.kv_all = static_cast<__half*>(kv);
    }
    // sizing pass on zero inputs: tiles every weight for its call sites, measures the activation arena
    {
        void *s, *t, *c, *ti = nullptr, *te = nullptr, *o;
        const size_t ns = static_cast<size_t>(u.B) * cfg->in_channels * u.H * u.W;
        B200SD_CHECK_CUDA(cudaMalloc(&s, ns * 2));
        B200SD_CHECK_CUDA(cudaMalloc(&t, u.B * 4));
        B200SD_CHECK_CUDA(cudaMalloc(&c, static_cast<size_t>(u.B) * cfg->cross_attention_dim * u.S * 2));
        B200SD_CHECK_CUDA(cudaMalloc(&o, static_cast<size_t>(u.B) * cfg->out_channels * u.H * u.W * 4));
        cudaMemsetAsync(s, 0, ns * 2, u.st);
        cudaMemsetAsync(t, 0, u.B * 4, u.st);
        cudaMemsetAsync(c, 0, static_cast<size_t>(u.B) * cfg->cross_attention_dim * u.S * 2, u.st);
        if (u.xl) {
            const size_t pooled = cfg->projection_class_embeddings_input_dim - u.cfg.num_time_ids * cfg->addition_time_embed_dim;
            B200SD_CHECK_CUDA(cudaMalloc(&ti, static_cast<size_t>(u.B) * u.cfg.num_time_ids * 4));
            B200SD_CHECK_CUDA(cudaMalloc(&te, static_cast<size_t>(u.B) * pooled * 4));
            cudaMemsetAsync(ti, 0, static_cast<size_t>(u.B) * u.cfg.num_time_ids * 4, u.st);
            cudaMemsetAsync(te, 0, static_cast<size_t>(u.B) * pooled * 4, u.st);
        }
        const int rc = u.forward(s, 0, static_cast<float*>(t), c, static_cast<float*>(ti), static_cast<float*>(te), nullptr, static_cast<float*>(o));
        cudaStreamSynchronize(u.st);
        cudaFree(s), cudaFree(t), cudaFree(c), cudaFree(o);
        if (ti) cudaFree(ti);
        if (te) cudaFree(te);
        if (rc) return rc;
        u.kv_ready = false;
        if (int rc2 = u.finalize()) return rc2;
    }
    *out = h.release();
    return 0;
}

extern "C" int b200sd_unet_prepare_prompt(b200sd_unet* h, const void* encoder_hidden_states, void* stream) {
    B200SD_REQUIRE(h && encoder_hidden_states, "b200sd_unet_prepare_prompt: null argument");
    h->impl.st = static_cast<cudaStream_t>(stream);
    h->impl.arena_off = 0;
    if (int rc = h->impl.prepare_prompt(encoder_hidden_states)) return rc;
    h->impl.kv_ready = true;
    return 0;
}

extern "C" int b200sd_unet_forward(b200sd_unet* h, const void* sample, int32_t sample_f32, const float* timesteps,
                                   const void* encoder_hidden_states, const float* time_ids, const float* text_embeds,
                                   const void* const* additional_residuals, float* noise_pred, void* stream) {
    B200SD_REQUIRE(h && sample && timesteps && noise_pred, "b200sd_unet_forward: null argument");
    B200SD_REQUIRE(!additional_residuals || h->impl.cfg.support_controlnet, "b200sd_unet_forward: this UNet was not created with support_controlnet");
    h->impl.st = static_cast<cudaStream_t>(stream);
    return h->impl.forward(sample, sample_f32, timesteps, encoder_hidden_states, time_ids, text_embeds, additional_residuals, noise_pred);
}

extern "C" int b200sd_unet_set_attention_impl(b200sd_unet* h, int32_t impl) {
    B200SD_REQUIRE(h && impl >= 0 && impl <= 2, "b200sd_unet_set_attention_impl: impl must be 0 (ORIGINAL), 1 (SPLIT_EINSUM) or 2 (SPLIT_EINSUM_V2)");
    h->impl.attn_impl = impl;
    return 0;
}

extern "C" size_t b200sd_unet_device_bytes(const b200sd_unet* h) {
    return h ? h->impl.arena_cap + h->impl.scratch_bytes : 0;
}

extern "C" void b200sd_destroy(b200sd_unet* h) { delete h; }
