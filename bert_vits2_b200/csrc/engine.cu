// libbv2: engine (weights, workspace, stage orchestration) and the C ABI declared in include/bv2.h.
// Orchestrates the path of reference models.SynthesizerTrn.infer (models.py:1026-1074).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <functional>
#include <cuda_fp16.h>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/bv2.h"
#include "common.cuh"
#include "kernels_simt.cuh"
#include "tc_conv.cuh"
#include "tc_gen.cuh"
#include "gen_stream.cuh"
#include "tc_attn.cuh"
#include "kernels_tok.cuh"

namespace bv2 {

struct HostTensor {
    std::vector<float> data;
    std::vector<int64_t> shape;
    int64_t numel() const { int64_t n = 1; for (auto s : shape) n *= s; return n; }
};

struct ConvW { float* w = nullptr; float* b = nullptr; int Cin = 0, Cout = 0, Cout_w = 0, K = 1; TcConvW tc; };
struct LnW { float* g = nullptr; float* b = nullptr; int C = 0; };
struct EncLayerW { ConvW qkv, o, f1, f2; LnW n1, n2; float* relk = nullptr; float* relv = nullptr; };
struct EncoderW { std::vector<EncLayerW> layers; int g_off = 0; int kernel = 3; };
struct DdsW { std::vector<float*> sep_w, sep_b; std::vector<ConvW> c1; std::vector<LnW> n1, n2; };
struct ConvFlowW { float* pre_w = nullptr; float* pre_b = nullptr; DdsW dds; ConvW proj; };
struct CouplingW {
    ConvW pre, post; int s = 0;  // orientation (Flip folded into weights)
    EncoderW enc;                // transformer flow
    std::vector<ConvW> wn_in, wn_res, wn_skip; int wn_g_off = 0;  // WN flow
};
struct ResBlockW { std::vector<ConvW> c1, c2; int k = 3; std::vector<int> dil; };
struct UpW { float* w = nullptr; float* b = nullptr; int Cin = 0, Cout = 0, K = 0, u = 0; TcConvW tc; };

struct DebugBuf { const float* p; int B, C, T; int c4; };

class Arena {
public:
    ~Arena() { if (base_) cudaFree(base_); }
    void reset() { off_ = 0; }
    // Sticky high-water mark: the arena only ever grows, and when it must it grows to 1.5x the request (the frame count of an
    // utterance varies with the duration noise), so a steady workload allocates during its first call(s) and never again.
    // Regrowth is a device-wide sync + cudaFree + cudaMalloc; bv2_reserve() sizes the arenas up front so that serving loops never hit it.
    // The sync also waits for the work of every other engine on the device (siblings included): correct, but a stall for them, so a
    // server reserves each sibling too.
    void ensure(size_t bytes) {
        if (bytes <= cap_) return;
        bytes += bytes / 2;
        if (base_) { cudaDeviceSynchronize(); cudaFree(base_); base_ = nullptr; cap_ = 0; }
        BV2_CUDA(cudaMalloc(&base_, bytes));
        cap_ = bytes;
        grows_++;
    }
    int grows() const { return grows_; }
    float* alloc(size_t nfloats) {
        size_t bytes = (nfloats * sizeof(float) + 255) & ~(size_t)255;
        BV2_CHECK(off_ + bytes <= cap_, "workspace overflow");
        float* p = reinterpret_cast<float*>(static_cast<char*>(base_) + off_);
        off_ += bytes;
        return p;
    }
    Act act(int B, int C, int T) { Act a; a.B = B; a.C = C; a.T = T; a.p = alloc((size_t)B * C * T); return a; }
    size_t cap() const { return cap_; }
    size_t used() const { return off_; }
    void release(size_t mark) { off_ = mark; }  // stack discipline; safe because all users are stream-ordered
private:
    void* base_ = nullptr; size_t cap_ = 0, off_ = 0; int grows_ = 0;
};

// One device error flag per device for the whole process.  tc_init_device() points the device-global g_tc_err_flag at a pinned int;
// re-pointing it would leave every older engine reading a flag the device no longer raises, so the first finalize on a device creates
// it, and it is never re-pointed or freed.  Every engine on the device reads the same flag: the first to see it raised consumes it
// under g_err_mu (clears both flags) and bumps the generation.  Once g_tc_err_dev is set every in-flight wait on the device drains
// early, so every call that was in flight at that moment has invalid results: a call fails if the generation changed since it began.
struct DeviceErrFlag { int* host = nullptr; uint64_t generation = 0; };
std::mutex g_err_mu;
std::unordered_map<int, DeviceErrFlag> g_err_flags;

}  // namespace bv2

using namespace bv2;

// Everything finalize() builds that stays fixed afterwards: the device weight arena and the layout bookkeeping that points into it.
// A sibling engine (bv2_create_sibling) copies this struct whole; the arena itself is shared and freed with the family's last member.
struct DeviceWeights {
    std::shared_ptr<uint8_t> warena_owner;
    uint8_t* warena = nullptr; size_t warena_bytes = 0;
    float *emb = nullptr, *temb = nullptr, *lemb = nullptr, *emb_g = nullptr;
    ConvW bert_proj, enc_proj;
    EncoderW enc_p;
    ConvW sdp_pre, sdp_proj; DdsW sdp_dds; std::vector<ConvFlowW> sdp_flows;  // index by flow id (1,3,5,7)
    float ea_m[2] = {0, 0}, ea_logs[2] = {0, 0};
    ConvW dp_c1, dp_c2, dp_proj; LnW dp_n1, dp_n2;
    std::vector<CouplingW> flows;
    ConvW conv_pre; std::vector<UpW> ups; std::vector<ResBlockW> resblocks; float* conv_post_w = nullptr;
    PostW<16, 7> conv_post_h{};  // host copy of conv_post's weights (kernel-parameter operand of k_conv_post_tanh_h8), read back in finalize()
    float *gproj_w = nullptr, *gproj_b = nullptr; int gproj_n = 0;
    int goff_dec = 0, goff_sdp = 0, goff_dp = 0;
    float dconst = 0.f;
    int hop = 512;
    int flow_tc = 0;       // 0 SIMT fp32, 1 TF32 wgmma, 2 FP16 wgmma + fused attention (finalize)
    int use_g2 = 0;        // FP16 Generator on 16-bit activation tensors (tc_gen.cuh)
    std::vector<std::pair<std::string, std::vector<int64_t>>> shape_table;  // kept for bv2_save_packed
};

struct bv2_engine : DeviceWeights {
    bv2_config cfg{};
    int device = 0;
    std::mutex mu;
    std::string err;
    std::unordered_map<std::string, HostTensor> host;
    bool finalized = false;
    int64_t launches = 0;
    int num_sms = 132;
    uint64_t call_gen = 0;  // device error generation when the current call began (check_device_error)

    // ---- workspace / per-call state
    Arena ws, persist;  // persist: state kept between infer_begin and infer_finish
    std::map<std::string, DebugBuf> dbg;
    struct {
        bool active = false, finished = false; int B = 0, T = 0, F = 0;
        float* stats = nullptr; int* cum = nullptr; long long* ylen = nullptr; int* ylen32 = nullptr; int* lens = nullptr;
        float* gproj = nullptr; float* w_ceil = nullptr;
        float* noise_scale = nullptr;  // [B] per-item noise scale of bv2_infer_begin_items (persist arena), nullptr after bv2_infer_begin
    } st;
    // Open Generator stream (bv2_infer_finish_stream .. the bv2_stream_advance that reaches Fg).  Every tensor of the Generator stays
    // in the workspace for the stream's lifetime, because later windows read the rows behind each layer's done pointer: the input z
    // plus conv_pre's output plus, per upsampling stage, the stage sum S, the upsampled xu and one tensor per resblock conv except the
    // last of each chain (2 + 3 * (3 + 2) = 17 tensors per stage at the default configuration), against the one-shot Generator's
    // per-stage release.
    //   fp32 / TF32 Generator: whole fp32 c4 tensors, 4 * (512 + 17 * (256*8 + 128*64 + 64*128 + 32*256 + 16*512)) = 2,369,536 bytes
    //                          per frame at the default configuration, besides z itself.
    //   FP16 Generator: every tensor, the input included, is an H8 tensor of gen_stream_rows() rows of storage, and the input is
    //                   converted from z chunk by chunk.  With chunks of at most max_chunk frames < Fg (a bounded stream) that is
    //                   gen_stream_capacity(), independent of Fg, and a slide (k_g2_slide) moves a tensor's live rows to the front of its
    //                   storage when a chunk would run past its end.  Otherwise every tensor is whole and never slides:
    //                   2 * (192 + 512 + 17 * (256*8 + 128*64 + 64*128 + 32*256 + 16*512)) = 1,185,152 bytes per frame plus the halos.
    // The stream also reads the per-batch conditioning and the lengths in the persist arena.  Any call that resets the workspace, and a
    // bv2_reserve that regrows either arena, closes the stream.
    struct {
        bool open = false; int B = 0, Fg = 0, frontier = 0;
        GenGraph g; std::vector<H8> t; std::vector<Act> a;  // tensors of the FP16 Generator (t) / of the fp32 c4 Generator (a)
        float* o = nullptr; const float* gdec = nullptr; int g_stride = 0; const int* lens = nullptr;
        int max_chunk = 0;      // > 0: bounded stream
        bool ragged = false;    // FP16: item b runs at its own length min(lens[b], Fg) (bv2_infer_finish_stream_ragged)
        std::vector<int> rows;  // FP16: rows of storage per tensor (gen_stream_rows)
        Act z;                  // FP16: the Generator input z (fp32 c4), converted per chunk
    } gs;
    void ws_reset() { gs.open = false; ws.reset(); }
    long long* h_ylen = nullptr;  // pinned: y_lengths[B <= 4096] + the input-validation mask
    void ensure_h_ylen() { if (!h_ylen) BV2_CUDA(cudaMallocHost(&h_ylen, 4100 * sizeof(long long))); }
    // side streams: the MRF's resblocks (k = 3, 7, 11) of one Generator stage are independent chains of 6 convs
    cudaStream_t side[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev_fork = nullptr, ev_rb[4] = {nullptr, nullptr, nullptr, nullptr};
    void ensure_side_streams() {
        if (ev_fork) return;
        for (int i = 0; i < 4; i++) { BV2_CUDA(cudaStreamCreateWithFlags(&side[i], cudaStreamNonBlocking)); BV2_CUDA(cudaEventCreateWithFlags(&ev_rb[i], cudaEventDisableTiming)); }
        BV2_CUDA(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    }
    bool profiling = false;
    struct StageEv { cudaEvent_t a = nullptr, b = nullptr; bool rec = false; };
    std::map<std::string, StageEv> stage_ev;
    void stage_begin(const char* n, cudaStream_t s) {
        if (!profiling) return;
        StageEv& ev = stage_ev[n];
        if (!ev.a) { BV2_CUDA(cudaEventCreate(&ev.a)); BV2_CUDA(cudaEventCreate(&ev.b)); }
        BV2_CUDA(cudaEventRecord(ev.a, s)); ev.rec = false;
    }
    void stage_end(const char* n, cudaStream_t s) {
        if (!profiling) return;
        StageEv& ev = stage_ev[n];
        BV2_CUDA(cudaEventRecord(ev.b, s)); ev.rec = true;
    }

    ~bv2_engine() {
        if (h_ylen) cudaFreeHost(h_ylen);
        for (int i = 0; i < 4; i++) { if (side[i]) cudaStreamDestroy(side[i]); if (ev_rb[i]) cudaEventDestroy(ev_rb[i]); }
        if (ev_fork) cudaEventDestroy(ev_fork);
        for (auto& kv : stage_ev) { if (kv.second.a) cudaEventDestroy(kv.second.a); if (kv.second.b) cudaEventDestroy(kv.second.b); }
    }

    // ---------------------------------------------------------------- weights
    const HostTensor& W(const std::string& k) const {
        auto it = host.find(k);
        if (it == host.end()) throw Error(BV2_ERR_STATE, "missing weight: " + k);
        return it->second;
    }
    // ---- weight arena.  Every device-resident weight image (SIMT packs, wgmma stage images, embeddings, LayerNorm vectors)
    // lives in ONE allocation filled by ONE cudaMemcpy.  build_weights() runs twice: a measuring pass (sizes only, packing
    // loops skipped) and the real pass that writes into a host mirror at the same offsets.  bv2_save_packed() dumps that
    // arena; bv2_load_packed() re-runs the structure pass with the packing loops skipped and copies the file in (SURVEY 8f.4).
    size_t woff = 0;
    std::vector<uint8_t> wmirror;
    bool wmeasure = false, wfill = true;
    bool packing() const { return wfill && !wmeasure; }  // false: skip the expensive fold / repack loops (only sizes matter)
    float* upload(const std::vector<float>& v) {
        const size_t bytes = (std::max<size_t>(v.size(), 4) * sizeof(float) + 255) & ~(size_t)255;
        const size_t o = woff;
        woff += bytes;
        if (wmeasure) return reinterpret_cast<float*>(o + 256);  // never dereferenced; discarded with the measuring pass
        BV2_CHECK(woff <= warena_bytes, "weight arena overflow");
        if (wfill) std::memcpy(wmirror.data() + o, v.data(), v.size() * sizeof(float));
        return reinterpret_cast<float*>(warena + o);
    }
    // torch.nn.utils.weight_norm fold, dim=0: w = g * v / ||v|| over dims (1,2)  (SURVEY.md §7 H6)
    std::vector<float> fold_wn(const std::string& name, std::vector<int64_t>* shape) const {
        const HostTensor& v = W(name + ".weight_v");
        const HostTensor& g = W(name + ".weight_g");
        int64_t d0 = v.shape[0], inner = v.numel() / d0;
        BV2_CHECK(g.numel() == d0, "weight_g shape " + name);
        std::vector<float> w(v.data.size());
        *shape = v.shape;
        if (!packing()) return w;
        for (int64_t i = 0; i < d0; i++) {
            double n = 0;
            for (int64_t j = 0; j < inner; j++) { double x = v.data[i * inner + j]; n += x * x; }
            float norm = (float)std::sqrt(n);
            float s = g.data[i] / norm;
            for (int64_t j = 0; j < inner; j++) w[i * inner + j] = v.data[i * inner + j] * s;
        }
        *shape = v.shape;
        return w;
    }
    // [Cout][Cin][K] -> packed [Cin][K][Cout_w], Cout_w = Cout rounded up to 4 (+ zero pad)
    ConvW make_conv(const std::vector<float>& w, int Cout, int Cin, int K, const std::vector<float>* bias, int tc_mode = 0, int tc_nt = 0, int tc_kc = 0) {
        ConvW c; c.Cin = Cin; c.Cout = (Cout + 3) / 4 * 4; c.Cout_w = c.Cout; c.K = K;
        std::vector<float> p((size_t)Cin * K * c.Cout_w, 0.f);
        if (packing())
            for (int co = 0; co < Cout; co++)
                for (int ci = 0; ci < Cin; ci++)
                    for (int j = 0; j < K; j++) p[((size_t)ci * K + j) * c.Cout_w + co] = w[((size_t)co * Cin + ci) * K + j];
        c.w = upload(p);
        std::vector<float> b(c.Cout, 0.f);
        if (bias) for (int co = 0; co < Cout; co++) b[co] = (*bias)[co];
        c.b = upload(b);
        if (tc_mode && Cout % 16 == 0) c.tc = tc_pack_weights(*this_uploader(), w, Cout, Cin, K, tc_nt, tc_mode == 2 ? 1 : 0, tc_kc, packing());  // tc_mode: 1 = TF32, 2 = FP16 operands
        return c;
    }
    // uploader functor handed to tc_conv.cuh
    std::function<float*(const std::vector<float>&)>* this_uploader() {
        if (!uploader_) uploader_.reset(new std::function<float*(const std::vector<float>&)>([this](const std::vector<float>& v) { return upload(v); }));
        return uploader_.get();
    }
    std::unique_ptr<std::function<float*(const std::vector<float>&)>> uploader_;

    ConvW conv_from(const std::string& name, bool wn = false, int tc_mode = 0, int tc_nt = 0, int tc_kc = 0) {
        std::vector<int64_t> shp;
        std::vector<float> w;
        if (wn) w = fold_wn(name, &shp);
        else { const HostTensor& t = W(name + ".weight"); w = t.data; shp = t.shape; }
        BV2_CHECK(shp.size() == 3 || shp.size() == 2, "conv weight rank " + name);
        int Cout = (int)shp[0], Cin = (int)shp[1], K = shp.size() == 3 ? (int)shp[2] : 1;
        const std::vector<float>* b = host.count(name + ".bias") ? &W(name + ".bias").data : nullptr;
        return make_conv(w, Cout, Cin, K, b, tc_mode, tc_nt, tc_kc);
    }
    LnW ln_from(const std::string& name) {
        LnW l; l.C = (int)W(name + ".gamma").numel(); l.g = upload(W(name + ".gamma").data); l.b = upload(W(name + ".beta").data);
        return l;
    }
    EncoderW encoder_from(const std::string& name, int n_layers, int kernel, std::vector<float>& gw, std::vector<float>& gb, int tc_mode = 0) {
        EncoderW e; e.kernel = kernel;
        const int H = cfg.hidden_channels, dk = H / cfg.n_heads;
        e.g_off = append_gproj(name + ".spk_emb_linear", gw, gb);
        for (int i = 0; i < n_layers; i++) {
            EncLayerW L;
            std::string a = name + ".attn_layers." + std::to_string(i);
            // fused QKV projection; 1/sqrt(dk) of attentions.py:280 folded into the q rows
            std::vector<float> w((size_t)3 * H * H), b(3 * H);
            const float qs = 1.f / std::sqrt((float)dk);
            const char* nm[3] = {".conv_q", ".conv_k", ".conv_v"};
            for (int p = 0; p < 3; p++) {
                const HostTensor& wt = W(a + nm[p] + ".weight");
                const HostTensor& bt = W(a + nm[p] + ".bias");
                float s = p == 0 ? qs : 1.f;
                for (int i2 = 0; i2 < H * H; i2++) w[(size_t)p * H * H + i2] = wt.data[i2] * s;
                for (int i2 = 0; i2 < H; i2++) b[p * H + i2] = bt.data[i2] * s;
            }
            L.qkv = make_conv(w, 3 * H, H, 1, &b, tc_mode, 96, 64);
            L.o = conv_from(a + ".conv_o", false, tc_mode, tc_mode == 2 ? H : 48, 64);  // FP16 flow: one N tile = all channels (LayerNorm fused into the tail)
            L.relk = upload(W(a + ".emb_rel_k").data);
            L.relv = upload(W(a + ".emb_rel_v").data);
            L.n1 = ln_from(name + ".norm_layers_1." + std::to_string(i));
            L.f1 = conv_from(name + ".ffn_layers." + std::to_string(i) + ".conv_1", false, tc_mode, 128, 64);
            L.f2 = conv_from(name + ".ffn_layers." + std::to_string(i) + ".conv_2", false, tc_mode, 32, 64);  // (one 192-column N tile with the LayerNorm in the tail measured 10 us per layer slower)
            L.n2 = ln_from(name + ".norm_layers_2." + std::to_string(i));
            e.layers.push_back(L);
        }
        return e;
    }
    DdsW dds_from(const std::string& name, int n_layers, int tc_mode = 0) {
        DdsW d;
        for (int i = 0; i < n_layers; i++) {
            std::string s = std::to_string(i);
            d.sep_w.push_back(upload(W(name + ".convs_sep." + s + ".weight").data));  // [C][1][3]
            d.sep_b.push_back(upload(W(name + ".convs_sep." + s + ".bias").data));
            d.c1.push_back(conv_from(name + ".convs_1x1." + s, false, tc_mode, 32));
            d.n1.push_back(ln_from(name + ".norms_1." + s));
            d.n2.push_back(ln_from(name + ".norms_2." + s));
        }
        return d;
    }
    int append_gproj(const std::string& name, std::vector<float>& gw, std::vector<float>& gb, bool wn = false) {
        std::vector<int64_t> shp; std::vector<float> w;
        if (wn) w = fold_wn(name, &shp); else { w = W(name + ".weight").data; shp = W(name + ".weight").shape; }
        BV2_CHECK((int)shp[1] == cfg.gin_channels, "gproj Cin " + name);
        int off = (int)gb.size();
        gw.insert(gw.end(), w.begin(), w.end());
        const auto& b = W(name + ".bias").data;
        gb.insert(gb.end(), b.begin(), b.end());
        return off;
    }

    void finalize(const uint8_t* packed = nullptr, size_t packed_bytes = 0);
    void build_weights();
    void reset_weights() {
        enc_p = EncoderW(); sdp_dds = DdsW(); sdp_flows.clear(); flows.clear(); ups.clear(); resblocks.clear();
        bert_proj = enc_proj = sdp_pre = sdp_proj = dp_c1 = dp_c2 = dp_proj = conv_pre = ConvW();
    }

    // ---------------------------------------------------------------- launch helpers
    int tc_out_tf32 = 0, tc_skip_xform = 0, tc_in_f16 = 0, tc_out_f16 = 0;  // one-shot modifiers for the next tensor-core conv() call
    const LnW* tc_ln = nullptr;                                               // one-shot: LayerNorm fused into the tail
    int tc_gate = 0;                                                          // one-shot: WN gate fused into the tail
    void conv(const ConvW& cw, const Act& x, const Act& y, cudaStream_t s, ConvArgs extra = ConvArgs(), int cin_off = 0,
              int cout_off = 0, bool allow_tc = false) {
        if (allow_tc && cw.tc.w) {
            TcEpi e;
            e.in_slope = extra.in_slope; e.in_mask = extra.in_mask; e.relu = extra.act == 1; e.res_mode = extra.res_mode; e.res = extra.res;
            e.res_C_total = extra.res_C_total; e.res_c_off = extra.res_c_off; e.accumulate = extra.accumulate; e.out_scale = extra.out_scale;
            e.out_mask = extra.out_mask; e.lens = extra.lens; e.bias_b = extra.bias_b; e.bias_b_stride = extra.bias_b_stride;
            e.cin_off = cin_off; e.cout_off = cout_off; e.dil = extra.dil ? extra.dil : 1; e.t_begin = extra.t_begin; e.t_end = extra.t_end;
            e.out_tf32 = tc_out_tf32; e.skip_xform = tc_skip_xform; e.in_f16 = tc_in_f16; e.out_f16 = tc_out_f16;
            BV2_CHECK(x.T == y.T && x.B == y.B, "conv T/B mismatch");
            if (tc_ln) { e.ln_gamma = tc_ln->g; e.ln_beta = tc_ln->b; }
            e.gate = tc_gate; tc_gate = 0;
            tc_out_tf32 = 0; tc_skip_xform = 0; tc_in_f16 = 0; tc_out_f16 = 0; tc_ln = nullptr;
            tc_conv1d(cw.tc, cw.b, x, y, e, s, num_sms);
            launches++;
            return;
        }
        ConvArgs a = extra;
        a.x = x.p; a.Cin_total = x.C; a.cin_off = cin_off; a.Cin = cw.Cin;
        a.w = cw.w; a.Cout_w = cw.Cout_w; a.bias = cw.b;
        a.y = y.p; a.Cout_total = y.C; a.cout_off = cout_off; a.Cout = cw.Cout;
        a.T = x.T; a.B = x.B; a.K = cw.K;
        if (extra.dil == 0) a.dil = 1;
        a.pad = (cw.K - 1) / 2 * a.dil;
        BV2_CHECK(x.T == y.T && x.B == y.B, "conv T/B mismatch");
        launch_conv1d(a, s);
        launches++;
    }
    // token-rate FP32 conv through the cluster split-K kernel (kernels_tok.cuh); false -> caller uses the generic path
    bool tok_conv(const ConvW& cw, const Act& x, const Act& y, cudaStream_t s, const ConvArgs& e, const LnW* ln = nullptr, const float* ln_res = nullptr,
                  int mask_pre = 0, int cout_off = 0) {
        TokGemmArgs a{};
        a.x = x.p; a.Cin_total = x.C; a.cin_off = 0; a.Cin = cw.Cin;
        a.w = cw.w; a.Cout_w = cw.Cout_w; a.bias = cw.b; a.bias_b = e.bias_b; a.bias_b_stride = e.bias_b_stride;
        a.y = y.p; a.Cout_total = y.C; a.cout_off = cout_off;
        a.res = ln_res; a.res_C_total = 192; a.gamma = ln ? ln->g : nullptr; a.beta = ln ? ln->b : nullptr;
        a.lens = e.lens; a.T = x.T; a.B = x.B; a.relu = e.act == 1; a.in_mask = e.in_mask; a.out_mask = e.out_mask; a.mask_pre = mask_pre;
        if (e.res || e.accumulate || e.in_slope != 1.f || e.out_scale != 1.f || (e.dil != 0 && e.dil != 1) || cw.Cin % 16) return false;
        if (!launch_tok_gemm(a, cw.K, cw.Cout, s)) return false;
        launches++;
        return true;
    }
    void layernorm(const LnW& w, const Act& x, const float* add, const Act& y, cudaStream_t s, int gelu, const float* post_res,
                   const int* lens, int out_mask) {
        LnArgs a; a.x = x.p; a.add = add; a.gamma = w.g; a.beta = w.b; a.y = y.p; a.post_res = post_res; a.C = x.C; a.T = x.T;
        a.B = x.B; a.gelu = gelu; a.relu_in = 0; a.out_mask = out_mask; a.lens = lens; a.eps = 1e-5f;
        BV2_CHECK(w.C == x.C, "LN C");
        launch_layernorm(a, s);
        launches++;
    }
    static dim3 grid_tcb(int T, int C, int B) { return dim3(cdiv(T, 128), C / 4, B); }

    void debug(const std::string& name, const Act& a, int c4 = 1) { dbg[name] = DebugBuf{a.p, a.B, a.C, a.T, c4}; }
    void debug_plain(const std::string& name, const float* p, int B, int C, int T) { dbg[name] = DebugBuf{p, B, C, T, 0}; }

    // ---------------------------------------------------------------- stages
    void run_gproj(const float* g, int B, float* out, cudaStream_t s) {
        dim3 grid(cdiv(gproj_n, 8), B);
        k_linear_g<<<grid, 256, 0, s>>>(gproj_w, gproj_b, g, out, gproj_n, cfg.gin_channels);
        BV2_CUDA(cudaGetLastError()); launches++;
    }
    void run_encoder(const EncoderW& E, Act x, const int* lens, const float* gproj, cudaStream_t s, int tc);  // tc: 0 SIMT, 1 TF32, 2 FP16 + fused attention
    void run_dds(const DdsW& D, Act x, const int* lens, cudaStream_t s);
    void run_text_encoder(int B, int T, const int64_t* x, const int64_t* tone, const int64_t* lang, const float* bert,
                          const float* ja, const float* en, const int* lens, const float* gproj, Act& h, Act& stats, cudaStream_t s);
    void run_durations(Act h, const int* lens, const float* gproj, const float* noise_w, float nsw, const float* nsw_b, float* z,
                       Act& dp_out, int* zch, cudaStream_t s);
    void run_dp(Act h, const int* lens, const float* gproj, Act& dp_out, Act xg, Act d1, Act d2, cudaStream_t s);
    void run_flow(Act z, const int* lens, const float* gproj, cudaStream_t s);
    // ragged: batch item b runs at its own length lens[b] (clamped to z.T) instead of z.T: FP16 Generator only, else BV2_ERR_ARG
    void run_generator(Act z, const int* lens_or_null, const float* gdec, int g_stride, float* o, cudaStream_t s, bool ragged = false);
    void run_generator_g2(Act z, const int* lens_or_null, const float* gdec, int g_stride, float* o, cudaStream_t s, bool ragged);
    H8 g2_h8(int B, int C, int T, int rows = -1);
    H8 g2_input(Act z, const int* lens_or_null, cudaStream_t s);
    size_t stream_bytes(int B, int Fg, int max_chunk) const;
    void gen_stream_open(Act z, const int* lens_or_null, const float* gdec, int g_stride, float* o, int max_chunk, bool ragged);
    void g2_stream_prepare(int done, int target, cudaStream_t s);
    void gen_windows(const GenGraph& g, const std::vector<GenWin>& w, std::vector<Act>& t, bool stream, const int* lens_or_null, const float* gdec,
                     int g_stride, float* o, cudaStream_t s);
    void g2_windows(const GenGraph& g, const std::vector<GenWin>& w, std::vector<H8>& t, bool stream, const float* gdec, int g_stride,
                    float* o, cudaStream_t s, const int* ragged_lens = nullptr);
    int* lens_to_device(const int64_t* x_lengths_dev, int B, Arena& ar, cudaStream_t s);
    // ids inside their tables, 1 <= lengths <= T (the reference raises IndexError / a shape error): device-side check into *err_dev
    void launch_validate(int B, int T, const int64_t* x, const int64_t* tone, const int64_t* lang, const int64_t* sid, const int64_t* lens,
                         int* err_dev, cudaStream_t s) {
        BV2_CUDA(cudaMemsetAsync(err_dev, 0, sizeof(int), s));
        const int n = B * std::max(T, 1);
        k_validate_inputs<<<std::min(cdiv(n, 256), 64), 256, 0, s>>>(reinterpret_cast<const long long*>(x), reinterpret_cast<const long long*>(tone),
                                                                   reinterpret_cast<const long long*>(lang), reinterpret_cast<const long long*>(sid),
                                                                   reinterpret_cast<const long long*>(lens), B, T, cfg.n_vocab, cfg.num_tones,
                                                                   cfg.num_languages, cfg.n_speakers, err_dev);
        BV2_CUDA(cudaGetLastError()); launches++;
    }
    static void throw_if_bad_inputs(int mask) {
        if (!mask) return;
        const char* weight = "non-finite speaker-mix weight";
        if (!(mask & 31)) throw Error(BV2_ERR_ARG, weight);  // no "index out of range": a ValueError in Python, not an IndexError
        std::string m = "index out of range:";
        if (mask & 1) m += " phoneme id (n_vocab)";
        if (mask & 2) m += " tone id";
        if (mask & 4) m += " language id";
        if (mask & 8) m += " speaker id (n_speakers)";
        if (mask & 16) m += " x_lengths (need 1 <= len <= T)";
        if (mask & 32) m += std::string("; ") + weight;
        throw Error(BV2_ERR_ARG, m);
    }
    // stage entry points (not on the hot path): validate, read the verdict back synchronously
    void validate_sync(int B, int T, const int64_t* x, const int64_t* tone, const int64_t* lang, const int64_t* sid, const int64_t* lens, cudaStream_t s) {
        int* d = reinterpret_cast<int*>(ws.alloc(4));
        launch_validate(B, T, x, tone, lang, sid, lens, d, s);
        int h = 0;
        BV2_CUDA(cudaMemcpyAsync(&h, d, sizeof(int), cudaMemcpyDeviceToHost, s));
        BV2_CUDA(cudaStreamSynchronize(s));
        throw_if_bad_inputs(h);
    }
    // wave [B][L] fp32 -> int16 (peak-normalised per utterance over n_valid samples; ylen given in units of `unit` samples)
    void pcm16(const float* wave, int B, long long L, const long long* ylen, int unit, long long* nval_scratch, unsigned* peak, int16_t* out, cudaStream_t s) {
        const long long* nv = ylen;
        if (ylen && unit != 1) {
            k_scale_i64<<<cdiv(B, 128), 128, 0, s>>>(ylen, nval_scratch, unit, B);
            BV2_CUDA(cudaGetLastError()); launches++;
            nv = nval_scratch;
        }
        BV2_CUDA(cudaMemsetAsync(peak, 0, (size_t)B * sizeof(unsigned), s));
        dim3 g1((unsigned)std::min<long long>((L + 255) / 256, 256), B), g2((unsigned)((L + 255) / 256), B);
        k_wave_peak<<<g1, 256, 0, s>>>(wave, L, nv, peak);
        k_wave_to_pcm16<<<g2, 256, 0, s>>>(wave, L, nv, peak, reinterpret_cast<short*>(out));
        BV2_CUDA(cudaGetLastError()); launches += 2;
    }
    void begin_call() {
        std::lock_guard<std::mutex> lk(g_err_mu);
        call_gen = g_err_flags[device].generation;
    }
    void check_device_error() {
        std::lock_guard<std::mutex> lk(g_err_mu);
        DeviceErrFlag& f = g_err_flags[device];
        if (f.host && *reinterpret_cast<volatile int*>(f.host)) {
            *f.host = 0;
            tc_clear_error();
            f.generation++;
        }
        if (f.generation != call_gen)
            throw Error(BV2_ERR_INTERNAL, "device-side barrier timeout in a wgmma kernel on this device (results of this call are invalid)");
    }
};

// ------------------------------------------------------------------------------------------------
__global__ void k_i64_to_i32(const long long* __restrict__ a, int* __restrict__ b, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) b[i] = (int)a[i];
}
// lengths clamped to [1, hi] (bv2_generator_ragged: an out-of-range length never becomes an out-of-range row)
__global__ void k_lengths_clamp(const long long* __restrict__ a, int* __restrict__ b, int n, int hi) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) b[i] = (int)max(1ll, min((long long)hi, a[i]));
}
// b = a * s over blockIdx.y = item rows of per_item elements; s_item ([items], bv2_infer_begin_items): item y's own s
__global__ void k_scale_copy(const float* __restrict__ a, float* __restrict__ b, float s, const float* __restrict__ s_item, int per_item) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= per_item) return;
    size_t i = (size_t)blockIdx.y * per_item + j;
    if (s_item) s = s_item[blockIdx.y];
    b[i] = a[i] * s;
}

int* bv2_engine::lens_to_device(const int64_t* xl, int B, Arena& ar, cudaStream_t s) {
    int* lens = reinterpret_cast<int*>(ar.alloc(B));
    k_i64_to_i32<<<cdiv(B, 128), 128, 0, s>>>(reinterpret_cast<const long long*>(xl), lens, B);
    BV2_CUDA(cudaGetLastError()); launches++;
    return lens;
}

void bv2_engine::finalize(const uint8_t* packed, size_t packed_bytes) {
    const bv2_config& c = cfg;
    const int H = c.hidden_channels, I = c.inter_channels;
    BV2_CHECK(H % 4 == 0 && I % 8 == 0 && c.filter_channels % 4 == 0 && c.gin_channels % 4 == 0, "channel multiples of 4");
    BV2_CHECK(H / c.n_heads == 96, "head dim 96 is the only instantiated attention kernel");
    BV2_CHECK(c.window_size <= 4, "window_size <= 4 (relative-position tables of the attention kernels hold 9 slots)");
    BV2_CHECK(c.n_flows >= 1 && c.n_flows <= 16, "n_flows");
    BV2_CHECK(c.sdp_num_bins == 10 && c.sdp_kernel == 3, "sdp spline bins/kernel");
    BV2_CUDA(cudaSetDevice(device));
    {   // > 48 KB dynamic shared memory opt-in (a per-device function attribute) + the device error flag: once per device and process
        std::lock_guard<std::mutex> lk(g_err_mu);
        DeviceErrFlag& f = g_err_flags[device];
        if (!f.host) f.host = tc_init_device();
    }
    tok_init_device();
    shape_table.clear();
    for (const auto& kv : host) shape_table.emplace_back(kv.first, kv.second.shape);
    std::sort(shape_table.begin(), shape_table.end());
    // pass 1: sizes
    wmeasure = true; woff = 0;
    build_weights();
    const size_t total = woff;
    reset_weights();
    BV2_CUDA(cudaMalloc(reinterpret_cast<void**>(&warena), total));
    warena_owner.reset(warena, [](uint8_t* p) { cudaFree(p); });
    warena_bytes = total;
    wmeasure = false; woff = 0;
    if (packed) {
        BV2_CHECK(packed_bytes == total, "packed weight file does not match this configuration (arena size)");
        wfill = false;
        build_weights();
        BV2_CUDA(cudaMemcpy(warena, packed, total, cudaMemcpyHostToDevice));
    } else {
        wmirror.assign(total, 0);
        wfill = true;
        build_weights();
        BV2_CUDA(cudaMemcpy(warena, wmirror.data(), total, cudaMemcpyHostToDevice));
        std::vector<uint8_t>().swap(wmirror);
    }
    ensure_h_ylen();
    if (use_g2) {  // same bytes whichever way the arena was filled (state_dict or packed file)
        BV2_CHECK(c.upsample_initial_channel >> c.n_ups == 16, "conv_post kernel instantiated for 16 input channels, 7 taps");
        BV2_CUDA(cudaMemcpy(conv_post_h.w, conv_post_w, sizeof(conv_post_h.w), cudaMemcpyDeviceToHost));
    }
    host.clear();
    finalized = true;
}

void bv2_engine::build_weights() {
    const bv2_config& c = cfg;
    const int H = c.hidden_channels, I = c.inter_channels;
    std::vector<float> gw, gb;
    // Precision policy: stages that feed ceil(durations) never run on the tensor-core path: a TF32 / FP16 product carries an 11-bit
    // significand, so the error grows with the reduction length and misses the fp32-class accuracy ceil() needs.  These
    // stages therefore stay on FP32 FMA (SIMT) in every engine (x3 = 0: no tensor-core weight image is packed for them).
    const int x3 = 0;
    // ---- enc_p (reference models.py:333-375)
    emb = upload(W("enc_p.emb.weight").data);
    temb = upload(W("enc_p.tone_emb.weight").data);
    lemb = upload(W("enc_p.language_emb.weight").data);
    {
        // three 1024->H projections concatenated along Cin (one K=3*1024 contraction)
        const char* nm[3] = {"enc_p.bert_proj", "enc_p.ja_bert_proj", "enc_p.en_bert_proj"};
        const int D = c.bert_dim;
        std::vector<float> w((size_t)H * 3 * D), b(H, 0.f);
        for (int p = 0; p < 3; p++) {
            const HostTensor& wt = W(std::string(nm[p]) + ".weight");
            const HostTensor& bt = W(std::string(nm[p]) + ".bias");
            for (int co = 0; co < H; co++) {
                for (int ci = 0; ci < D; ci++) w[(size_t)co * 3 * D + p * D + ci] = wt.data[(size_t)co * D + ci];
                b[co] += bt.data[co];
            }
        }
        bert_proj = make_conv(w, H, 3 * D, 1, &b, x3, 32);
    }
    enc_p = encoder_from("enc_p.encoder", c.n_layers, c.kernel_size, gw, gb, x3);
    enc_proj = conv_from("enc_p.proj", false, x3, 32);
    // ---- sdp (reference models.py:148-195); flows[1] is the dropped "useless vflow" (:247)
    sdp_pre = conv_from("sdp.pre", false, x3, 32);
    sdp_proj = conv_from("sdp.proj", false, x3, 32);
    sdp_dds = dds_from("sdp.convs", c.sdp_dds_layers, x3);
    goff_sdp = append_gproj("sdp.cond", gw, gb);
    sdp_flows.resize(2 * c.sdp_n_flows + 1);
    for (int i = 2; i <= c.sdp_n_flows; i++) {
        std::string f = "sdp.flows." + std::to_string(2 * i - 1);
        ConvFlowW cf;
        cf.pre_w = upload(W(f + ".pre.weight").data);
        cf.pre_b = upload(W(f + ".pre.bias").data);
        cf.dds = dds_from(f + ".convs", c.sdp_dds_layers, x3);
        cf.proj = conv_from(f + ".proj", false, x3, 32);
        sdp_flows[2 * i - 1] = cf;
    }
    for (int i = 0; i < 2; i++) { ea_m[i] = W("sdp.flows.0.m").data[i]; ea_logs[i] = W("sdp.flows.0.logs").data[i]; }
    dconst = (float)std::log(std::exp(1.0 - 1e-3) - 1.0);  // transforms.py:69
    // ---- dp (reference models.py:259-299)
    dp_c1 = conv_from("dp.conv_1", false, x3, 32); dp_c2 = conv_from("dp.conv_2", false, x3, 32); dp_proj = conv_from("dp.proj");
    dp_n1 = ln_from("dp.norm_1"); dp_n2 = ln_from("dp.norm_2");
    goff_dp = append_gproj("dp.cond", gw, gb);
    // ---- flow (reference models.py:82-145 / 403-445): Flip folded into pre/post channel order
    const int half = I / 2, n = c.n_flows;
    flows.resize(n);
    // generator_precision: 0 = fp32 SIMT everywhere; 1 = TF32 wgmma (flow + Generator); 2 = FP16-operand wgmma Generator
    // (same 11-bit significand as TF32, fp32 accumulate, 16-bit activations in HBM: k_g2_conv, tc_gen.cuh) + TF32 flow
    // 3 = FP16 operands in the flow too, with the fused attention kernel (tc_attn.cuh)
    const int tc = c.generator_precision == 3 ? 2 : (c.generator_precision ? 1 : 0);
    const int gtc = c.generator_precision >= 2 ? 2 : tc;
    flow_tc = tc;
    if (tc == 2) tc_flow_attn_init_device();
    use_g2 = gtc == 2 ? 1 : 0;
    if (use_g2) g2_init_device();
    for (int i = 0; i < n; i++) {
        CouplingW& fl = flows[i];
        std::string f = "flow.flows." + std::to_string(2 * i);
        fl.s = ((n - 1 - i) % 2 == 0) ? 1 : 0;
        const HostTensor& pw = W(f + ".pre.weight");   // [H][half][1]
        const HostTensor& pb = W(f + ".pre.bias");
        const HostTensor& qw = W(f + ".post.weight");  // [half][H][1]
        const HostTensor& qb = W(f + ".post.bias");
        BV2_CHECK((int)qw.shape[0] == half, "mean_only coupling expected");
        std::vector<float> w1(pw.data), w2(qw.data), b2(qb.data);
        if (fl.s) {
            for (int co = 0; co < H; co++)
                for (int ci = 0; ci < half; ci++) w1[(size_t)co * half + ci] = pw.data[(size_t)co * half + (half - 1 - ci)];
            for (int co = 0; co < half; co++) {
                for (int ci = 0; ci < H; ci++) w2[(size_t)co * H + ci] = qw.data[(size_t)(half - 1 - co) * H + ci];
                b2[co] = qb.data[half - 1 - co];
            }
        }
        fl.pre = make_conv(w1, H, half, 1, &pb.data, tc, 96);
        fl.post = make_conv(w2, half, H, 1, &b2, tc, 48);
        if (c.use_transformer_flow) {
            fl.enc = encoder_from(f + ".enc", c.n_layers_trans_flow, c.flow_kernel_size, gw, gb, tc);
        } else {
            const int L = c.wn_layers;
            fl.wn_g_off = append_gproj(f + ".enc.cond_layer", gw, gb, true);
            if (tc == 2) {
                // FP16 engine: the gate runs in the in_layer conv's tail, which needs tanh / sigmoid pre-activations of a channel in adjacent
                // accumulator columns -> interleave the output rows (c, H + c) of every in_layer and of its slice of cond_layer
                for (int l = 0; l < L; l++) {
                    const size_t G = (size_t)c.gin_channels;
                    std::vector<float> tw(gw.begin() + ((size_t)fl.wn_g_off + 2 * (size_t)H * l) * G, gw.begin() + ((size_t)fl.wn_g_off + 2 * (size_t)H * (l + 1)) * G);
                    std::vector<float> tb(gb.begin() + fl.wn_g_off + 2 * H * l, gb.begin() + fl.wn_g_off + 2 * H * (l + 1));
                    for (int ch = 0; ch < H; ch++)
                        for (int hf = 0; hf < 2; hf++) {
                            std::copy(tw.begin() + ((size_t)hf * H + ch) * G, tw.begin() + ((size_t)hf * H + ch + 1) * G, gw.begin() + ((size_t)fl.wn_g_off + 2 * (size_t)H * l + 2 * ch + hf) * G);
                            gb[fl.wn_g_off + 2 * H * l + 2 * ch + hf] = tb[hf * H + ch];
                        }
                }
            }
            for (int l = 0; l < L; l++) {
                if (tc == 2) {
                    std::vector<int64_t> shp;
                    std::vector<float> w = fold_wn(f + ".enc.in_layers." + std::to_string(l), &shp), wi(w.size());
                    const auto& b = W(f + ".enc.in_layers." + std::to_string(l) + ".bias").data;
                    std::vector<float> bi(b.size());
                    const size_t row = (size_t)shp[1] * shp[2];
                    for (int ch = 0; ch < H; ch++)
                        for (int hf = 0; hf < 2; hf++) {
                            if (packing()) std::copy(w.begin() + ((size_t)hf * H + ch) * row, w.begin() + ((size_t)hf * H + ch + 1) * row, wi.begin() + ((size_t)2 * ch + hf) * row);
                            bi[2 * ch + hf] = b[hf * H + ch];
                        }
                    fl.wn_in.push_back(make_conv(wi, 2 * H, H, (int)shp[2], &bi, tc, 128));
                } else
                fl.wn_in.push_back(conv_from(f + ".enc.in_layers." + std::to_string(l), true, tc, 128));
                std::vector<int64_t> shp;
                std::vector<float> w = fold_wn(f + ".enc.res_skip_layers." + std::to_string(l), &shp);
                const auto& b = W(f + ".enc.res_skip_layers." + std::to_string(l) + ".bias").data;
                if (l < L - 1) {
                    std::vector<float> wr(w.begin(), w.begin() + (size_t)H * H), ws(w.begin() + (size_t)H * H, w.end());
                    std::vector<float> br(b.begin(), b.begin() + H), bs(b.begin() + H, b.end());
                    fl.wn_res.push_back(make_conv(wr, H, H, 1, &br, tc, 96));
                    fl.wn_skip.push_back(make_conv(ws, H, H, 1, &bs, tc, 96));
                } else {
                    fl.wn_skip.push_back(make_conv(w, H, H, 1, &b, tc, 96));
                }
            }
        }
    }
    // ---- dec (reference models.py:490-564)
    conv_pre = conv_from("dec.conv_pre", false, gtc, 128, use_g2 ? g2_kc(I) : 0);
    goff_dec = append_gproj("dec.cond", gw, gb);
    int ch = c.upsample_initial_channel;
    for (int i = 0; i < c.n_ups; i++) {
        std::vector<int64_t> shp;
        std::vector<float> w = fold_wn("dec.ups." + std::to_string(i), &shp);  // [Cin][Cout][K]
        UpW u; u.Cin = (int)shp[0]; u.Cout = (int)shp[1]; u.K = (int)shp[2]; u.u = c.upsample_rates[i];
        BV2_CHECK(u.K % u.u == 0 && u.K <= 16 && u.Cin == ch && u.Cout == ch / 2 && (u.K - u.u) % 2 == 0, "upsample config");
        std::vector<float> p((size_t)u.Cin * u.K * u.Cout);
        if (packing())
        for (int ci = 0; ci < u.Cin; ci++)
            for (int co = 0; co < u.Cout; co++)
                for (int j = 0; j < u.K; j++) p[((size_t)ci * u.K + j) * u.Cout + co] = w[((size_t)ci * u.Cout + co) * u.K + j];
        u.w = upload(p); u.b = upload(W("dec.ups." + std::to_string(i) + ".bias").data);
        if (use_g2) u.tc = tc_pack_upsample(*this_uploader(), w, u.Cin, u.Cout, u.K, u.u, g2_kc(u.Cin), 1, packing(), 128);
        else if (gtc) u.tc = tc_pack_upsample(*this_uploader(), w, u.Cin, u.Cout, u.K, u.u, 32, 0, packing());
        ups.push_back(u);
        ch /= 2;
        for (int j = 0; j < c.n_resblock_kernels; j++) {
            ResBlockW rb; rb.k = c.resblock_kernel_sizes[j];
            std::string r = "dec.resblocks." + std::to_string(i * c.n_resblock_kernels + j);
            for (int d = 0; d < c.n_dilations; d++) {
                rb.dil.push_back(c.resblock_dilation_sizes[j][d]);
                const int kc = use_g2 ? g2_kc(ch) : 32;  // persistent kernels hide latency with deep rings: fewer, larger chunks
                const int nt0 = use_g2 ? g2_nt(ch) : 0;
                rb.c1.push_back(conv_from(r + ".convs1." + std::to_string(d), true, gtc, nt0, kc));
                rb.c2.push_back(conv_from(r + ".convs2." + std::to_string(d), true, gtc, nt0, kc));
            }
            resblocks.push_back(rb);
        }
    }
    BV2_CHECK(ch == 16, "conv_post kernel instantiated for 16 input channels");
    hop = 1; for (int i = 0; i < c.n_ups; i++) hop *= c.upsample_rates[i];
    conv_post_w = upload(W("dec.conv_post.weight").data);  // [1][16][7]
    emb_g = upload(W("emb_g.weight").data);
    gproj_n = (int)gb.size();
    gproj_w = upload(gw); gproj_b = upload(gb);
}

// ------------------------------------------------------------------------------------------------
// attentions.Encoder.forward (reference attentions.py:103-120)
void bv2_engine::run_encoder(const EncoderW& E, Act x, const int* lens, const float* gproj, cudaStream_t s, int tc) {
    const int B = x.B, T = x.T, H = x.C, Fc = cfg.filter_channels, nh = cfg.n_heads;
    const size_t mark = ws.used();
    Act qkv = ws.act(B, 3 * H, T), att = ws.act(B, H, T), y = ws.act(B, H, T), f = ws.act(B, Fc, T);
    const int nl = (int)E.layers.size();
    for (int i = 0; i < nl; i++) {
        const EncLayerW& L = E.layers[i];
        if (i == cfg.cond_layer_idx) {
            k_add_bvec_mask<<<grid_tcb(T, H, B), 128, 0, s>>>(x.p, gproj + E.g_off, gproj_n, H, T, lens);
            BV2_CUDA(cudaGetLastError()); launches++;
        }
        if (tc == 2) {
            // FP16 engine: the QKV projection's epilogue writes 16-bit c8 q|k|v (the operand images of the fused attention kernel),
            // the attention kernel writes a 16-bit c8 output that conv_o consumes without a prologue
            const size_t mk = ws.used();
            Act qkv16; qkv16.B = B; qkv16.C = 3 * H; qkv16.T = T; qkv16.p = ws.alloc((size_t)B * 3 * H * T / 2);
            Act att16; att16.B = B; att16.C = H; att16.T = T; att16.p = ws.alloc((size_t)B * H * T / 2);
            tc_out_f16 = 1;
            conv(L.qkv, x, qkv16, s, ConvArgs(), 0, 0, true);
            tc_flow_attn(qkv16, att16, L.relk, L.relv, lens, nh, (int)cfg.window_size, s, num_sms); launches++;
            {   // x = norm_1(x + conv_o(att)): LayerNorm runs in the conv's tail; the residual tile is staged in shared memory by TMA (small grids)
                // or pre-loaded into the accumulator (more CTAs than SMs)
                ConvArgs ao; ao.res = x.p; ao.res_mode = 1; ao.res_C_total = H;
                tc_in_f16 = 1; tc_ln = &L.n1;
                conv(L.o, att16, x, s, ao, 0, 0, true);
            }
            ws.release(mk);
            {
                // FFN hidden tensor as the 16-bit operand image of conv_2 (relu and x_mask applied by conv_1's tail, the conv's zero padding
                // cleared in the staged tile): conv_2 runs without an operand prologue (no fp32 -> f16 conversion of its 768-channel input)
                Act f16 = f;  // same workspace block, half of it used
                ConvArgs a1; a1.in_mask = 1; a1.act = 1; a1.out_mask = 1; a1.lens = lens;
                tc_out_f16 = 1;
                conv(L.f1, x, f16, s, a1, 0, 0, true);
                ConvArgs a2; a2.out_mask = 1; a2.lens = lens;
                tc_in_f16 = 1;
                conv(L.f2, f16, y, s, a2, 0, 0, true);
                layernorm(L.n2, x, y.p, x, s, 0, nullptr, lens, i == nl - 1 ? 1 : 0);
            }
            continue;
        }
        if (tc == 0 && H == 192) {
            // FP32 token-rate layer: 5 launches (qkv | attention | conv_o + residual + LayerNorm | FFN conv_1 + relu | FFN conv_2 + mask +
            // residual + LayerNorm) instead of 7, the dense convs on the cluster split-K kernel
            if (!tok_conv(L.qkv, x, qkv, s, ConvArgs())) conv(L.qkv, x, qkv, s, ConvArgs());
            dim3 grid(cdiv(T, 16), nh, B);
            k_attention_rel<96><<<grid, 128, 0, s>>>(qkv.p, L.relk, L.relv, att.p, H, T, lens, cfg.window_size);
            BV2_CUDA(cudaGetLastError()); launches++;
            if (!tok_conv(L.o, att, x, s, ConvArgs(), &L.n1, x.p)) {
                conv(L.o, att, y, s, ConvArgs());
                layernorm(L.n1, x, y.p, x, s, 0, nullptr, lens, 0);
            }
            ConvArgs a1; a1.in_mask = 1; a1.act = 1; a1.lens = lens;
            if (!tok_conv(L.f1, x, f, s, a1)) conv(L.f1, x, f, s, a1);
            ConvArgs a2; a2.in_mask = 1; a2.lens = lens; a2.out_mask = i == nl - 1 ? 1 : 0;
            if (!tok_conv(L.f2, f, x, s, a2, &L.n2, x.p, 1)) {
                ConvArgs a2b; a2b.in_mask = 1; a2b.out_mask = 1; a2b.lens = lens;
                conv(L.f2, f, y, s, a2b);
                layernorm(L.n2, x, y.p, x, s, 0, nullptr, lens, i == nl - 1 ? 1 : 0);
            }
            continue;
        }
        tc_out_tf32 = tc ? 1 : 0;  // q, k, v feed tensor-core GEMMs directly
        conv(L.qkv, x, qkv, s, ConvArgs(), 0, 0, tc);
        tc_out_tf32 = 0;
        if (tc) {
            // tensor-core attention: S = Q.K^T (wgmma) -> softmax + relative terms (SIMT) -> att += P.V (wgmma)
            const size_t mk = ws.used();
            const int Fp = (T + 127) / 128 * 128;
            Act S = ws.act(B * nh, Fp, T);
            float* vt = ws.alloc((size_t)B * nh * Fp * 96);
            dim3 gv(cdiv(Fp, 128), 24, B * nh);
            launch_pdl(k_pack_vt<96>, gv, dim3(128), 0, s, (const float*)qkv.p, vt, H, nh, T, Fp, lens); launches++;
            tc_attn_qk(qkv, H, nh, S, s); launches++;
            dim3 gs(cdiv(T, 32), B * nh);
            launch_pdl(k_attn_softmax<96, 16>, gs, dim3(512), 0, s, (const float*)qkv.p, S.p, (const float*)L.relk, (const float*)L.relv, att.p, H, nh, T, Fp,
                       lens, (int)cfg.window_size);
            launches++;
            tc_attn_pv(S, vt, H, nh, att, s); launches++;
            ws.release(mk);
        } else {
            dim3 grid(cdiv(T, 16), nh, B);
            k_attention_rel<96><<<grid, 128, 0, s>>>(qkv.p, L.relk, L.relv, att.p, H, T, lens, cfg.window_size);
            BV2_CUDA(cudaGetLastError()); launches++;
        }
        tc_skip_xform = tc ? 1 : 0;  // att was rounded by the P.V tail
        conv(L.o, att, y, s, ConvArgs(), 0, 0, tc);
        tc_skip_xform = 0;
        layernorm(L.n1, x, y.p, x, s, 0, nullptr, lens, 0);
        ConvArgs a1; a1.in_mask = 1; a1.act = 1; a1.lens = lens;
        conv(L.f1, x, f, s, a1, 0, 0, tc);
        ConvArgs a2; a2.in_mask = 1; a2.out_mask = 1; a2.lens = lens;
        conv(L.f2, f, y, s, a2, 0, 0, tc);
        layernorm(L.n2, x, y.p, x, s, 0, nullptr, lens, i == nl - 1 ? 1 : 0);
    }
    ws.release(mark);
}

// modules.DDSConv.forward without the optional g add (reference modules.py:118-130)
void bv2_engine::run_dds(const DdsW& D, Act x, const int* lens, cudaStream_t s) {
    const int B = x.B, T = x.T, C = x.C;
    const size_t mark = ws.used();
    const int nl0 = (int)D.c1.size();
    if (C == 192 && nl0 >= 2) {
        // one launch per layer (kernels_tok.cuh); the layer reads a +-dilation halo, so it ping-pongs between buffers and the last
        // layer lands in x again
        Act tmp[2] = {ws.act(B, C, T), ws.act(B, C, T)};
        int dil = 1;
        for (int i = 0; i < nl0; i++) {
            DdsArgs a;
            a.x = i == 0 ? x.p : tmp[(i - 1) & 1].p; a.y = i == nl0 - 1 ? x.p : tmp[i & 1].p;
            a.dw_w = D.sep_w[i]; a.dw_b = D.sep_b[i]; a.w1 = D.c1[i].w; a.b1 = D.c1[i].b;
            a.g1 = D.n1[i].g; a.be1 = D.n1[i].b; a.g2 = D.n2[i].g; a.be2 = D.n2[i].b;
            a.lens = lens; a.T = T; a.B = B; a.dil = dil; a.last = i == nl0 - 1;
            launch_dds_layer(a, C, s); launches++;
            dil *= cfg.sdp_kernel;
        }
        ws.release(mark);
        return;
    }
    Act y = ws.act(B, C, T), y2 = ws.act(B, C, T);
    const int nl = (int)D.c1.size();
    int dil = 1;
    for (int i = 0; i < nl; i++) {
        {   // depthwise dilated conv + LayerNorm + GELU in one launch (the output row of the conv is the LN row)
            LnArgs a; a.x = x.p; a.add = nullptr; a.gamma = D.n1[i].g; a.beta = D.n1[i].b; a.y = y.p; a.post_res = nullptr; a.C = C; a.T = T;
            a.B = B; a.gelu = 1; a.relu_in = 0; a.out_mask = 0; a.lens = lens; a.eps = 1e-5f;
            a.dw_w = D.sep_w[i]; a.dw_b = D.sep_b[i]; a.dw_dil = dil;
            launch_layernorm(a, s); launches++;
        }
        conv(D.c1[i], y, y2, s, ConvArgs(), 0, 0, true);
        layernorm(D.n2[i], y2, nullptr, x, s, 1, x.p, lens, i == nl - 1 ? 1 : 0);
        dil *= cfg.sdp_kernel;
    }
    ws.release(mark);
}

// TextEncoder.forward (reference models.py:377-400)
void bv2_engine::run_text_encoder(int B, int T, const int64_t* x, const int64_t* tone, const int64_t* lang, const float* bert,
                                  const float* ja, const float* en, const int* lens, const float* gproj, Act& h, Act& stats,
                                  cudaStream_t s) {
    const int H = cfg.hidden_channels, D = cfg.bert_dim;
    Act proj = ws.act(B, H, T);
    bool done = false;
    if (H == 192) {
        // BERT ingest (SURVEY.md section 8f.3): the three [B,1024,T] feature tensors are read in the layout get_text hands them over,
        // one K = 3072 contraction on the cluster split-K kernel (no staging transposes, no intermediate tensor)
        TokGemmArgs a{};
        a.plain[0] = bert; a.plain[1] = ja; a.plain[2] = en; a.plain_C = D;
        a.Cin_total = 3 * D; a.Cin = 3 * D; a.w = bert_proj.w; a.Cout_w = bert_proj.Cout_w; a.bias = bert_proj.b;
        a.y = proj.p; a.Cout_total = H; a.T = T; a.B = B;
        done = launch_tok_gemm(a, 1, H, s);
        if (done) launches++;
    }
    if (!done) {
        Act bc = ws.act(B, 3 * D, T);
        const float* srcs[3] = {bert, ja, en};
        for (int p = 0; p < 3; p++) {
            k_plain_to_c4<<<grid_tcb(T, D, B), 128, 0, s>>>(srcs[p], D, (long long)D * T, T, bc.p, 3 * D, p * D, T, nullptr, 1.f);
            BV2_CUDA(cudaGetLastError()); launches++;
        }
        conv(bert_proj, bc, proj, s, ConvArgs(), 0, 0, true);
    }
    k_embed_sum<<<grid_tcb(T, H, B), 128, 0, s>>>(proj.p, reinterpret_cast<const long long*>(x), reinterpret_cast<const long long*>(tone),
                                                  reinterpret_cast<const long long*>(lang), emb, temb, lemb, h.p, H, T, lens,
                                                  std::sqrt((float)H), cfg.n_vocab, cfg.num_tones, cfg.num_languages);
    BV2_CUDA(cudaGetLastError()); launches++;
    run_encoder(enc_p, h, lens, gproj, s, 0);  // feeds ceil(durations): FP32 FMA only
    ConvArgs a; a.out_mask = 1; a.lens = lens;
    if (!tok_conv(enc_proj, h, stats, s, a)) conv(enc_proj, h, stats, s, a, 0, 0, true);
}

// StochasticDurationPredictor(reverse) + DurationPredictor (reference models.py:197-204,245-256, 285-299)
void bv2_engine::run_durations(Act h, const int* lens, const float* gproj, const float* noise_w, float nsw, const float* nsw_b, float* z,
                               Act& dp_out, int* zch_out, cudaStream_t s) {
    const int B = h.B, T = h.T, Cf = cfg.sdp_filter;
    // ---- DP on a side stream (buffers allocated before the SDP's stack-disciplined temporaries)
    ensure_side_streams();
    {
        const int Cd = cfg.dp_filter;
        Act xg = ws.act(B, h.C, T), d1 = ws.act(B, Cd, T), d2 = ws.act(B, Cd, T);
        BV2_CUDA(cudaEventRecord(ev_fork, s));
        BV2_CUDA(cudaStreamWaitEvent(side[3], ev_fork, 0));
        run_dp(h, lens, gproj, dp_out, xg, d1, d2, side[3]);
        BV2_CUDA(cudaEventRecord(ev_rb[3], side[3]));
    }
    // ---- SDP conditioning
    Act c = ws.act(B, Cf, T), cond = ws.act(B, Cf, T);
    ConvArgs a0; a0.bias_b = gproj + goff_sdp; a0.bias_b_stride = gproj_n;
    if (!tok_conv(sdp_pre, h, c, s, a0)) conv(sdp_pre, h, c, s, a0, 0, 0, true);
    run_dds(sdp_dds, c, lens, s);
    ConvArgs a1; a1.out_mask = 1; a1.lens = lens;
    if (!tok_conv(sdp_proj, c, cond, s, a1)) conv(sdp_proj, c, cond, s, a1, 0, 0, true);
    debug("sdp_cond", cond);
    {
        k_scale_copy<<<dim3(cdiv(2 * T, 256), B), 256, 0, s>>>(noise_w, z, nsw, nsw_b, 2 * T);
        BV2_CUDA(cudaGetLastError()); launches++;
    }
    Act hh = ws.act(B, Cf, T), pp = ws.act(B, 32, T);
    int sflip = 0;
    for (int i = cfg.sdp_n_flows; i >= 2; i--) {
        sflip ^= 1;  // Flip
        const ConvFlowW& cf = sdp_flows[2 * i - 1];
        const int x0ch = sflip ? 1 : 0;
        k_flow_pre<<<grid_tcb(T, Cf, B), 128, 0, s>>>(z, x0ch, cf.pre_w, cf.pre_b, cond.p, hh.p, Cf, T);
        BV2_CUDA(cudaGetLastError()); launches++;
        run_dds(cf.dds, hh, lens, s);
        conv(cf.proj, hh, pp, s, ConvArgs(), 0, 0, true);
        dim3 grid(cdiv(T, 128), B);
        k_spline_inverse<10><<<grid, 128, 0, s>>>(pp.p, 32, z, 1 - x0ch, T, lens, 1.f / std::sqrt((float)Cf), cfg.sdp_tail_bound, dconst);
        BV2_CUDA(cudaGetLastError()); launches++;
    }
    sflip ^= 1;  // final Flip before ElementwiseAffine
    *zch_out = sflip ? 1 : 0;  // physical channel holding logical channel 0
    BV2_CUDA(cudaStreamWaitEvent(s, ev_rb[3], 0));  // join the DP chain
}

// DurationPredictor (reference models.py:285-299); independent of the SDP chain -> runs on a side stream
void bv2_engine::run_dp(Act h, const int* lens, const float* gproj, Act& dp_out, Act xg, Act d1, Act d2, cudaStream_t s) {
    const int B = h.B, T = h.T;
    BV2_CUDA(cudaMemcpyAsync(xg.p, h.p, h.elems() * sizeof(float), cudaMemcpyDeviceToDevice, s));
    k_add_bvec_mask<<<grid_tcb(T, h.C, B), 128, 0, s>>>(xg.p, gproj + goff_dp, gproj_n, h.C, T, lens);
    BV2_CUDA(cudaGetLastError()); launches++;
    ConvArgs r; r.act = 1;
    conv(dp_c1, xg, d1, s, r, 0, 0, true);
    layernorm(dp_n1, d1, nullptr, d1, s, 0, nullptr, lens, 0);
    ConvArgs r2; r2.act = 1; r2.in_mask = 1; r2.lens = lens;
    conv(dp_c2, d1, d2, s, r2, 0, 0, true);
    layernorm(dp_n2, d2, nullptr, d2, s, 0, nullptr, lens, 0);
    ConvArgs r3; r3.in_mask = 1; r3.out_mask = 1; r3.lens = lens;
    conv(dp_proj, d2, dp_out, s, r3);
}

// {Transformer,Residual}CouplingBlock reverse (reference models.py:142-145, 442-445; modules.py:437-456, 561-580)
void bv2_engine::run_flow(Act z, const int* lens, const float* gproj, cudaStream_t s) {
    const int B = z.B, F = z.T, H = cfg.hidden_channels, half = cfg.inter_channels / 2;
    const bool tcf = cfg.generator_precision != 0;
    const size_t mark = ws.used();
    Act h = ws.act(B, H, F);
    for (int i = cfg.n_flows - 1; i >= 0; i--) {
        CouplingW& fl = flows[i];
        const int in_off = fl.s ? half : 0, out_off = fl.s ? 0 : half;
        ConvArgs a; a.out_mask = 1; a.lens = lens;
        conv(fl.pre, z, h, s, a, in_off, 0, tcf);
        Act m_in = h;
        if (cfg.use_transformer_flow) {
            run_encoder(fl.enc, h, lens, gproj, s, flow_tc);
        } else {
            const int L = cfg.wn_layers;
            Act xin = ws.act(B, 2 * H, F), acts = ws.act(B, H, F), out = ws.act(B, H, F);
            for (int l = 0; l < L; l++) {
                if (flow_tc == 2) {
                    // in_layer conv with the gate (tanh * sigmoid, speaker conditioning as per-batch bias) in its tail; acts is a 16-bit c8
                    // tensor that the two 1x1 convs below consume as their operand image
                    ConvArgs ag; ag.bias_b = gproj + fl.wn_g_off + 2 * H * l; ag.bias_b_stride = gproj_n;
                    tc_gate = 1;
                    conv(fl.wn_in[l], h, acts, s, ag, 0, 0, true);
                    if (l < L - 1) {
                        ConvArgs ar; ar.res_mode = 1; ar.res = h.p; ar.res_C_total = H; ar.out_mask = 1; ar.lens = lens;
                        tc_in_f16 = 1;
                        conv(fl.wn_res[l], acts, h, s, ar, 0, 0, true);
                    }
                    ConvArgs as; as.accumulate = l > 0 ? 1 : 0;
                    tc_in_f16 = 1;
                    conv(fl.wn_skip[l], acts, out, s, as, 0, 0, true);
                    continue;
                }
                conv(fl.wn_in[l], h, xin, s, ConvArgs(), 0, 0, tcf);
                k_wn_gate<<<grid_tcb(F, H, B), 128, 0, s>>>(xin.p, gproj + fl.wn_g_off + 2 * H * l, gproj_n, acts.p, H, F);
                BV2_CUDA(cudaGetLastError()); launches++;
                if (l < L - 1) {
                    ConvArgs ar; ar.res_mode = 1; ar.res = h.p; ar.res_C_total = H; ar.out_mask = 1; ar.lens = lens;
                    conv(fl.wn_res[l], acts, h, s, ar, 0, 0, tcf);
                }
                ConvArgs as; as.accumulate = l > 0 ? 1 : 0;
                conv(fl.wn_skip[l], acts, out, s, as, 0, 0, tcf);
            }
            m_in = out;
        }
        ConvArgs p; p.in_mask = cfg.use_transformer_flow ? 0 : 1; p.res_mode = 2; p.res = z.p; p.res_C_total = z.C; p.res_c_off = out_off;
        p.out_mask = 1; p.lens = lens;
        conv(fl.post, m_in, z, s, p, 0, out_off, tcf);
    }
    if (cfg.n_flows % 2 == 1) {
        Act t = ws.act(B, z.C, F);
        k_flip_c4<<<grid_tcb(F, z.C, B), 128, 0, s>>>(z.p, t.p, z.C, F);
        BV2_CUDA(cudaMemcpyAsync(z.p, t.p, z.elems() * sizeof(float), cudaMemcpyDeviceToDevice, s));
        launches++;
    }
    ws.release(mark);
}

// Generator.forward (reference models.py:538-557) + ResBlock1.forward (modules.py:296-309).  The one-shot run is the one-chunk plan of a
// stream (gen_stream.cuh): every window covers its whole layer.
void bv2_engine::run_generator(Act z, const int* lens, const float* gdec, int g_stride, float* o, cudaStream_t s, bool ragged) {
    if (use_g2) { run_generator_g2(z, lens, gdec, g_stride, o, s, ragged); return; }
    if (ragged) throw Error(BV2_ERR_ARG, "a ragged batch needs the FP16 Generator (precision fp16 or fp16g)");
    const GenGraph g = gen_graph(cfg, z.T);
    std::vector<Act> t(g.tensor_len.size());
    t[0] = z;
    gen_windows(g, gen_stream_plan(g, z.T, 0, z.T), t, false, lens, gdec, g_stride, o, s);
}

// fp32 c4 Generator (SIMT, or TF32 wgmma with generator_precision 1) over the windows of w, on the tensors t (one per GenGraph tensor;
// t[0] is the input z).  stream = false: a one-shot run over whole layers; the stage temporaries are bump-allocated per stage and
// released after the join.  stream = true: a chunk of a stream, on tensors that live as long as the stream.  Zero padding is the
// kernels' bounds check against each tensor's full length, so a window reads final rows or padding only (gen_stream.cuh).
void bv2_engine::gen_windows(const GenGraph& g, const std::vector<GenWin>& w, std::vector<Act>& t, bool stream, const int* lens, const float* gdec,
                             int g_stride, float* o, cudaStream_t s) {
    const int B = t[0].B;
    const bool tc = cfg.generator_precision != 0;
    int li = 0;
    // runs layer li over its window (nothing for an empty one) with the epilogue a
    auto conv_layer = [&](const ConvW& cw, ConvArgs a, cudaStream_t sj) {
        const GenLayer& l = g.layers[li];
        const GenWin& wi = w[li++];
        if (wi.t_end <= wi.t_begin) return;
        a.t_begin = wi.t_begin; a.t_end = wi.t_end;
        if (l.res >= 0) { a.res_mode = 1; a.res = t[l.res].p; a.res_C_total = t[l.res].C; }
        conv(cw, t[l.in], t[l.out], sj, a, 0, 0, tc);
    };
    if (!stream) t[g.layers[0].out] = ws.act(B, cfg.upsample_initial_channel, g.layers[0].L_out);
    {
        ConvArgs a; a.bias_b = gdec; a.bias_b_stride = g_stride;
        if (lens) { a.in_mask = 1; a.lens = lens; }
        conv_layer(conv_pre, a, s);
    }
    const int nk = cfg.n_resblock_kernels, nd = cfg.n_dilations;
    BV2_CHECK(nk <= 4, "at most 4 resblock kernels");
    ensure_side_streams();
    for (int i = 0; i < cfg.n_ups; i++) {
        const UpW& u = ups[i];
        const GenLayer& lu = g.layers[li];
        BV2_CHECK(lu.kind == GenLayer::UPS && lu.stage == i, "Generator plan order");
        auto layer_of = [&](int j, int d, int c2) -> const GenLayer& { return g.layers[li + 1 + 2 * (j * nd + d) + c2]; };
        size_t mark_after_S = 0;
        if (!stream) {
            const int Lo = lu.L_out;
            t[layer_of(0, nd - 1, 1).out] = ws.act(B, u.Cout, Lo);  // S: the next stage's input stays
            mark_after_S = ws.used();
            t[lu.out] = ws.act(B, u.Cout, Lo);
            for (int j = 0; j < nk; j++) {
                const Act xt = ws.act(B, u.Cout, Lo), ra = ws.act(B, u.Cout, Lo), rb = ws.act(B, u.Cout, Lo);
                for (int d = 0; d < nd; d++) {
                    t[layer_of(j, d, 0).out] = xt;
                    if (d < nd - 1) t[layer_of(j, d, 1).out] = d % 2 ? rb : ra;
                }
            }
        }
        {
            const Act& x = t[lu.in];
            const Act& xu = t[lu.out];
            const GenWin& wi = w[li++];
            if (wi.t_end > wi.t_begin) {
                if (tc) {
                    TcEpi eu; eu.in_slope = 0.1f; eu.t_begin = wi.t_begin; eu.t_end = wi.t_end;
                    tc_conv1d(u.tc, u.b, x, xu, eu, s, num_sms); launches++;
                } else {
                    ConvTArgs ct; ct.x = x.p; ct.Cin = u.Cin; ct.Tin = x.T; ct.w = u.w; ct.bias = u.b; ct.y = xu.p; ct.Cout = u.Cout; ct.Tout = xu.T;
                    ct.K = u.K; ct.u = u.u; ct.p = (u.K - u.u) / 2; ct.B = B; ct.in_slope = 0.1f; ct.n_begin = wi.t_begin; ct.n_end = wi.t_end;
                    dim3 grid(cdiv(wi.t_end - wi.t_begin, 128), cdiv(u.Cout, 64), B);
                    k_convT_c4<<<grid, 256, 0, s>>>(ct);
                    BV2_CUDA(cudaGetLastError()); launches++;
                }
            }
        }
        // fork: resblock j runs on its own stream; only the last conv of each chain (the MRF running sum) is ordered
        BV2_CUDA(cudaEventRecord(ev_fork, s));
        for (int j = 0; j < nk; j++) {
            cudaStream_t sj = j == 0 ? s : side[j];
            if (j) BV2_CUDA(cudaStreamWaitEvent(sj, ev_fork, 0));
            const ResBlockW& R = resblocks[i * nk + j];
            for (int d = 0; d < nd; d++) {
                const bool last = d == nd - 1;
                ConvArgs c1; c1.in_slope = 0.1f; c1.dil = R.dil[d];
                conv_layer(R.c1[d], c1, sj);
                if (last && j > 0) BV2_CUDA(cudaStreamWaitEvent(sj, ev_rb[j - 1], 0));  // S += ... after resblock j-1 wrote S
                ConvArgs c2; c2.in_slope = 0.1f;  // residual: the chain's input (GenLayer::res)
                if (last) { c2.accumulate = j > 0; c2.out_scale = (j == nk - 1) ? 1.f / nk : 1.f; }
                conv_layer(R.c2[d], c2, sj);
            }
            BV2_CUDA(cudaEventRecord(ev_rb[j], sj));
        }
        // join: the caller's stream continues after the last resblock (which itself waited for all earlier ones)
        if (nk > 1) BV2_CUDA(cudaStreamWaitEvent(s, ev_rb[nk - 1], 0));
        if (!stream) {
            if (i == 0) debug("gen_stage0", t[layer_of(0, nd - 1, 1).out]);
            ws.release(mark_after_S);
        }
    }
    const GenLayer& lp = g.layers[li];
    BV2_CHECK(lp.kind == GenLayer::CONV_POST && li + 1 == (int)g.layers.size(), "Generator plan order");
    const GenWin& wp = w[li];
    if (wp.t_end > wp.t_begin) {
        dim3 grid(cdiv(wp.t_end - wp.t_begin, 256), B);
        k_conv_post_tanh<16, 7><<<grid, 256, 0, s>>>(t[lp.in].p, conv_post_w, o, lp.L_out, 0.01f, wp.t_begin, wp.t_end);
        BV2_CUDA(cudaGetLastError()); launches++;
    }
}

// Generator on 16-bit activation tensors (tc_gen.cuh): every tensor between conv_pre and conv_post is an H8 operand image
// (f16(lrelu_0.1(x)), zero halos); 96 launches of ONE kernel (k_g2_conv) + conv_post.  The one-shot run is the one-chunk plan of a
// stream (gen_stream.cuh): every window covers its whole layer.
// ragged: item b's rows stop at min(lens[b], z.T) frames in every layer, each followed by its own zero halo, so it computes exactly what a
// run of that item alone at that length computes (same launches, same workspace; samples past its length are 0).
void bv2_engine::run_generator_g2(Act z, const int* lens, const float* gdec, int g_stride, float* o, cudaStream_t s, bool ragged) {
    BV2_CHECK(!ragged || lens, "ragged Generator without lengths");
    const GenGraph g = gen_graph(cfg, z.T);
    std::vector<H8> t(g.tensor_len.size());
    t[0] = g2_input(z, lens, s);
    g2_windows(g, gen_stream_plan(g, z.T, 0, z.T), t, false, gdec, g_stride, o, s, ragged ? lens : nullptr);
}

// rows >= 0: storage for only that many rows (a stream's tensor, H8::base); else the whole tensor
H8 bv2_engine::g2_h8(int B, int C, int T, int rows) {
    H8 t; t.B = B; t.C = C; t.T = T; t.Tp = G2_PADL + (rows >= 0 ? rows : T) + G2_PADR;
    t.p = reinterpret_cast<uint4*>(ws.alloc(H8::bytes(B, C, t.Tp - G2_PADL - G2_PADR) / 4)) + G2_PADL;
    return t;
}

// z * y_mask as the raw f16 H8 tensor conv_pre reads (zero halos: every producer clears the halo rows of its own output)
H8 bv2_engine::g2_input(Act z, const int* lens, cudaStream_t s) {
    H8 zh = g2_h8(z.B, z.C, z.T);
    k_c4_to_h8<<<dim3(cdiv(z.T, 128), z.C / 8, z.B), 128, 0, s>>>(reinterpret_cast<const float4*>(z.p), zh.p, z.C, z.T, zh.Tp, lens, 0, z.T, 0);
    BV2_CUDA(cudaGetLastError()); launches++;
    return zh;
}

// Workspace bytes of the tensors of a stream over Fg frames with chunks of at most max_chunk frames: all but the waveform, which the
// caller owns, and, for the fp32 Generator, the input z, which the caller allocated.  Only the FP16 Generator bounds its storage, so a
// cap below the frame count on any other is a BV2_ERR_ARG.
size_t bv2_engine::stream_bytes(int B, int Fg, int max_chunk) const {
    if (!use_g2 && gen_stream_bounded(Fg, max_chunk))
        throw Error(BV2_ERR_ARG, "a chunk cap below the frame count needs the FP16 Generator (precision fp16 or fp16g)");
    const GenGraph g = gen_graph(cfg, Fg);
    const std::vector<int> rows = gen_stream_rows(cfg, g, max_chunk);
    size_t n = 0;
    for (size_t i = use_g2 ? 0 : 1; i + 1 < rows.size(); i++) {
        const int C = g.tensor_ch[i];
        n += ((use_g2 ? H8::bytes(B, C, rows[i]) : (size_t)B * C * rows[i] * sizeof(float)) + 255) & ~(size_t)255;
    }
    return n;
}

void bv2_engine::gen_stream_open(Act z, const int* lens, const float* gdec, int g_stride, float* o, int max_chunk, bool ragged) {
    BV2_CHECK(!ragged || (use_g2 && lens), "a ragged stream needs the FP16 Generator and the lengths");
    gs.g = gen_graph(cfg, z.T);
    const size_t n = gs.g.tensor_len.size();
    gs.t.clear(); gs.a.clear(); gs.rows.clear();
    if (use_g2) {
        gs.rows = gen_stream_rows(cfg, gs.g, max_chunk);
        gs.t.assign(n, H8());
        for (size_t i = 0; i + 1 < n; i++) gs.t[i] = g2_h8(z.B, gs.g.tensor_ch[i], gs.g.tensor_len[i], gs.rows[i]);
    } else {
        gs.a.assign(n, Act());
        gs.a[0] = z;
        for (size_t i = 1; i + 1 < n; i++) gs.a[i] = ws.act(z.B, gs.g.tensor_ch[i], gs.g.tensor_len[i]);
    }
    gs.max_chunk = gen_stream_bounded(z.T, max_chunk) ? max_chunk : 0;
    gs.B = z.B; gs.Fg = z.T; gs.frontier = 0; gs.o = o; gs.gdec = gdec; gs.g_stride = g_stride; gs.lens = lens; gs.z = z;
    gs.ragged = ragged;
    gs.open = true;
}

// Before the windows of the chunk done -> target of an FP16 stream: one slide launch for the tensors whose storage the chunk would
// overrun (gen_stream_slides; none while every tensor is whole), then the conversion of the input rows the chunk reads.
void bv2_engine::g2_stream_prepare(int done, int target, cudaStream_t s) {
    const size_t n = gs.t.size();
    std::vector<int> base(n);
    for (size_t i = 0; i < n; i++) base[i] = gs.t[i].base;
    const std::vector<GenSlide> sl = gen_stream_slides(gs.g, gs.Fg, gs.rows, base, done, target);
    for (size_t k = 0; k < sl.size(); k += G2_SLIDE_MAX) {  // one launch at the default configuration (87 tensors)
        G2SlideParams sp{};
        int most = 0;
        for (size_t j = k; j < sl.size() && sp.n < G2_SLIDE_MAX; j++) {
            const H8& t = gs.t[sl[j].tensor];
            sp.d[sp.n++] = G2SlideDesc{t.p, t.B * (t.C / 8), t.Tp, sl[j].src, sl[j].dst, sl[j].rows};
            most = std::max(most, t.B * (t.C / 8) * sl[j].rows);
        }
        launch_pdl(k_g2_slide, dim3(std::min(32, cdiv(most, 256)), sp.n), dim3(256), 0, s, sp);
        launches++;
    }
    for (size_t i = 0; i < n; i++) gs.t[i].base = base[i];
    const int a = gen_needs(gs.g, gs.Fg, done).tensor[0], b = gen_needs(gs.g, gs.Fg, target).tensor[0];
    if (b > a) {
        const Act& z = gs.z;
        k_c4_to_h8<<<dim3(cdiv(b - a, 128), z.C / 8, z.B), 128, 0, s>>>(reinterpret_cast<const float4*>(z.p), gs.t[0].p, z.C, z.T, gs.t[0].Tp, gs.lens,
                                                                      a, b, gs.t[0].base);
        BV2_CUDA(cudaGetLastError()); launches++;
    }
}

// Runs every Generator layer over its window of w (GenGraph launch order; empty windows launch nothing) on the H8 tensors t, one per
// GenGraph tensor.  stream = false: a one-shot run over whole layers; t holds only the input, and the stage temporaries are
// bump-allocated per stage and released after the join (the convs of one resblock chain share one temporary and two ping-pong
// buffers).  stream = true: a chunk of a stream, on tensors that live as long as the stream and hold the rows of gen_stream_rows().
// Every tensor is addressed by logical row through its base (0 for a whole tensor).  ragged_lens (device, frames per item; null: every
// item has all g.tensor_len[0] frames): every layer stores item b's rows below its length only, at the layer's rows per frame, followed
// by its zero halo (one-shot) or, in a stream, by zeros in every later row of each window (G2_RAGGED_STREAM; conv_post and the input
// conversion already store zeros past an item's end inside their windows and nothing outside them).
void bv2_engine::g2_windows(const GenGraph& g, const std::vector<GenWin>& w, std::vector<H8>& t, bool stream, const float* gdec, int g_stride,
                            float* o, cudaStream_t s, const int* ragged_lens) {
    const int B = t[0].B;
    int li = 0;
    auto conv = [&](const TcConvW& cw, const float* bias, G2Epi e, cudaStream_t sj) {
        const GenLayer& l = g.layers[li];
        const GenWin& wi = w[li++];
        if (wi.t_end <= wi.t_begin) return;
        e.t_begin = wi.t_begin; e.t_end = wi.t_end;
        if (ragged_lens) { e.lens = ragged_lens; e.lens_scale = l.L_in / g.tensor_len[0]; e.ragged_stream = stream; }  // the M axis is the input's time axis
        if (l.res >= 0) e.res = &t[l.res];
        g2_conv(cw, bias, t[l.in], t[l.out], e, sj, num_sms); launches++;
    };
    if (!stream) t[g.layers[0].out] = g2_h8(B, cfg.upsample_initial_channel, g.layers[0].L_out);
    {
        G2Epi e; e.bias_b = gdec; e.bias_b_stride = g_stride;
        conv(conv_pre.tc, conv_pre.b, e, s);
    }
    const int nk = cfg.n_resblock_kernels, nd = cfg.n_dilations;
    BV2_CHECK(nk <= 4, "at most 4 resblock kernels");
    ensure_side_streams();
    for (int i = 0; i < cfg.n_ups; i++) {
        const UpW& u = ups[i];
        const GenLayer& lu = g.layers[li];
        BV2_CHECK(lu.kind == GenLayer::UPS && lu.stage == i, "Generator plan order");
        auto layer_of = [&](int j, int d, int c2) -> const GenLayer& { return g.layers[li + 1 + 2 * (j * nd + d) + c2]; };
        size_t mark_after_S = 0;
        if (!stream) {
            const int Lo = lu.L_out;
            t[layer_of(0, nd - 1, 1).out] = g2_h8(B, u.Cout, Lo);  // S: the next stage's input stays
            mark_after_S = ws.used();
            t[lu.out] = g2_h8(B, u.Cout, Lo);
            for (int j = 0; j < nk; j++) {
                const H8 xt = g2_h8(B, u.Cout, Lo), ra = g2_h8(B, u.Cout, Lo), rb = g2_h8(B, u.Cout, Lo);
                for (int d = 0; d < nd; d++) {
                    t[layer_of(j, d, 0).out] = xt;
                    if (d < nd - 1) t[layer_of(j, d, 1).out] = d % 2 ? rb : ra;
                }
            }
        }
        conv(u.tc, u.b, G2Epi(), s);
        BV2_CUDA(cudaEventRecord(ev_fork, s));
        for (int j = 0; j < nk; j++) {
            cudaStream_t sj = j == 0 ? s : side[j];
            if (j) BV2_CUDA(cudaStreamWaitEvent(sj, ev_fork, 0));
            const ResBlockW& R = resblocks[i * nk + j];
            for (int d = 0; d < nd; d++) {
                const bool last = d == nd - 1;
                G2Epi e1; e1.dil = R.dil[d];
                conv(R.c1[d].tc, R.c1[d].b, e1, sj);
                if (last && j > 0) BV2_CUDA(cudaStreamWaitEvent(sj, ev_rb[j - 1], 0));  // S += ... after resblock j-1 wrote S
                G2Epi e2;  // residual: the chain's input (GenLayer::res)
                if (last) { e2.accumulate = j > 0; e2.out_scale = (j == nk - 1) ? 1.f / nk : 1.f; }
                conv(R.c2[d].tc, R.c2[d].b, e2, sj);
            }
            BV2_CUDA(cudaEventRecord(ev_rb[j], sj));
        }
        if (nk > 1) BV2_CUDA(cudaStreamWaitEvent(s, ev_rb[nk - 1], 0));
        if (!stream) ws.release(mark_after_S);
    }
    const GenLayer& lp = g.layers[li];
    BV2_CHECK(lp.kind == GenLayer::CONV_POST && li + 1 == (int)g.layers.size(), "Generator plan order");
    const H8& x = t[lp.in];
    BV2_CHECK(x.C == 16, "conv_post kernel instantiated for 16 input channels");
    const GenWin& wp = w[li];
    if (wp.t_end > wp.t_begin) {
        BV2_CHECK((x.base == 0 || wp.t_begin - 3 >= x.base) && std::min(wp.t_end + 3, x.T + G2_PADR) <= x.lim(), "conv_post input rows not resident");
        PostW<16, 7> pw = conv_post_h;
        if (ragged_lens) { pw.lens = ragged_lens; pw.lens_scale = g.hop; }
        launch_pdl(ragged_lens ? k_conv_post_tanh_h8<16, 7, true> : k_conv_post_tanh_h8<16, 7>, dim3(cdiv(wp.t_end - wp.t_begin, 512), B), dim3(256), 0, s, (const uint4*)x.p, x.Tp, x.base, pw, o,
                   lp.L_out, wp.t_begin, wp.t_end);
        launches++;
    }
}

// ================================================================================================
// C ABI
// ================================================================================================
#define BV2_API_BEGIN(e)                                  \
    if (!(e)) return BV2_ERR_ARG;                         \
    std::lock_guard<std::mutex> _lk((e)->mu);             \
    try {                                                 \
        BV2_CUDA(cudaSetDevice((e)->device));             \
        (e)->begin_call();
#define BV2_API_END(e)                                    \
    }                                                     \
    catch (const bv2::Error& ex) { (e)->err = ex.what(); return ex.code; } \
    catch (const std::exception& ex) { (e)->err = ex.what(); return BV2_ERR_INTERNAL; } \
    return BV2_OK;

// Workspace of a call, in two parts (generous upper bounds; every buffer is bump-allocated per call): the encoder, durations and flow,
// and the one-shot Generator's stage temporaries.  A Generator stream needs the first part plus its own tensors (stream_bytes).
static size_t ws_enc_flow_bytes(const bv2_config& c, int B, int T, int F) {
    size_t tok = (size_t)B * T, frm = (size_t)B * std::max(F, 1);
    size_t enc = tok * (3 * c.bert_dim + 16 * c.hidden_channels + c.filter_channels + 2 * c.dp_filter + 64) * 4;
    size_t flow = frm * (12 * c.hidden_channels + c.filter_channels + 4 * c.inter_channels) * 4 +
                  (size_t)B * c.n_heads * ((size_t)F + 128) * ((size_t)F + 96) * 4 + (1u << 20);  // attention S/P + V^T
    return enc + flow + (64u << 20);
}
static size_t ws_gen_bytes(const bv2_config& c, int B, int F) {
    const size_t frm = (size_t)B * std::max(F, 1);
    return frm * ((size_t)c.upsample_initial_channel + 8192ull * (5 + 10) + 4096) * 4;  // 5 stage outputs + 10 temporaries (3 resblock chains)
}
static size_t ws_bytes_for(const bv2_config& c, int B, int T, int F) { return ws_enc_flow_bytes(c, B, T, F) + ws_gen_bytes(c, B, F); }

// Workspace a stream over F frames (Fg of them through the Generator) ensures.  max_chunk <= 0: the unbounded stream, which has always
// reserved the one-shot Generator's part as well; a cap: the encoder/flow part plus the stream's own tensors.
static size_t ws_stream_bytes(const bv2_engine* e, int B, int T, int F, int Fg, int max_chunk) {
    return (max_chunk <= 0 ? ws_bytes_for(e->cfg, B, T, F) : ws_enc_flow_bytes(e->cfg, B, T, F)) + e->stream_bytes(B, Fg, max_chunk);
}

static size_t persist_bytes_for(const bv2_config& c, int B, int T, int gproj_n) {
    return (size_t)B * T * (2 * c.inter_channels + 8) * 4 + (size_t)B * (gproj_n + c.gin_channels + 16) * 4 + (1 << 20);
}

extern "C" {

const char* bv2_version(void) { return "bv2-b200 0.1 (sm_90a)"; }

int bv2_create(bv2_engine** out, const bv2_config* cfg, int cuda_device) {
    if (!out || !cfg) return BV2_ERR_ARG;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || cuda_device < 0 || cuda_device >= n) return BV2_ERR_CUDA;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, cuda_device) != cudaSuccess) return BV2_ERR_CUDA;
    if (prop.major != 9) return BV2_ERR_CUDA;  // sm_90a only: no fallback path exists
    bv2_engine* e = new bv2_engine();
    e->cfg = *cfg;
    e->device = cuda_device;
    e->num_sms = prop.multiProcessorCount;
    *out = e;
    return BV2_OK;
}

int bv2_create_sibling(bv2_engine** out, bv2_engine* src) {
    if (!out || !src) return BV2_ERR_ARG;
    *out = nullptr;
    std::lock_guard<std::mutex> lk(src->mu);
    if (!src->finalized) { src->err = "create_sibling needs a finalized engine (bv2_finalize or bv2_load_packed)"; return BV2_ERR_STATE; }
    std::unique_ptr<bv2_engine> e(new bv2_engine());
    e->cfg = src->cfg;
    e->device = src->device;
    e->num_sms = src->num_sms;
    static_cast<DeviceWeights&>(*e) = static_cast<const DeviceWeights&>(*src);
    e->finalized = true;  // bv2_set_weight / bv2_finalize / bv2_load_packed return BV2_ERR_STATE on a sibling
    try {
        BV2_CUDA(cudaSetDevice(e->device));
        e->ensure_h_ylen();
    } catch (const bv2::Error& ex) { src->err = ex.what(); return ex.code; }
    *out = e.release();
    return BV2_OK;
}

int bv2_set_weight(bv2_engine* e, const char* key, const void* host_ptr, const int64_t* shape, int ndim, int dtype) {
    if (!e || !key || !host_ptr || ndim < 0 || ndim > 4) return BV2_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    if (e->finalized) { e->err = "set_weight after finalize"; return BV2_ERR_STATE; }
    if (std::strncmp(key, "enc_q.", 6) == 0) return BV2_OK;
    HostTensor t;
    int64_t n = 1;
    for (int i = 0; i < ndim; i++) { t.shape.push_back(shape[i]); n *= shape[i]; }
    t.data.resize((size_t)n);
    if (dtype == 0) std::memcpy(t.data.data(), host_ptr, (size_t)n * 4);
    else if (dtype == 1) { const __half* h = static_cast<const __half*>(host_ptr); for (int64_t i = 0; i < n; i++) t.data[i] = __half2float(h[i]); }
    else { e->err = "dtype"; return BV2_ERR_ARG; }
    e->host[key] = std::move(t);
    return BV2_OK;
}

int bv2_finalize(bv2_engine* e) {
    BV2_API_BEGIN(e)
    BV2_CHECK(!e->finalized, "already finalized");
    e->finalize();
    BV2_API_END(e)
}

// ---- packed engine weight file (SURVEY.md section 8f.4; the reference's counterpart is compress_model.py:44-53, which only drops enc_q and
// casts to fp16): header | reference state_dict key/shape table | arena image (weight-norm folded, Flip folded, SIMT + wgmma packs).
namespace {
struct PackHeader {
    char magic[8];
    uint32_t version, cfg_bytes;
    uint64_t arena_bytes;
    uint32_t n_keys, reserved;
    float ea_m[2], ea_logs[2];
};
const char kPackMagic[8] = {'B', 'V', '2', 'P', 'A', 'C', 'K', '2'};
}  // namespace

int bv2_save_packed(bv2_engine* e, const char* path) {
    BV2_API_BEGIN(e)
    BV2_CHECK(e->finalized && path, "save_packed needs a finalized engine");
    std::vector<uint8_t> img(e->warena_bytes);
    BV2_CUDA(cudaDeviceSynchronize());
    BV2_CUDA(cudaMemcpy(img.data(), e->warena, e->warena_bytes, cudaMemcpyDeviceToHost));
    FILE* f = std::fopen(path, "wb");
    if (!f) throw Error(BV2_ERR_ARG, std::string("cannot open ") + path);
    PackHeader h{};
    std::memcpy(h.magic, kPackMagic, 8);
    h.version = 2; h.cfg_bytes = (uint32_t)sizeof(bv2_config); h.arena_bytes = e->warena_bytes; h.n_keys = (uint32_t)e->shape_table.size();
    for (int i = 0; i < 2; i++) { h.ea_m[i] = e->ea_m[i]; h.ea_logs[i] = e->ea_logs[i]; }
    bool ok = std::fwrite(&h, sizeof(h), 1, f) == 1 && std::fwrite(&e->cfg, sizeof(bv2_config), 1, f) == 1;
    for (const auto& kv : e->shape_table) {
        const uint32_t kl = (uint32_t)kv.first.size(), nd = (uint32_t)kv.second.size();
        ok = ok && std::fwrite(&kl, 4, 1, f) == 1 && std::fwrite(kv.first.data(), 1, kl, f) == kl && std::fwrite(&nd, 4, 1, f) == 1;
        if (nd) ok = ok && std::fwrite(kv.second.data(), sizeof(int64_t), nd, f) == nd;
    }
    ok = ok && std::fwrite(img.data(), 1, img.size(), f) == img.size();
    ok = (std::fclose(f) == 0) && ok;
    if (!ok) throw Error(BV2_ERR_INTERNAL, std::string("short write to ") + path);
    BV2_API_END(e)
}

int bv2_load_packed(bv2_engine* e, const char* path) {
    BV2_API_BEGIN(e)
    BV2_CHECK(!e->finalized && path, "load_packed replaces set_weight + finalize on a fresh engine");
    FILE* f = std::fopen(path, "rb");
    if (!f) throw Error(BV2_ERR_ARG, std::string("cannot open ") + path);
    struct Closer { FILE* f; ~Closer() { std::fclose(f); } } closer{f};
    PackHeader h{};
    bv2_config fc{};
    if (std::fread(&h, sizeof(h), 1, f) != 1 || std::memcmp(h.magic, kPackMagic, 8) != 0 || h.version != 2 || h.cfg_bytes != sizeof(bv2_config) ||
        std::fread(&fc, sizeof(fc), 1, f) != 1)
        throw Error(BV2_ERR_ARG, "not a bv2 packed weight file (magic / version / config size)");
    if (std::memcmp(&fc, &e->cfg, sizeof(fc)) != 0) throw Error(BV2_ERR_ARG, "packed weight file was written for a different configuration / precision");
    e->host.clear();
    for (uint32_t i = 0; i < h.n_keys; i++) {
        uint32_t kl = 0, nd = 0;
        if (std::fread(&kl, 4, 1, f) != 1 || kl > 512) throw Error(BV2_ERR_ARG, "corrupt key table");
        std::string key(kl, '\0');
        if (std::fread(&key[0], 1, kl, f) != kl || std::fread(&nd, 4, 1, f) != 1 || nd > 4) throw Error(BV2_ERR_ARG, "corrupt key table");
        HostTensor t;
        t.shape.resize(nd);
        if (nd && std::fread(t.shape.data(), sizeof(int64_t), nd, f) != nd) throw Error(BV2_ERR_ARG, "corrupt key table");
        t.data.assign((size_t)t.numel(), 0.f);  // structure only: the packing loops are skipped, the images come from the file
        e->host[key] = std::move(t);
    }
    std::vector<uint8_t> img(h.arena_bytes);
    if (std::fread(img.data(), 1, img.size(), f) != img.size()) throw Error(BV2_ERR_ARG, "truncated packed weight file");
    e->finalize(img.data(), img.size());
    for (int i = 0; i < 2; i++) { e->ea_m[i] = h.ea_m[i]; e->ea_logs[i] = h.ea_logs[i]; }
    BV2_API_END(e)
}

// items: the settings are per-item device arrays [B] (bv2_infer_begin_items) instead of the scalars, which are then ignored
struct ItemSettings { const float *noise_scale_w, *length_scale, *sdp_ratio, *noise_scale; };
// mix: g is each item's weighted sum of K emb_g rows (bv2_infer_begin_mix) instead of the row of sid, which is then ignored
struct SpeakerMix { int K; const int64_t* sid; const float* weight; };

static int infer_begin_impl(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, const int64_t* sid,
                            const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert,
                            const float* en_bert, const float* noise_w, float noise_scale_w, float length_scale, float sdp_ratio,
                            const ItemSettings* items, const float* w_ceil_override, void* stream, int64_t* y_lengths_host,
                            int32_t* f_max, const SpeakerMix* mix = nullptr) {
    BV2_API_BEGIN(e)
    BV2_CHECK(e->finalized, "not finalized");
    BV2_CHECK(B >= 1 && B <= 4096 && T >= 1 && x && x_lengths && (sid || mix) && tone && language && bert && ja_bert && en_bert &&
                  noise_w && y_lengths_host && f_max, "infer_begin args");
    if (items && !(items->noise_scale_w && items->length_scale && items->sdp_ratio && items->noise_scale))
        throw Error(BV2_ERR_ARG, "infer_begin_items: every setting array must be given");
    if (mix && !(mix->K >= 1 && (int64_t)B * mix->K <= INT32_MAX && mix->sid && mix->weight))
        throw Error(BV2_ERR_ARG, "infer_begin_mix: need K >= 1, B*K <= INT32_MAX and both mix arrays");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bv2_config& c = e->cfg;
    const int H = c.hidden_channels, I = c.inter_channels;
    e->dbg.clear();
    e->ws.ensure(ws_bytes_for(c, B, T, 0));
    e->ws_reset();
    e->persist.ensure(persist_bytes_for(c, B, T, e->gproj_n));
    e->persist.reset();
    auto& st = e->st;
    st.active = false; st.finished = false; st.B = B; st.T = T; st.F = 0;
    e->stage_begin("encoder_duration", s);
    st.ylen = reinterpret_cast<long long*>(e->persist.alloc(2 * (size_t)B + 4));  // [B] y_lengths, then the input-validation mask
    int* err_dev = reinterpret_cast<int*>(st.ylen + B);
    st.noise_scale = nullptr;
    if (items) {  // finish reads it; a copy, not a kernel, so the launches are those of bv2_infer_begin
        st.noise_scale = e->persist.alloc(B);
        BV2_CUDA(cudaMemcpyAsync(st.noise_scale, items->noise_scale, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, s));
    }
    e->launch_validate(B, T, x, tone, language, mix ? nullptr : sid, x_lengths, err_dev, s);  // k_speaker_mix checks a mix's ids
    st.lens = e->lens_to_device(x_lengths, B, e->persist, s);
    float* g = e->persist.alloc((size_t)B * c.gin_channels);
    st.gproj = e->persist.alloc((size_t)B * e->gproj_n);
    if (mix)
        k_speaker_mix<<<B, 128, 0, s>>>(e->emb_g, reinterpret_cast<const long long*>(mix->sid), mix->weight, mix->K, g, c.gin_channels,
                                        c.n_speakers, err_dev);
    else
        k_gather_rows<<<B, 128, 0, s>>>(e->emb_g, reinterpret_cast<const long long*>(sid), g, c.gin_channels, c.n_speakers);
    BV2_CUDA(cudaGetLastError()); e->launches++;
    e->debug_plain("g", g, B, c.gin_channels, 1);
    e->run_gproj(g, B, st.gproj, s);
    Act h = e->ws.act(B, H, T);
    Act stats; stats.B = B; stats.C = 2 * I; stats.T = T; stats.p = e->persist.alloc(stats.elems());
    st.stats = stats.p;
    e->run_text_encoder(B, T, x, tone, language, bert, ja_bert, en_bert, st.lens, st.gproj, h, stats, s);
    e->debug("x", h); e->debug("stats", stats);
    float* z = e->ws.alloc((size_t)B * 2 * T);
    Act dp = e->ws.act(B, 4, T);
    int zch = 0;
    e->run_durations(h, st.lens, st.gproj, noise_w, noise_scale_w, items ? items->noise_scale_w : nullptr, z, dp, &zch, s);
    float* lsdp = e->ws.alloc((size_t)B * T); float* ldp = e->ws.alloc((size_t)B * T);
    st.w_ceil = e->persist.alloc((size_t)B * T);
    st.cum = reinterpret_cast<int*>(e->persist.alloc((size_t)B * T));
    k_durations<<<B, 1024, 0, s>>>(z, zch, e->ea_m[0], e->ea_logs[0], dp.p, sdp_ratio, length_scale, items ? items->sdp_ratio : nullptr,
                                   items ? items->length_scale : nullptr, st.lens, T, lsdp, ldp, st.w_ceil, st.cum, st.ylen, w_ceil_override);
    BV2_CUDA(cudaGetLastError()); e->launches++;
    e->debug_plain("logw_sdp", lsdp, B, 1, T); e->debug_plain("logw_dp", ldp, B, 1, T); e->debug_plain("w_ceil", st.w_ceil, B, 1, T);
    e->stage_end("encoder_duration", s);
    BV2_CUDA(cudaMemcpyAsync(e->h_ylen, st.ylen, ((size_t)B + 1) * sizeof(long long), cudaMemcpyDeviceToHost, s));
    BV2_CUDA(cudaStreamSynchronize(s));
    bv2_engine::throw_if_bad_inputs((int)(e->h_ylen[B] & 0xffffffffll));
    e->check_device_error();
    int fm = 1;
    for (int b = 0; b < B; b++) { y_lengths_host[b] = e->h_ylen[b]; fm = std::max<long long>(fm, e->h_ylen[b]); }
    *f_max = fm; st.F = fm;
    st.ylen32 = e->lens_to_device(reinterpret_cast<const int64_t*>(st.ylen), B, e->persist, s);
    st.active = true;
    BV2_API_END(e)
}

int bv2_infer_begin(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, const int64_t* sid,
                    const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert,
                    const float* en_bert, const float* noise_w, float noise_scale_w, float length_scale, float sdp_ratio,
                    const float* w_ceil_override, void* stream, int64_t* y_lengths_host, int32_t* f_max) {
    return infer_begin_impl(e, B, T, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, noise_w, noise_scale_w, length_scale,
                            sdp_ratio, nullptr, w_ceil_override, stream, y_lengths_host, f_max);
}

int bv2_infer_begin_items(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, const int64_t* sid,
                          const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert,
                          const float* en_bert, const float* noise_w, const float* noise_scale_w, const float* length_scale,
                          const float* sdp_ratio, const float* noise_scale, const float* w_ceil_override, void* stream,
                          int64_t* y_lengths_host, int32_t* f_max) {
    const ItemSettings items{noise_scale_w, length_scale, sdp_ratio, noise_scale};
    return infer_begin_impl(e, B, T, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, noise_w, 1.f, 1.f, 0.f, &items,
                            w_ceil_override, stream, y_lengths_host, f_max);
}

int bv2_infer_begin_mix(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, int K, const int64_t* mix_sid,
                        const float* mix_weight, const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert,
                        const float* en_bert, const float* noise_w, const float* noise_scale_w, const float* length_scale,
                        const float* sdp_ratio, const float* noise_scale, const float* w_ceil_override, void* stream,
                        int64_t* y_lengths_host, int32_t* f_max) {
    const ItemSettings items{noise_scale_w, length_scale, sdp_ratio, noise_scale};
    const SpeakerMix mix{K, mix_sid, mix_weight};
    return infer_begin_impl(e, B, T, x, x_lengths, nullptr, tone, language, bert, ja_bert, en_bert, noise_w, 1.f, 1.f, 0.f, &items,
                            w_ceil_override, stream, y_lengths_host, f_max, &mix);
}

// open_stream: stop after the flow and open a Generator stream over o instead of running the Generator (bv2_infer_finish_stream)
// ragged: the Generator runs each utterance at its own length (bv2_infer_finish_ragged; with open_stream, a ragged stream:
// bv2_infer_finish_stream_ragged)
static int infer_finish_impl(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len, float* o, int16_t* o16,
                             float* attn, float* y_mask, float* z_out, float* z_p, float* m_p, float* logs_p, void* stream, bool open_stream = false,
                             int max_chunk = 0, bool ragged = false) {
    BV2_API_BEGIN(e)
    auto& st = e->st;
    BV2_CHECK(st.active, "infer_finish without infer_begin");
    BV2_CHECK(noise_z && (o || o16) && noise_ld >= st.F, "infer_finish args");
    if (ragged && !e->use_g2) throw Error(BV2_ERR_ARG, "a ragged batch needs the FP16 Generator (precision fp16 or fp16g)");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bv2_config& c = e->cfg;
    const int B = st.B, T = st.T, F = st.F, I = c.inter_channels;
    const int Fg = (max_len > 0 && max_len < F) ? max_len : F;
    e->ws.ensure(open_stream ? ws_stream_bytes(e, B, T, F, Fg, max_chunk) : ws_bytes_for(c, B, T, F));
    e->ws_reset();
    float* m_tmp = m_p ? m_p : e->ws.alloc((size_t)B * I * F);
    float* l_tmp = logs_p ? logs_p : e->ws.alloc((size_t)B * I * F);
    float* zp_tmp = z_p ? z_p : e->ws.alloc((size_t)B * I * F);
    Act z = e->ws.act(B, I, F);
    {
        dim3 grid(cdiv(F, 128), I / 4, B);
        k_expand_prior<<<grid, 128, 0, s>>>(st.stats, st.cum, st.ylen, st.lens, noise_z, (long long)I * noise_ld, (int)noise_ld, noise_scale,
                                            st.noise_scale, I, T, F, m_tmp, l_tmp, zp_tmp, z.p, y_mask);
        BV2_CUDA(cudaGetLastError()); e->launches++;
    }
    if (attn) {
        dim3 grid(cdiv(T, 128), F, B);
        k_attn_path<<<grid, 128, 0, s>>>(st.cum, st.ylen, st.lens, attn, T, F);
        BV2_CUDA(cudaGetLastError()); e->launches++;
    }
    e->stage_begin("flow", s);
    e->run_flow(z, st.ylen32, st.gproj, s);
    e->stage_end("flow", s);
    e->debug("z", z);
    if (z_out) {
        k_c4_to_plain<<<bv2_engine::grid_tcb(F, I, B), 128, 0, s>>>(z.p, I, 0, F, z_out, I, F);
        BV2_CUDA(cudaGetLastError()); e->launches++;
    }
    Act zg = z;
    if (Fg < F) {
        zg = e->ws.act(B, I, Fg);
        // slice [:, :, :max_len] (reference models.py:1073): c4 rows are contiguous per (b, cg)
        BV2_CUDA(cudaMemcpy2DAsync(zg.p, (size_t)Fg * 16, z.p, (size_t)F * 16, (size_t)Fg * 16, (size_t)B * I / 4, cudaMemcpyDeviceToDevice, s));
    }
    if (open_stream) {
        e->gen_stream_open(zg, st.ylen32, st.gproj + e->goff_dec, e->gproj_n, o, max_chunk, ragged);
        st.active = false; st.finished = true;
        return BV2_OK;
    }
    e->stage_begin("generator", s);
    if (o16) {
        // 16-bit PCM epilogue (SURVEY.md section 8f.4): the float waveform stays in the workspace, only int16 leaves the engine
        // (halves the D2H / peer-store bytes); peak-normalised exactly like the reference's convert_to_16_bit_wav (webui.py:86)
        const long long L = (long long)Fg * e->hop;
        float* wf = e->ws.alloc((size_t)B * L);
        unsigned* peak = reinterpret_cast<unsigned*>(e->ws.alloc(B));
        long long* nval = reinterpret_cast<long long*>(e->ws.alloc(2 * (size_t)B));
        e->run_generator(zg, st.ylen32, st.gproj + e->goff_dec, e->gproj_n, wf, s, ragged);
        e->pcm16(wf, B, L, st.ylen, e->hop, nval, peak, o16, s);
    } else {
        e->run_generator(zg, st.ylen32, st.gproj + e->goff_dec, e->gproj_n, o, s, ragged);
    }
    e->stage_end("generator", s);
    st.active = false; st.finished = true;
    BV2_API_END(e)
}

int bv2_infer_finish(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len, float* o,
                     float* attn, float* y_mask, float* z_out, float* z_p, float* m_p, float* logs_p, void* stream) {
    if (!o) return BV2_ERR_ARG;
    return infer_finish_impl(e, noise_z, noise_ld, noise_scale, max_len, o, nullptr, attn, y_mask, z_out, z_p, m_p, logs_p, stream);
}

int bv2_infer_finish_pcm16(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len, int16_t* o16,
                           float* attn, float* y_mask, float* z_out, float* z_p, float* m_p, float* logs_p, void* stream) {
    if (!o16) return BV2_ERR_ARG;
    return infer_finish_impl(e, noise_z, noise_ld, noise_scale, max_len, nullptr, o16, attn, y_mask, z_out, z_p, m_p, logs_p, stream);
}

int bv2_infer_finish_ragged(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len, float* o, int16_t* o16,
                            float* attn, float* y_mask, float* z_out, float* z_p, float* m_p, float* logs_p, void* stream) {
    if (!o == !o16) return BV2_ERR_ARG;  // exactly one output
    return infer_finish_impl(e, noise_z, noise_ld, noise_scale, max_len, o, o16, attn, y_mask, z_out, z_p, m_p, logs_p, stream, false, 0, true);
}

int bv2_infer_finish_stream_bounded(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len, int32_t max_chunk_frames,
                                    float* o, float* attn, float* y_mask, float* z_out, float* z_p, float* m_p, float* logs_p, void* stream) {
    if (!o) return BV2_ERR_ARG;
    return infer_finish_impl(e, noise_z, noise_ld, noise_scale, max_len, o, nullptr, attn, y_mask, z_out, z_p, m_p, logs_p, stream, true,
                             std::max<int32_t>(max_chunk_frames, 0));
}

int bv2_infer_finish_stream_ragged(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len, int32_t max_chunk_frames,
                                   float* o, float* attn, float* y_mask, float* z_out, float* z_p, float* m_p, float* logs_p, void* stream) {
    if (!o) return BV2_ERR_ARG;
    return infer_finish_impl(e, noise_z, noise_ld, noise_scale, max_len, o, nullptr, attn, y_mask, z_out, z_p, m_p, logs_p, stream, true,
                             std::max<int32_t>(max_chunk_frames, 0), true);
}

int bv2_infer_finish_stream(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len, float* o,
                            float* attn, float* y_mask, float* z_out, float* z_p, float* m_p, float* logs_p, void* stream) {
    return bv2_infer_finish_stream_bounded(e, noise_z, noise_ld, noise_scale, max_len, 0, o, attn, y_mask, z_out, z_p, m_p, logs_p, stream);
}

int bv2_stream_advance(bv2_engine* e, int32_t frames, void* stream, int64_t* samples_ready) {
    BV2_API_BEGIN(e)
    auto& gs = e->gs;
    if (!gs.open) throw Error(BV2_ERR_STATE, "stream_advance without an open stream");
    if (frames <= gs.frontier) throw Error(BV2_ERR_STATE, "stream_advance: frames must exceed the frames already final");
    if (gs.max_chunk && (int64_t)frames - gs.frontier > gs.max_chunk)
        throw Error(BV2_ERR_ARG, "stream_advance: the chunk exceeds the stream's max_chunk_frames");
    const int f = std::min<int>(frames, gs.Fg);
    const std::vector<GenWin> w = gen_stream_plan(gs.g, gs.Fg, gs.frontier, f);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    e->stage_begin("generator", s);
    if (e->use_g2) {
        e->g2_stream_prepare(gs.frontier, f, s);
        e->g2_windows(gs.g, w, gs.t, true, gs.gdec, gs.g_stride, gs.o, s, gs.ragged ? gs.lens : nullptr);
    } else {
        e->gen_windows(gs.g, w, gs.a, true, gs.lens, gs.gdec, gs.g_stride, gs.o, s);
    }
    e->stage_end("generator", s);
    gs.frontier = f;
    if (samples_ready) *samples_ready = (int64_t)f * e->hop;
    if (f == gs.Fg) gs.open = false;
    BV2_API_END(e)
}

int bv2_attn_path(bv2_engine* e, float* attn, void* stream) {
    BV2_API_BEGIN(e)
    auto& st = e->st;
    BV2_CHECK(attn && (st.active || st.finished) && st.F > 0, "attn_path needs a preceding infer_begin");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    dim3 grid(cdiv(st.T, 128), st.F, st.B);
    k_attn_path<<<grid, 128, 0, s>>>(st.cum, st.ylen, st.lens, attn, st.T, st.F);
    BV2_CUDA(cudaGetLastError()); e->launches++;
    BV2_API_END(e)
}

int bv2_wave_to_pcm16(bv2_engine* e, int B, int64_t L, const float* wave, const int64_t* n_valid, int16_t* out, void* stream) {
    BV2_API_BEGIN(e)
    BV2_CHECK(e->finalized && B >= 1 && L >= 1 && wave && out, "wave_to_pcm16 args");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    unsigned* peak = nullptr;
    BV2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&peak), (size_t)B * sizeof(unsigned), s));
    e->pcm16(wave, B, L, reinterpret_cast<const long long*>(n_valid), 1, nullptr, peak, out, s);
    BV2_CUDA(cudaFreeAsync(peak, s));
    BV2_API_END(e)
}

// Workspace that covers every call within (B, T, F_cap) and, with with_stream, every stream with chunks of at most max_chunk frames
// (max_chunk <= 0: unbounded streams).  A stream over Fg <= max_chunk frames is unbounded, and its tensors are no larger than the
// bounded storage for max_chunk; the workspace needs grow with F otherwise.
static size_t reserve_bytes(const bv2_engine* e, int B, int T, int F_cap, bool with_stream, int max_chunk) {
    size_t need = ws_bytes_for(e->cfg, B, T, F_cap);
    if (!with_stream) return need;
    need = std::max(need, ws_stream_bytes(e, B, T, F_cap, F_cap, max_chunk));
    if (max_chunk >= 1) need = std::max(need, ws_enc_flow_bytes(e->cfg, B, T, F_cap) + e->stream_bytes(B, std::min(F_cap, max_chunk), max_chunk));
    return need;
}

static int reserve_impl(bv2_engine* e, int B, int T, int F_cap, bool with_stream, int max_chunk) {
    BV2_API_BEGIN(e)
    BV2_CHECK(e->finalized && B >= 1 && T >= 1 && F_cap >= 1, "reserve args");
    const bv2_config& c = e->cfg;
    const size_t need = reserve_bytes(e, B, T, F_cap, with_stream, max_chunk);
    const size_t pneed = persist_bytes_for(c, B, T, e->gproj_n);
    if (need > e->ws.cap() || pneed > e->persist.cap()) e->gs.open = false;  // regrowing an arena frees what an open stream reads
    e->ws.ensure(need);
    e->persist.ensure(pneed);
    BV2_API_END(e)
}

int bv2_reserve(bv2_engine* e, int B, int T, int F_cap) { return reserve_impl(e, B, T, F_cap, false, 0); }

int bv2_reserve_stream(bv2_engine* e, int B, int T, int F_cap, int32_t max_chunk_frames) {
    return reserve_impl(e, B, T, F_cap, true, std::max<int32_t>(max_chunk_frames, 0));
}

int64_t bv2_stream_bytes(const bv2_engine* e, int B, int32_t Fg, int32_t max_chunk_frames) {
    if (!e || !e->finalized || B < 1 || Fg < 1) return BV2_ERR_ARG;
    const int32_t cap = std::max<int32_t>(max_chunk_frames, 0);
    if (((int64_t)std::max(Fg, cap) + 1024) * e->hop > INT32_MAX) return BV2_ERR_ARG;  // rows of the waveform must fit an int
    try {
        return (int64_t)e->stream_bytes(B, Fg, cap);
    } catch (const Error& ex) { return ex.code == BV2_ERR_ARG ? BV2_ERR_ARG : BV2_ERR_INTERNAL; }  // ARG: a cap the Generator cannot bound
    catch (const std::exception&) { return BV2_ERR_INTERNAL; }
}

int bv2_text_encoder(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, const int64_t* sid,
                     const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert, const float* en_bert,
                     float* x_out, float* m_out, float* logs_out, void* stream) {
    BV2_API_BEGIN(e)
    BV2_CHECK(e->finalized, "not finalized");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bv2_config& c = e->cfg;
    const int H = c.hidden_channels, I = c.inter_channels;
    BV2_CHECK(B >= 1 && B <= 4096 && T >= 1 && x && x_lengths && sid && tone && language && bert && ja_bert && en_bert && x_out && m_out && logs_out,
              "text_encoder args");
    e->dbg.clear(); e->st.active = false;
    e->ws.ensure(ws_bytes_for(c, B, T, 0)); e->ws_reset();
    e->validate_sync(B, T, x, tone, language, sid, x_lengths, s);
    int* lens = e->lens_to_device(x_lengths, B, e->ws, s);
    float* g = e->ws.alloc((size_t)B * c.gin_channels);
    float* gp = e->ws.alloc((size_t)B * e->gproj_n);
    k_gather_rows<<<B, 128, 0, s>>>(e->emb_g, reinterpret_cast<const long long*>(sid), g, c.gin_channels, c.n_speakers);
    e->launches++;
    e->run_gproj(g, B, gp, s);
    Act h = e->ws.act(B, H, T), stats = e->ws.act(B, 2 * I, T);
    e->run_text_encoder(B, T, x, tone, language, bert, ja_bert, en_bert, lens, gp, h, stats, s);
    k_c4_to_plain<<<bv2_engine::grid_tcb(T, H, B), 128, 0, s>>>(h.p, H, 0, T, x_out, H, T);
    k_c4_to_plain<<<bv2_engine::grid_tcb(T, I, B), 128, 0, s>>>(stats.p, 2 * I, 0, T, m_out, I, T);
    k_c4_to_plain<<<bv2_engine::grid_tcb(T, I, B), 128, 0, s>>>(stats.p, 2 * I, I, T, logs_out, I, T);
    BV2_CUDA(cudaGetLastError()); e->launches += 3;
    BV2_API_END(e)
}

int bv2_duration(bv2_engine* e, int B, int T, const float* x, const int64_t* x_lengths, const int64_t* sid, const float* noise_w,
                 float noise_scale_w, float* logw_sdp, float* logw_dp, void* stream) {
    BV2_API_BEGIN(e)
    BV2_CHECK(e->finalized, "not finalized");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bv2_config& c = e->cfg;
    const int H = c.hidden_channels;
    BV2_CHECK(B >= 1 && B <= 4096 && T >= 1 && x && x_lengths && sid && noise_w && logw_sdp && logw_dp, "duration args");
    e->dbg.clear(); e->st.active = false;
    e->ws.ensure(ws_bytes_for(c, B, T, 0)); e->ws_reset();
    e->validate_sync(B, T, nullptr, nullptr, nullptr, sid, x_lengths, s);
    int* lens = e->lens_to_device(x_lengths, B, e->ws, s);
    float* g = e->ws.alloc((size_t)B * c.gin_channels);
    float* gp = e->ws.alloc((size_t)B * e->gproj_n);
    k_gather_rows<<<B, 128, 0, s>>>(e->emb_g, reinterpret_cast<const long long*>(sid), g, c.gin_channels, c.n_speakers);
    e->launches++;
    e->run_gproj(g, B, gp, s);
    Act h = e->ws.act(B, H, T);
    k_plain_to_c4<<<bv2_engine::grid_tcb(T, H, B), 128, 0, s>>>(x, H, (long long)H * T, T, h.p, H, 0, T, nullptr, 1.f);
    e->launches++;
    float* z = e->ws.alloc((size_t)B * 2 * T);
    Act dp = e->ws.act(B, 4, T);
    int zch = 0;
    e->run_durations(h, lens, gp, noise_w, noise_scale_w, nullptr, z, dp, &zch, s);
    float* wc = e->ws.alloc((size_t)B * T);
    int* cum = reinterpret_cast<int*>(e->ws.alloc((size_t)B * T));
    long long* yl = reinterpret_cast<long long*>(e->ws.alloc(2 * (size_t)B + 2));
    k_durations<<<B, 1024, 0, s>>>(z, zch, e->ea_m[0], e->ea_logs[0], dp.p, 0.5f, 1.f, nullptr, nullptr, lens, T, logw_sdp, logw_dp, wc, cum, yl,
                                   nullptr);
    BV2_CUDA(cudaGetLastError()); e->launches++;
    BV2_API_END(e)
}

int bv2_flow_reverse(bv2_engine* e, int B, int F, const float* z_p, const int64_t* y_lengths, const int64_t* sid, float* z_out,
                     void* stream) {
    BV2_API_BEGIN(e)
    BV2_CHECK(e->finalized, "not finalized");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bv2_config& c = e->cfg;
    const int I = c.inter_channels;
    BV2_CHECK(B >= 1 && B <= 4096 && F >= 1 && z_p && y_lengths && sid && z_out, "flow_reverse args");
    e->dbg.clear(); e->st.active = false;
    e->ws.ensure(ws_bytes_for(c, B, 1, F)); e->ws_reset();
    e->validate_sync(B, F, nullptr, nullptr, nullptr, sid, y_lengths, s);
    int* lens = e->lens_to_device(y_lengths, B, e->ws, s);
    float* g = e->ws.alloc((size_t)B * c.gin_channels);
    float* gp = e->ws.alloc((size_t)B * e->gproj_n);
    k_gather_rows<<<B, 128, 0, s>>>(e->emb_g, reinterpret_cast<const long long*>(sid), g, c.gin_channels, c.n_speakers);
    e->launches++;
    e->run_gproj(g, B, gp, s);
    Act z = e->ws.act(B, I, F);
    k_plain_to_c4<<<bv2_engine::grid_tcb(F, I, B), 128, 0, s>>>(z_p, I, (long long)I * F, F, z.p, I, 0, F, nullptr, 1.f);
    e->launches++;
    e->run_flow(z, lens, gp, s);
    k_c4_to_plain<<<bv2_engine::grid_tcb(F, I, B), 128, 0, s>>>(z.p, I, 0, F, z_out, I, F);
    BV2_CUDA(cudaGetLastError()); e->launches++;
    BV2_API_END(e)
}

// lengths (device, may be null): a ragged batch, item b at its own length clamped to [1, F]
static int generator_impl(bv2_engine* e, int B, int F, const float* z_in, const float* g, const int64_t* lengths, float* o, void* stream) {
    BV2_API_BEGIN(e)
    BV2_CHECK(e->finalized, "not finalized");
    BV2_CHECK(B >= 1 && F >= 1 && z_in && g && o, "generator args");
    if (lengths && !e->use_g2) throw Error(BV2_ERR_ARG, "a ragged batch needs the FP16 Generator (precision fp16 or fp16g)");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bv2_config& c = e->cfg;
    const int I = c.inter_channels;
    e->dbg.clear(); e->st.active = false;
    e->ws.ensure(ws_bytes_for(c, B, 1, F)); e->ws_reset();
    int* lens = nullptr;
    if (lengths) {
        lens = reinterpret_cast<int*>(e->ws.alloc(B));
        k_lengths_clamp<<<cdiv(B, 128), 128, 0, s>>>(reinterpret_cast<const long long*>(lengths), lens, B, F);
        BV2_CUDA(cudaGetLastError()); e->launches++;
    }
    float* gp = e->ws.alloc((size_t)B * e->gproj_n);
    e->run_gproj(g, B, gp, s);
    Act z = e->ws.act(B, I, F);
    k_plain_to_c4<<<bv2_engine::grid_tcb(F, I, B), 128, 0, s>>>(z_in, I, (long long)I * F, F, z.p, I, 0, F, nullptr, 1.f);
    BV2_CUDA(cudaGetLastError()); e->launches++;
    e->stage_begin("generator", s);
    e->run_generator(z, lens, gp + e->goff_dec, e->gproj_n, o, s, lengths != nullptr);
    e->stage_end("generator", s);
    BV2_API_END(e)
}

int bv2_generator(bv2_engine* e, int B, int F, const float* z_in, const float* g, float* o, void* stream) {
    return generator_impl(e, B, F, z_in, g, nullptr, o, stream);
}

int bv2_generator_ragged(bv2_engine* e, int B, int F, const float* z_in, const float* g, const int64_t* lengths, float* o, void* stream) {
    if (!lengths) return BV2_ERR_ARG;
    return generator_impl(e, B, F, z_in, g, lengths, o, stream);
}

int64_t bv2_debug_read(bv2_engine* e, const char* name, float* host_out, int64_t capacity) {
    if (!e || !name || !host_out) return BV2_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    try {
        BV2_CUDA(cudaSetDevice(e->device));
        auto it = e->dbg.find(name);
        if (it == e->dbg.end()) { e->err = std::string("no debug buffer ") + name; return BV2_ERR_ARG; }
        const DebugBuf& d = it->second;
        int64_t n = (int64_t)d.B * d.C * d.T;
        if (n > capacity) { e->err = "capacity"; return BV2_ERR_ARG; }
        BV2_CUDA(cudaDeviceSynchronize());
        if (!d.c4) {
            BV2_CUDA(cudaMemcpy(host_out, d.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
        } else {
            float* tmp = nullptr;
            BV2_CUDA(cudaMalloc(&tmp, (size_t)n * 4));
            k_c4_to_plain<<<bv2_engine::grid_tcb(d.T, d.C, d.B), 128>>>(d.p, d.C, 0, d.T, tmp, d.C, d.T);
            cudaError_t er = cudaMemcpy(host_out, tmp, (size_t)n * 4, cudaMemcpyDeviceToHost);
            cudaFree(tmp);
            BV2_CUDA(er);
        }
        return n;
    } catch (const bv2::Error& ex) { e->err = ex.what(); return ex.code; }
}

int bv2_set_profiling(bv2_engine* e, int enable) {
    if (!e) return BV2_ERR_ARG;
    std::lock_guard<std::mutex> lk(e->mu);
    e->profiling = enable != 0;
    return BV2_OK;
}

float bv2_stage_ms(bv2_engine* e, const char* stage) {
    if (!e || !stage) return -1.f;
    std::lock_guard<std::mutex> lk(e->mu);
    auto it = e->stage_ev.find(stage);
    if (it == e->stage_ev.end() || !it->second.rec) return -1.f;
    cudaSetDevice(e->device);
    if (cudaEventSynchronize(it->second.b) != cudaSuccess) return -1.f;
    float ms = -1.f;
    if (cudaEventElapsedTime(&ms, it->second.a, it->second.b) != cudaSuccess) return -1.f;
    return ms;
}

int64_t bv2_launch_count(const bv2_engine* e) { return e ? e->launches : 0; }
int64_t bv2_workspace_bytes(const bv2_engine* e) { return e ? (int64_t)(e->ws.cap() + e->persist.cap()) : 0; }
int64_t bv2_workspace_grows(const bv2_engine* e) { return e ? (int64_t)(e->ws.grows() + e->persist.grows()) : 0; }
// ---- peer output slab (multi-GPU exchange step): plain CUDA IPC plumbing, no engine state
static_assert(sizeof(cudaIpcMemHandle_t) == BV2_IPC_HANDLE_BYTES, "IPC handle size");
int bv2_peer_slab_alloc(int dev, int64_t bytes, void** dptr, unsigned char* handle_out) {
    if (!dptr || !handle_out || bytes <= 0) return BV2_ERR_ARG;
    *dptr = nullptr;
    if (cudaSetDevice(dev) != cudaSuccess) return BV2_ERR_CUDA;
    void* p = nullptr;
    if (cudaMalloc(&p, (size_t)bytes) != cudaSuccess) return BV2_ERR_CUDA;
    cudaIpcMemHandle_t h;
    if (cudaMemset(p, 0, (size_t)bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess ||
        cudaIpcGetMemHandle(&h, p) != cudaSuccess) { cudaFree(p); return BV2_ERR_CUDA; }
    memcpy(handle_out, &h, sizeof(h));
    *dptr = p;
    return BV2_OK;
}
int bv2_peer_slab_open(int dev, const unsigned char* handle, void** dptr) {
    if (!dptr || !handle) return BV2_ERR_ARG;
    *dptr = nullptr;
    if (cudaSetDevice(dev) != cudaSuccess) return BV2_ERR_CUDA;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    void* p = nullptr;
    if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); return BV2_ERR_CUDA; }
    *dptr = p;
    return BV2_OK;
}
int bv2_peer_slab_close(int dev, void* dptr) {
    if (!dptr) return BV2_ERR_ARG;
    if (cudaSetDevice(dev) != cudaSuccess || cudaIpcCloseMemHandle(dptr) != cudaSuccess) return BV2_ERR_CUDA;
    return BV2_OK;
}
int bv2_peer_slab_free(int dev, void* dptr) {
    if (!dptr) return BV2_ERR_ARG;
    if (cudaSetDevice(dev) != cudaSuccess || cudaFree(dptr) != cudaSuccess) return BV2_ERR_CUDA;
    return BV2_OK;
}
int bv2_peer_write(int dev, void* dst, const void* src, int64_t bytes, void* stream) {
    if (!dst || !src || bytes < 0) return BV2_ERR_ARG;
    if (cudaSetDevice(dev) != cudaSuccess) return BV2_ERR_CUDA;
    if (bytes && cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream) != cudaSuccess) return BV2_ERR_CUDA;
    return BV2_OK;
}

const char* bv2_last_error(const bv2_engine* e) { return e ? e->err.c_str() : "null engine"; }
void bv2_destroy(bv2_engine* e) { delete e; }

}  // extern "C"
