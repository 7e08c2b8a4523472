// Kernel test harness: a thin extern "C" layer over the product headers, loaded by tests/test_kernels_gpu.py through ctypes.
// Python builds every device layout with numpy (c4 [B][C/4][T][4] fp32, c8 [B][C/8][T][8] halves, H8 with its zero halo rows) and passes
// raw host buffers; the harness uploads them, packs the weights with the product packers, launches one kernel, synchronises and copies
// the output back.  Every output buffer sits between two guard regions filled with a byte pattern; the caller supplies the output's
// initial contents (NaN where the kernel writes, old values where it must not or where it accumulates) and gets back the whole
// buffer plus a guard check.  The kh_*_plan entry points run the host planning only (no device access).
// Built with the product flags by bert_vits2_b200/_lib.py (build_harness); see tests/kernel_harness.py.
#include <cstring>
#include <functional>
#include <string>
#include <vector>
#include "../../bert_vits2_b200/csrc/tc_attn.cuh"
#include "../../bert_vits2_b200/csrc/tc_gen.cuh"

using namespace bv2;

namespace {
constexpr size_t GUARD = 4096;            // bytes before and after every output buffer
constexpr unsigned char GUARD_BYTE = 0xA5;
thread_local std::string g_err;
int* g_flag = nullptr;                    // host view of the device error flag (barrier timeout)
bool g_init = false;

struct Arena {
    std::vector<void*> ptrs;
    ~Arena() { for (void* p : ptrs) cudaFree(p); }
    void* alloc(size_t bytes) {
        void* p = nullptr;
        BV2_CUDA(cudaMalloc(&p, bytes < 16 ? 16 : bytes));
        ptrs.push_back(p);
        return p;
    }
    template <typename T> T* up(const T* h, size_t n) {
        if (!h) return nullptr;
        T* d = static_cast<T*>(alloc(n * sizeof(T)));
        BV2_CUDA(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
        return d;
    }
    // guarded output: [GUARD][bytes][GUARD], the middle initialised from `init`
    uint8_t* guarded(const void* init, size_t bytes) {
        uint8_t* d = static_cast<uint8_t*>(alloc(bytes + 2 * GUARD));
        BV2_CUDA(cudaMemset(d, GUARD_BYTE, bytes + 2 * GUARD));
        BV2_CUDA(cudaMemcpy(d + GUARD, init, bytes, cudaMemcpyHostToDevice));
        return d + GUARD;
    }
};
// copies the output back and returns 1 if both guard regions are intact
int read_guarded(const uint8_t* d, void* out, size_t bytes) {
    std::vector<uint8_t> h(bytes + 2 * GUARD);
    BV2_CUDA(cudaMemcpy(h.data(), d - GUARD, h.size(), cudaMemcpyDeviceToHost));
    std::memcpy(out, h.data() + GUARD, bytes);
    for (size_t i = 0; i < GUARD; i++)
        if (h[i] != GUARD_BYTE || h[GUARD + bytes + i] != GUARD_BYTE) return 0;
    return 1;
}
void init_device() {
    if (g_init) return;
    g_flag = tc_init_device();
    tc_flow_attn_init_device();
    g2_init_device();
    g_init = true;
}
void finish(int* err_flag) {
    BV2_CUDA(cudaGetLastError());
    BV2_CUDA(cudaDeviceSynchronize());
    *err_flag = *g_flag;
    if (*g_flag) { *g_flag = 0; tc_clear_error(); }
}
template <typename F>
int guarded_call(F&& f) {
    try {
        f();
        return 0;
    } catch (const std::exception& ex) {
        g_err = ex.what();
        return -1;
    }
}
// uploader for the packers; without an arena it hands out a non-null dummy pointer (planning only, no device access)
std::function<float*(const std::vector<float>&)> uploader(Arena* a) {
    if (!a) return [](const std::vector<float>&) { return reinterpret_cast<float*>(256); };
    return [a](const std::vector<float>& v) { return a->up(v.data(), v.size()); };
}
float* const DUMMY = reinterpret_cast<float*>(256);
}  // namespace

extern "C" {

// ---- tc_conv1d ----------------------------------------------------------------------------------------------------
struct KhTcArgs {
    int B, T, Cin, Cout, K, u;  // u > 0: polyphase ConvTranspose1d, weights [Cin][Cout][K]; else weights [Cout][Cin][K]
    int x_C, y_C;               // channels of the x / y tensors (windows via cin_off / cout_off)
    int nt, kc, f16, num_sms;
    float in_slope; int in_mask, relu, res_mode, res_C_total, res_c_off, accumulate;
    float out_scale; int out_mask, bias_b_stride, cin_off, cout_off, dil, out_tf32, skip_xform, in_f16, out_f16, gate;
    int res_is_y;               // the residual is the output tensor itself (in-place update, as the engine does)
    const float* w; const float* bias; const void* x; long long x_bytes;
    const float* res; long long res_elems;
    const int* lens; const float* bias_b; long long bias_b_elems; const float* ln_gamma; const float* ln_beta;
};
struct KhTcPlan { int kind, gen, f16, res_smem, nas, nws, grid_x, grid_y, grid_z, threads, mtiles, ntiles, total, tiles_per_cta, nt; long long smem; };

// The product objects of one case: packed weights, epilogue, tensors.  ar = nullptr: planning only (dummy pointers, no device access).
struct TcCase { TcConvW cw; TcEpi e; Act x, y; };
static TcCase tc_case(const KhTcArgs& a, Arena* ar, const void* dx, void* dy, const float* dres, const int* dlens, const float* dbias_b,
                      const float* dg, const float* db) {
    TcCase c;
    auto up = uploader(ar);
    const size_t nw = (size_t)a.Cin * a.Cout * a.K;
    const std::vector<float> w = ar ? std::vector<float>(a.w, a.w + nw) : std::vector<float>(nw, 0.f);
    c.cw = a.u ? tc_pack_upsample(up, w, a.Cin, a.Cout, a.K, a.u, a.kc, a.f16, ar != nullptr, a.nt ? a.nt : 128)
               : tc_pack_weights(up, w, a.Cout, a.Cin, a.K, a.nt, a.f16, a.kc, ar != nullptr);
    TcEpi& e = c.e;
    e.in_slope = a.in_slope; e.in_mask = a.in_mask; e.relu = a.relu; e.res_mode = a.res_mode; e.res = dres;
    e.res_C_total = a.res_C_total; e.res_c_off = a.res_c_off; e.accumulate = a.accumulate; e.out_scale = a.out_scale;
    e.out_mask = a.out_mask; e.lens = dlens; e.bias_b = dbias_b; e.bias_b_stride = a.bias_b_stride;
    e.cin_off = a.cin_off; e.cout_off = a.cout_off; e.dil = a.dil ? a.dil : 1;
    e.out_tf32 = a.out_tf32; e.skip_xform = a.skip_xform; e.in_f16 = a.in_f16; e.out_f16 = a.out_f16; e.gate = a.gate;
    e.ln_gamma = dg; e.ln_beta = db;
    c.x.p = (float*)dx; c.x.B = a.B; c.x.C = a.x_C; c.x.T = a.T;
    c.y.p = (float*)dy; c.y.B = a.B; c.y.C = a.y_C; c.y.T = a.T * (a.u ? a.u : 1);
    return c;
}
static void fill_plan(const TcConvPlan& pl, const TcConvW& cw, KhTcPlan* o) {
    o->kind = pl.kind; o->gen = pl.gen; o->f16 = pl.f16; o->res_smem = pl.res_smem; o->nas = pl.nas; o->nws = pl.nws;
    o->grid_x = (int)pl.grid.x; o->grid_y = (int)pl.grid.y; o->grid_z = (int)pl.grid.z; o->threads = (int)pl.block.x;
    o->mtiles = pl.mtiles; o->ntiles = pl.ntiles; o->total = pl.total;
    o->tiles_per_cta = pl.kind == TC_ONE_TILE ? 1 : (pl.total + (int)pl.grid.x - 1) / (int)pl.grid.x;
    o->nt = cw.nt;
    o->smem = (long long)pl.smem;
}

// Host planning only: which kernel / pipeline shape tc_conv1d would launch.  Returns 0, or -1 with kh_last_error().
int kh_tc_plan(const KhTcArgs* a, KhTcPlan* out) {
    return guarded_call([&] {
        const TcCase c = tc_case(*a, nullptr, DUMMY, DUMMY, (a->res || a->res_is_y) ? DUMMY : nullptr, a->lens ? (const int*)DUMMY : nullptr,
                                 a->bias_b ? DUMMY : nullptr, a->ln_gamma ? DUMMY : nullptr, a->ln_beta ? DUMMY : nullptr);
        TcParams p;
        fill_plan(tc_conv_plan(c.cw, DUMMY, c.x, c.y, c.e, a->num_sms, p), c.cw, out);
    });
}

// One tc_conv1d launch.  y: in = initial contents of the output tensor (y_bytes), out = its contents after the kernel.
int kh_tc_conv1d(const KhTcArgs* a, void* y, long long y_bytes, KhTcPlan* plan, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        const void* dx = ar.up(static_cast<const uint8_t*>(a->x), (size_t)a->x_bytes);
        uint8_t* dy = ar.guarded(y, (size_t)y_bytes);
        const float* dres = a->res_is_y ? reinterpret_cast<const float*>(dy) : ar.up(a->res, (size_t)a->res_elems);
        const TcCase c = tc_case(*a, &ar, dx, dy, dres, ar.up(a->lens, (size_t)a->B), ar.up(a->bias_b, (size_t)a->bias_b_elems),
                                 ar.up(a->ln_gamma, (size_t)a->Cout), ar.up(a->ln_beta, (size_t)a->Cout));
        const float* dbias = ar.up(a->bias, (size_t)a->Cout);
        TcParams p;
        fill_plan(tc_conv_plan(c.cw, dbias, c.x, c.y, c.e, a->num_sms, p), c.cw, plan);
        tc_conv1d(c.cw, dbias, c.x, c.y, c.e, 0, a->num_sms);  // the product launcher (it re-plans to the same result)
        finish(err_flag);
        *guard_ok = read_guarded(dy, y, (size_t)y_bytes);
    });
}

// ---- fused flow attention ------------------------------------------------------------------------------------------
// qkv: 16-bit c8 [B][3H/8][T][8]; att: 16-bit c8 [B][H/8][T][8] (in = initial contents, out = result); rel_k / rel_v [2w+1][H/heads]
int kh_flow_attn(const void* qkv, const float* rel_k, const float* rel_v, const int* lens, int B, int T, int H, int heads, int window,
                 int ks_override, int num_sms, void* att, int* ks_used, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        const int dk = H / heads, nrel = 2 * window + 1;
        const size_t qkv_bytes = (size_t)B * 3 * H * T * 2, att_bytes = (size_t)B * H * T * 2;
        Act q; q.p = (float*)ar.up(static_cast<const uint8_t*>(qkv), qkv_bytes); q.B = B; q.C = 3 * H; q.T = T;
        Act o; o.p = (float*)ar.guarded(att, att_bytes); o.B = B; o.C = H; o.T = T;
        const float* dk_ = ar.up(rel_k, (size_t)nrel * dk);
        const float* dv_ = ar.up(rel_v, (size_t)nrel * dk);
        const int* dl = ar.up(lens, (size_t)B);
        // the key split tc_flow_attn picks (same rule; ks_override wins)
        const int qtiles = cdiv(T, 128), ctas = qtiles * heads * B;
        int ks = 1;
        while (ks < 4 && 2 * ks <= qtiles && ctas * 2 * ks <= num_sms) ks *= 2;
        *ks_used = ks_override > 0 ? ks_override : ks;
        tc_flow_attn(q, o, dk_, dv_, dl, heads, window, 0, num_sms, ks_override);
        finish(err_flag);
        *guard_ok = read_guarded(reinterpret_cast<const uint8_t*>(o.p), att, att_bytes);
    });
}

// ---- Generator conv on H8 tensors ----------------------------------------------------------------------------------------
struct KhG2Args {
    int B, T, Cin, Cout, K, u, dil;  // u > 0: polyphase ConvTranspose1d, weights [Cin][Cout][K]; else [Cout][Cin][K]
    int residual, accumulate; float out_scale; int bias_b_stride, st_override, num_sms;
    const float* w; const float* bias; const float* bias_b; long long bias_b_elems;
    const void* x;    // H8 [B][Cin/8][PADL + T + PADR][8] halves (halo rows included)
    const void* res;  // H8 like y, or null
};
struct KhG2Plan { int resident, NG, MG, nas, nws, grid_x, grid_y, grid_z, nt, kc; long long smem; };

static G2Plan g2_plan_of(const KhG2Args& a, Arena* ar, const H8& x, const H8& y, const H8* res, const float* dbias, const float* dbias_b,
                         G2Params& p, TcConvW& cw) {
    auto up = uploader(ar);
    std::vector<float> w;
    const size_t nw = (size_t)a.Cin * a.Cout * a.K;
    if (ar) w.assign(a.w, a.w + nw);
    else w.assign(nw, 0.f);
    cw = a.u ? tc_pack_upsample(up, w, a.Cin, a.Cout, a.K, a.u, g2_kc(a.Cin), 1, ar != nullptr, 128)
             : tc_pack_weights(up, w, a.Cout, a.Cin, a.K, g2_nt(a.Cout), 1, g2_kc(a.Cin), ar != nullptr);
    G2Epi e;
    e.res = res; e.accumulate = a.accumulate; e.out_scale = a.out_scale; e.bias_b = dbias_b; e.bias_b_stride = a.bias_b_stride;
    e.dil = a.dil ? a.dil : 1; e.st_override = a.st_override;
    return g2_conv_plan(cw, dbias, x, y, e, a.num_sms, p);
}
static void fill_g2(const G2Plan& pl, const TcConvW& cw, KhG2Plan* o) {
    o->resident = pl.resident; o->NG = pl.NG; o->MG = pl.MG; o->nas = pl.nas; o->nws = pl.nws;
    o->grid_x = (int)pl.grid.x; o->grid_y = (int)pl.grid.y; o->grid_z = (int)pl.grid.z; o->nt = cw.nt; o->kc = cw.KC; o->smem = (long long)pl.smem;
}
static H8 h8_view(uint4* base, int B, int C, int T) {
    H8 t; t.B = B; t.C = C; t.T = T; t.Tp = G2_PADL + T + G2_PADR; t.p = base ? base + G2_PADL : nullptr;
    return t;
}

int kh_g2_plan(const KhG2Args* a, KhG2Plan* out) {
    return guarded_call([&] {
        const int To = a->T * (a->u ? a->u : 1);
        uint4* dummy = reinterpret_cast<uint4*>(4096);
        H8 x = h8_view(dummy, a->B, a->Cin, a->T), y = h8_view(dummy, a->B, a->Cout, To), r = h8_view(dummy, a->B, a->Cout, To);
        G2Params p; TcConvW cw;
        const G2Plan pl = g2_plan_of(*a, nullptr, x, y, a->res ? &r : nullptr, DUMMY, a->bias_b ? DUMMY : nullptr, p, cw);
        fill_g2(pl, cw, out);
    });
}

// One g2_conv launch.  y: H8 output with halo rows (in = initial contents, out = result).
int kh_g2_conv(const KhG2Args* a, void* y, KhG2Plan* plan, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        const int To = a->T * (a->u ? a->u : 1);
        const size_t xb = H8::bytes(a->B, a->Cin, a->T), yb = H8::bytes(a->B, a->Cout, To);
        H8 x = h8_view(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(a->x), xb)), a->B, a->Cin, a->T);
        H8 yy = h8_view(reinterpret_cast<uint4*>(ar.guarded(y, yb)), a->B, a->Cout, To);
        H8 r;
        if (a->res) r = h8_view(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(a->res), yb)), a->B, a->Cout, To);
        const float* dbias = ar.up(a->bias, (size_t)a->Cout);
        const float* dbias_b = ar.up(a->bias_b, (size_t)a->bias_b_elems);
        G2Params p; TcConvW cw;
        const G2Plan pl = g2_plan_of(*a, &ar, x, yy, a->res ? &r : nullptr, dbias, dbias_b, p, cw);
        fill_g2(pl, cw, plan);
        G2Epi e;
        e.res = a->res ? &r : nullptr; e.accumulate = a->accumulate; e.out_scale = a->out_scale; e.bias_b = dbias_b; e.bias_b_stride = a->bias_b_stride;
        e.dil = a->dil ? a->dil : 1; e.st_override = a->st_override;
        g2_conv(cw, dbias, x, yy, e, 0, a->num_sms);
        finish(err_flag);
        *guard_ok = read_guarded(reinterpret_cast<const uint8_t*>(yy.p - G2_PADL), y, yb);
    });
}

const char* kh_last_error() { return g_err.c_str(); }
int kh_g2_padl() { return G2_PADL; }
int kh_g2_padr() { return G2_PADR; }

}  // extern "C"
