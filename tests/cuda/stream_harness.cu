// Streaming harness: the kernel harness (kernel_harness.cu, included whole) plus the Generator's time-window launches and the
// wavefront planner of gen_stream.cuh, loaded by tests/test_stream_*.py through ctypes.  Same buffer conventions as the kernel
// harness: every output sits between two guard regions and the caller supplies its initial contents.
// Built with the product flags by bert_vits2_b200/_lib.py (build_harness(stream=True)); see tests/stream_harness.py.
#include "kernel_harness.cu"
#include "../../bert_vits2_b200/csrc/gen_stream.cuh"
#include "../../bert_vits2_b200/csrc/kernels_simt.cuh"

extern "C" {

// ---- planner (host only, no device access) --------------------------------------------------------------------------------
// Layers of the Generator graph for Fg frames: desc[n][11] = kind, stage, branch, dil_idx, in, out, res, reach, u, L_in, L_out;
// tensor_len[n_tensors].  Returns the number of layers (or -1), writes *n_tensors and *hop.
int kh_gen_graph(const bv2_config* c, int Fg, int* desc, int cap, int* tensor_len, int tcap, int* n_tensors, int* hop) {
    int n = -1;
    guarded_call([&] {
        const GenGraph g = gen_graph(*c, Fg);
        BV2_CHECK((int)g.layers.size() <= cap && (int)g.tensor_len.size() <= tcap, "kh_gen_graph capacity");
        for (size_t i = 0; i < g.layers.size(); i++) {
            const GenLayer& l = g.layers[i];
            const int v[11] = {l.kind, l.stage, l.branch, l.dil_idx, l.in, l.out, l.res, l.reach, l.u, l.L_in, l.L_out};
            std::memcpy(desc + 11 * i, v, sizeof(v));
        }
        for (size_t i = 0; i < g.tensor_len.size(); i++) tensor_len[i] = g.tensor_len[i];
        *n_tensors = (int)g.tensor_len.size(); *hop = g.hop;
        n = (int)g.layers.size();
    });
    return n;
}

// The windows of the chunk that takes the stream from `done` to `target` frames: win[n][2] = t_begin, t_end.  Returns n or -1.
int kh_gen_stream_plan(const bv2_config* c, int Fg, int done, int target, int* win, int cap) {
    int n = -1;
    guarded_call([&] {
        const GenGraph g = gen_graph(*c, Fg);
        const std::vector<GenWin> w = gen_stream_plan(g, Fg, done, target);
        BV2_CHECK((int)w.size() <= cap, "kh_gen_stream_plan capacity");
        for (size_t i = 0; i < w.size(); i++) { win[2 * i] = w[i].t_begin; win[2 * i + 1] = w[i].t_end; }
        n = (int)w.size();
    });
    return n;
}

// ---- window launches --------------------------------------------------------------------------------------------------------
// One g2_conv launch over the output window [t_begin, t_end) (t_end = -1: the whole output).  As kh_g2_conv otherwise.
int kh_g2_conv_window(const KhG2Args* a, int t_begin, int t_end, void* y, KhG2Plan* plan, int* guard_ok, int* err_flag) {
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
        g2_plan_of(*a, &ar, x, yy, a->res ? &r : nullptr, dbias, dbias_b, p, cw);  // packs the weights
        G2Epi e;
        e.res = a->res ? &r : nullptr; e.accumulate = a->accumulate; e.out_scale = a->out_scale; e.bias_b = dbias_b; e.bias_b_stride = a->bias_b_stride;
        e.dil = a->dil ? a->dil : 1; e.st_override = a->st_override; e.t_begin = t_begin; e.t_end = t_end;
        fill_g2(g2_conv_plan(cw, dbias, x, yy, e, a->num_sms, p), cw, plan);
        g2_conv(cw, dbias, x, yy, e, 0, a->num_sms);
        finish(err_flag);
        *guard_ok = read_guarded(reinterpret_cast<const uint8_t*>(yy.p - G2_PADL), y, yb);
    });
}

// conv_post + tanh (16 channels, 7 taps) on an H8 input x (halo rows included) over the output window [t_begin, t_end) of T samples.
// w: [16][7]; y: [B][T] fp32 (in = initial contents, out = result).
int kh_conv_post_window(const void* x, const float* w, int B, int T, int t_begin, int t_end, float* y, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        BV2_CHECK(0 <= t_begin && t_begin < t_end && t_end <= T, "conv_post window");
        Arena ar;
        const size_t xb = H8::bytes(B, 16, T), yb = (size_t)B * T * sizeof(float);
        H8 xx = h8_view(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(x), xb)), B, 16, T);
        uint8_t* dy = ar.guarded(y, yb);
        PostW<16, 7> pw;
        std::memcpy(pw.w, w, sizeof(pw.w));
        launch_pdl(k_conv_post_tanh_h8<16, 7>, dim3(cdiv(t_end - t_begin, 512), B), dim3(256), 0, (cudaStream_t)0, (const uint4*)xx.p, xx.Tp, 0, pw,
                   reinterpret_cast<float*>(dy), T, t_begin, t_end);
        finish(err_flag);
        *guard_ok = read_guarded(dy, y, yb);
    });
}

// One tc_conv1d launch over the output window [t_begin, t_end) (t_end = -1: the whole output).  As kh_tc_conv1d otherwise.
int kh_tc_conv1d_window(const KhTcArgs* a, int t_begin, int t_end, void* y, long long y_bytes, KhTcPlan* plan, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        const void* dx = ar.up(static_cast<const uint8_t*>(a->x), (size_t)a->x_bytes);
        uint8_t* dy = ar.guarded(y, (size_t)y_bytes);
        const float* dres = a->res_is_y ? reinterpret_cast<const float*>(dy) : ar.up(a->res, (size_t)a->res_elems);
        TcCase c = tc_case(*a, &ar, dx, dy, dres, ar.up(a->lens, (size_t)a->B), ar.up(a->bias_b, (size_t)a->bias_b_elems),
                           ar.up(a->ln_gamma, (size_t)a->Cout), ar.up(a->ln_beta, (size_t)a->Cout));
        c.e.t_begin = t_begin; c.e.t_end = t_end;
        const float* dbias = ar.up(a->bias, (size_t)a->Cout);
        TcParams p;
        fill_plan(tc_conv_plan(c.cw, dbias, c.x, c.y, c.e, a->num_sms, p), c.cw, plan);
        tc_conv1d(c.cw, dbias, c.x, c.y, c.e, 0, a->num_sms);
        finish(err_flag);
        *guard_ok = read_guarded(dy, y, (size_t)y_bytes);
    });
}

// SIMT fp32 Generator kernels on c4 tensors, each over an output window (t_end = -1: the whole output).
// k_conv1d_c4 through launch_conv1d: w [Cout][Cin][K]; residual (c4 like y) optional; y: c4 [B][Cout/4][T][4] (in = initial contents).
int kh_conv1d_window(int B, int T, int Cin, int Cout, int K, int dil, float in_slope, const float* w, const float* bias, const float* x,
                     const float* res, int accumulate, float out_scale, int t_begin, int t_end, float* y, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        std::vector<float> wp((size_t)Cin * K * Cout);  // [Cin][K][Cout]
        for (int co = 0; co < Cout; co++)
            for (int ci = 0; ci < Cin; ci++)
                for (int j = 0; j < K; j++) wp[((size_t)ci * K + j) * Cout + co] = w[((size_t)co * Cin + ci) * K + j];
        const size_t yb = (size_t)B * Cout * T * sizeof(float);
        uint8_t* dy = ar.guarded(y, yb);
        ConvArgs a;
        a.x = ar.up(x, (size_t)B * Cin * T); a.Cin_total = Cin; a.Cin = Cin;
        a.w = ar.up(wp.data(), wp.size()); a.Cout_w = Cout; a.bias = ar.up(bias, (size_t)Cout);
        a.y = reinterpret_cast<float*>(dy); a.Cout_total = Cout; a.Cout = Cout;
        a.T = T; a.B = B; a.K = K; a.dil = dil; a.pad = (K - 1) / 2 * dil; a.in_slope = in_slope;
        if (res) { a.res_mode = 1; a.res = ar.up(res, (size_t)B * Cout * T); a.res_C_total = Cout; }
        a.accumulate = accumulate; a.out_scale = out_scale; a.t_begin = t_begin; a.t_end = t_end;
        launch_conv1d(a, 0);
        finish(err_flag);
        *guard_ok = read_guarded(dy, y, yb);
    });
}

// k_convT_c4: w [Cin][Cout][K] (ConvTranspose1d layout), stride u, padding (K-u)/2, input lrelu slope 0.1; y c4 [B][Cout/4][T*u][4].
int kh_convT_window(int B, int T, int Cin, int Cout, int K, int u, const float* w, const float* bias, const float* x, int n_begin, int n_end,
                    float* y, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        std::vector<float> wp((size_t)Cin * K * Cout);  // [Cin][K][Cout]
        for (int ci = 0; ci < Cin; ci++)
            for (int co = 0; co < Cout; co++)
                for (int j = 0; j < K; j++) wp[((size_t)ci * K + j) * Cout + co] = w[((size_t)ci * Cout + co) * K + j];
        const int To = T * u;
        const size_t yb = (size_t)B * Cout * To * sizeof(float);
        uint8_t* dy = ar.guarded(y, yb);
        ConvTArgs a;
        a.x = ar.up(x, (size_t)B * Cin * T); a.Cin = Cin; a.Tin = T; a.w = ar.up(wp.data(), wp.size()); a.bias = ar.up(bias, (size_t)Cout);
        a.y = reinterpret_cast<float*>(dy); a.Cout = Cout; a.Tout = To; a.K = K; a.u = u; a.p = (K - u) / 2; a.B = B; a.in_slope = 0.1f;
        a.n_begin = n_begin; a.n_end = n_end;
        const int ne = n_end < 0 ? To : n_end;
        k_convT_c4<<<dim3(cdiv(ne - n_begin, 128), cdiv(Cout, 64), B), 256>>>(a);
        finish(err_flag);
        *guard_ok = read_guarded(dy, y, yb);
    });
}

// k_conv_post_tanh (16 channels, 7 taps, slope 0.01) on a c4 input x [B][4][T][4]; w [16][7]; y [B][T].
int kh_conv_post_simt_window(const float* x, const float* w, int B, int T, int t_begin, int t_end, float* y, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        BV2_CHECK(0 <= t_begin && t_begin < t_end && t_end <= T, "conv_post window");
        Arena ar;
        const size_t yb = (size_t)B * T * sizeof(float);
        uint8_t* dy = ar.guarded(y, yb);
        k_conv_post_tanh<16, 7><<<dim3(cdiv(t_end - t_begin, 256), B), 256>>>(ar.up(x, (size_t)B * 16 * T), ar.up(w, 16 * 7),
                                                                             reinterpret_cast<float*>(dy), T, 0.01f, t_begin, t_end);
        finish(err_flag);
        *guard_ok = read_guarded(dy, y, yb);
    });
}

}  // extern "C"
