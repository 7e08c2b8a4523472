// Bounded-stream harness: the kernel harness (kernel_harness.cu, included whole) plus the resident-range planner of gen_stream.cuh
// (resident rows, capacities, slides) and the launches on tensors held as a resident row range (k_g2_conv, conv_post, k_g2_slide),
// loaded by tests/test_stream_bounded_*.py through ctypes.  Same buffer conventions as the kernel harness: every output sits between
// two guard regions and the caller supplies its initial contents.
// Built with the product flags by bert_vits2_b200/_lib.py (build_harness(bounded=True)); see tests/stream_bounded_harness.py.
#include "kernel_harness.cu"
#include "../../bert_vits2_b200/csrc/gen_stream.cuh"

extern "C" {

// ---- bounded streams (host only) ----------------------------------------------------------------------------------------------
// Per-tensor vectors of gen_stream.cuh; each returns the number of tensors (or -1).
// need[n]: gen_needs(...).tensor, the rows of each tensor that are final once the frontier is at `frontier` frames
int kh_gen_tensor_need(const bv2_config* c, int Fg, int frontier, int* out, int cap) {
    int n = -1;
    guarded_call([&] {
        const std::vector<int> v = gen_needs(gen_graph(*c, Fg), Fg, frontier).tensor;
        BV2_CHECK((int)v.size() <= cap, "kh_gen_tensor_need capacity");
        std::memcpy(out, v.data(), v.size() * sizeof(int));
        n = (int)v.size();
    });
    return n;
}
int kh_gen_resident_begin(const bv2_config* c, int Fg, int done, int* out, int cap) {
    int n = -1;
    guarded_call([&] {
        const std::vector<int> v = gen_resident_begin(gen_graph(*c, Fg), Fg, done);
        BV2_CHECK((int)v.size() <= cap, "kh_gen_resident_begin capacity");
        std::memcpy(out, v.data(), v.size() * sizeof(int));
        n = (int)v.size();
    });
    return n;
}
int kh_gen_stream_capacity(const bv2_config* c, int max_chunk_frames, int* out, int cap) {
    int n = -1;
    guarded_call([&] {
        const std::vector<int> v = gen_stream_capacity(*c, max_chunk_frames);
        BV2_CHECK((int)v.size() <= cap, "kh_gen_stream_capacity capacity");
        std::memcpy(out, v.data(), v.size() * sizeof(int));
        n = (int)v.size();
    });
    return n;
}
// The slides before the chunk done -> target: base[n_tensors] (in: current bases, out: after the chunk's slides), slides[k][4] =
// tensor, src, dst, rows.  Returns k (or -1).
int kh_gen_stream_slides(const bv2_config* c, int Fg, const int* capv, int* base, int done, int target, int* slides, int cap) {
    int n = -1;
    guarded_call([&] {
        const GenGraph g = gen_graph(*c, Fg);
        const size_t nt = g.tensor_len.size();
        std::vector<int> cv(capv, capv + nt), bv(base, base + nt);
        const std::vector<GenSlide> s = gen_stream_slides(g, Fg, cv, bv, done, target);
        BV2_CHECK((int)s.size() <= cap, "kh_gen_stream_slides capacity");
        for (size_t i = 0; i < s.size(); i++) { const int v[4] = {s[i].tensor, s[i].src, s[i].dst, s[i].rows}; std::memcpy(slides + 4 * i, v, sizeof(v)); }
        std::memcpy(base, bv.data(), nt * sizeof(int));
        n = (int)s.size();
    });
    return n;
}

// ---- resident-range launches (device) --------------------------------------------------------------------------------------
// H8 storage of `rows` resident rows starting at logical row `base` of a T-row tensor: [B][C/8][PADL + rows + PADR][8] halves
static H8 h8_resident(uint4* storage, int B, int C, int T, int base, int rows) {
    H8 t; t.B = B; t.C = C; t.T = T; t.Tp = G2_PADL + rows + G2_PADR; t.base = base; t.p = storage + G2_PADL;
    return t;
}

// One g2_conv launch over the output window [t_begin, t_end) on resident storages: a->x holds rows x_rows of the input from x_base,
// a->res (optional) res_rows of the residual from res_base, y (in = initial contents, out = result) y_rows of the output from y_base.
int kh_g2_conv_resident(const KhG2Args* a, int t_begin, int t_end, int x_base, int x_rows, int y_base, int y_rows, int res_base, int res_rows,
                        void* y, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        const int To = a->T * (a->u ? a->u : 1);
        const size_t xb = H8::bytes(a->B, a->Cin, x_rows), yb = H8::bytes(a->B, a->Cout, y_rows);
        H8 x = h8_resident(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(a->x), xb)), a->B, a->Cin, a->T, x_base, x_rows);
        H8 yy = h8_resident(reinterpret_cast<uint4*>(ar.guarded(y, yb)), a->B, a->Cout, To, y_base, y_rows);
        H8 r;
        if (a->res) r = h8_resident(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(a->res), H8::bytes(a->B, a->Cout, res_rows))), a->B, a->Cout, To,
                                    res_base, res_rows);
        const float* dbias = ar.up(a->bias, (size_t)a->Cout);
        const float* dbias_b = ar.up(a->bias_b, (size_t)a->bias_b_elems);
        G2Params p; TcConvW cw;
        auto whole = [](H8 t) { t.base = 0; t.Tp = G2_PADL + t.T + G2_PADR; return t; };  // the packing call plans the whole output
        const H8 xw = whole(x), yw = whole(yy), rw = whole(r);
        g2_plan_of(*a, &ar, xw, yw, a->res ? &rw : nullptr, dbias, dbias_b, p, cw);  // packs the weights
        G2Epi e;
        e.res = a->res ? &r : nullptr; e.accumulate = a->accumulate; e.out_scale = a->out_scale; e.bias_b = dbias_b; e.bias_b_stride = a->bias_b_stride;
        e.dil = a->dil ? a->dil : 1; e.st_override = a->st_override; e.t_begin = t_begin; e.t_end = t_end;
        g2_conv(cw, dbias, x, yy, e, 0, a->num_sms);
        finish(err_flag);
        *guard_ok = read_guarded(reinterpret_cast<const uint8_t*>(yy.p - G2_PADL), y, yb);
    });
}

// conv_post + tanh over [t_begin, t_end) of T samples, the input held as x_rows resident rows from x_base (storage with halo rows).
int kh_conv_post_resident(const void* x, int x_base, int x_rows, const float* w, int B, int T, int t_begin, int t_end, float* y, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        BV2_CHECK(0 <= t_begin && t_begin < t_end && t_end <= T, "conv_post window");
        Arena ar;
        const size_t xb = H8::bytes(B, 16, x_rows), yb = (size_t)B * T * sizeof(float);
        H8 xx = h8_resident(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(x), xb)), B, 16, T, x_base, x_rows);
        uint8_t* dy = ar.guarded(y, yb);
        PostW<16, 7> pw;
        std::memcpy(pw.w, w, sizeof(pw.w));
        launch_pdl(k_conv_post_tanh_h8_resident<16, 7>, dim3(cdiv(t_end - t_begin, 512), B), dim3(256), 0, (cudaStream_t)0, (const uint4*)xx.p, xx.Tp, xx.base, pw,
                   reinterpret_cast<float*>(dy), T, t_begin, t_end);
        finish(err_flag);
        *guard_ok = read_guarded(dy, y, yb);
    });
}

// One k_g2_slide launch over n H8 storages bufs[i] (in = initial contents, out = result; bytes[i] each, halo rows included): rows
// [src, src + rows) of each of its blocks[i] row blocks (row stride Tp[i], physical rows counted from the first non-halo row) move to dst.
int kh_g2_slide(int n, void** bufs, const long long* bytes, const int* blocks, const int* Tp, const int* src, const int* dst, const int* rows,
                int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        BV2_CHECK(n >= 1 && n <= G2_SLIDE_MAX, "kh_g2_slide: descriptors");
        Arena ar;
        G2SlideParams sp{};
        std::vector<uint8_t*> d(n);
        int most = 0;
        for (int i = 0; i < n; i++) {
            d[i] = ar.guarded(bufs[i], (size_t)bytes[i]);
            sp.d[i] = G2SlideDesc{reinterpret_cast<uint4*>(d[i]) + G2_PADL, blocks[i], Tp[i], src[i], dst[i], rows[i]};
            most = std::max(most, blocks[i] * rows[i]);
        }
        sp.n = n;
        launch_pdl(k_g2_slide, dim3(std::max(1, std::min(32, cdiv(most, 256))), n), dim3(256), 0, (cudaStream_t)0, sp);
        finish(err_flag);
        int ok = 1;
        for (int i = 0; i < n; i++) ok &= read_guarded(d[i], bufs[i], (size_t)bytes[i]);
        *guard_ok = ok;
    });
}


}  // extern "C"
