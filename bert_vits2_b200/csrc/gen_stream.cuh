// Wavefront plan of the Generator (reference models.py:538-557) for streaming synthesis: host-only, pure functions of the
// configuration and the frame counts (no device access), so tests can enumerate them.
//
// The Generator is purely convolutional, so output sample t of a layer depends on a bounded range of input rows around it.  A
// stream advances a frontier of frames whose audio must be final; each chunk runs every layer over a time window [done, need)
// of its output, where need is back-propagated from the frontier through what each layer reads:
//   conv with padding p:                 need_in = need_out + p
//   polyphase ConvTranspose (stride u):  output rows are computed u at a time (the need rounds up to a multiple of u), and input row r
//                                        feeds outputs r*u .. r*u + u - 1 from input rows r - half .. r + half (half = ups_half)
//   a residual is read at the output's own rows; everything is clamped to each tensor's length.
// A layer's done pointer is its need at the previous frontier, so the windows of one layer over a stream are contiguous and disjoint
// and every output element is computed exactly once.  The last conv of every MRF branch writes the same stage sum S, so its window
// is the same for every branch and the running sum S += ... (branches j = 0, 1, 2, then the 1/nk scale) keeps its per-column order.
#pragma once
#include <algorithm>
#include <vector>
#include "../../include/bv2.h"
#include "tc_conv.cuh"

namespace bv2 {

// One Generator layer, in launch order.  Tensors are numbered in allocation order: 0 is the Generator input z (all F frames are
// final before a stream opens), then the layers' outputs; the last tensor is the waveform.
struct GenLayer {
    enum Kind { CONV_PRE = 0, UPS = 1, RB_C1 = 2, RB_C2 = 3, CONV_POST = 4 };
    int kind, stage, branch, dil_idx;
    int in, out, res;  // tensor ids (res = -1: no residual)
    int reach;         // output row r reads input rows r - reach .. r + reach (ConvTranspose: r counts groups of u outputs)
    int u;             // ConvTranspose stride; 1 for a conv
    int L_in, L_out;   // rows of the input / output tensor
};
struct GenGraph {
    std::vector<GenLayer> layers;
    std::vector<int> tensor_len, tensor_ch;  // rows and channels of each tensor
    int hop = 1;  // waveform samples per frame
};
struct GenWin { int t_begin = 0, t_end = 0; };  // output rows [t_begin, t_end); empty: no launch

constexpr int GEN_PRE_POST_REACH = 3;  // conv_pre and conv_post: 7 taps, padding 3

inline GenGraph gen_graph(const bv2_config& c, int Fg) {
    GenGraph g;
    auto tensor = [&](int L, int C) { g.tensor_len.push_back(L); g.tensor_ch.push_back(C); return (int)g.tensor_len.size() - 1; };
    auto layer = [&](int kind, int stage, int j, int d, int in, int out, int res, int reach, int u) {
        g.layers.push_back(GenLayer{kind, stage, j, d, in, out, res, reach, u, g.tensor_len[in], g.tensor_len[out]});
    };
    int L = Fg, C = c.upsample_initial_channel;
    const int z = tensor(L, c.inter_channels);
    int x = tensor(L, C);
    layer(GenLayer::CONV_PRE, -1, 0, 0, z, x, -1, GEN_PRE_POST_REACH, 1);
    for (int i = 0; i < c.n_ups; i++) {
        const int u = c.upsample_rates[i], Lo = L * u;
        C /= 2;  // every upsampling stage halves the channels
        const int S = tensor(Lo, C), xu = tensor(Lo, C);
        layer(GenLayer::UPS, i, 0, 0, x, xu, -1, ups_half(c.upsample_kernel_sizes[i], u), u);
        for (int j = 0; j < c.n_resblock_kernels; j++) {
            const int k = c.resblock_kernel_sizes[j];
            int cur = xu;
            for (int d = 0; d < c.n_dilations; d++) {
                const int xt = tensor(Lo, C), nxt = d == c.n_dilations - 1 ? S : tensor(Lo, C);
                layer(GenLayer::RB_C1, i, j, d, cur, xt, -1, (k - 1) / 2 * c.resblock_dilation_sizes[j][d], 1);
                layer(GenLayer::RB_C2, i, j, d, xt, nxt, cur, (k - 1) / 2, 1);
                cur = nxt;
            }
        }
        x = S; L = Lo; g.hop *= u;
    }
    layer(GenLayer::CONV_POST, -1, 0, 0, x, tensor(L, 1), -1, GEN_PRE_POST_REACH, 1);
    return g;
}

// End of the output range every layer (layer) and every tensor (tensor: the rows its consumers read) must have computed for
// `frontier` (clamped to [0, Fg]) frames of final audio.
struct GenNeed { std::vector<int> layer, tensor; };
inline GenNeed gen_needs(const GenGraph& g, int Fg, int frontier) {
    GenNeed r;
    std::vector<int>& tneed = r.tensor;
    std::vector<int>& lneed = r.layer;
    tneed.assign(g.tensor_len.size(), 0); lneed.assign(g.layers.size(), 0);
    tneed[g.layers.back().out] = std::min(std::max(frontier, 0), Fg) * g.hop;
    for (int li = (int)g.layers.size() - 1; li >= 0; li--) {  // consumers come after their producers in launch order
        const GenLayer& l = g.layers[li];
        int n = tneed[l.out];
        if (n <= 0) continue;
        if (l.u > 1) n = std::min(l.L_out, (n + l.u - 1) / l.u * l.u);
        lneed[li] = n;
        tneed[l.out] = n;
        tneed[l.in] = std::max(tneed[l.in], std::min(l.L_in, n / l.u + l.reach));
        if (l.res >= 0) tneed[l.res] = std::max(tneed[l.res], n);
    }
    return r;
}
inline std::vector<int> gen_need(const GenGraph& g, int Fg, int frontier) { return gen_needs(g, Fg, frontier).layer; }

// The windows of one chunk: everything that makes frames [done, target) of audio final, given that frames [0, done) already are.
inline std::vector<GenWin> gen_stream_plan(const GenGraph& g, int Fg, int done, int target) {
    const std::vector<int> a = gen_need(g, Fg, done), b = gen_need(g, Fg, target);
    std::vector<GenWin> w(g.layers.size());
    for (size_t i = 0; i < w.size(); i++) { w[i].t_begin = a[i]; w[i].t_end = std::max(a[i], b[i]); }
    return w;
}

// ---- bounded streams: every tensor but the waveform keeps only a range of its rows resident.
// Logical row t of a tensor lives at physical row t - base of a storage of `capacity` rows (plus the zero halos).  After the frontier
// reaches `done`, no future window reads a row below resident_begin: a conv consumer with done pointer d reads from d / u - reach, a
// residual read from d.  The rows [resident_begin(done), need(done)) are final and still read; the rows below are dead.
inline std::vector<int> gen_resident_begin(const GenGraph& g, int Fg, int done) {
    const std::vector<int> d = gen_need(g, Fg, done);
    std::vector<int> lo(g.tensor_len);  // a tensor nobody reads any more keeps nothing
    for (size_t li = 0; li < g.layers.size(); li++) {
        const GenLayer& l = g.layers[li];
        lo[l.in] = std::min(lo[l.in], d[li] / l.u - l.reach);
        if (l.res >= 0) lo[l.res] = std::min(lo[l.res], d[li]);
    }
    for (size_t i = 0; i < lo.size(); i++) lo[i] = std::max(0, std::min(lo[i], g.tensor_len[i]));
    return lo;
}

// Rows of storage each tensor needs for any chunk schedule whose chunks are at most max_chunk_frames >= 1 frames, for any Fg.  A chunk
// done -> target touches the rows [resident_begin(done), need(target)) of a tensor; away from the ends of the utterance both bounds
// are affine in the frame count (every rate is a whole multiple of the ConvTranspose strides), so that span is rows_per_frame *
// max_chunk_frames + keep, with keep = need(done) - resident_begin(done) the rows a slide carries over.  The capacity is span + keep:
// a slide happens only when the span no longer fits behind the current base, which then drops more than `keep` rows, so a slide's
// source never overlaps its destination.  Near the ends the clamps to [0, L] only shrink both terms.  The one exception is the first
// chunk: at frontier 0 every done pointer is 0 rather than affine, so it touches need(max_chunk_frames) rows from row 0.  The
// waveform (the caller's buffer) gets 0.
inline std::vector<int> gen_stream_capacity(const bv2_config& c, int max_chunk_frames) {
    BV2_CHECK(max_chunk_frames >= 1, "gen_stream_capacity: cap >= 1");
    for (int d0 = 64;; d0 *= 2) {  // a frontier far enough from both ends that no clamp applies
        const int Fv = 2 * d0 + max_chunk_frames;
        const GenGraph g = gen_graph(c, Fv);
        const std::vector<int> lo = gen_resident_begin(g, Fv, d0), n0 = gen_needs(g, Fv, d0).tensor, n1 = gen_needs(g, Fv, d0 + max_chunk_frames).tensor;
        const size_t nt = g.tensor_len.size();
        bool interior = true;
        for (size_t i = 0; i + 1 < nt; i++) interior = interior && lo[i] > 0 && n1[i] < g.tensor_len[i];
        if (!interior) { BV2_CHECK(d0 < (1 << 20), "gen_stream_capacity"); continue; }
        // the first chunk starts from nothing (every done pointer is 0, so it runs the whole lead of the wavefront) and never slides
        const std::vector<int> first = gen_needs(g, Fv, max_chunk_frames).tensor;
        std::vector<int> cap(nt, 0);
        for (size_t i = 0; i + 1 < nt; i++) cap[i] = std::max((n1[i] - lo[i]) + (n0[i] - lo[i]), first[i]);
        return cap;
    }
}

// A stream over Fg frames is bounded when its chunk cap lies in [1, Fg).
inline bool gen_stream_bounded(int Fg, int max_chunk_frames) { return max_chunk_frames >= 1 && max_chunk_frames < Fg; }

// Rows of storage of every tensor of a stream over g (Fg = g.tensor_len[0] frames) with chunks of at most max_chunk_frames: the
// capacities of a bounded stream, else every tensor whole (L rows, so gen_stream_slides never slides it).  The waveform gets 0.
inline std::vector<int> gen_stream_rows(const bv2_config& c, const GenGraph& g, int max_chunk_frames) {
    if (gen_stream_bounded(g.tensor_len[0], max_chunk_frames)) return gen_stream_capacity(c, max_chunk_frames);
    std::vector<int> rows(g.tensor_len);
    rows.back() = 0;
    return rows;
}

// One slide: rows [src, src + rows) of every row block of tensor `tensor` move to [dst, dst + rows) (physical rows, dst < src).
struct GenSlide { int tensor, src, dst, rows; };

// Slides that let the chunk done -> target fit in the storage rows cap (gen_stream_rows), given the current bases (updated in place;
// the waveform, the last tensor, is never bounded).  A tensor slides only when the chunk's rows would run past its storage; its base
// then becomes resident_begin(done) and the final rows it still reads, [resident_begin(done), need(done)), move to the front.
inline std::vector<GenSlide> gen_stream_slides(const GenGraph& g, int Fg, const std::vector<int>& cap, std::vector<int>& base, int done, int target) {
    std::vector<GenSlide> s;
    const std::vector<int> lo = gen_resident_begin(g, Fg, done), n0 = gen_needs(g, Fg, done).tensor, n1 = gen_needs(g, Fg, target).tensor;
    for (size_t i = 0; i + 1 < g.tensor_len.size(); i++) {
        if (n1[i] - base[i] <= cap[i]) continue;
        const int keep = std::max(0, n0[i] - lo[i]), drop = lo[i] - base[i];
        BV2_CHECK(n1[i] - lo[i] <= cap[i] && drop >= keep, "bounded stream: a chunk exceeds the capacity it was planned for");
        if (keep > 0) s.push_back(GenSlide{(int)i, drop, 0, keep});
        base[i] = lo[i];
    }
    return s;
}

}  // namespace bv2
