"""CPU checks of streaming synthesis: the Generator's wavefront planner (gen_stream.cuh, through the streaming harness; no device
access) and a float64 restatement of a streamed Generator on the oracle."""
import pytest
import torch
import torch.nn.functional as F

from bert_vits2_b200.spec import ModelConfig
from stream_harness import Graph
from util import model_for

FGS = [1, 13, 14, 15, 127, 128, 129, 1000]


def schedules(Fg):
    """name -> increasing frontiers ending at Fg"""
    geo, f, step = [], 0, 32
    while f < Fg:
        f = min(f + step, Fg)
        geo.append(f)
        step *= 2
    edges = sorted({m * e + d for e in (2, 16, 128) for m in range(1, Fg // e + 2) for d in (-1, 0, 1) if 0 < m * e + d < Fg})
    return {"every_frame": list(range(1, Fg + 1)), "chunks_of_7": list(range(7, Fg, 7)) + [Fg], "geometric_32": geo, "one_chunk": [Fg],
            "tile_edges": edges + [Fg]}


def _reads(l, a, b):
    """input rows a layer reads to compute output rows [a, b)"""
    u, r = l["u"], l["reach"]
    return a // u - r, b // u + r


@pytest.mark.parametrize("Fg", FGS)
def test_planner_properties(Fg):
    g = Graph(ModelConfig(), Fg)
    layers, n = g.layers, len(g.layers)
    consumers = {}
    for li, l in enumerate(layers):
        consumers.setdefault(l["in_"], []).append((li, "in"))
        if l["res"] >= 0:
            consumers.setdefault(l["res"], []).append((li, "res"))
    for name, sched in schedules(Fg).items():
        end = [0] * n  # every layer's done pointer
        prev = 0
        for f in sched:
            w = g.plan(prev, f)
            assert len(w) == n
            for li, (a, b) in enumerate(w):
                assert a == end[li] and b >= a, (name, f, li)  # contiguous and disjoint
                if layers[li]["u"] > 1:
                    assert a % layers[li]["u"] == 0 and (b % layers[li]["u"] == 0 or b == layers[li]["L_out"])
                end[li] = b
            done = {0: g.tensor_len[0]}  # the Generator input is final before the stream starts
            for li, l in enumerate(layers):
                done[l["out"]] = end[li]
            # every read lies inside the producer's finished range (producers launch first) or outside [0, L) (the zero halo)
            for li, (a, b) in enumerate(w):
                if b == a:
                    continue
                l = layers[li]
                lo, hi = _reads(l, a, b)
                assert min(hi, l["L_in"]) <= done[l["in_"]], (name, f, li, a, b, done[l["in_"]])
                if l["res"] >= 0:
                    assert b <= done[l["res"]]
            # all MRF branches write identical S windows
            for li, l in enumerate(layers):
                if l["kind"] == 3 and l["dil_idx"] == max(x["dil_idx"] for x in layers):
                    writers = [w[k] for k, x in enumerate(layers) if x["out"] == l["out"]]
                    assert len(writers) == 3 and len(set(writers)) == 1
            # conv_post ends at exactly min(frontier, Fg) * hop
            assert end[-1] == min(f, Fg) * g.hop
            # no layer computes beyond what its consumers need (rounded up to whole ConvTranspose phases)
            for li, l in enumerate(layers[:-1]):
                need = 0
                for ci, how in consumers.get(l["out"], []):
                    if end[ci] == 0:
                        continue
                    c = layers[ci]
                    need = max(need, min(c["L_in"], _reads(c, 0, end[ci])[1]) if how == "in" else end[ci])
                if l["u"] > 1:
                    need = min(l["L_out"], -(-need // l["u"]) * l["u"])
                assert end[li] == need, (name, f, li, end[li], need)
            prev = f
        assert end == [l["L_out"] for l in layers], name  # every layer covered [0, L) exactly


def test_planner_one_chunk_is_whole_layers():
    g = Graph(ModelConfig(), 300)
    assert g.plan(0, 300) == [(0, l["L_out"]) for l in g.layers]
    assert g.plan(0, 10_000) == g.plan(0, 300)
    assert all(a == b for a, b in g.plan(300, 400))  # past the end: nothing left


def test_streamed_oracle_generator_float64():
    """Every layer computed only over its planned windows (frontiers 3, 10, 40 of F = 40), each from full-length producer buffers
    whose unfinished rows are NaN, with zero padding at the true edges, matches the one-shot oracle Generator."""
    from oracle import vits2_oracle as O
    cfg, sd32 = model_for(True, 0)
    sd = {k: v.double() for k, v in sd32.items() if k.startswith("dec.")}
    Fg, nk = 40, len(cfg.resblock_kernel_sizes)
    z = torch.randn(1, cfg.inter_channels, Fg, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    ref = O.generator(sd, cfg, z, None)

    g = Graph(cfg, Fg)
    buf = {i: torch.full((1, 1, L), float("nan"), dtype=torch.float64) for i, L in enumerate(g.tensor_len)}
    buf[0] = z
    branch = {}  # (stage, j) -> this branch's resblock output, the term of the stage sum
    lr = lambda x: F.leaky_relu(x, O.LRELU_SLOPE)  # noqa: E731

    def full(l):
        x = buf[l["in_"]]
        i, j, d = l["stage"], l["branch"], l["dil_idx"]
        if l["kind"] == 0:
            return O.conv1d(sd, "dec.conv_pre", x, padding=3)
        if l["kind"] == 1:
            k, u = cfg.upsample_kernel_sizes[i], cfg.upsample_rates[i]
            return F.conv_transpose1d(lr(x), O.wn_weight(sd, f"dec.ups.{i}"), sd[f"dec.ups.{i}.bias"], stride=u, padding=(k - u) // 2)
        name, k = f"dec.resblocks.{i * nk + j}", cfg.resblock_kernel_sizes[j]
        if l["kind"] == 2:
            dil = cfg.resblock_dilation_sizes[j][d]
            return F.conv1d(lr(x), O.wn_weight(sd, f"{name}.convs1.{d}"), sd[f"{name}.convs1.{d}.bias"], padding=(k * dil - dil) // 2, dilation=dil)
        if l["kind"] == 3:
            return F.conv1d(lr(x), O.wn_weight(sd, f"{name}.convs2.{d}"), sd[f"{name}.convs2.{d}.bias"], padding=(k - 1) // 2) + buf[l["res"]]
        return torch.tanh(F.conv1d(F.leaky_relu(x), sd["dec.conv_post.weight"], None, padding=3))

    prev = 0
    for f in (3, 10, 40):
        for l, (a, b) in zip(g.layers, g.plan(prev, f)):
            if b == a:
                continue
            y = full(l)[..., a:b]
            out = l["out"]
            if buf[out].shape[1] != y.shape[1]:
                buf[out] = torch.full((1, y.shape[1], g.tensor_len[out]), float("nan"), dtype=torch.float64)
            last = l["kind"] == 3 and l["dil_idx"] == len(cfg.resblock_dilation_sizes[l["branch"]]) - 1
            if not last:
                buf[out][..., a:b] = y
                continue
            branch[(l["stage"], l["branch"])] = y  # S = ((r_0 + r_1) + r_2) / nk, per column as the oracle sums
            if l["branch"] == nk - 1:
                s = branch[(l["stage"], 0)]
                for jj in range(1, nk):
                    s = s + branch[(l["stage"], jj)]
                buf[out][..., a:b] = s / nk
        prev = f
    got = buf[len(g.tensor_len) - 1]
    assert got.shape == ref.shape and torch.isfinite(got).all()
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-12
