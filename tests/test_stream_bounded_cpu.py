"""CPU checks of the bounded-stream planner (gen_stream.cuh, through the bounded-stream harness; no device access): under any schedule whose
chunks stay within the cap, every row a chunk reads or writes lies inside its tensor's resident storage, slides never overlap, and the
storage does not depend on the utterance's length."""
import numpy as np
import pytest

from bert_vits2_b200.spec import ModelConfig
from stream_bounded_harness import BoundedGraph as Graph

FGS = [1, 7, 33, 1023, 4096, 20000]
CAPS = [1, 7, 32, 256]
PADL = PADR = 32  # G2_PADL / G2_PADR: zero halo rows of every H8 tensor


def schedules(Fg, cap):
    """name -> increasing frontiers ending at Fg whose steps are at most cap"""
    geo, f, step = [], 0, 1
    while f < Fg:
        f = min(f + step, Fg)
        geo.append(f)
        step = min(2 * step, cap)
    fixed = min(7, cap)
    rng = np.random.default_rng(Fg * 1000 + cap)
    rnd, f = [], 0
    while f < Fg:
        f = min(f + int(rng.integers(1, cap + 1)), Fg)
        rnd.append(f)
    out = {"geometric": geo, "fixed_7": list(range(fixed, Fg, fixed)) + [Fg], "random": rnd}
    uniq = {}
    for k, v in out.items():  # with cap = 1 all three are the same schedule
        if v not in uniq.values():
            uniq[k] = v
    return uniq


def _check_schedule(g, cap_frames, sched):
    layers = g.layers
    nt = len(g.tensor_len)
    L = np.array(g.tensor_len)
    cap = g.capacity(cap_frames)
    assert len(cap) == nt and cap[-1] == 0 and (cap[:-1] > 0).all()
    base = np.zeros(nt, np.int32)
    lin = np.array([l["in_"] for l in layers])
    lout = np.array([l["out"] for l in layers])
    lres = np.array([l["res"] for l in layers])
    reach = np.array([l["reach"] for l in layers])
    u = np.array([l["u"] for l in layers])
    bounded = np.arange(nt) < nt - 1  # the waveform is the caller's buffer

    def inside(t, lo, hi):
        """rows [lo, hi) of tensor t are in its storage: physical rows [-PADL, cap + PADR) relative to base (the halo rows below 0 exist
        only while base is 0, and rows at and past L are the zero halo)"""
        lo_ok = lo >= base[t] or (base[t] == 0 and lo >= -PADL)
        hi_ok = hi <= base[t] + cap[t] or (hi <= L[t] + PADR and L[t] - base[t] <= cap[t])
        return lo_ok and hi_ok

    prev = 0
    need_prev = g.tensor_need(0)
    for f in sched:
        assert 0 < f - prev <= cap_frames
        old = base.copy()
        lo_prev = g.resident_begin(prev)
        slides = g.slides(cap, base, prev, f)
        for t, src, dst, rows in slides:
            assert bounded[t] and dst == 0 and rows > 0
            assert dst + rows <= src, ("slide overlaps", t, src, dst, rows)
            assert base[t] == lo_prev[t] and src == base[t] - old[t] and rows == need_prev[t] - lo_prev[t]
        moved = {s[0] for s in slides}
        for t in np.nonzero(base != old)[0]:  # a base that advances without rows to carry over keeps nothing final
            assert t in moved or need_prev[t] == lo_prev[t]
        need = g.tensor_need(f)
        # every live row survives: rows [resident_begin(prev), need(prev)) stay addressable
        for t in np.nonzero(bounded)[0]:
            assert inside(t, lo_prev[t], need_prev[t]), ("live rows dropped", t)
            assert need[t] - base[t] <= cap[t], ("chunk overruns storage", t, f)
        # the input conversion of the chunk
        assert inside(0, need_prev[0], need[0])
        w = np.array(g.plan(prev, f))
        a, b = w[:, 0], w[:, 1]
        for li in np.nonzero(b > a)[0]:
            r0, r1 = a[li] // u[li] - reach[li], b[li] // u[li] + reach[li]  # input rows the window reads (halo included)
            assert inside(lin[li], r0, min(r1, L[lin[li]] + PADR)), ("read", li, f)
            if bounded[lout[li]]:
                assert inside(lout[li], a[li], b[li]), ("write", li, f)
                if b[li] == L[lout[li]]:
                    assert inside(lout[li], L[lout[li]], L[lout[li]] + PADR), ("halo", li, f)
                if a[li] == 0:
                    assert base[lout[li]] == 0
            if lres[li] >= 0:
                assert inside(lres[li], a[li], b[li]), ("residual", li, f)
        # the rows resident after the chunk fit the storage
        lo = g.resident_begin(f)
        assert (need[bounded] - lo[bounded] <= cap[bounded]).all()
        prev, need_prev = f, need
    assert prev == g.Fg


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("Fg", FGS)
def test_bounded_plan_properties(Fg, cap):
    g = Graph(ModelConfig(), Fg)
    for name, sched in schedules(Fg, cap).items():
        _check_schedule(g, cap, sched)


@pytest.mark.parametrize("cap", CAPS)
def test_capacity_independent_of_length(cap):
    cfg = ModelConfig()
    ref = Graph(cfg, cap + 1).capacity(cap)
    for Fg in FGS + [cap + 1, cap + 2, 3 * cap + 5]:
        if Fg > cap:
            assert np.array_equal(Graph(cfg, Fg).capacity(cap), ref)


@pytest.mark.parametrize("Fg", FGS)
def test_cap_at_least_length_never_slides(Fg):
    """With the cap >= Fg the stream keeps whole tensors: the storage a cap gives already holds every row, and nothing slides."""
    cfg = ModelConfig()
    g = Graph(cfg, Fg)
    L = np.array(g.tensor_len)
    for cap_frames in (Fg, Fg + 1, 2 * Fg):
        cap = g.capacity(cap_frames)
        assert (cap[:-1] >= L[:-1]).all()
        base = np.zeros(len(L), np.int32)
        prev = 0
        for f in schedules(Fg, cap_frames)["geometric"]:
            assert g.slides(cap, base, prev, f) == [] and not base.any()
            prev = f


def test_capacity_grows_with_the_cap():
    cfg = ModelConfig()
    g = Graph(cfg, 300)
    caps = [g.capacity(c) for c in (1, 2, 7, 32, 256)]
    for lo, hi in zip(caps, caps[1:]):
        assert (hi >= lo).all() and (hi[:-1] > lo[:-1]).all()
