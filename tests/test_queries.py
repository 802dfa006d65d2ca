"""Queries at any frame, tracked forward and backward in time (pips_b200.chain.track_queries).

A query (t, x, y) is the reference chain (chain_demo.py:40-83) on the clip from frame t on, and the same chain on the
time-reversed clip from frame t back to frame 0.  CPU: the slice-and-flip composition around the oracle's chain
(tests/golden/make_golden_queries.py), its visibility rule, and the batched host
logic (with the oracle as the 8-frame tracker) against the reference's recording, and input validation.  GPU: the
CUDA path against the recording, the backward-window decode of the kernels and of engine.refine against forward
windows over the flipped clip, and bit-exact invariants of the batched rounds."""
import os

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from tests.golden.make_golden import CHAIN_CASE, chain_inputs
from tests.golden.make_golden_queries import QUERY_TIMES, chain_track_vis, query_inputs, track_queries as oracle_queries

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_queries.npz"))
DEV = "cuda:0"
S = 8


def _unflatten(a, n):
    lens, flat, out, k = a[:n], a[n:], [], 0
    for L_ in lens:
        out.append(list(flat[k:k + L_]))
        k += L_
    return out


def _gold_skips():
    n = len(QUERY_TIMES)
    return _unflatten(GOLD["skips_fwd"], n), _unflatten(GOLD["skips_bwd"], n)


def _oracle_window(sd, c):
    def window(xys, seq, feat_init):
        with torch.no_grad():
            o = po.forward(sd, xys, seq, iters=c["iters"], stride=c["stride"], feat_init=feat_init, return_feat=True)
        return o[0], o[2], o[3]
    return window


def _window_frames(base, T):
    """The frames step s = 0..7 of a window reads (csrc/corr_common.cuh window_frame): base >= 0 forward from base,
    base < 0 backward from ~base."""
    s = torch.arange(S)
    return (base + s).clamp(max=T - 1) if base >= 0 else (~base - s).clamp(min=0)


def test_oracle_queries_match_reference_recording():
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    rgbs, queries = query_inputs(c)
    trajs, vis, skips = oracle_queries(_oracle_window(sd, c), rgbs, queries, iters=c["iters"])
    fwd, bwd = _gold_skips()
    assert [f for f, _ in skips] == fwd and [b for _, b in skips] == bwd
    assert np.abs(trajs.numpy() - GOLD["trajs"]).max() < 1e-3
    assert np.abs(vis.numpy() - GOLD["vis"]).max() < 1e-4


def test_chain_visibility_follows_the_overwrite_rule():
    """chain_track_vis: a frame's visibility is that of the window that last wrote it.  A fake 8-frame tracker that is
    visible only at step 5 makes every skip 5, so frame f is last written by window f // 5 at step f % 5."""
    T, N = 12, 2
    calls = []

    def window(xys, seq, feat_init):
        k = len(calls)
        calls.append(k)
        logits = -(1.0 + k + 0.01 * torch.arange(S, dtype=torch.float32))
        logits[5] = 5.0
        preds = [xys.reshape(1, 1, 1, 2).repeat(1, S, 1, 1) + k]
        return preds, logits.view(1, S, 1), torch.zeros(1, 1, 128)

    rgbs, xy0 = torch.zeros(1, T, 3, 8, 8), torch.rand(1, N, 2)
    trajs, skips, vis = chain_track_vis(window, rgbs, xy0)
    assert skips == [[5, 5, 5]] * N
    for n in range(N):
        for f in range(T):
            k = 3 * n + f // 5
            logits = -(1.0 + k + 0.01 * torch.arange(S, dtype=torch.float32))
            assert torch.equal(vis[0, f, n], torch.sigmoid(logits[f % 5]))
    calls.clear()
    t2, s2 = po.chain_track(window, rgbs, xy0)
    assert torch.equal(t2, trajs) and s2 == skips


def test_batched_queries_host_logic_on_cpu():
    """track_queries with the CUDA engine replaced by the oracle, one 8-frame window per track read through
    ``frame_base`` as the kernels decode it: forward and backward tracks, their truncation at either end of the
    clip, the carried feature and the threshold sweep reproduce the reference's per-query slice-and-flip chains
    (same skips per direction, same trajectories and visibilities)."""
    from pips_b200.chain import track_queries
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    rgbs, queries = query_inputs(c)
    T = rgbs.shape[1]
    log = []

    class Engine:
        def refine(self, module, fmaps, coords, feat_init, iters, stride, frame_base=None, reuse_pyramid=False):
            B, _, na, _ = coords.shape
            assert B == 1 and fmaps.shape[1] == T and frame_base.shape == (1, na) and frame_base.dtype == torch.int32
            assert reuse_pyramid == (len(log) > 0)
            preds = torch.zeros(iters, 1, S, na, 2)
            vis = torch.zeros(1, S, na)
            ffeat = torch.zeros(1, na, 128)
            for n in range(na):
                idx = _window_frames(int(frame_base[0, n]), T)
                fi = None if feat_init is None else feat_init[:, n:n + 1]
                with torch.no_grad():
                    o = po.forward(sd, coords[:, 0, n:n + 1] * stride, torch.zeros(1, S, 3, c["H"], c["W"]), iters=iters,
                                   stride=int(stride), fmaps=fmaps[:, idx], feat_init=fi, return_feat=True)
                preds[:, :, :, n] = torch.stack(o[0])[:, :, :, 0]
                vis[:, :, n] = o[2][:, :, 0]
                ffeat[:, n] = o[3][:, 0]
            log.append(frame_base[0].tolist())
            return preds, vis, ffeat

    class Model:
        stride = c["stride"]
        engine = Engine()

        def encode(self, clip):
            Bc, Tc = clip.shape[:2]
            x = 2 * (clip / 255.0) - 1.0
            with torch.no_grad():
                f = po.fnet(sd, x.reshape(Bc * Tc, 3, c["H"], c["W"]), c["stride"])
            return f.reshape(Bc, Tc, 128, c["H"] // c["stride"], c["W"] // c["stride"])

    trajs, vis, rounds = track_queries(Model(), rgbs, queries, iters=c["iters"], return_rounds=True)
    fwd, bwd = _gold_skips()
    # tracks: every query forward, then the queries with t > 0 backward; window starts are the cumulative skips
    tracks = [(t, +1, h) for t, h in zip(QUERY_TIMES, fwd)] + [(t, -1, h) for t, h in zip(QUERY_TIMES, bwd) if t > 0]
    assert rounds == max(len(h) for _, _, h in tracks)
    starts = [[t + d * int(s) for s in [0] + list(np.cumsum(h)[:-1])] for t, d, h in tracks]
    for r, bases in enumerate(log):
        assert bases == [st[r] if d > 0 else ~st[r] for (_, d, _), st in zip(tracks, starts) if len(st) > r]
    assert trajs.shape == (1, T, len(QUERY_TIMES), 2) and vis.shape == (1, T, len(QUERY_TIMES))
    err = np.abs(trajs.numpy() - GOLD["trajs"]).max()
    print("batched queries host logic (oracle windows) vs reference recording: max err px", err)
    assert err < 1e-3
    assert np.abs(vis.numpy() - GOLD["vis"]).max() < 1e-4


@pytest.mark.parametrize("case", ["rgbs_4d", "rgbs_not_rgb", "batch_2", "queries_2d", "queries_xy_only", "queries_batch_2",
                                  "no_queries", "t_fractional", "t_negative", "t_past_end", "t_nan", "x_nan", "y_inf"])
def test_track_queries_rejects_bad_input(case):
    from pips_b200.chain import track_queries

    class Model:                  # never reached: validation comes before any work
        stride = 4
        engine = None

        def encode(self, clip):
            raise AssertionError("encoded despite bad input")

    T = 5
    rgbs = torch.zeros(1, T, 3, 16, 16)
    q = torch.tensor([[[0.0, 3.0, 4.0], [4.0, 1.0, 2.0]]])
    if case == "rgbs_4d":
        rgbs = rgbs[0]
    elif case == "rgbs_not_rgb":
        rgbs = torch.zeros(1, T, 1, 16, 16)
    elif case == "batch_2":
        rgbs = torch.zeros(2, T, 3, 16, 16)
        q = q.repeat(2, 1, 1)
    elif case == "queries_2d":
        q = q[0]
    elif case == "queries_xy_only":
        q = q[:, :, 1:]
    elif case == "queries_batch_2":
        q = q.repeat(2, 1, 1)
    elif case == "no_queries":
        q = q[:, :0]
    elif case == "t_fractional":
        q[0, 1, 0] = 2.5
    elif case == "t_negative":
        q[0, 1, 0] = -1.0
    elif case == "t_past_end":
        q[0, 1, 0] = float(T)
    elif case == "t_nan":
        q[0, 0, 0] = float("nan")
    elif case == "x_nan":
        q[0, 1, 1] = float("nan")
    elif case == "y_inf":
        q[0, 0, 2] = float("inf")
    with pytest.raises(ValueError):
        track_queries(Model(), rgbs, q)


# ------------------------------------------------------------------------------------------------ GPU

def _model(precision):
    from pips_b200 import Pips
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    model = Pips(S=8, stride=c["stride"], precision=precision).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    return model


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_queries_match_reference_recording(precision):
    from pips_b200.chain import track_queries
    c = CHAIN_CASE
    model = _model(precision)
    rgbs, queries = query_inputs(c)
    trajs, vis, rounds = track_queries(model, rgbs.to(DEV), queries.to(DEV), iters=c["iters"], return_rounds=True)
    assert trajs.shape == (1, c["T"], len(QUERY_TIMES), 2) and vis.shape == (1, c["T"], len(QUERY_TIMES))
    err = np.abs(trajs.cpu().numpy() - GOLD["trajs"]).max()
    verr = np.abs(vis.cpu().numpy() - GOLD["vis"]).max()
    fwd, bwd = _gold_skips()
    longest = max(len(h) for h in fwd + bwd)
    print(f"queries {precision}: {rounds} batched rounds (longest reference chain {longest}, "
          f"{sum(len(h) for h in fwd + bwd)} model calls), max err {err:.2e} px, vis {verr:.2e}")
    assert rounds == longest
    assert err < 2e-3
    assert verr < 5e-3


def _pyramid(fm):
    """(frames, 128, H, W) on the host -> the 4 device levels, fp32 and bf16."""
    from pips_b200 import _lib as L
    lib = L.load()
    frames, _, H, W = fm.shape
    f32, bf, h, w = [], [], H, W
    for _ in range(L.LEVELS):
        f32.append(torch.full((frames, h, w, 128), float("nan"), device=DEV))
        bf.append(torch.full((frames, h, w, 128), float("nan"), dtype=torch.bfloat16, device=DEV))
        h, w = h // 2, w // 2
    src = fm.contiguous().to(DEV)
    L.check(lib.pips_pyramid_build(L.ptr(src), frames, H, W, L.ptr_array(f32), L.ptr_array(bf),
                                   torch.cuda.current_stream().cuda_stream))
    return f32, bf


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32).cpu()


def _window_case(B, N, T, H, W, seed):
    """A clip per batch element, the same clips reversed in time, and query frames with t = 0, t = T-1 and t < 7
    (backward windows that clamp at frame 0) among them; tracks with even n run backward, odd n forward."""
    g = torch.Generator().manual_seed(seed)
    fm = torch.randn(B, T, 128, H, W, generator=g)
    t = torch.randint(0, T, (B, N), generator=g, dtype=torch.int32)
    t.view(-1)[:4] = torch.tensor([0, T - 1, min(3, T - 1), min(6, T - 1)], dtype=torch.int32)
    back = (torch.arange(N) % 2 == 0).view(1, N).expand(B, N)
    coords = torch.rand(B, S, N, 2, generator=g) * torch.tensor([W + 6.0, H + 6.0]) - 3.0
    ff_rows = torch.randn(B * N, S, 128, generator=g)
    return fm, t, back, coords, ff_rows


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["fp32", "bf16"])
@pytest.mark.parametrize("T", [3, 13, 20])
def test_backward_windows_equal_forward_windows_over_reversed_clip(feat, T):
    """pips_corr_gather and pips_init_gather with frame_base ~t (a backward window from frame t) write the same bits
    as with frame_base T-1-t over the pyramid of the time-reversed clips; the forward tracks of the same call write
    the bits of a call with forward windows only."""
    from pips_b200 import _lib as L
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    B, N, H, W = 2, 12, 16, 24
    fm, t, back, coords, ff_rows = _window_case(B, N, T, H, W, 300 + T)
    mixed = torch.where(back, ~t, t)
    rows = back.reshape(B * N)
    times = po.times_axis(S).to(DEV)
    cd, fd = coords.to(DEV).contiguous(), ff_rows.to(DEV).contiguous()

    def run(levels, fb):
        lv = levels[1] if feat == "bf16" else levels[0]
        fbd = fb.to(DEV).contiguous()
        x = torch.full((B * N * S, 576), float("nan"), device=DEV)
        L.check(lib.pips_corr_gather(L.ptr_array(lv), L.FEAT_DTYPES[feat], B, S, N, H, W, L.ptr(cd), L.ptr(fd), L.ptr(times),
                                     L.ptr(fbd), T, None, None, L.ptr(x), 576, st))
        ffeat, ffeats = torch.full((B * N, 128), float("nan"), device=DEV), torch.full((B * N, S, 128), float("nan"), device=DEV)
        L.check(lib.pips_init_gather(L.ptr(levels[0][0]), B, S, N, H, W, L.ptr(cd), L.ptr(fbd), T, L.ptr(ffeat), L.ptr(ffeats), st))
        torch.cuda.synchronize()
        return x.view(B * N, S, 576), ffeat, ffeats

    pyr = _pyramid(fm.reshape(B * T, 128, H, W))
    rev = _pyramid(fm.flip(1).reshape(B * T, 128, H, W))
    got = run(pyr, mixed)
    want_b = run(rev, (T - 1 - t))
    want_f = run(pyr, t)
    for g, wb, wf in zip(got, want_b, want_f):
        assert bool(torch.isfinite(g).all())
        assert torch.equal(_bits(g[rows]), _bits(wb[rows])), "backward windows differ from forward windows over the reversed clip"
        assert torch.equal(_bits(g[~rows]), _bits(wf[~rows])), "forward windows changed next to backward ones"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_refine_backward_windows_equal_forward_windows_over_flipped_fmaps(precision):
    """engine.refine with frame_base ~t over the clip's fmaps == frame_base T-1-t over the time-flipped fmaps: every
    iteration's predictions, the visibility logits and the initial features, bit for bit."""
    c = CHAIN_CASE
    model = _model(precision)
    rgbs, _ = chain_inputs(c)
    with torch.no_grad():
        fmaps = model.encode(rgbs.to(DEV)).contiguous()
    T, H8, W8 = fmaps.shape[1], fmaps.shape[3], fmaps.shape[4]
    g = torch.Generator().manual_seed(11)
    N = 40
    t = torch.randint(0, T, (1, N), generator=g, dtype=torch.int32)
    t.view(-1)[:4] = torch.tensor([0, T - 1, 3, 6], dtype=torch.int32)
    coords = (torch.rand(1, 1, N, 2, generator=g) * torch.tensor([W8 - 1.0, H8 - 1.0])).repeat(1, S, 1, 1).to(DEV)
    eng = model.engine
    with torch.no_grad():
        got = eng.refine(model, fmaps, coords, None, c["iters"], float(c["stride"]), frame_base=~t)
        want = eng.refine(model, fmaps.flip(1).contiguous(), coords, None, c["iters"], float(c["stride"]),
                          frame_base=T - 1 - t)
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert bool(torch.isfinite(a).all())
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_queries_at_frame_zero_reproduce_track_chain(precision):
    from pips_b200.chain import track_chain, track_queries
    c = CHAIN_CASE
    model = _model(precision)
    rgbs, xy0 = chain_inputs(c)
    rgbs, xy0 = rgbs.to(DEV), xy0.to(DEV)
    want, want_rounds = track_chain(model, rgbs, xy0, iters=c["iters"], return_rounds=True)
    q = torch.cat([torch.zeros(1, xy0.shape[1], 1, device=DEV), xy0], dim=2)
    trajs, vis, rounds = track_queries(model, rgbs, q, iters=c["iters"], return_rounds=True)
    assert rounds == want_rounds
    assert torch.equal(_bits(trajs), _bits(want))
    assert bool(((vis > 0) & (vis < 1)).all())


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_query_outputs_do_not_depend_on_the_other_queries(precision):
    """Each recorded query alone == the same query inside a batch of 40 queries at random frames, bit for bit."""
    from pips_b200.chain import track_queries
    c = CHAIN_CASE
    model = _model(precision)
    rgbs, queries = query_inputs(c)
    rgbs = rgbs.to(DEV)
    g = torch.Generator().manual_seed(12)
    n_other = 34
    other = torch.cat([torch.randint(0, c["T"], (1, n_other, 1), generator=g).float(),
                       po.random_queries(1, n_other, c["H"], c["W"], seed=13)], dim=2)
    slots = torch.randperm(n_other + len(QUERY_TIMES), generator=g)[:len(QUERY_TIMES)]
    batch = torch.empty(1, n_other + len(QUERY_TIMES), 3)
    keep = torch.ones(batch.shape[1], dtype=torch.bool)
    keep[slots] = False
    batch[:, slots], batch[:, keep] = queries, other
    trajs, vis = track_queries(model, rgbs, batch.to(DEV), iters=c["iters"])
    for i, s in enumerate(slots.tolist()):
        t1, v1 = track_queries(model, rgbs, queries[:, i:i + 1].to(DEV), iters=c["iters"])
        assert torch.equal(_bits(t1[:, :, 0]), _bits(trajs[:, :, s])), f"query {i} (t={QUERY_TIMES[i]}) trajectory differs"
        assert torch.equal(_bits(v1[:, :, 0]), _bits(vis[:, :, s])), f"query {i} (t={QUERY_TIMES[i]}) visibility differs"
