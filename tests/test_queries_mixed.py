"""Queries in videos of different frame sizes in one batch (pips_b200.chain.track_queries_mixed) and the grouped mode
of the window kernels under it.

The clips are grouped by frame size, one pyramid per group; each track carries {first, count, group} and reads its
windows inside its clip of its group's pyramid (pips_corr_gather_groups / pips_init_gather_groups,
engine.refine(fmaps=[...], clip=(B, N, 3))).  CPU: the host logic with the oracle as the 8-frame tracker reproduces
track_queries clip by clip, the size cap splits a batch into sub-batches, input validation, the table check and the
new C entry points' argument checks.  GPU: the grouped kernels against the clip kernels over each group's own pyramid,
engine.refine with groups against per-group refine(clip=), and track_queries_mixed against per-clip track_queries,
bit for bit."""
import ctypes as C

import pytest
import torch

from oracle import pips_oracle as po
from tests.golden.make_golden import CHAIN_CASE
from tests.test_queries_batch import _OracleModel, _bases, _bits, _model, _pyramid, _window_frames

DEV = "cuda:0"
S = 8


class _MixedOracleModel(_OracleModel):
    """_OracleModel for frames of any size: the oracle encodes each frame at its own size, and a refinement call with
    feature maps in groups reads track n's window inside its clip of its group only -- every other frame of that group
    is NaN to it, and no other group is read.  ``encodes`` records the (H, W) of every encode call; ``calls`` records
    (frame_base, clip table) of every refinement call."""

    def __init__(self):
        super().__init__()
        self.encodes = []

    def encode(self, clip):
        Bc, Tc, _, H, W = clip.shape
        assert Bc == 1 and Tc <= 32
        self.encoded += Tc
        self.encodes.append((H, W))
        x = 2 * (clip.float() / 255.0) - 1.0
        st = self.c["stride"]
        with torch.no_grad():
            f = torch.cat([po.fnet(self.sd, x[:, k], st) for k in range(Tc)])
        return f.reshape(Bc, Tc, 128, H // st, W // st)

    def _refine(self, fmaps, coords, feat_init, iters, stride, frame_base, clip):
        B, _, na, _ = coords.shape
        grouped = isinstance(fmaps, list)
        assert B == 1 and frame_base.shape == (1, na) and frame_base.dtype == torch.int32
        assert (clip is not None and clip.shape == (1, na, 3)) if grouped else clip is None
        self.calls.append((frame_base[0].tolist(), None if clip is None else clip[0].tolist()))
        preds = torch.zeros(iters, 1, S, na, 2)
        vis = torch.zeros(1, S, na)
        ffeat = torch.zeros(1, na, 128)
        for n in range(na):
            base = int(frame_base[0, n])
            if grouped:
                first, count, group = (int(v) for v in clip[0, n])
                fm = fmaps[group]
                own = torch.full_like(fm, float("nan"))
                own[:, first:first + count] = fm[:, first:first + count]
                fm = own[:, first + _window_frames(base, count)]
            else:
                fm = fmaps[:, _window_frames(base, fmaps.shape[1])]
            H, W = fm.shape[3] * int(stride), fm.shape[4] * int(stride)
            fi = None if feat_init is None else feat_init[:, n:n + 1]
            with torch.no_grad():
                o = po.forward(self.sd, coords[:, 0, n:n + 1] * stride, torch.zeros(1, S, 3, H, W),
                               iters=iters, stride=int(stride), fmaps=fm, feat_init=fi, return_feat=True)
            preds[:, :, :, n] = torch.stack(o[0])[:, :, :, 0]
            vis[:, :, n] = o[2][:, :, 0]
            ffeat[:, n] = o[3][:, 0]
        return preds, vis, ffeat


def _clip(T, H, W, seed, n):
    """A smooth clip (T, 3, H, W) and n queries (n, 3) at frames 0, T-1 and random ones."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, T, (n,), generator=g).float()
    t[0], t[-1] = 0.0, float(T - 1)
    q = torch.cat([t.view(n, 1), po.random_queries(1, n, H, W, seed=seed + 1)[0]], dim=1)
    return po.smooth_video(1, T, H, W, seed=seed)[0], q


def _mixed_case():
    """Five clips at three sizes (stride 4: 8x10, 10x8 and 12x12 feature maps), of 9, 1, 6 (shorter than a window),
    4 and 3 frames; the clips of one size are not adjacent."""
    spec = [(9, 32, 40), (1, 40, 32), (6, 32, 40), (4, 48, 48), (3, 40, 32)]
    pairs = [_clip(T, H, W, 300 + 7 * i, 2 + i % 2) for i, (T, H, W) in enumerate(spec)]
    return [p[0] for p in pairs], [p[1] for p in pairs]


def _check_against_track_queries(m, clips, queries, outs):
    from pips_b200.chain import track_queries
    per = []
    for (trajs, vis), v, q in zip(outs, clips, queries):
        T, N = v.shape[0], q.shape[0]
        assert trajs.shape == (1, T, N, 2) and vis.shape == (1, T, N)
        assert bool(torch.isfinite(trajs).all()) and bool(torch.isfinite(vis).all())
        wt, wv, r = track_queries(m, v.unsqueeze(0), q.unsqueeze(0), iters=2, return_rounds=True)
        per.append(r)
        assert torch.equal(trajs, wt)
        assert torch.allclose(vis, wv, rtol=0, atol=4 * 2 ** -24)
    return per


def test_mixed_host_logic_equals_track_queries_per_clip_on_cpu():
    """track_queries_mixed with the oracle as tracker == track_queries on each clip alone: the same trajectories bit for
    bit, visibilities within a few ulps (as in the one-size batch), in as many rounds as the longest clip's chain, one
    refinement call per round.  Every frame is encoded once, every encode call sees one frame size, and every track
    reads only its own clip of its own group (the oracle makes everything else NaN, and the results are finite)."""
    from pips_b200.chain import track_queries_mixed
    clips, queries = _mixed_case()
    m = _MixedOracleModel()
    outs, rounds = track_queries_mixed(m, clips, queries, iters=2, return_rounds=True)
    assert m.encoded == sum(v.shape[0] for v in clips)
    sizes = {tuple(v.shape[-2:]) for v in clips}
    assert set(m.encodes) == sizes                                    # one size per encode call, each group encoded
    calls = list(m.calls)
    assert all(cl is not None and len(cl[0]) == 3 for _, cl in calls)
    assert {row[2] for _, cl in calls for row in cl} == set(range(len(sizes)))
    m.calls.clear()
    per = _check_against_track_queries(m, clips, queries, outs)
    assert rounds == max(per)


def test_mixed_size_cap_runs_sub_batches_on_cpu(monkeypatch):
    """With the size cap lowered to 2, four sizes run as two sub-batches of two groups each, with the results of the
    uncapped run."""
    import pips_b200.chain as ch
    spec = [(5, 32, 40), (3, 40, 32), (4, 48, 48), (2, 36, 44), (6, 32, 40)]
    pairs = [_clip(T, H, W, 500 + 5 * i, 2) for i, (T, H, W) in enumerate(spec)]
    clips, queries = [p[0] for p in pairs], [p[1] for p in pairs]
    m = _MixedOracleModel()
    want, r_all = ch.track_queries_mixed(m, clips, queries, iters=1, return_rounds=True)
    assert max(row[2] for _, cl in m.calls for row in cl) == 3
    monkeypatch.setattr(ch, "MAX_GROUPS", 2)
    m2 = _MixedOracleModel()
    got, r_cap = ch.track_queries_mixed(m2, clips, queries, iters=1, return_rounds=True)
    assert max(row[2] for _, cl in m2.calls for row in cl) == 1
    assert m2.encoded == sum(v.shape[0] for v in clips)
    assert r_cap > r_all
    for (a, av), (b, bv) in zip(got, want):
        assert torch.equal(a, b)
        assert torch.allclose(av, bv, rtol=0, atol=4 * 2 ** -24)


@pytest.mark.parametrize("case", ["count_mismatch", "empty", "clip_not_rgb", "clip_batch_2", "clip_no_frames",
                                  "queries_xy_only", "no_queries", "t_past_clip", "t_fractional", "x_nan",
                                  "map_under_8x8_high", "map_under_8x8_wide"])
def test_track_queries_mixed_rejects_bad_input(case):
    from pips_b200.chain import track_queries_mixed

    class Model:                  # never reached: validation comes before any work
        stride = 4
        engine = None

        def parameters(self):
            return iter([torch.zeros(1)])

        def encode(self, clip):
            raise AssertionError("encoded despite bad input")

    clips = [torch.zeros(5, 3, 32, 40), torch.zeros(1, 3, 3, 48, 32), torch.zeros(9, 3, 32, 32, dtype=torch.uint8)]
    queries = [torch.tensor([[0.0, 3.0, 4.0], [4.0, 1.0, 2.0]]), torch.tensor([[[2.0, 3.0, 4.0]]]),
               torch.tensor([[8.0, 1.0, 1.0]])]
    if case == "count_mismatch":
        queries = queries[:2]
    elif case == "empty":
        clips, queries = [], []
    elif case == "clip_not_rgb":
        clips[1] = torch.zeros(3, 1, 32, 32)
    elif case == "clip_batch_2":
        clips[1] = torch.zeros(2, 3, 3, 32, 32)
    elif case == "clip_no_frames":
        clips[0] = clips[0][:0]
    elif case == "queries_xy_only":
        queries[0] = queries[0][:, 1:]
    elif case == "no_queries":
        queries[2] = queries[2][:0]
    elif case == "t_past_clip":
        queries[1] = torch.tensor([[[3.0, 3.0, 4.0]]])
    elif case == "t_fractional":
        queries[0][1, 0] = 2.5
    elif case == "x_nan":
        queries[2][0, 1] = float("nan")
    elif case == "map_under_8x8_high":
        clips[2] = torch.zeros(9, 3, 31, 64, dtype=torch.uint8)         # 7 x 16 at stride 4
    elif case == "map_under_8x8_wide":
        clips[0] = torch.zeros(5, 3, 64, 28)                            # 16 x 7
    with pytest.raises(ValueError):
        track_queries_mixed(Model(), clips, queries)


def test_track_queries_mixed_rejects_sharded_models():
    from pips_b200.chain import track_queries_mixed

    class Model:
        _shard = (0, 2, None)

    with pytest.raises(RuntimeError):
        track_queries_mixed(Model(), [torch.zeros(4, 3, 32, 32)], [torch.tensor([[0.0, 3.0, 4.0]])])


def test_group_entry_points_validate_arguments_without_gpu():
    """pips_corr_gather_groups, pips_init_gather_groups and pips_refine_iter_groups reject NULL pointers, a missing
    table or frame_base, G outside 1..PIPS_MAX_GROUPS, a group under 8x8 or without frames and a NULL level, before
    any launch."""
    from pips_b200 import _lib as L
    lib = L.load()
    fake = 256

    def groups(G=2, H=16, W=16, frames=3, null_level=False):
        g = L.Groups()
        g.G = G
        for k in range(min(G, L.MAX_GROUPS)):
            for l in range(L.LEVELS):
                g.lvl[k][l] = None if null_level and k == 1 and l == 2 else fake
            g.H[k], g.W[k], g.frames[k] = H, W, frames
        return g

    def corr(g, fb=fake, table=fake):
        return lib.pips_corr_gather_groups(None if g is None else C.byref(g), 0, 1, S, 1, fake, fake, fake, fb, table,
                                           None, None, fake, 576, None)

    def init(g, fb=fake, table=fake):
        return lib.pips_init_gather_groups(None if g is None else C.byref(g), 1, S, 1, fake, fb, table, fake, fake, None)

    for fn, who in ((corr, b"pips_corr_gather_groups"), (init, b"pips_init_gather_groups")):
        assert fn(None) != 0 and who + b": null pointer" in lib.pips_last_error()
        assert fn(groups(), table=None) != 0 and b"needs frame_base and a table" in lib.pips_last_error()
        assert fn(groups(), fb=None) != 0 and b"needs frame_base and a table" in lib.pips_last_error()
        for G in (0, L.MAX_GROUPS + 1):
            assert fn(groups(G=G)) != 0 and b"1 <= G <= PIPS_MAX_GROUPS" in lib.pips_last_error()
        assert fn(groups(H=7)) != 0 and b"at least 8x8" in lib.pips_last_error()
        assert fn(groups(W=7)) != 0 and b"at least 8x8" in lib.pips_last_error()
        assert fn(groups(frames=0)) != 0 and b"frames >= 1" in lib.pips_last_error()
    assert corr(groups(null_level=True)) != 0 and b"null level pointer" in lib.pips_last_error()
    g = groups()
    assert lib.pips_corr_gather_groups(C.byref(g), 7, 1, S, 1, fake, fake, fake, fake, fake, None, None, fake, 576,
                                       None) != 0
    assert b"unknown feat_dtype" in lib.pips_last_error()
    prob, w, ws = L.Problem(), L.Weights(), L.Workspace()
    prob.B, prob.S, prob.N = 1, S, 1
    assert lib.pips_refine_iter_groups(None, C.byref(g), fake, C.byref(w), C.byref(ws), fake, None) != 0
    assert b"pips_refine_iter_groups: null argument" in lib.pips_last_error()
    assert lib.pips_refine_iter_groups(C.byref(prob), None, fake, C.byref(w), C.byref(ws), fake, None) != 0
    assert b"needs groups and a table" in lib.pips_last_error()
    assert lib.pips_refine_iter_groups(C.byref(prob), C.byref(g), None, C.byref(w), C.byref(ws), fake, None) != 0
    assert b"needs groups and a table" in lib.pips_last_error()


def test_engine_checks_the_group_table():
    """refine()'s grouped mode checks the (B, N, 3) table on the host and hands the kernels (B, N, 4) rows."""
    from pips_b200 import _lib as L
    from pips_b200.engine import RefineEngine
    fb = torch.zeros(1, 2, dtype=torch.int32)
    check = RefineEngine._check_groups
    ok = torch.tensor([[[0, 5, 1], [2, 4, 0]]], dtype=torch.int32)
    assert torch.equal(check(ok, fb, 1, 2, [6, 5], "cpu"), torch.tensor([[[0, 5, 1, 0], [2, 4, 0, 0]]], dtype=torch.int32))
    for bad in ([[0, 5, 1], [3, 4, 0]], [[-1, 3, 0], [0, 1, 0]], [[0, 0, 0], [0, 1, 0]], [[0, 1, 2], [0, 1, 0]],
                [[0, 1, -1], [0, 1, 0]], [[0, 6, 1], [0, 1, 0]]):
        with pytest.raises(L.PipsCudaError):
            check(torch.tensor([bad], dtype=torch.int32), fb, 1, 2, [6, 5], "cpu")
    with pytest.raises(L.PipsCudaError):
        check(ok[..., :2], fb, 1, 2, [6, 5], "cpu")
    with pytest.raises(L.PipsCudaError):
        check(ok.float(), fb, 1, 2, [6, 5], "cpu")


# ------------------------------------------------------------------------------------------------ GPU

def _groups_struct(pyrs, feat, f32_level0=False):
    """pips_groups over per-group (f32 levels, bf16 levels) pairs: fp32 level 0 for init_gather, else feat's levels."""
    from pips_b200 import _lib as L
    g = L.Groups()
    g.G = len(pyrs)
    for k, (f32, bf) in enumerate(pyrs):
        lv = f32 if (f32_level0 or feat == "fp32") else bf
        for l in range(L.LEVELS):
            g.lvl[k][l] = L.ptr(lv[l])
        g.H[k], g.W[k], g.frames[k] = f32[0].shape[1], f32[0].shape[2], f32[0].shape[0]
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["fp32", "bf16"])
def test_group_kernels_equal_clip_kernels_per_group(feat):
    """pips_corr_gather_groups and pips_init_gather_groups over three pyramids (16x24, 8x9 -- level 3 one pixel --
    and 12x20 maps), each holding several clips, with the tracks of all groups interleaved in one call, write for every
    track the bits pips_corr_gather_clips / pips_init_gather_clips write over the track's own group's pyramid."""
    from pips_b200 import _lib as L
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator().manual_seed(61)
    spec = [((16, 24), [3, 9]), ((8, 9), [1, 5, 2]), ((12, 20), [11])]
    per = 12
    fms, pyrs, rows, base, coords = [], [], [], [], []
    for k, ((H, W), lens) in enumerate(spec):
        fm = torch.randn(sum(lens), 128, H, W, generator=g)
        fms.append(fm)
        pyrs.append(_pyramid(fm))
        first = torch.tensor([0] + lens).cumsum(0)[:-1].tolist()
        for f0, T in zip(first, lens):
            base.append(_bases(T, per, g))
            rows += [[f0, T, k, 0]] * per
            coords.append(torch.rand(1, S, per, 2, generator=g) * torch.tensor([W + 6.0, H + 6.0]) - 3.0)
    table = torch.tensor(rows, dtype=torch.int32)
    base = torch.cat(base)
    coords = torch.cat(coords, dim=2)
    N = base.numel()
    order = torch.randperm(N, generator=g)                         # not sorted by group
    table, base, coords = table[order].contiguous(), base[order].contiguous(), coords[:, :, order].contiguous()
    ff_rows = torch.randn(N, S, 128, generator=g)
    times = po.times_axis(S).to(DEV)

    def bufs(n):
        return (torch.full((n * S, 576), float("nan"), device=DEV), torch.full((n, 128), float("nan"), device=DEV),
                torch.full((n, S, 128), float("nan"), device=DEV))

    cd, fd, fbd, td = coords.to(DEV), ff_rows.to(DEV), base.to(DEV), table.to(DEV)
    x, ffeat, ffeats = bufs(N)
    gl, g0 = _groups_struct(pyrs, feat), _groups_struct(pyrs, feat, f32_level0=True)
    L.check(lib.pips_corr_gather_groups(C.byref(gl), L.FEAT_DTYPES[feat], 1, S, N, L.ptr(cd), L.ptr(fd), L.ptr(times),
                                        L.ptr(fbd), L.ptr(td), None, None, L.ptr(x), 576, st))
    L.check(lib.pips_init_gather_groups(C.byref(g0), 1, S, N, L.ptr(cd), L.ptr(fbd), L.ptr(td), L.ptr(ffeat),
                                        L.ptr(ffeats), st))
    torch.cuda.synchronize()
    got = (x.view(N, S, 576), ffeat, ffeats)
    for k, ((H, W), lens) in enumerate(spec):
        mine = (table[:, 2] == k).nonzero().flatten()
        n = mine.numel()
        cl = table[mine, :2].contiguous().to(DEV)
        c_k = coords[:, :, mine].contiguous().to(DEV)
        f_k, b_k = ff_rows[mine].contiguous().to(DEV), base[mine].contiguous().to(DEV)
        f32, bf = pyrs[k]
        lv = bf if feat == "bf16" else f32
        xw, fw, fsw = bufs(n)
        F = sum(lens)
        L.check(lib.pips_corr_gather_clips(L.ptr_array(lv), L.FEAT_DTYPES[feat], 1, S, n, H, W, L.ptr(c_k), L.ptr(f_k),
                                           L.ptr(times), L.ptr(b_k), F, L.ptr(cl), None, None, L.ptr(xw), 576, st))
        L.check(lib.pips_init_gather_clips(L.ptr(f32[0]), 1, S, n, H, W, L.ptr(c_k), L.ptr(b_k), F, L.ptr(cl),
                                           L.ptr(fw), L.ptr(fsw), st))
        torch.cuda.synchronize()
        md = mine.to(DEV)
        for a, b in zip(got, (xw.view(n, S, 576), fw, fsw)):
            a = a[md]
            assert bool(torch.isfinite(a).all())
            assert torch.equal(_bits(a), _bits(b)), f"group {k} ({H}x{W}) differs from its own pyramid"


@pytest.mark.gpu
@pytest.mark.parametrize("precision,feat,max_seqs", [("bf16x3", "fp32", 32768), ("bf16x3", "bf16", 7),
                                                     ("bf16", "fp32", 7), ("fp32", "fp32", 7)])
def test_refine_with_groups_equals_refine_per_group(precision, feat, max_seqs):
    """engine.refine over three groups of feature maps of different sizes (a (B, N, 3) table, tracks interleaved) ==
    engine.refine(clip=) over each group's maps alone, for every iteration's predictions, the visibility logits and the
    features, bit for bit; with gathered and carried features, and with N split into chunks (max_seqs 7)."""
    c = CHAIN_CASE
    model = _model(precision, feat, max_seqs)
    spec = [((96, 128), [(0, 19), (19, 24)]), ((40, 36), [(0, 1), (1, 9)]), ((64, 96), [(0, 12)])]
    g = torch.Generator().manual_seed(45)
    fms, rows, base, coords = [], [], [], []
    per = 10                                                        # _bases' 8 edge cases and 2 random ones
    for k, ((H, W), cuts) in enumerate(spec):
        rgbs = po.smooth_video(1, cuts[-1][1], H, W, seed=46 + k)
        with torch.no_grad():
            fm = model.encode(rgbs.to(DEV)).contiguous()
        fms.append(fm)
        H8, W8 = fm.shape[3], fm.shape[4]
        for a, b in cuts:
            base.append(_bases(b - a, per, g))
            rows += [[a, b - a, k]] * per
            coords.append((torch.rand(1, 1, per, 2, generator=g) * torch.tensor([W8 - 1.0, H8 - 1.0])).repeat(1, S, 1, 1))
    table = torch.tensor(rows, dtype=torch.int32)
    base = torch.cat(base)
    coords = torch.cat(coords, dim=2)
    N = base.numel()
    order = torch.randperm(N, generator=g)
    table, base, coords = table[order], base[order], coords[:, :, order].to(DEV)
    eng, it, st = model.engine, c["iters"], float(c["stride"])
    with torch.no_grad():
        got = eng.refine(model, fms, coords, None, it, st, frame_base=base.view(1, N), clip=table.view(1, N, 3))
        feat_k = got[2]
        got_c = eng.refine(model, fms, coords, feat_k, it, st, frame_base=base.view(1, N), clip=table.view(1, N, 3),
                           reuse_pyramid=True)
        for k in range(len(spec)):
            mine = (table[:, 2] == k).nonzero().flatten()
            md = mine.to(DEV)
            cl = table[mine, :2].reshape(1, -1, 2)
            want = eng.refine(model, fms[k], coords[:, :, md], None, it, st, frame_base=base[mine].view(1, -1), clip=cl)
            want_c = eng.refine(model, fms[k], coords[:, :, md], feat_k[:, md], it, st, frame_base=base[mine].view(1, -1),
                                clip=cl, reuse_pyramid=True)
            for x, y in ((got, want), (got_c, want_c)):
                assert torch.equal(_bits(x[0][:, :, :, md]), _bits(y[0]))
                assert torch.equal(_bits(x[1][:, :, md]), _bits(y[1]))
                assert torch.equal(_bits(x[2][:, md]), _bits(y[2]))
    for x in got:
        assert bool(torch.isfinite(x).all())


def _gpu_mixed():
    """Six clips at four sizes (stride 4), of 19, 5, 1, 40, 9 and 3 frames, with queries at frames 0, T-1 and random
    ones; clips of one size are not adjacent."""
    spec = [(19, 96, 128), (5, 64, 96), (1, 96, 128), (40, 40, 36), (9, 64, 96), (3, 72, 48)]
    pairs = [_clip(T, H, W, 700 + 11 * i, 3 + i) for i, (T, H, W) in enumerate(spec)]
    return [p[0] for p in pairs], [p[1] for p in pairs]


@pytest.mark.gpu
@pytest.mark.parametrize("precision,feat", [("bf16x3", "fp32"), ("bf16x3", "bf16"), ("fp32", "fp32")])
def test_track_queries_mixed_equals_track_queries_per_clip(precision, feat):
    from pips_b200.chain import track_queries, track_queries_mixed
    model = _model(precision, feat)
    clips, queries = _gpu_mixed()
    dc = [v.to(DEV) for v in clips]
    dq = [q.to(DEV) for q in queries]
    outs, rounds = track_queries_mixed(model, dc, dq, iters=CHAIN_CASE["iters"], return_rounds=True)
    per = []
    for (trajs, vis), v, q in zip(outs, dc, dq):
        wt, wv, r = track_queries(model, v.unsqueeze(0), q.unsqueeze(0), iters=CHAIN_CASE["iters"], return_rounds=True)
        per.append(r)
        assert trajs.shape == wt.shape and vis.shape == wv.shape
        assert bool(torch.isfinite(trajs).all())
        assert torch.equal(_bits(trajs), _bits(wt))
        assert torch.equal(_bits(vis), _bits(wv))
    assert rounds == max(per)
    print(f"mixed {precision}/{feat}: {rounds} rounds for the batch, {sum(per)} one clip at a time")


@pytest.mark.gpu
def test_track_queries_mixed_host_uint8_permuted_and_one_size():
    """Host uint8 clips give the bits of device float clips; permuting the clips permutes the results and changes no
    bits; a batch of one size gives track_queries_batch's bits."""
    from pips_b200.chain import track_queries_batch, track_queries_mixed
    model = _model("bf16x3")
    clips, queries = _gpu_mixed()
    want = track_queries_mixed(model, [v.to(DEV) for v in clips], [q.to(DEV) for q in queries])
    host = [v.to(torch.uint8) for v in clips]
    host[1] = host[1].unsqueeze(0)
    qs = list(queries)
    qs[2] = qs[2].unsqueeze(0)
    got = track_queries_mixed(model, host, qs)
    for (a, av), (b, bv) in zip(got, want):
        assert a.device == b.device
        assert torch.equal(_bits(a), _bits(b)) and torch.equal(_bits(av), _bits(bv))
    perm = [3, 5, 1, 0, 4, 2]
    got = track_queries_mixed(model, [clips[p].to(DEV) for p in perm], [queries[p].to(DEV) for p in perm])
    for k, p in enumerate(perm):
        assert torch.equal(_bits(got[k][0]), _bits(want[p][0])) and torch.equal(_bits(got[k][1]), _bits(want[p][1]))
    one = [0, 2]                                                    # the two 96x128 clips
    got = track_queries_mixed(model, [clips[i].to(DEV) for i in one], [queries[i].to(DEV) for i in one])
    ref = track_queries_batch(model, [clips[i].to(DEV) for i in one], [queries[i].to(DEV) for i in one])
    for (a, av), (b, bv) in zip(got, ref):
        assert torch.equal(_bits(a), _bits(b)) and torch.equal(_bits(av), _bits(bv))
