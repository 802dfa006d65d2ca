"""Queries in many videos at once (pips_b200.chain.track_queries_batch) and the per-track clip table under it.

Several clips are concatenated in one pyramid; each track carries its clip {first, count} and reads its windows inside
that clip (pips_corr_gather_clips / pips_init_gather_clips, engine.refine(clip=)).  CPU: the host logic with the
oracle as the 8-frame tracker reproduces track_queries clip by clip and never reads another clip's frames; input
validation; the new C entry points' argument checks.  GPU: the clip-aware kernels against the frame_base kernels over
each clip's own pyramid, engine.refine(clip=) against per-clip refine(frame_base=), and track_queries_batch against
per-clip track_queries, bit for bit."""
import ctypes as C

import pytest
import torch

from oracle import pips_oracle as po
from tests.golden.make_golden import CHAIN_CASE
from tests.golden.make_golden_queries import query_inputs

DEV = "cuda:0"
S = 8


def _window_frames(base, T):
    """The frames step s = 0..7 of a window reads inside a clip of T frames (csrc/corr_common.cuh window_frame)."""
    s = torch.arange(S)
    return (base + s).clamp(max=T - 1) if base >= 0 else (~base - s).clamp(min=0)


def _batch_case():
    """Three clips cut from CHAIN_CASE's video -- 19 frames, 6 frames (shorter than a window) and a single frame -- with
    6, 3 and 2 queries."""
    c = CHAIN_CASE
    rgbs, q19 = query_inputs(c)
    q6 = torch.cat([torch.tensor([0.0, 2.0, 5.0]).view(1, 3, 1), po.random_queries(1, 3, c["H"], c["W"], seed=71)], dim=2)
    q1 = torch.cat([torch.zeros(1, 2, 1), po.random_queries(1, 2, c["H"], c["W"], seed=72)], dim=2)
    return [rgbs[0], rgbs[0, 4:10], rgbs[0, 11:12]], [q19[0], q6[0], q1[0]]


class _OracleModel:
    """The oracle as encoder (one frame at a time, so a frame's maps do not depend on its chunk) and as the 8-frame
    tracker, one window per track read through frame_base -- inside the track's clip when the call carries a clip
    table, as the kernels decode it.  With a clip table every frame outside the track's clip is NaN to that track.
    ``calls`` records (frame_base, clip) of every refinement call."""

    def __init__(self):
        c = CHAIN_CASE
        self.c = c
        self.sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
        self.stride = c["stride"]
        self.calls = []
        self.encoded = 0
        model = self

        class Engine:
            def refine(self, module, fmaps, coords, feat_init, iters, stride, frame_base=None, reuse_pyramid=False,
                       clip=None):
                return model._refine(fmaps, coords, feat_init, iters, stride, frame_base, clip)

        self.engine = Engine()

    def parameters(self):
        return iter([torch.zeros(1)])

    def encode(self, clip):
        c = self.c
        Bc, Tc = clip.shape[:2]
        assert Bc == 1 and Tc <= 32
        self.encoded += Tc
        x = 2 * (clip.float() / 255.0) - 1.0
        with torch.no_grad():
            f = torch.cat([po.fnet(self.sd, x[:, k], c["stride"]) for k in range(Tc)])
        return f.reshape(Bc, Tc, 128, c["H"] // c["stride"], c["W"] // c["stride"])

    def _refine(self, fmaps, coords, feat_init, iters, stride, frame_base, clip):
        c = self.c
        B, _, na, _ = coords.shape
        F = fmaps.shape[1]
        assert B == 1 and frame_base.shape == (1, na) and frame_base.dtype == torch.int32
        if clip is not None:
            assert clip.shape == (1, na, 2) and clip.dtype == torch.int32
        self.calls.append((frame_base[0].tolist(), None if clip is None else clip[0].tolist()))
        preds = torch.zeros(iters, 1, S, na, 2)
        vis = torch.zeros(1, S, na)
        ffeat = torch.zeros(1, na, 128)
        for n in range(na):
            base = int(frame_base[0, n])
            if clip is None:
                fm = fmaps[:, _window_frames(base, F)]
            else:
                first, count = (int(v) for v in clip[0, n])
                own = torch.full_like(fmaps, float("nan"))
                own[:, first:first + count] = fmaps[:, first:first + count]
                fm = own[:, first + _window_frames(base, count)]
            fi = None if feat_init is None else feat_init[:, n:n + 1]
            with torch.no_grad():
                o = po.forward(self.sd, coords[:, 0, n:n + 1] * stride, torch.zeros(1, S, 3, c["H"], c["W"]),
                               iters=iters, stride=int(stride), fmaps=fm, feat_init=fi, return_feat=True)
            preds[:, :, :, n] = torch.stack(o[0])[:, :, :, 0]
            vis[:, :, n] = o[2][:, :, 0]
            ffeat[:, n] = o[3][:, 0]
        return preds, vis, ffeat


def test_batch_host_logic_equals_track_queries_per_clip_on_cpu():
    """track_queries_batch with the oracle as tracker == track_queries on each clip alone, with the same tracker: the
    same trajectories bit for bit, visibilities within a few ulps (torch's CPU sigmoid rounds its vectorised body and
    its scalar tail differently, and a track's position in the call differs), and as many rounds as the longest
    clip's chain.  Every window reads its own clip only: the other clips' frames are NaN to it, and the results are
    finite.  All frames are encoded once."""
    from pips_b200.chain import track_queries, track_queries_batch
    clips, queries = _batch_case()
    m = _OracleModel()
    outs, rounds = track_queries_batch(m, clips, queries, iters=CHAIN_CASE["iters"], return_rounds=True)
    assert m.encoded == sum(v.shape[0] for v in clips)
    batch_calls = list(m.calls)
    assert all(cl is not None for _, cl in batch_calls)
    assert len(outs) == len(clips)
    per_rounds = []
    for (trajs, vis), v, q in zip(outs, clips, queries):
        T, N = v.shape[0], q.shape[0]
        assert trajs.shape == (1, T, N, 2) and vis.shape == (1, T, N)
        assert bool(torch.isfinite(trajs).all()) and bool(torch.isfinite(vis).all())
        m.calls.clear()
        wt, wv, r = track_queries(m, v.unsqueeze(0), q.unsqueeze(0), iters=CHAIN_CASE["iters"], return_rounds=True)
        assert all(cl is None for _, cl in m.calls)              # the one-clip path passes no clip table
        per_rounds.append(r)
        assert torch.equal(trajs, wt)
        assert torch.allclose(vis, wv, rtol=0, atol=4 * 2 ** -24)
    assert rounds == max(per_rounds) == len(batch_calls)
    # clip tables: clip i spans frames offset_i .. offset_i + T_i - 1 of the batch
    offsets = torch.tensor([0] + [v.shape[0] for v in clips]).cumsum(0).tolist()
    spans = {(offsets[i], clips[i].shape[0]) for i in range(len(clips))}
    for bases, cl in batch_calls:
        assert {tuple(x) for x in cl} <= spans


def test_batch_of_one_clip_is_track_queries_on_cpu():
    from pips_b200.chain import track_queries, track_queries_batch
    clips, queries = _batch_case()
    m = _OracleModel()
    (got,) = track_queries_batch(m, clips[1:2], queries[1:2], iters=2)
    want = track_queries(m, clips[1].unsqueeze(0), queries[1].unsqueeze(0), iters=2)
    assert torch.equal(got[0], want[0])


@pytest.mark.parametrize("case", ["count_mismatch", "empty", "sizes_differ", "clip_not_rgb", "clip_batch_2",
                                  "clip_no_frames", "queries_xy_only", "queries_batch_2", "no_queries",
                                  "t_past_second_clip", "t_fractional", "x_nan"])
def test_track_queries_batch_rejects_bad_input(case):
    from pips_b200.chain import track_queries_batch

    class Model:                  # never reached: validation comes before any work
        stride = 4
        engine = None

        def parameters(self):
            return iter([torch.zeros(1)])

        def encode(self, clip):
            raise AssertionError("encoded despite bad input")

    clips = [torch.zeros(5, 3, 16, 16), torch.zeros(1, 3, 3, 16, 16), torch.zeros(9, 3, 16, 16, dtype=torch.uint8)]
    queries = [torch.tensor([[0.0, 3.0, 4.0], [4.0, 1.0, 2.0]]), torch.tensor([[[2.0, 3.0, 4.0]]]),
               torch.tensor([[8.0, 1.0, 1.0]])]
    if case == "count_mismatch":
        queries = queries[:2]
    elif case == "empty":
        clips, queries = [], []
    elif case == "sizes_differ":
        clips[2] = torch.zeros(9, 3, 16, 20)
    elif case == "clip_not_rgb":
        clips[1] = torch.zeros(3, 1, 16, 16)
    elif case == "clip_batch_2":
        clips[1] = torch.zeros(2, 3, 3, 16, 16)
    elif case == "clip_no_frames":
        clips[0] = clips[0][:0]
    elif case == "queries_xy_only":
        queries[0] = queries[0][:, 1:]
    elif case == "queries_batch_2":
        queries[1] = queries[1].repeat(2, 1, 1)
    elif case == "no_queries":
        queries[2] = queries[2][:0]
    elif case == "t_past_second_clip":
        queries[1] = torch.tensor([[[3.0, 3.0, 4.0]]])          # clip 1 has 3 frames; 3 is inside clip 0 and 2
    elif case == "t_fractional":
        queries[0][1, 0] = 2.5
    elif case == "x_nan":
        queries[2][0, 1] = float("nan")
    with pytest.raises(ValueError):
        track_queries_batch(Model(), clips, queries)


def test_track_queries_batch_rejects_sharded_models():
    from pips_b200.chain import track_queries_batch

    class Model:
        _shard = (0, 2, None)

    with pytest.raises(RuntimeError):
        track_queries_batch(Model(), [torch.zeros(4, 3, 16, 16)], [torch.tensor([[0.0, 3.0, 4.0]])])


def test_clip_entry_points_validate_arguments_without_gpu():
    """pips_corr_gather_clips, pips_init_gather_clips and pips_refine_iter_clips reject NULL pointers, and a clip table
    without frame_base, before any launch."""
    from pips_b200 import _lib as L
    lib = L.load()
    fake = 256
    lvl = (C.c_void_p * L.LEVELS)(*([fake] * L.LEVELS))
    assert lib.pips_corr_gather_clips(None, 0, 1, S, 1, 16, 16, 0, 0, 0, None, 0, None, 0, 0, 0, 576, None) != 0
    assert b"pips_corr_gather_clips: null pointer" in lib.pips_last_error()
    assert lib.pips_corr_gather_clips(lvl, 0, 1, S, 1, 16, 16, fake, fake, fake, None, 0, fake, 0, 0, fake, 576, None) != 0
    assert b"clip table needs frame_base" in lib.pips_last_error()
    assert lib.pips_init_gather_clips(None, 1, S, 1, 16, 16, 0, None, 0, None, 0, 0, None) != 0
    assert b"pips_init_gather_clips: null pointer" in lib.pips_last_error()
    assert lib.pips_init_gather_clips(fake, 1, S, 1, 16, 16, fake, None, 0, fake, fake, fake, None) != 0
    assert b"clip table needs frame_base" in lib.pips_last_error()
    assert lib.pips_refine_iter_clips(None, None, None, None, 0, None) != 0
    assert b"pips_refine_iter_clips: null argument" in lib.pips_last_error()
    prob, w, ws = L.Problem(), L.Weights(), L.Workspace()
    prob.B, prob.S, prob.N = 1, S, 1
    assert lib.pips_refine_iter_clips(C.byref(prob), fake, C.byref(w), C.byref(ws), fake, None) != 0
    assert b"clip table needs frame_base" in lib.pips_last_error()


def test_engine_checks_the_clip_table():
    """refine(clip=) checks the table on the host, before any kernel: the kernels read pyramid frames through it."""
    from pips_b200 import _lib as L
    from pips_b200.engine import RefineEngine
    fb = torch.zeros(1, 2, dtype=torch.int32)
    check = RefineEngine._check_clip
    ok = torch.tensor([[[0, 5], [5, 4]]], dtype=torch.int32)
    assert torch.equal(check(ok, fb, 1, 2, 9, "cpu"), ok)
    for bad in ([[0, 5], [5, 5]], [[-1, 3], [0, 1]], [[0, 0], [0, 1]]):
        with pytest.raises(L.PipsCudaError):
            check(torch.tensor([bad], dtype=torch.int32), fb, 1, 2, 9, "cpu")
    with pytest.raises(L.PipsCudaError):
        check(ok, None, 1, 2, 9, "cpu")                                     # a clip table needs frame_base
    with pytest.raises(L.PipsCudaError):
        check(ok[:, :1], fb, 1, 2, 9, "cpu")                                # one row per track
    with pytest.raises(L.PipsCudaError):
        check(ok.float(), fb, 1, 2, 9, "cpu")


# ------------------------------------------------------------------------------------------------ GPU

def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32).cpu()


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


def _bases(T, n, g):
    """Window starts inside a clip of T frames: forward and backward, at and past either end, and random ones."""
    edge = [0, T - 1, T + 3, ~0, ~(T - 1), ~(T + 2), min(3, T - 1), ~min(6, T - 1)]
    rnd = torch.randint(0, T, (n - len(edge),), generator=g)
    rnd = torch.where(torch.rand(rnd.shape, generator=g) < 0.5, rnd, ~rnd)
    return torch.cat([torch.tensor(edge), rnd]).to(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["fp32", "bf16"])
def test_clip_kernels_equal_frame_base_kernels_per_clip(feat):
    """pips_corr_gather_clips and pips_init_gather_clips over clips of 3, 13, 1 and 9 frames concatenated in one
    pyramid write, for every track, the bits pips_corr_gather / pips_init_gather write with frame_base over the track's
    clip alone.  Each clip is checked on a pyramid whose other clips' frames are NaN, so a window that left its clip
    would show."""
    from pips_b200 import _lib as L
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    lens, per, H, W = [3, 13, 1, 9], 14, 16, 24
    g = torch.Generator().manual_seed(41)
    F = sum(lens)
    first = torch.tensor([0] + lens).cumsum(0)[:-1].tolist()
    fm = torch.randn(F, 128, H, W, generator=g)
    N = per * len(lens)
    base = torch.cat([_bases(T, per, g) for T in lens])
    clip = torch.tensor([[f, T] for f, T in zip(first, lens) for _ in range(per)], dtype=torch.int32)
    order = torch.randperm(N, generator=g)                        # tracks of all clips interleaved in one call
    base, clip = base[order].contiguous(), clip[order].contiguous()
    coords = torch.rand(1, S, N, 2, generator=g) * torch.tensor([W + 6.0, H + 6.0]) - 3.0
    ff_rows = torch.randn(N, S, 128, generator=g)
    times = po.times_axis(S).to(DEV)

    def run(levels, fb, cl, frames, idx):
        n = idx.numel()
        lv = levels[1] if feat == "bf16" else levels[0]
        cd = coords[:, :, idx].to(DEV).contiguous()
        fd = ff_rows[idx].to(DEV).contiguous()
        fbd = fb[idx].to(DEV).contiguous()
        cld = None if cl is None else cl[idx].to(DEV).contiguous()
        x = torch.full((n * S, 576), float("nan"), device=DEV)
        ffeat, ffeats = torch.full((n, 128), float("nan"), device=DEV), torch.full((n, S, 128), float("nan"), device=DEV)
        if cld is None:
            L.check(lib.pips_corr_gather(L.ptr_array(lv), L.FEAT_DTYPES[feat], 1, S, n, H, W, L.ptr(cd), L.ptr(fd),
                                         L.ptr(times), L.ptr(fbd), frames, None, None, L.ptr(x), 576, st))
            L.check(lib.pips_init_gather(L.ptr(levels[0][0]), 1, S, n, H, W, L.ptr(cd), L.ptr(fbd), frames, L.ptr(ffeat),
                                         L.ptr(ffeats), st))
        else:
            L.check(lib.pips_corr_gather_clips(L.ptr_array(lv), L.FEAT_DTYPES[feat], 1, S, n, H, W, L.ptr(cd), L.ptr(fd),
                                               L.ptr(times), L.ptr(fbd), frames, L.ptr(cld), None, None, L.ptr(x), 576, st))
            L.check(lib.pips_init_gather_clips(L.ptr(levels[0][0]), 1, S, n, H, W, L.ptr(cd), L.ptr(fbd), frames,
                                               L.ptr(cld), L.ptr(ffeat), L.ptr(ffeats), st))
        torch.cuda.synchronize()
        return x.view(n, S, 576), ffeat, ffeats

    all_idx = torch.arange(N)
    for i, (f0, T) in enumerate(zip(first, lens)):
        mine = (clip[:, 0] == f0).nonzero().flatten()
        alone = fm.clone()
        alone[:f0] = float("nan")
        alone[f0 + T:] = float("nan")
        got = run(_pyramid(alone), base, clip, F, all_idx)
        want = run(_pyramid(fm[f0:f0 + T]), base, None, T, mine)
        for a, b in zip(got, want):
            a = a[mine]
            assert bool(torch.isfinite(a).all()), f"clip {i} ({T} frames): a window read another clip's frames"
            assert torch.equal(_bits(a), _bits(b)), f"clip {i} ({T} frames) differs from its own pyramid"


def _model(precision, feat="fp32", max_seqs=32768):
    from pips_b200 import Pips
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    model = Pips(S=8, stride=c["stride"], precision=precision, feat_dtype=feat, max_seqs=max_seqs).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    return model


@pytest.mark.gpu
@pytest.mark.parametrize("max_seqs", [32768, 7])
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_refine_with_clips_equals_refine_per_clip(precision, max_seqs):
    """engine.refine(clip=) over the concatenated feature maps of four clips == engine.refine(frame_base=) over each
    clip's own maps, for every iteration's predictions, the visibility logits and the features, bit for bit; also
    when N is split into chunks (max_seqs 7)."""
    c = CHAIN_CASE
    model = _model(precision, max_seqs=max_seqs)
    rgbs = po.smooth_video(1, 30, c["H"], c["W"], seed=43)
    with torch.no_grad():
        fm = model.encode(rgbs.to(DEV)).contiguous()
    cuts = [(0, 19), (19, 24), (24, 25), (25, 30)]                  # 19, 5, 1 and 5 frames
    H8, W8 = fm.shape[3], fm.shape[4]
    g = torch.Generator().manual_seed(44)
    per = 9
    base = torch.cat([_bases(b - a, per, g) for a, b in cuts])
    clip = torch.tensor([[a, b - a] for a, b in cuts for _ in range(per)], dtype=torch.int32)
    N = base.numel()
    order = torch.randperm(N, generator=g)
    base, clip = base[order], clip[order]
    coords = (torch.rand(1, 1, N, 2, generator=g) * torch.tensor([W8 - 1.0, H8 - 1.0])).repeat(1, S, 1, 1).to(DEV)
    eng, it, st = model.engine, c["iters"], float(c["stride"])
    with torch.no_grad():
        got = eng.refine(model, fm, coords, None, it, st, frame_base=base.view(1, N), clip=clip.view(1, N, 2))
        feat = got[2]
        got_c = eng.refine(model, fm, coords, feat, it, st, frame_base=base.view(1, N), clip=clip.view(1, N, 2),
                           reuse_pyramid=True)                       # carried features
        for a, b in cuts:
            mine = (clip[:, 0] == a).nonzero().flatten()
            md = mine.to(DEV)
            own = fm[:, a:b].contiguous()
            want = eng.refine(model, own, coords[:, :, md], None, it, st, frame_base=base[mine].view(1, -1))
            want_c = eng.refine(model, own, coords[:, :, md], feat[:, md], it, st, frame_base=base[mine].view(1, -1),
                                reuse_pyramid=True)
            for x, y in ((got, want), (got_c, want_c)):
                assert torch.equal(_bits(x[0][:, :, :, md]), _bits(y[0]))
                assert torch.equal(_bits(x[1][:, :, md]), _bits(y[1]))
                assert torch.equal(_bits(x[2][:, md]), _bits(y[2]))
    for x in got:
        assert bool(torch.isfinite(x).all())


def _gpu_batch(n_frames=(19, 5, 1, 40)):
    """Four clips of 19, 5, 1 and 40 frames (65 in all: encoder chunks cross clip boundaries) with queries at random
    frames, t = 0 and t = T-1 among them."""
    c = CHAIN_CASE
    clips, queries = [], []
    for i, T in enumerate(n_frames):
        clips.append(po.smooth_video(1, T, c["H"], c["W"], seed=80 + i)[0])
        n = 3 + 2 * i
        g = torch.Generator().manual_seed(90 + i)
        t = torch.randint(0, T, (n,), generator=g).float()
        t[0], t[-1] = 0.0, float(T - 1)
        queries.append(torch.cat([t.view(n, 1), po.random_queries(1, n, c["H"], c["W"], seed=100 + i)[0]], dim=1))
    return clips, queries


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["fp32", "bf16"])
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_track_queries_batch_equals_track_queries_per_clip(precision, feat):
    from pips_b200.chain import track_queries, track_queries_batch
    model = _model(precision, feat)
    clips, queries = _gpu_batch()
    dc = [v.to(DEV) for v in clips]
    dq = [q.to(DEV) for q in queries]
    outs, rounds = track_queries_batch(model, dc, dq, iters=CHAIN_CASE["iters"], return_rounds=True)
    per = []
    for (trajs, vis), v, q in zip(outs, dc, dq):
        wt, wv, r = track_queries(model, v.unsqueeze(0), q.unsqueeze(0), iters=CHAIN_CASE["iters"], return_rounds=True)
        per.append(r)
        assert trajs.shape == wt.shape and vis.shape == wv.shape
        assert bool(torch.isfinite(trajs).all())
        assert torch.equal(_bits(trajs), _bits(wt))
        assert torch.equal(_bits(vis), _bits(wv))
    assert rounds == max(per)
    print(f"batch {precision}/{feat}: {rounds} rounds for the batch, {sum(per)} one clip at a time")


@pytest.mark.gpu
def test_track_queries_batch_host_uint8_and_permuted_clips():
    """Host uint8 clips give the bits of device float clips, with (T, 3, H, W) and (1, T, 3, H, W) clips and (N, 3) and
    (1, N, 3) queries mixed; permuting the clips permutes the results and changes no bits."""
    from pips_b200.chain import track_queries_batch
    model = _model("bf16x3")
    clips, queries = _gpu_batch()
    want = track_queries_batch(model, [v.to(DEV) for v in clips], [q.to(DEV) for q in queries])
    host = [v.to(torch.uint8) for v in clips]
    host[1] = host[1].unsqueeze(0)
    qs = list(queries)
    qs[2] = qs[2].unsqueeze(0)
    got = track_queries_batch(model, host, qs)
    for (a, av), (b, bv) in zip(got, want):
        assert a.device == b.device
        assert torch.equal(_bits(a), _bits(b)) and torch.equal(_bits(av), _bits(bv))
    perm = [3, 1, 0, 2]
    got = track_queries_batch(model, [clips[p].to(DEV) for p in perm], [queries[p].to(DEV) for p in perm])
    for k, p in enumerate(perm):
        assert torch.equal(_bits(got[k][0]), _bits(want[p][0])) and torch.equal(_bits(got[k][1]), _bits(want[p][1]))
