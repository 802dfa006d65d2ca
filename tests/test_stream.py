"""Streamed tracking in bounded device memory (pips_b200.stream: TrackStream, track_queries_stream).

CPU: the stream's host logic with the oracle as the 8-frame tracker and the oracle's fnet as the encoder, against
track_queries' host logic and the reference's recording; the bound on the frames a refinement call sees and the
stream retains; the rules of the returned blocks; input validation.  GPU: bit equality with track_queries and
track_chain at every chunk size, precision and pyramid dtype, uint8 host chunks against float device chunks, and peak
device memory that does not grow with the length of the video."""
import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from tests.golden.make_golden import CHAIN_CASE
from tests.golden.make_golden_queries import QUERY_TIMES, query_inputs
from tests.test_queries import GOLD, _gold_skips, _window_frames

DEV = "cuda:0"
S = 8


def _chunks(rgbs, k, reverse=False):
    """rgbs (1, T, 3, H, W) as chunks of k frames (k, 3, H, W), in time order or from the last frame back."""
    clip = rgbs[0].flip(0) if reverse else rgbs[0]
    return [clip[i:i + k] for i in range(0, clip.shape[0], k)]


class _OracleModel:
    """The oracle's fnet as the encoder (each frame encoded once, looked up by its pixels) and the oracle's 8-frame
    model as the tracker, one window per track read through frame_base as the kernels decode it.  ``log`` records
    every refinement call: frames held, and for every track the clip frame of its window's step 0 and its direction."""
    stride = CHAIN_CASE["stride"]

    def __init__(self):
        c = CHAIN_CASE
        self.c = c
        self.sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
        self.rgbs, self.queries = query_inputs(c)
        with torch.no_grad():
            x = 2 * (self.rgbs[0] / 255.0) - 1.0
            self.fm = po.fnet(self.sd, x, c["stride"])                                  # (T, 128, H8, W8)
        self.log = []
        self.engine = self

    def parameters(self):
        return iter([torch.zeros(1)])

    def _frame(self, rgb):
        return next(j for j in range(self.rgbs.shape[1]) if torch.equal(self.rgbs[0, j], rgb))

    def encode(self, clip):
        return self.fm[[self._frame(clip[0, i]) for i in range(clip.shape[1])]].unsqueeze(0)

    def refine(self, module, fmaps, coords, feat_init, iters, stride, frame_base=None, reuse_pyramid=False):
        c, sd = self.c, self.sd
        B, F, na = 1, fmaps.shape[1], coords.shape[2]
        assert coords.shape[0] == B and frame_base.shape == (1, na) and frame_base.dtype == torch.int32
        clip = [next(j for j in range(self.fm.shape[0]) if torch.equal(self.fm[j], fmaps[0, i])) for i in range(F)]
        preds = torch.zeros(iters, 1, S, na, 2)
        vis = torch.zeros(1, S, na)
        ffeat = torch.zeros(1, na, 128)
        starts = []
        for n in range(na):
            idx = _window_frames(int(frame_base[0, n]), F)
            fi = None if feat_init is None else feat_init[:, n:n + 1]
            with torch.no_grad():
                o = po.forward(sd, coords[:, 0, n:n + 1] * stride, torch.zeros(1, S, 3, c["H"], c["W"]), iters=iters,
                               stride=int(stride), fmaps=fmaps[:, idx], feat_init=fi, return_feat=True)
            if iters > 0:
                preds[:, :, :, n] = torch.stack(o[0])[:, :, :, 0]
            vis[:, :, n] = o[2][:, :, 0]
            ffeat[:, n] = o[3][:, 0]
            starts.append(clip[int(idx[0])])
        direction = 1 if F < 2 or clip[1] > clip[0] else -1
        self.log.append(dict(frames=F, iters=iters, reuse=reuse_pyramid, starts=starts, direction=direction))
        return preds, vis, ffeat


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _ulps(a, b):
    """Largest distance in units in the last place between two same-signed fp32 tensors."""
    return int((_bits(a).long() - _bits(b).long()).abs().max())


@pytest.mark.parametrize("chunk", [1, 3, 8, 19])
def test_stream_host_logic_matches_track_queries_and_reference_recording(chunk):
    """track_queries_stream with the oracle as the tracker == track_queries' host logic with the same tracker: the same
    trajectories bit for bit, both within the recording's tolerances; every track's windows start where the reference's
    skips put them, in both directions; no refinement call holds more than chunk + 7 frames.  Visibilities agree to
    4 ulps: torch's CPU sigmoid rounds an element of its vectorised body and of its scalar tail differently (up to
    2 ulps apart on random logits), so on the host a visibility's last bits depend on its place in the round's batch.
    The GPU tests check visibilities bit for bit."""
    from pips_b200.chain import track_queries
    from pips_b200.stream import track_queries_stream
    m = _OracleModel()
    want_t, want_v = track_queries(m, m.rgbs, m.queries, iters=m.c["iters"])
    m.log.clear()
    trajs, vis = track_queries_stream(m, _chunks(m.rgbs, chunk), _chunks(m.rgbs, chunk, reverse=True), m.queries,
                                      iters=m.c["iters"])
    assert trajs.shape == want_t.shape and vis.shape == want_v.shape
    assert torch.equal(_bits(trajs), _bits(want_t)) and _ulps(vis, want_v) <= 4
    assert np.abs(trajs.numpy() - GOLD["trajs"]).max() < 1e-3
    assert np.abs(vis.numpy() - GOLD["vis"]).max() < 1e-4
    assert max(e["frames"] for e in m.log) <= chunk + S - 1
    fwd, bwd = _gold_skips()
    for d, skips in ((1, fwd), (-1, bwd)):
        want = sorted(t + d * int(s) for t, h in zip(QUERY_TIMES, skips) if d > 0 or t > 0
                      for s in [0] + list(np.cumsum(h)[:-1]))
        got = sorted(s for e in m.log if e["direction"] == d and e["iters"] > 0 for s in e["starts"])
        assert got == want, f"direction {d}: window starts differ from the reference's skips"


@pytest.mark.parametrize("chunk", [1, 4, 8])
def test_stream_blocks_and_retained_frames(chunk):
    """TrackStream on the recorded clip: push and finish blocks continue one another and cover frames 0..T-1 once;
    frames before a query's t are NaN and all later frames finite; at most 7 frames' feature maps are retained after
    any push; the result is the forward half of track_queries (visibilities to 4 ulps, as above)."""
    from pips_b200.chain import track_queries
    from pips_b200.stream import TrackStream
    m = _OracleModel()
    T, N = m.rgbs.shape[1], m.queries.shape[1]
    want_t, want_v = track_queries(m, m.rgbs, m.queries, iters=m.c["iters"])
    m.log.clear()
    s = TrackStream(m, m.queries, iters=m.c["iters"])
    blocks = []
    for ch in _chunks(m.rgbs, chunk):
        blocks.append(s.push(ch))
        assert s._held.shape[1] <= S - 1
    blocks.append(s.finish())
    assert s._held is None
    nxt = 0
    for f0, tr, v in blocks:
        assert f0 == nxt and tr.shape == (tr.shape[0], N, 2) and v.shape == (tr.shape[0], N)
        assert tr.device.type == "cpu" and v.device.type == "cpu"
        nxt += tr.shape[0]
    assert nxt == T
    trajs = torch.cat([b[1] for b in blocks])
    vis = torch.cat([b[2] for b in blocks])
    before = torch.arange(T).view(T, 1) < torch.tensor(QUERY_TIMES).view(1, N)
    assert bool(trajs[before].isnan().all()) and bool(vis[before].isnan().all())
    assert bool(torch.isfinite(trajs[~before]).all()) and bool(torch.isfinite(vis[~before]).all())
    assert torch.equal(_bits(trajs[~before]), _bits(want_t[0][~before]))
    assert _ulps(vis[~before], want_v[0][~before]) <= 4
    assert max(e["frames"] for e in m.log) <= chunk + S - 1


@pytest.mark.parametrize("case", ["queries_1d", "queries_xy_only", "queries_batch_2", "no_queries", "t_fractional",
                                  "t_negative", "t_nan", "t_inf", "x_nan", "y_inf"])
def test_stream_rejects_bad_queries(case):
    from pips_b200.stream import TrackStream
    q = torch.tensor([[0.0, 3.0, 4.0], [4.0, 1.0, 2.0]])
    if case == "queries_1d":
        q = q[0]
    elif case == "queries_xy_only":
        q = q[:, 1:]
    elif case == "queries_batch_2":
        q = q.unsqueeze(0).repeat(2, 1, 1)
    elif case == "no_queries":
        q = q[:0]
    elif case == "t_fractional":
        q[1, 0] = 2.5
    elif case == "t_negative":
        q[1, 0] = -1.0
    elif case == "t_nan":
        q[0, 0] = float("nan")
    elif case == "t_inf":
        q[0, 0] = float("inf")
    elif case == "x_nan":
        q[1, 1] = float("nan")
    elif case == "y_inf":
        q[0, 2] = float("inf")
    with pytest.raises(ValueError):
        TrackStream(_OracleModel(), q)


@pytest.mark.parametrize("case", ["chunk_3d", "chunk_not_rgb", "chunk_batch_2", "empty_chunk", "size_changes",
                                  "push_after_finish", "finish_twice", "query_never_arrives", "no_frames"])
def test_stream_rejects_bad_chunks_and_calls(case):
    from pips_b200.stream import TrackStream
    m = _OracleModel()
    s = TrackStream(m, m.queries[:, :2], iters=1)       # queries at frames 0 and 1
    frames = m.rgbs[0, :2]
    if case == "no_frames":
        with pytest.raises(ValueError):
            s.finish()
        return
    if case == "query_never_arrives":                   # the query at frame 1 needs two frames
        s.push(frames[:1])
        with pytest.raises(ValueError):
            s.finish()
        return
    s.push(frames)
    if case in ("push_after_finish", "finish_twice"):
        s.finish()
        with pytest.raises(ValueError):
            s.push(frames) if case == "push_after_finish" else s.finish()
        return
    bad = {"chunk_3d": frames[0], "chunk_not_rgb": frames[:, :1], "chunk_batch_2": torch.stack([frames, frames]),
           "empty_chunk": frames[:0], "size_changes": frames[..., :-4]}[case]
    with pytest.raises(ValueError):
        s.push(bad)


def test_stream_rejects_sharded_models():
    from pips_b200.stream import TrackStream

    class Model:
        _shard = (0, 2, None)

    with pytest.raises(RuntimeError):
        TrackStream(Model(), torch.tensor([[0.0, 3.0, 4.0]]))


def test_backward_pass_must_deliver_the_forward_pass_frames():
    """track_queries_stream: a backward pass with fewer or more frames than the forward pass, or other frame sizes,
    is a ValueError."""
    from pips_b200.stream import track_queries_stream
    m = _OracleModel()
    fwd = _chunks(m.rgbs, 8)
    bwd = _chunks(m.rgbs, 8, reverse=True)
    for wrong in (bwd[:-1], bwd + [bwd[0][:1]], [b[..., :-4] for b in bwd]):
        with pytest.raises(ValueError):
            track_queries_stream(m, fwd, wrong, m.queries, iters=1)


# ------------------------------------------------------------------------------------------------ GPU

def _model(precision, feat="fp32"):
    from pips_b200 import Pips
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    model = Pips(S=8, stride=8, precision=precision, feat_dtype=feat).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    return model


def _clip_and_queries(T=40, N=64, H=128, W=160, seed=41):
    """A T-frame clip and N queries at random frames, among them frames 0 and T-1 and both sides of the chunk
    boundaries of chunk sizes 7, 8 and 32."""
    rgbs = po.smooth_video(1, T, H, W, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    t = torch.randint(0, T, (N,), generator=g)
    fixed = torch.tensor([0, T - 1, 6, 7, 8, 13, 14, 15, 16, 31, 32, 33, T - 8, T - 7])
    fixed = fixed[fixed < T]
    t[:fixed.numel()] = fixed
    q = torch.cat([t.float().view(1, N, 1), po.random_queries(1, N, H, W, seed=seed + 2)], dim=2)
    return rgbs, q


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["fp32", "bf16"])
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_stream_equals_track_queries_bit_for_bit(precision, feat):
    from pips_b200.chain import track_queries
    from pips_b200.stream import track_queries_stream
    model = _model(precision, feat)
    rgbs, q = _clip_and_queries()
    rgbs = rgbs.to(DEV)
    want_t, want_v = track_queries(model, rgbs, q.to(DEV), iters=6)
    assert bool(torch.isfinite(want_t).all())
    for chunk in (1, 7, 8, 32):
        trajs, vis = track_queries_stream(model, _chunks(rgbs, chunk), _chunks(rgbs, chunk, reverse=True), q, iters=6)
        assert torch.equal(_bits(trajs), _bits(want_t)), f"chunk {chunk}: trajectories differ"
        assert torch.equal(_bits(vis), _bits(want_v)), f"chunk {chunk}: visibilities differ"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_stream_from_frame_zero_equals_track_chain(precision):
    from pips_b200.chain import track_chain
    from pips_b200.stream import TrackStream
    model = _model(precision)
    rgbs, q = _clip_and_queries(T=37, N=48)
    rgbs = rgbs.to(DEV)
    xy0 = q[:, :, 1:3]
    want = track_chain(model, rgbs, xy0.to(DEV), iters=6)[0]
    q[:, :, 0] = 0
    s = TrackStream(model, q, iters=6)
    blocks = [s.push(ch) for ch in _chunks(rgbs, 5)] + [s.finish()]
    trajs = torch.cat([b[1] for b in blocks])
    assert torch.equal(_bits(trajs), _bits(want))


@pytest.mark.gpu
def test_uint8_host_chunks_equal_float_device_chunks():
    from pips_b200.stream import track_queries_stream
    model = _model("bf16x3")
    rgbs, q = _clip_and_queries(T=24, N=32)
    u8 = rgbs.round().clamp(0, 255).to(torch.uint8)
    f32 = u8.float().to(DEV)
    want = track_queries_stream(model, _chunks(f32, 8), _chunks(f32, 8, reverse=True), q, iters=6)
    got = track_queries_stream(model, _chunks(u8, 8), _chunks(u8, 8, reverse=True), q, iters=6)
    for a, b in zip(got, want):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.gpu
def test_stream_memory_does_not_grow_with_the_video():
    """Peak device memory above the model's baseline: 32 and 160 frames streamed in chunks of 8 agree within 2 MiB,
    and stay below what track_queries holds for the 160-frame clip."""
    from pips_b200.chain import track_queries
    from pips_b200.stream import track_queries_stream
    model = _model("bf16x3")
    H, W, N = 128, 160, 64

    def frames(T, reverse=False):
        for i in range(0, T, 8):
            idx = torch.arange(i, min(T, i + 8), device=DEV)
            idx = T - 1 - idx if reverse else idx
            yield 127.5 + 120 * torch.sin(idx.view(-1, 1, 1, 1) * 0.1 + torch.arange(3, device=DEV).view(1, 3, 1, 1)
                                           + torch.linspace(0, 6, H * W, device=DEV).view(1, 1, H, W))

    def queries(T):
        g = torch.Generator().manual_seed(T)
        return torch.cat([torch.randint(0, T, (N, 1), generator=g).float(), po.random_queries(1, N, H, W, seed=T)[0]], 1)

    def peak(fn):
        fn()                                                            # warm-up: encoder plans, workspaces
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        return (torch.cuda.max_memory_allocated() - base) / 2 ** 20

    p = {T: peak(lambda: track_queries_stream(model, frames(T), frames(T, True), queries(T))) for T in (32, 160)}
    clip = torch.cat(list(frames(160))).unsqueeze(0)
    whole = peak(lambda: track_queries(model, clip, queries(160).unsqueeze(0).to(DEV)))
    print(f"stream peak: 32 frames {p[32]:.2f} MiB, 160 frames {p[160]:.2f} MiB; track_queries 160 frames {whole:.2f} MiB")
    assert abs(p[160] - p[32]) <= 2.0
    assert p[160] < whole
