"""Many videos streamed at once (pips_b200.stream.MultiStream): live videos of any frame sizes share the rounds.

Per video, the concatenated blocks must be what a TrackStream on that video alone returns for the same chunks (with a
query added live in the column it has in a TrackStream opened with all the video's queries).  CPU: the host logic with
the oracle as encoder and tracker over uneven schedules -- chunk sizes 1, 3 and 8, ticks that skip videos, a video
opened late, videos ended early or in the same tick as another's push, a one-frame video -- the rounds of each tick,
the frames a refinement call holds and a video retains, live queries, the size cap, and every rejection.  GPU: bit
equality with per-video TrackStreams in every precision, uint8 host chunks, live queries, and a peak that does not grow
with the length of the videos."""
import pytest
import torch

from oracle import pips_oracle as po
from tests.golden.make_golden import CHAIN_CASE
from tests.test_queries_batch import _bits, _model
from tests.test_queries_mixed import _clip, _MixedOracleModel

DEV = "cuda:0"
S = 8


class _LoggingOracle(_MixedOracleModel):
    """_MixedOracleModel that also records the frames every refinement call holds, summed over its groups, and answers
    the calls of no iteration that gather the features of tracks starting beside carried ones."""

    def __init__(self):
        super().__init__()
        self.frames = []

    def _refine(self, fmaps, coords, feat_init, iters, stride, frame_base, clip):
        self.frames.append(sum(f.shape[1] for f in fmaps) if isinstance(fmaps, list) else fmaps.shape[1])
        preds, vis, ffeat = super()._refine(fmaps, coords, feat_init, max(iters, 1), stride, frame_base, clip)
        return preds[:iters], vis, ffeat


def _ulps(a, b):
    """Largest distance in units in the last place between two fp32 tensors with NaN in the same places."""
    assert torch.equal(a.isnan(), b.isnan())
    a, b = a[~a.isnan()], b[~b.isnan()]
    return int((_bits(a).long() - _bits(b).long()).abs().max()) if a.numel() else 0


def _drive(model, clips, queries, ticks, iters, adds=(), retained=None):
    """Runs ``ticks`` through one MultiStream and through one TrackStream per video.  A tick is ({video: k}, {videos
    that end}): the next k frames of each named video, then the end of the listed ones.  A video is opened before the
    first tick that names it; ``adds`` holds (tick, video, queries) added live before that tick, and the video's
    TrackStream is opened with all its queries in order of addition.  Returns per video the concatenated blocks of both
    (f0s, trajs, vis), and per tick (shared rounds, rounds of each video's TrackStream, most frames of a refinement call,
    sum(k_v + 7) over the tick's videos)."""
    from pips_b200.stream import MultiStream, TrackStream
    ms = MultiStream(model, iters=iters)
    allq = {v: torch.cat([queries[v]] + [q for _, w, q in adds if w == v]) for v in clips}
    ids, pos, lone = {}, {}, {}
    got = {v: [] for v in clips}
    want = {v: [] for v in clips}
    stats = []
    for i, (ks, end) in enumerate(ticks):
        for v in list(ks) + sorted(end):
            if v not in ids:
                ids[v], pos[v] = ms.open(queries[v]), 0
                lone[v] = TrackStream(model, allq[v], iters=iters)
        for j, v, q in adds:
            if j == i:
                ms.add_queries(ids[v], q)
        frames = {v: clips[v][pos[v]:pos[v] + k] for v, k in ks.items()}
        for v, k in ks.items():
            pos[v] += k
        log = getattr(model, "frames", None)
        n0 = 0 if log is None else len(log)
        r0 = ms.rounds
        out = ms.push({ids[v]: f for v, f in frames.items()}, end={ids[v] for v in end})
        most = 0 if log is None else max(log[n0:], default=0)
        assert set(out) == {ids[v] for v in set(ks) | set(end)}
        for v in set(ks) | set(end):
            got[v].append(out[ids[v]])
        lr = {}
        for v in set(ks) | set(end):
            r = lone[v].rounds
            if v in ks:
                want[v].append(lone[v].push(frames[v]))
            if v in end:
                want[v].append(lone[v].finish())
            lr[v] = lone[v].rounds - r
        bound = sum(ks.get(v, 0) + S - 1 for v in set(ks) | set(end))
        stats.append((ms.rounds - r0, lr, most, bound, bool(end)))
        if retained is not None:
            retained.append(max([0] + [x.held.shape[1] for x in ms._videos.values() if x.held is not None]))
    res = {}
    for v in clips:
        n = allq[v].shape[0]

        def cat(bl):     # blocks returned before a query was added lack its column: NaN there, frames before its t
            pad = [torch.full((b[1].shape[0], n - b[1].shape[1]), float("nan")) for b in bl]
            return (torch.cat([torch.cat([b[1], p.unsqueeze(2).expand(-1, -1, 2)], 1) for b, p in zip(bl, pad)]),
                    torch.cat([torch.cat([b[2], p], 1) for b, p in zip(bl, pad)]))
        nxt = 0
        for f0, tr, vi in got[v]:
            assert f0 == nxt and tr.device.type == "cpu" and vi.shape == tr.shape[:2]
            nxt += tr.shape[0]
        res[v] = (cat(got[v]), cat(want[v]))
    return res, stats


def _cpu_case():
    """Four videos at two sizes (stride 4: 8x10 and 10x8 feature maps): A 13 frames in chunks of 1, B 11 frames in
    chunks of 3 and ended two ticks after its last one while the others push, C 17 frames in chunks of 8 opened late
    and pushed every other tick, D a single frame ended in its first tick; A ends in the same tick as C's last push."""
    spec = {"A": (13, 32, 40, 3), "B": (11, 40, 32, 2), "C": (17, 32, 40, 3), "D": (1, 40, 32, 2)}
    clips, queries = {}, {}
    for i, (v, (T, H, W, n)) in enumerate(spec.items()):
        clips[v], queries[v] = _clip(T, H, W, 900 + 13 * i, n)
    ticks = []
    for i in range(13):
        ks = {"A": 1}
        if i < 4:
            ks["B"] = 3 if i < 3 else 2
        if i in (3, 5, 7):
            ks["C"] = 8 if i < 7 else 1
        if i == 2:
            ks["D"] = 1
        end = {"D"} if i == 2 else {"B"} if i == 5 else {"A", "C"} if i == 12 else set()
        ticks.append((ks, end))
    return clips, queries, ticks


def _check(res, stats, vis_ulps):
    for v, ((gt, gv), (wt, wv)) in res.items():
        assert gt.shape == wt.shape and gv.shape == wv.shape, f"video {v}: blocks cover other frames"
        assert torch.equal(_bits(gt), _bits(wt)), f"video {v}: trajectories differ from its TrackStream"
        assert _ulps(gv, wv) <= vis_ulps, f"video {v}: visibilities differ from its TrackStream"
    for shared, lone, most, bound, ends in stats:
        assert most <= bound
        # the tracks of every video run as in their own stream, so a tick takes its slowest video's rounds; a video
        # that ends in the tick of a push runs both loops of its stream in one here
        assert shared == max(lone.values(), default=0) if not ends else shared <= max(lone.values(), default=0)


def test_multistream_equals_per_video_track_streams_on_cpu():
    """Per video the blocks are its TrackStream's: trajectories bit for bit, visibilities within 4 ulps (the CPU
    sigmoid caveat of test_stream.py); every tick takes its slowest video's rounds; no refinement call holds more than
    sum(k_v + 7) frames of the tick's videos; no video retains more than 7 frames."""
    clips, queries, ticks = _cpu_case()
    m = _LoggingOracle()
    retained = []
    res, stats = _drive(m, clips, queries, ticks, iters=1, retained=retained)
    _check(res, stats, 4)
    assert max(retained) <= S - 1
    assert sum(s[0] for s in stats) < sum(sum(s[1].values()) for s in stats)     # the videos did share rounds
    for v, ((gt, _), _) in res.items():
        T = clips[v].shape[0]
        before = torch.arange(T).view(T, 1) < queries[v][:, 0].view(1, -1)
        assert gt.shape[0] == T and bool(gt[before].isnan().all()) and bool(torch.isfinite(gt[~before]).all())


def _pendings(model, clips, queries, ticks, at):
    """pending(v) before tick j for every (j, v) of ``at``, from a run of the schedule."""
    from pips_b200.stream import MultiStream
    ms, ids, pos, out = MultiStream(model, iters=1), {}, {}, {}
    for i, (ks, end) in enumerate(ticks):
        for v in list(ks) + sorted(end):
            if v not in ids:
                ids[v], pos[v] = ms.open(queries[v]), 0
        for j, v in at:
            if j == i:
                out[(j, v)] = ms.pending(ids[v])
        ms.push({ids[v]: clips[v][pos[v]:pos[v] + k] for v, k in ks.items()}, end={ids[v] for v in end})
        for v, k in ks.items():
            pos[v] += k
    return out


def _live_adds(model, clips, queries, ticks, at, offsets, seed):
    """Queries added before tick j to video v for every (j, v) of ``at``: one at pending(v) + o for each of
    ``offsets``, at most the video's last frame."""
    pend = _pendings(model, clips, queries, ticks, at)
    adds = []
    for k, (j, v) in enumerate(at):
        T, H, W = clips[v].shape[0], clips[v].shape[-2], clips[v].shape[-1]
        t = torch.tensor([min(pend[(j, v)] + o, T - 1) for o in offsets], dtype=torch.float32).view(-1, 1)
        adds.append((j, v, torch.cat([t, po.random_queries(1, len(offsets), H, W, seed=seed + k)[0]], dim=1)))
    return adds


def test_multistream_live_queries_on_cpu():
    """Queries added while the videos run -- at pending(vid) and later -- give the columns of a TrackStream opened with
    them from the start; a query before pending(vid) is a ValueError that names that frame."""
    from pips_b200.stream import MultiStream
    clips, queries, ticks = _cpu_case()
    m = _LoggingOracle()
    adds = _live_adds(m, clips, queries, ticks, [(4, "A"), (6, "C"), (3, "B"), (9, "A")], (0, 2), 1500)
    assert any(q[0, 0] > 0 for _, _, q in adds)
    res, stats = _drive(m, clips, queries, ticks, iters=1, adds=adds)
    _check(res, stats, 4)
    ms = MultiStream(m, iters=1)
    a = ms.open(queries["A"][:1])
    ms.push({a: clips["A"][:9]})
    p = ms.pending(a)
    assert 0 < p <= 9 and ms.frames(a) == 9
    with pytest.raises(ValueError, match=f"frame {p}"):
        ms.add_queries(a, torch.tensor([[p - 1.0, 3.0, 3.0]]))
    ms.add_queries(a, torch.tensor([[float(p), 3.0, 3.0]]))


def test_multistream_size_cap_runs_successive_loops_on_cpu(monkeypatch):
    """With MAX_GROUPS lowered to 2, a tick of three frame sizes runs as two round loops with unchanged results."""
    import pips_b200.chain as ch
    spec = {"A": (10, 32, 40), "B": (9, 40, 32), "C": (11, 36, 44)}
    clips, queries = {}, {}
    for i, (v, (T, H, W)) in enumerate(spec.items()):
        clips[v], queries[v] = _clip(T, H, W, 1300 + 7 * i, 2)
    ticks = [({"A": 5, "B": 5, "C": 5}, set()), ({"A": 5, "B": 4, "C": 6}, {"A", "B", "C"})]
    m = _LoggingOracle()
    want, _ = _drive(m, clips, queries, ticks, iters=1)
    assert max(row[2] for _, cl in m.calls if cl is not None for row in cl) == 2
    monkeypatch.setattr(ch, "MAX_GROUPS", 2)
    m2 = _LoggingOracle()
    got, stats = _drive(m2, clips, queries, ticks, iters=1)
    assert max(row[2] for _, cl in m2.calls if cl is not None for row in cl) == 1
    assert any(cl is None for _, cl in m2.calls)                     # the third size alone: the plain calls
    for v in clips:
        (a, av), _ = got[v]
        (b, bv), _ = want[v]
        assert torch.equal(_bits(a), _bits(b)) and _ulps(av, bv) <= 4
    assert sum(s[0] for s in stats) > 0


class _NoWork:
    """A model that must not be reached: every rejection comes before any encoding or refinement."""
    stride = 4
    engine = None

    def parameters(self):
        return iter([torch.zeros(1)])

    def encode(self, clip):
        raise AssertionError("encoded despite bad input")


@pytest.mark.parametrize("case", ["not_a_dict", "unknown_id", "unknown_end", "ended_id", "chunk_3d", "chunk_not_rgb",
                                  "chunk_batch_2", "empty_chunk", "size_changes", "map_under_8x8_high",
                                  "map_under_8x8_wide", "query_past_end", "bad_id_beside_good_chunk"])
def test_multistream_rejects_bad_pushes_before_any_work(case):
    from pips_b200.stream import MultiStream
    m = _LoggingOracle()
    ms = MultiStream(m, iters=1)
    a = ms.open(torch.tensor([[0.0, 3.0, 4.0]]))
    b = ms.open(torch.tensor([[5.0, 3.0, 4.0]]))
    frames = torch.zeros(4, 3, 32, 40)
    ms.push({a: frames[:2], b: frames[:2]})
    ended = ms.open(torch.zeros(0, 3))
    ms.push({}, end={ended})
    n_enc, n_calls = m.encoded, len(m.calls)
    bad = {"not_a_dict": ([a, frames], ()), "unknown_id": ({7: frames}, ()), "unknown_end": ({a: frames}, {9}),
           "ended_id": ({ended: frames}, ()), "chunk_3d": ({a: frames[0]}, ()), "chunk_not_rgb": ({a: frames[:, :1]}, ()),
           "chunk_batch_2": ({a: torch.stack([frames, frames])}, ()), "empty_chunk": ({a: frames[:0]}, ()),
           "size_changes": ({a: frames[..., :-4]}, ()), "query_past_end": ({a: frames[:2]}, {b}),
           "bad_id_beside_good_chunk": ({a: frames, "b": frames}, ())}
    if case.startswith("map_under"):
        c = ms.open(torch.tensor([[0.0, 3.0, 4.0]]))
        bad[case] = ({a: frames, c: torch.zeros(2, 3, 28, 64) if case.endswith("high") else torch.zeros(2, 3, 64, 28)},
                     ())
    chunks, end = bad[case]
    with pytest.raises(ValueError):
        ms.push(chunks, end=end)
    assert (m.encoded, len(m.calls)) == (n_enc, n_calls)
    assert ms.frames(a) == 2 and ms.frames(b) == 2


def test_multistream_rejects_bad_queries_ids_and_sharded_models():
    from pips_b200.stream import MultiStream
    ms = MultiStream(_NoWork())
    for q in (torch.tensor([0.0, 3.0, 4.0]), torch.tensor([[0.0, 3.0]]), torch.tensor([[2.5, 3.0, 4.0]]),
              torch.tensor([[-1.0, 3.0, 4.0]]), torch.tensor([[0.0, float("nan"), 4.0]]), torch.zeros(2, 1, 3)):
        with pytest.raises(ValueError):
            ms.open(q)
    a = ms.open(torch.zeros(0, 3))                                        # no queries yet
    b = ms.open(torch.tensor([[[1.0, 2.0, 3.0]]]))
    assert a != b and ms.pending(a) == 0 and ms.frames(b) == 0 and ms.rounds == 0
    ms.add_queries(a, torch.tensor([[3.0, 1.0, 1.0]]))
    with pytest.raises(ValueError):
        ms.add_queries(a, torch.tensor([[3.0, float("inf"), 1.0]]))
    for call in (lambda: ms.add_queries(5, torch.tensor([[3.0, 1.0, 1.0]])), lambda: ms.pending(5),
                 lambda: ms.frames(-1)):
        with pytest.raises(ValueError):
            call()
    assert ms.push({}) == {}                                              # an empty tick does nothing

    class Sharded:
        _shard = (0, 2, None)

    with pytest.raises(RuntimeError):
        MultiStream(Sharded())


def test_multistream_ended_video_is_released_and_its_id_not_reused():
    from pips_b200.stream import MultiStream
    m = _LoggingOracle()
    ms = MultiStream(m, iters=1)
    clip, q = _clip(9, 32, 40, 77, 2)
    a = ms.open(q)
    out = ms.push({a: clip}, end={a})
    f0, tr, vis = out[a]
    assert f0 == 0 and tr.shape == (9, 2, 2) and vis.shape == (9, 2)
    assert a not in ms._videos
    for call in (lambda: ms.push({a: clip}), lambda: ms.push({}, end={a}), lambda: ms.pending(a)):
        with pytest.raises(ValueError, match="ended"):
            call()
    assert ms.open(q) != a
    e = ms.open(torch.zeros(0, 3))                                        # no queries: empty blocks
    f0, tr, vis = ms.push({e: clip[:3]})[e]
    assert f0 == 0 and tr.shape == (3, 0, 2) and vis.shape == (3, 0)


# ------------------------------------------------------------------------------------------------ GPU

def _gpu_case():
    """Four videos at three sizes (stride 4): two 96x128, one 64x96, one 72x48 alone in its group; lengths 37, 23, 30
    and 9 frames, uneven chunks, a video opened late and videos ending at different ticks."""
    spec = {"A": (37, 96, 128, 24), "B": (23, 64, 96, 16), "C": (30, 96, 128, 20), "D": (9, 72, 48, 6)}
    clips, queries = {}, {}
    for i, (v, (T, H, W, n)) in enumerate(spec.items()):
        clips[v], queries[v] = _clip(T, H, W, 1700 + 17 * i, n)
    step = {"A": 5, "B": 3, "C": 8, "D": 2}
    pos = dict.fromkeys(spec, 0)
    ticks, i = [], 0
    while any(pos[v] < clips[v].shape[0] for v in spec):
        ks, end = {}, set()
        for v in spec:
            if (v == "C" and i < 2) or (v == "B" and i % 3 == 2):
                continue
            k = min(step[v] + (i % 2 if v == "A" else 0), clips[v].shape[0] - pos[v])
            if k > 0:
                ks[v] = k
                pos[v] += k
                if pos[v] == clips[v].shape[0] and v != "B":
                    end.add(v)
        if ks:
            ticks.append((ks, end))
        i += 1
    ticks.append(({}, {"B"}))
    return clips, queries, ticks


@pytest.mark.gpu
@pytest.mark.parametrize("precision,feat", [("bf16x3", "fp32"), ("bf16x3", "bf16"), ("fp32", "fp32")])
def test_multistream_equals_track_streams_bit_for_bit(precision, feat):
    model = _model(precision, feat)
    clips, queries, ticks = _gpu_case()
    dc = {v: c.to(DEV) for v, c in clips.items()}
    res, stats = _drive(model, dc, queries, ticks, iters=CHAIN_CASE["iters"])
    _check(res, stats, 0)
    shared = sum(s[0] for s in stats)
    print(f"multistream {precision}/{feat}: {shared} shared rounds, {sum(sum(s[1].values()) for s in stats)} in "
          f"per-video streams")


@pytest.mark.gpu
def test_multistream_uint8_host_chunks_and_live_queries():
    """uint8 host chunks give the bits of float device chunks; queries added live give a TrackStream's columns."""
    model = _model("bf16x3")
    clips, queries, ticks = _gpu_case()
    u8 = {v: c.round().clamp(0, 255).to(torch.uint8) for v, c in clips.items()}
    f32 = {v: c.float().to(DEV) for v, c in u8.items()}
    a, _ = _drive(model, u8, queries, ticks, iters=6)
    b, _ = _drive(model, f32, queries, ticks, iters=6)
    for v in clips:
        for x, y in zip(a[v][0], b[v][0]):
            assert torch.equal(_bits(x), _bits(y))
    adds = _live_adds(model, f32, queries, ticks, [(2, "A"), (4, "C"), (4, "B"), (6, "A")], (0, 0, 1, 3, 8), 2100)
    res, stats = _drive(model, f32, queries, ticks, iters=6, adds=adds)
    _check(res, stats, 0)


@pytest.mark.gpu
def test_multistream_memory_does_not_grow_with_the_videos():
    """Peak device memory above the model's baseline: the same schedule with every video 5x longer peaks within
    2 MiB of the short one."""
    from pips_b200.stream import MultiStream
    model = _model("bf16x3")
    sizes = [(96, 128), (96, 128), (64, 96), (72, 48)]
    N = 32

    def run(T):
        ms = MultiStream(model, iters=6)
        ids = []
        for i, (H, W) in enumerate(sizes):
            g = torch.Generator().manual_seed(T + i)
            q = torch.cat([torch.randint(0, T, (N, 1), generator=g).float(), po.random_queries(1, N, H, W, seed=T + i)[0]], 1)
            ids.append(ms.open(q))
        for t0 in range(0, T, 8):
            chunks = {}
            for vid, (H, W) in zip(ids, sizes):
                idx = torch.arange(t0, min(T, t0 + 8), device=DEV)
                chunks[vid] = 127.5 + 120 * torch.sin(idx.view(-1, 1, 1, 1) * 0.1 + vid
                                                      + torch.arange(3, device=DEV).view(1, 3, 1, 1)
                                                      + torch.linspace(0, 6, H * W, device=DEV).view(1, 1, H, W))
            ms.push(chunks, end=set(ids) if t0 + 8 >= T else ())

    def peak(T):
        run(T)                                                          # warm-up: encoder plans, workspaces, pyramids
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        run(T)
        torch.cuda.synchronize()
        return (torch.cuda.max_memory_allocated() - base) / 2 ** 20

    short, long = peak(32), peak(160)
    print(f"multistream peak: 32 frames per video {short:.2f} MiB, 160 frames {long:.2f} MiB")
    assert abs(long - short) <= 2.0
