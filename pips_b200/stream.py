"""Tracking videos of any length in bounded device memory: frames streamed through the chained tracker in chunks.

``track_chain`` and ``track_queries`` (chain.py) hold the whole clip's feature maps and their pyramid on the device, so
their memory grows with the clip.  A chained track only ever reads the 8-frame window at its cursor, and once every
track's cursor is past a frame nothing reads that frame again.  ``TrackStream`` therefore encodes each chunk of frames
as it arrives, runs every track whose window has arrived (the round loop of chain.py over the held frames), and keeps
only the last 7 frames' feature maps for the next chunk: device memory depends on the chunk size, not on the length
of the video.  Trajectories go to the host as their frames become final.  Results are the same bits as
``track_queries`` on the whole clip: a frame is encoded alone, a track's outputs do not depend on the other tracks in
its call, and a window reads the same frames whatever buffer holds them.

``MultiStream`` does the same for many videos at once, each arriving at its own pace and at its own frame size, with
queries added while a video runs: in every tick the new frames of all videos are encoded once and the tracks of all of
them share the rounds, through the grouped mode of the window kernels (one pyramid per frame size, every track reading
its own video's held and new frames).  A ``TrackStream`` is its one-video case.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Tuple

import torch

from . import chain
from .chain import S_WIN, _encode_batch, _run_rounds, _Tracks

# a track's length while the video has not ended: a runnable track's window has arrived, so nothing is truncated
_OPEN = 2 ** 62
_FIELDS = ("base0", "length", "row0", "pos", "cur", "started", "done")          # _Tracks' per-track tensors


def _as_queries(queries, allow_empty: bool = False) -> torch.Tensor:
    """(N, 3) or (1, N, 3) queries (t, x, y) -> (N, 3) float64 on the host, validated."""
    if not isinstance(queries, torch.Tensor) or queries.dim() not in (2, 3) or queries.shape[-1] != 3 \
            or (queries.dim() == 3 and queries.shape[0] != 1):
        raise ValueError(f"queries must be (N, 3) or (1, N, 3) as (t, x, y), got {tuple(getattr(queries, 'shape', ()))}")
    q = queries.reshape(-1, 3).detach().to(device="cpu", dtype=torch.float64)
    if q.shape[0] < 1 and not allow_empty:
        raise ValueError("queries holds no query")
    t = q[:, 0]
    if not bool((torch.isfinite(t) & (t == torch.round(t))).all()):
        raise ValueError("query frames t must be integral")
    if not bool((t >= 0).all()):
        raise ValueError("query frames t must not be negative")
    if not bool(torch.isfinite(q[:, 1:]).all()):
        raise ValueError("query positions x, y must be finite")
    return q


def _as_clip(chunk) -> torch.Tensor:
    """(k, 3, H, W) or (1, k, 3, H, W) frames -> a (1, k, 3, H, W) view, k >= 1."""
    if not isinstance(chunk, torch.Tensor) or chunk.dim() not in (4, 5) or chunk.shape[-3] != 3 \
            or (chunk.dim() == 5 and chunk.shape[0] != 1):
        raise ValueError(f"a chunk must be (k, 3, H, W) or (1, k, 3, H, W), got {tuple(getattr(chunk, 'shape', ()))}")
    clip = chunk if chunk.dim() == 5 else chunk.unsqueeze(0)
    if clip.shape[1] < 1:
        raise ValueError("empty chunk: a chunk holds at least one frame")
    return clip


def _check_model(model) -> None:
    from .chain import check_window
    check_window(model, "pips_b200.stream")
    shard = getattr(model, "_shard", None)
    if shard is not None and shard[1] > 1:
        raise RuntimeError("pips_b200.stream: chained tracking does not cover particle-sharded models")


class _Video:
    """One streamed video: its queries' tracks, its frames' bookkeeping and the feature maps it holds between ticks.
    Row r of tr.traj / tr.vis is frame p0 + r; frames p0 .. frames-1 have been received but not returned."""

    def __init__(self, q: torch.Tensor, device):
        self.t = q[:, 0].long()                      # query frames, on the host
        base0 = self.t.to(device)
        self.tr = _Tracks(base0, torch.full_like(base0, _OPEN), q[:, 1:3].to(device=device, dtype=torch.float32), 0,
                          want_vis=True, fill=float("nan"))
        self.tr.row0 = base0.clone()
        self.p0 = 0                                  # first frame not yet returned
        self.frames = 0                              # frames received
        self.f0 = 0                                  # during a tick: the frame of the first held map
        self.held: Optional[torch.Tensor] = None     # feature maps of the last <= 7 frames received
        self.hw: Optional[Tuple[int, int]] = None

    def add(self, q: torch.Tensor) -> None:
        """New queries (n, 3), t >= p0, as the next columns."""
        tr, n = self.tr, q.shape[0]
        dev = tr.base0.device
        base0 = q[:, 0].long().to(dev)
        self.t = torch.cat([self.t, q[:, 0].long()])
        tr.base0 = torch.cat([tr.base0, base0])
        tr.length = torch.cat([tr.length, torch.full_like(base0, _OPEN)])
        tr.row0 = torch.cat([tr.row0, base0 - self.p0])
        tr.pos = torch.cat([tr.pos, q[:, 1:3].to(device=dev, dtype=torch.float32)])
        tr.cur = torch.cat([tr.cur, torch.zeros_like(base0)])
        tr.started = torch.cat([tr.started, torch.zeros(n, dtype=torch.bool, device=dev)])
        tr.done = torch.cat([tr.done, torch.zeros(n, dtype=torch.bool, device=dev)])
        if tr.feat is not None:
            tr.feat = torch.cat([tr.feat, tr.feat.new_empty(n, tr.feat.shape[1])])
        tr.traj = torch.cat([tr.traj, tr.traj.new_full((tr.traj.shape[0], n, 2), float("nan"))], dim=1)
        tr.vis = torch.cat([tr.vis, tr.vis.new_full((tr.vis.shape[0], n), float("nan"))], dim=1)

    def begin(self, k: int, ended: bool) -> None:
        """Takes k new frames (and the end of the video when ``ended``) before the tick's rounds."""
        self.f0 = self.frames - (0 if self.held is None else self.held.shape[1])
        self.frames += k
        tr = self.tr
        grow = self.frames - self.p0 - tr.traj.shape[0]
        if grow > 0:
            n = tr.base0.numel()
            tr.traj = torch.cat([tr.traj, tr.traj.new_full((grow, n, 2), float("nan"))])
            tr.vis = torch.cat([tr.vis, tr.vis.new_full((grow, n), float("nan"))])
        if ended:
            tr.length = self.frames - tr.base0

    def settle(self, ended: bool) -> Tuple[int, torch.Tensor, torch.Tensor]:
        """After the tick's rounds: the frames that became final, (f0, trajs (k', N, 2), vis (k', N)) on the host."""
        tr = self.tr
        if ended or tr.base0.numel() == 0:
            last = self.frames
        else:
            # every track, started or not, still writes from frame base0 + cur on; after the rounds that is
            # at frame frames - 7 or later, so the last 7 frames' feature maps are all the next tick needs
            last = min(self.frames, int((tr.base0 + tr.cur).min()))
        k = last - self.p0
        out = (self.p0, tr.traj[:k].cpu(), tr.vis[:k].cpu())
        tr.traj, tr.vis = tr.traj[k:], tr.vis[k:]
        tr.row0 -= k
        self.p0 = last
        return out


def _join(trs: List[_Tracks], table: torch.Tensor) -> _Tracks:
    """The tracks of several videos as one _Tracks, video after video, with the (n, 3) group table ``table``."""
    tr = _Tracks.__new__(_Tracks)
    for f in _FIELDS:
        setattr(tr, f, torch.cat([getattr(t, f) for t in trs]))
    rows = max(t.traj.shape[0] for t in trs)
    tr.traj = torch.cat([torch.cat([t.traj, t.traj.new_full((rows - t.traj.shape[0],) + t.traj.shape[1:], float("nan"))])
                         for t in trs], dim=1)
    tr.vis = torch.cat([torch.cat([t.vis, t.vis.new_full((rows - t.vis.shape[0],) + t.vis.shape[1:], float("nan"))])
                        for t in trs], dim=1)
    feats = [t.feat for t in trs if t.feat is not None]
    tr.feat = None if not feats else torch.cat([t.feat if t.feat is not None else feats[0].new_empty(t.base0.numel(),
                                                                                                    feats[0].shape[1])
                                                for t in trs])
    tr.clip, tr.rounds = table, 0
    return tr


def _split(tr: _Tracks, trs: List[_Tracks]) -> None:
    """Hands the columns of a _join'ed _Tracks back to the videos' own."""
    c0 = 0
    for t in trs:
        c1 = c0 + t.base0.numel()
        for f in _FIELDS:
            setattr(t, f, getattr(tr, f)[c0:c1])
        t.traj, t.vis = tr.traj[:t.traj.shape[0], c0:c1], tr.vis[:t.vis.shape[0], c0:c1]
        t.feat = None if tr.feat is None else tr.feat[c0:c1]
        c0 = c1


def _round_loop(model, iters: int, vids: List[_Video], clips: List[torch.Tensor], ended: List[bool]) -> int:
    """Encodes the new frames ``clips`` ((k_v, 3, H_v, W_v), k_v >= 0) of videos of at most MAX_GROUPS sizes after their
    held maps, runs one round loop over all their tracks and leaves each video still open its last min(7, frames) maps.
    A lone video makes the plain calls (no clip table); several make grouped calls, one channels-last buffer per frame
    size laid out [held_v, new_v] per video, sized sum(7 + k_v) so that steady ticks keep one pyramid shape.  Returns
    the rounds run."""
    if len(vids) == 1:
        v = vids[0]
        fmaps = _encode_batch(model, clips, held=[v.held])                          # frames f0 .. f0 + F - 1
        v.held = None
        r0 = v.tr.rounds
        _run_rounds(model, fmaps, v.tr, iters, f0=v.f0, ended=ended[0])
        if not ended[0]:
            v.held = fmaps[:, -(S_WIN - 1):].clone()
        return v.tr.rounds - r0
    dev = vids[0].tr.base0.device
    fmaps, rows, order = [], [], []
    for g, hw in enumerate(dict.fromkeys(v.hw for v in vids)):
        mine = [i for i, v in enumerate(vids) if v.hw == hw]
        cap = sum(S_WIN - 1 + clips[i].shape[0] for i in mine)
        fmaps.append(_encode_batch(model, [clips[i] for i in mine], held=[vids[i].held for i in mine], frames=cap))
        first = 0
        for i in mine:
            vids[i].held = None
            count = vids[i].frames - vids[i].f0
            rows.append([first, count, g])
            order.append(i)
            first += count
    members = [vids[i] for i in order]
    n = torch.tensor([v.tr.base0.numel() for v in members], device=dev)
    table = torch.tensor(rows, dtype=torch.int32, device=dev).repeat_interleave(n, dim=0)
    f0 = torch.tensor([v.f0 for v in members], device=dev).repeat_interleave(n)
    frames = torch.tensor([v.frames for v in members], device=dev).repeat_interleave(n)
    end = torch.tensor([ended[i] for i in order], device=dev).repeat_interleave(n)
    tr = _join([v.tr for v in members], table)
    _run_rounds(model, fmaps, tr, iters, f0=f0, ended=end, frames=frames)
    _split(tr, [v.tr for v in members])
    for i, (first, count, g) in zip(order, rows):
        if not ended[i]:
            vids[i].held = fmaps[g][:, first + count - min(S_WIN - 1, count):first + count].clone()
    return tr.rounds


@torch.no_grad()
def _tick(model, iters: int, vids: List[_Video], clips: List[Optional[torch.Tensor]], ended: List[bool]):
    """One tick of streaming: video v takes the frames clips[v] ((k, 3, H, W) or None) and ends when ended[v]; every
    frame is encoded once and the tracks of all the videos run in shared rounds, in successive round loops of at most
    MAX_GROUPS frame sizes.  Returns (rounds run, one settle() block per video)."""
    for v, c, e in zip(vids, clips, ended):
        v.begin(0 if c is None else c.shape[0], e)
    work = [i for i, v in enumerate(vids) if v.frames > v.f0]                      # videos holding frames
    sizes = list(dict.fromkeys(vids[i].hw for i in work))
    rounds = 0
    for s0 in range(0, len(sizes), chain.MAX_GROUPS):
        part = [i for i in work if vids[i].hw in sizes[s0:s0 + chain.MAX_GROUPS]]
        new = [clips[i] if clips[i] is not None else torch.empty(0, 3, *vids[i].hw) for i in part]
        rounds += _round_loop(model, iters, [vids[i] for i in part], new, [ended[i] for i in part])
    return rounds, [v.settle(e) for v, e in zip(vids, ended)]


class TrackStream:
    """Tracks queries forward in time through a video that arrives in chunks of frames.

    ``queries`` (N, 3) or (1, N, 3) as (t, x, y): an integral frame index t >= 0 and a position in input pixels.  Each
    query is the reference chain (chain_demo.py:40-83) from frame t to the end of the video, with the rules of
    ``track_chain``: zero initial velocity, the track's own first-window feature carried, the threshold sweep of
    ``pick_skip``, a frame's visibility from the window that last wrote it.

    ``push(chunk)`` takes the next frames, (k, 3, H, W) or (1, k, 3, H, W), float 0..255 or uint8, on the host or the
    model's device, converted as ``Pips.encode`` converts them.  It returns ``(f0, trajs (k', N, 2), vis (k', N))`` on
    the host: the frames f0 .. f0+k'-1 that became final, k' >= 0, each block continuing the previous one.  A frame is
    final once every query at or before it has started and every started track's cursor has passed it.  Frames before
    a query's t are NaN in its column.  ``finish()`` ends the video, runs the remaining windows (clamped at the last
    frame, the reference's end-of-clip rule) and returns every frame still pending.  A query frame past the end of the
    video is a ValueError there.

    Device memory holds at most chunk + 7 frames' feature maps and their pyramid, the encoder's workspace for one
    chunk, and per-track state; it does not grow with the length of the video.  ``MultiStream`` is the same for many
    videos at once; a TrackStream is its one-video case."""

    def __init__(self, model, queries, iters: int = 6):
        _check_model(model)
        q = _as_queries(queries)
        self.model, self.iters = model, iters
        self.device = next(iter(model.parameters())).device
        self._v = _Video(q, self.device)
        self._rounds = 0
        self._finished = False

    @property
    def t(self) -> torch.Tensor:
        """The query frames (N,), on the host."""
        return self._v.t

    @property
    def frames(self) -> int:
        """The number of frames pushed so far."""
        return self._v.frames

    @property
    def rounds(self) -> int:
        """The number of batched rounds run so far."""
        return self._rounds

    @property
    def _hw(self):
        return self._v.hw

    @property
    def _held(self):
        return self._v.held

    @torch.no_grad()
    def push(self, chunk) -> Tuple[int, torch.Tensor, torch.Tensor]:
        if self._finished:
            raise ValueError("push after finish(): the stream has ended")
        clip = _as_clip(chunk)
        if self._v.hw is None:
            self._v.hw = tuple(clip.shape[-2:])
        elif tuple(clip.shape[-2:]) != self._v.hw:
            raise ValueError(f"chunk frames are {tuple(clip.shape[-2:])}, the stream's are {self._v.hw}")
        r, (out,) = _tick(self.model, self.iters, [self._v], [clip[0]], [False])
        self._rounds += r
        return out

    @torch.no_grad()
    def finish(self) -> Tuple[int, torch.Tensor, torch.Tensor]:
        if self._finished:
            raise ValueError("finish() called twice: the stream has ended")
        _check_end(self._v, 0)
        self._finished = True
        r, (out,) = _tick(self.model, self.iters, [self._v], [None], [True])
        self._rounds += r
        return out


def _check_end(v: _Video, k: int, who: str = "") -> None:
    """A video that ends after its next k frames: every query frame must have arrived."""
    T = v.frames + k
    late = v.t > T - 1
    if bool(late.any()):
        raise ValueError(f"{who}query frame {int(v.t[late][0])} never arrived: the video ended after {T} frames")


class MultiStream:
    """Tracks queries forward in time through any number of videos, each arriving in chunks at its own pace, the
    videos' frames of any sizes.  Per video the rules and results are TrackStream's; all videos share the rounds.

    ``open(queries)`` starts a video with (N, 3) or (1, N, 3) queries (t, x, y), validated as TrackStream validates
    them, N == 0 allowed, and returns its id (never reused).  ``add_queries(vid, queries)`` adds queries to an open
    video while it runs: each t at or after ``pending(vid)``, the video's first frame not yet returned; they take the
    video's next columns.  ``push(chunks, end=())`` is one tick: ``chunks`` maps video ids to their next frames,
    (k, 3, H, W) or (1, k, 3, H, W), float 0..255 or uint8, on the host or the model's device (converted as
    ``Pips.encode`` converts them), and ``end`` names videos that end in this tick, after their chunk if they have one.
    Every new frame is encoded once, frames of one size together in 32-frame chunks across videos, and then one round
    loop runs over the tracks of every video of the tick, of all sizes (successive loops beyond ``chain.MAX_GROUPS``
    sizes).  It returns {vid: (f0, trajs (k', N_v, 2), vis (k', N_v))} on the host for every video that got frames or
    ended: per video, the blocks TrackStream.push / finish return for the same chunks, bit for bit, with a query added
    live in the column it would have had in a TrackStream opened with all the video's queries.  An ended video's
    frames and tracks are released.

    Device memory: after a tick each open video holds at most 7 frames' feature maps; a tick holds at most
    sum(k_v + 7) frames' maps and their pyramids over the videos it touches, and the encoder's workspace.  Neither
    grows with the length of a video or the number of ticks."""

    def __init__(self, model, iters: int = 6):
        _check_model(model)
        self.model, self.iters = model, iters
        self.device = next(iter(model.parameters())).device
        self._videos: Dict[int, _Video] = {}
        self._next = 0
        self._rounds = 0

    @property
    def rounds(self) -> int:
        """The number of shared rounds run so far."""
        return self._rounds

    def _video(self, vid) -> _Video:
        v = self._videos.get(vid) if isinstance(vid, int) else None
        if v is None:
            state = "ended" if isinstance(vid, int) and 0 <= vid < self._next else "unknown"
            raise ValueError(f"video {vid!r} is {state}: not an open video of this stream")
        return v

    def open(self, queries) -> int:
        """Starts a video with its queries; returns its id."""
        v = _Video(_as_queries(queries, allow_empty=True), self.device)
        vid, self._next = self._next, self._next + 1
        self._videos[vid] = v
        return vid

    def add_queries(self, vid: int, queries) -> None:
        """Adds queries at frames at or after pending(vid) to an open video."""
        v = self._video(vid)
        q = _as_queries(queries, allow_empty=True)
        early = q[:, 0] < v.p0
        if bool(early.any()):
            raise ValueError(f"query frame {int(q[early][0, 0])} of video {vid} is before frame {v.p0}, its first frame "
                             f"not yet returned")
        if q.shape[0] > 0:
            v.add(q)

    def pending(self, vid: int) -> int:
        """The first frame of video ``vid`` not yet returned."""
        return self._video(vid).p0

    def frames(self, vid: int) -> int:
        """The number of frames video ``vid`` has received."""
        return self._video(vid).frames

    @torch.no_grad()
    def push(self, chunks, end: Iterable[int] = ()) -> Dict[int, Tuple[int, torch.Tensor, torch.Tensor]]:
        if not isinstance(chunks, dict):
            raise ValueError(f"chunks must be a dict of video id -> frames, got {type(chunks).__name__}")
        end = list(dict.fromkeys(end))
        stride = int(self.model.stride)
        clips, sizes = {}, {}
        for vid, chunk in chunks.items():
            v = self._video(vid)
            try:
                clip = _as_clip(chunk)[0]
            except ValueError as e:
                raise ValueError(f"video {vid}: {e}") from None
            hw = tuple(clip.shape[-2:])
            if v.hw is not None and hw != v.hw:
                raise ValueError(f"video {vid}: chunk frames are {hw}, the video's are {v.hw}")
            if hw[0] // stride < 8 or hw[1] // stride < 8:
                raise ValueError(f"video {vid}: frames are {hw[0]}x{hw[1]}: the feature map at stride {stride} is "
                                 f"{hw[0] // stride}x{hw[1] // stride}, under the 8x8 the 4-level pyramid needs")
            clips[vid], sizes[vid] = clip, hw
        for vid in end:
            _check_end(self._video(vid), 0 if vid not in clips else clips[vid].shape[0], f"video {vid}: ")
        ids = list(clips) + [vid for vid in end if vid not in clips]
        vids = [self._videos[vid] for vid in ids]
        for vid, v in zip(ids, vids):
            if v.hw is None and vid in sizes:
                v.hw = sizes[vid]
        ended = set(end)
        r, blocks = _tick(self.model, self.iters, vids, [clips.get(vid) for vid in ids], [vid in ended for vid in ids])
        self._rounds += r
        for vid in ended:
            del self._videos[vid]
        return dict(zip(ids, blocks))


@torch.no_grad()
def track_queries_stream(model, forward_chunks: Iterable, backward_chunks: Iterable, queries, iters: int = 6):
    """``track_queries`` over a video delivered in chunks, in bounded device memory: two passes of ``TrackStream``.

    ``forward_chunks`` yields frames 0 .. T-1 in order and ``backward_chunks`` the same frames T-1 .. 0, each chunked
    arbitrarily ((k, 3, H, W) or (1, k, 3, H, W), as ``TrackStream.push`` takes them).  ``queries`` (N, 3) or (1, N, 3)
    as (t, x, y), t in 0..T-1.  The first pass tracks every query forward from frame t; the second tracks the queries
    with t > 0 forward through the reversed video from frame T-1-t, which is the reference chain on the time-reversed
    clip.  ``backward_chunks`` is not read when every query is at frame 0.  Returns trajs (1, T, N, 2) and vis (1, T, N)
    on the host, merged as ``track_queries`` merges them: the same bits as ``track_queries`` on the whole clip."""
    q = _as_queries(queries)
    fwd = TrackStream(model, q, iters)
    blocks = [fwd.push(c) for c in forward_chunks]
    blocks.append(fwd.finish())
    trajs = torch.cat([b[1] for b in blocks])
    vis = torch.cat([b[2] for b in blocks])
    T = fwd.frames
    t = fwd.t
    back = (t > 0).nonzero().flatten()
    if back.numel() > 0:
        qb = q[back].clone()
        qb[:, 0] = T - 1 - qb[:, 0]
        bwd = TrackStream(model, qb, iters)
        blocks = []
        for c in backward_chunks:
            clip = _as_clip(c)
            if tuple(clip.shape[-2:]) != fwd._hw:
                raise ValueError(f"backward frames are {tuple(clip.shape[-2:])}, the forward pass's are {fwd._hw}")
            if bwd.frames + clip.shape[1] > T:
                raise ValueError(f"backward_chunks delivered more than the forward pass's {T} frames")
            blocks.append(bwd.push(clip))
        if bwd.frames != T:
            raise ValueError(f"backward_chunks delivered {bwd.frames} frames, the forward pass {T}")
        blocks.append(bwd.finish())
        # frame f of query n: its forward track when f >= t, else frame T-1-f of its backward track
        bt = torch.cat([b[1] for b in blocks]).flip(0)
        bv = torch.cat([b[2] for b in blocks]).flip(0)
        before = torch.arange(T).view(T, 1) < t[back].view(1, -1)
        trajs[:, back] = torch.where(before.unsqueeze(2), bt, trajs[:, back])
        vis[:, back] = torch.where(before, bv, vis[:, back])
    return trajs.unsqueeze(0), vis.unsqueeze(0)
