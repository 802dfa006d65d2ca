"""Batched visibility-aware chaining over long videos (SURVEY.md section 8f-1).

The reference tracks a long clip one particle at a time (chain_demo.py:40-83, identical logic in
test_on_badja.py:65-113): run the 8-frame model from the particle's current frame, keep the window's
estimate, jump to the latest frame of the window (index 2..7) whose visibility passes a threshold that
is lowered by 0.02 per sweep, repeat -- re-running fnet on every window of every particle.

Here all particles advance together: fnet runs ONCE per frame (exact: InstanceNorm is per frame,
nets/pips.py:412), the pyramid of the whole clip stays resident, and each round is one refinement call
in which every track reads its own window through a per-track frame offset (``frame_base`` of
pips_corr_gather); the threshold sweep is evaluated for all tracks at once.  Results are the same as
the per-particle loop up to fp32 noise.

``track_chain`` tracks points given at frame 0, forward in time, as the reference does.  ``track_queries`` takes
(t, x, y) queries at any frame and tracks each both ways: the reference chain on the clip from frame t on, and the
same chain on the time-reversed clip from frame t back to frame 0.  A backward track reads its windows through a
negative frame offset (``~t``), so both directions share the pyramid and the rounds.  ``track_queries_batch`` does the
same for many clips at once: their frames share one pyramid, and every track also carries its clip's place in it.
``track_queries_mixed`` takes clips of any frame sizes: one pyramid per size, and every track also names its pyramid.
"""
from __future__ import annotations

from typing import Optional

import torch

S_WIN = 8
# Distinct frame sizes one refinement call of track_queries_mixed reads (PIPS_MAX_GROUPS of the C library): a batch
# with more sizes runs as successive sub-batches of at most this many.
MAX_GROUPS = 32


def _threshold_table(n: int = 64) -> torch.Tensor:
    """thr = 0.9; thr -= 0.02 ... exactly as the Python loop accumulates it (chain_demo.py:64,75)."""
    vals, thr = [], 0.9
    for _ in range(n):
        vals.append(thr)
        thr -= 0.02
    return torch.tensor(vals, dtype=torch.float32)


def pick_skip(vis: torch.Tensor, thr_table: torch.Tensor) -> torch.Tensor:
    """vis (8, n) sigmoid visibilities -> (n,) frame index in [2, 7] chosen by chain_demo.py:63-76:
    scan si = 7..2 for vis > thr, lowering thr by 0.02 whenever the scan reaches si == 1."""
    cand = vis[2:S_WIN].unsqueeze(0) > thr_table.view(-1, 1, 1).to(vis.device)          # (K, 6, n)
    level_ok = cand.any(dim=1)                                                           # (K, n)
    if not bool(level_ok[-1].all()):
        raise RuntimeError("chain: visibility below every threshold (non-finite visibilities?)")
    k_star = level_ok.float().argmax(dim=0)                                              # first passing level
    sel = cand[k_star, :, torch.arange(vis.shape[1], device=vis.device)]                 # (n, 6)
    idx = torch.arange(2, S_WIN, device=vis.device).view(1, -1)
    return (sel.long() * idx).max(dim=1).values


def _encode_clip(model, rgbs: torch.Tensor, held: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The clip's feature maps (1, T, 128, H8, W8), encoded once per frame in chunks of 32 frames; after the ``held``
    feature maps (1, k, 128, H8, W8) of earlier frames when given."""
    T = rgbs.shape[1]
    parts = [] if held is None else [held]
    fmaps = torch.cat(parts + [model.encode(rgbs[:, t0:t0 + 32]) for t0 in range(0, T, 32)], dim=1)
    if not fmaps.is_contiguous() and not fmaps.reshape(-1, *fmaps.shape[2:]).permute(0, 2, 3, 1).is_contiguous():
        fmaps = fmaps.contiguous()
    return fmaps


class _Tracks:
    """Per-track state of the round loop.  Track k runs the reference chain from xy[k] (input pixels) over the
    length[k] frames of its direction.  Its first window is read through frame_base base0[k], counted in frames of the
    video: t for a forward track from frame t, ~t for a backward one (see window_frame in csrc/corr_common.cuh).  A
    window that starts c frames further on is base0[k] + c in both directions (~(t - c) == ~t + c).  Step s of the
    window at cursor c writes row row0[k] + c + s of traj (rows, n, 2) and vis (rows, n); vis holds sigmoid(vis_e) of
    the window that last wrote the row, and is None unless ``want_vis``.  ``clip`` (n, 2) int32 (optional): track k's
    clip {first, count} among the held frames when they hold several videos; base0[k] then counts inside that clip
    (clip_window_frame in csrc/corr_common.cuh).  With feature maps in groups (track_queries_mixed) ``clip`` is (n, 3)
    {first, count, group}: the clip among the frames of pyramid group ``group``."""

    def __init__(self, base0: torch.Tensor, length: torch.Tensor, xy: torch.Tensor, rows: int, want_vis: bool,
                 fill: float = 0.0, clip: Optional[torch.Tensor] = None):
        n = base0.numel()
        dev = base0.device
        self.base0, self.length, self.clip = base0, length, clip
        self.row0 = torch.zeros(n, dtype=torch.long, device=dev)
        self.pos = xy.float().clone()                                                # start of each track's next window
        self.cur = torch.zeros(n, dtype=torch.long, device=dev)
        self.started = torch.zeros(n, dtype=torch.bool, device=dev)
        self.done = torch.zeros(n, dtype=torch.bool, device=dev)
        self.feat: Optional[torch.Tensor] = None                                     # (n, 128) first-window features
        self.traj = torch.full((rows, n, 2), fill, dtype=torch.float32, device=dev)
        self.vis = torch.full((rows, n), fill, dtype=torch.float32, device=dev) if want_vis else None
        self.rounds = 0


def _run_rounds(model, fmaps: torch.Tensor, tr: _Tracks, iters: int, advance: Optional[int] = None, f0=0,
                ended=True, frames: Optional[torch.Tensor] = None) -> None:
    """The round loop shared by track_chain, track_queries, TrackStream and MultiStream.  fmaps (1, F, 128, H8, W8)
    holds frames f0 .. f0+F-1 of the video.  Every round is one refinement call over all runnable tracks, each reading
    its window through its frame_base rebased to the held frames; rounds repeat until no track is runnable.  A track is
    runnable while it is inside its clip and, unless the video has ``ended``, its whole window has arrived.  A window
    past the last held frame replicates that frame, which is the end-of-clip rule once the video has ended.  A track's
    first window gathers its own feature; later windows carry it (outs[3], chain_demo.py:57).  With a per-track clip
    (tr.clip) the refinement calls pass the runnable tracks' rows of it as ``clip``; without one they pass no clip.
    ``fmaps`` may also be a list of such tensors of different map sizes, one per pyramid group, with a 3-column
    tr.clip.  Tracks of several streamed videos take the per-track form: ``f0`` (n,) the video frame of the first held
    frame of each track's video (its clip's frame 0), ``frames`` (n,) the frames that video has delivered and
    ``ended`` (n,) bool; the scalars stand for every track, with frames = f0 + F."""
    grouped = isinstance(fmaps, (list, tuple))
    if frames is None and not grouped:
        frames = f0 + fmaps.shape[1]
    dev = (fmaps[0] if grouped else fmaps).device
    eng = model.engine
    stride = float(model.stride)
    thr = _threshold_table().to(dev)
    steps = torch.arange(S_WIN, device=dev).view(S_WIN, 1)
    built = False                                                                    # the pyramid of fmaps exists
    while True:
        live = ~tr.done
        if not isinstance(ended, bool):
            live &= ended | (tr.base0 + tr.cur + (S_WIN - 1) <= frames - 1)
        elif not ended:
            live &= tr.base0 + tr.cur + (S_WIN - 1) <= frames - 1
        run = live.nonzero().flatten()
        na = run.numel()
        if na == 0:
            return
        c = tr.cur[run]
        fb = (tr.base0[run] + c - (f0[run] if isinstance(f0, torch.Tensor) else f0)).view(1, na).to(torch.int32)
        coords = (tr.pos[run] / stride).view(1, 1, na, 2).repeat(1, S_WIN, 1, 1)    # zero-velocity init, :453
        new = ~tr.started[run]
        cl = None if tr.clip is None else tr.clip[run].view(1, na, tr.clip.shape[1])
        fi = None
        if not bool(new.all()):
            if bool(new.any()):
                # tracks starting beside carried ones: their first-window features alone (initial gather, no iteration)
                kw = {} if cl is None else {"clip": cl[:, new]}
                _, _, f_new = eng.refine(model, fmaps, coords[:, :, new], None, 0, stride, frame_base=fb[:, new],
                                         reuse_pyramid=built, **kw)
                built = True
                tr.feat[run[new]] = f_new[0]
                tr.started[run[new]] = True
            fi = tr.feat[run].unsqueeze(0)
        kw = {} if cl is None else {"clip": cl}
        preds, vis_e, ffeat = eng.refine(model, fmaps, coords, fi, iters, stride, frame_base=fb, reuse_pyramid=built, **kw)
        built = True
        if fi is None:
            if tr.feat is None:
                tr.feat = torch.empty(tr.base0.numel(), ffeat.shape[-1], dtype=ffeat.dtype, device=dev)
            tr.feat[run] = ffeat[0]
            tr.started[run] = True
        xys = preds[-1][0]                                                           # (8, na, 2)
        lim = tr.length[run]
        t_idx = c.view(1, na) + steps                                                # (8, na)
        ok = t_idx < lim.view(1, na)                                                 # S_local truncation, :61
        rows, cols = (tr.row0[run].view(1, na) + t_idx)[ok], run.view(1, na).expand(S_WIN, na)[ok]
        tr.traj[rows, cols] = xys[ok]
        v = torch.sigmoid(vis_e[0]) if tr.vis is not None or advance is None else None
        if tr.vis is not None:
            tr.vis[rows, cols] = v[ok]
        si = pick_skip(v, thr) if advance is None else torch.full_like(c, int(advance))
        nxt = c + si
        tr.cur[run] = nxt
        tr.pos[run] = xys[si, torch.arange(na, device=dev)]
        tr.done[run] = nxt >= lim
        tr.rounds += 1


def check_window(model, who: str = "pips_b200.chain") -> None:
    """Chained tracking moves 8-frame windows along the clip (chain_demo.py:52, test_on_badja.py:81): models of
    another window length are refused before any work."""
    S = getattr(model, "S", S_WIN)
    if S != S_WIN:
        raise ValueError(f"{who}: chained tracking needs a model of S={S_WIN} frames per window; this model has S={S}")


@torch.no_grad()
def track_chain(model, rgbs: torch.Tensor, xy0: torch.Tensor, iters: int = 6, return_rounds: bool = False,
                advance: Optional[int] = None):
    """rgbs (1, T, 3, H, W) float 0..255, xy0 (1, N, 2) start positions at frame 0 (input pixels).
    Returns trajs_e (1, T, N, 2).  Equivalent to chain_demo.py:run_model's per-particle loop.
    ``advance`` (2..7): every track moves on by that many frames per round instead of the visibility-driven
    choice -- a data-independent schedule (ceil((T-1)/advance) rounds) for throughput measurements (SURVEY.md 8d)."""
    check_window(model)
    if advance is not None and not 2 <= int(advance) <= S_WIN - 1:
        raise ValueError("advance must be in 2..7 (the reference's sweep never picks another frame, chain_demo.py:63-76)")
    B, T, C, H, W = rgbs.shape
    assert B == 1, "chained tracking follows the reference: one clip at a time"
    N = xy0.shape[1]
    dev = rgbs.device
    fmaps = _encode_clip(model, rgbs)
    tr = _Tracks(torch.zeros(N, dtype=torch.long, device=dev), torch.full((N,), T, dtype=torch.long, device=dev),
                 xy0[0], T, want_vis=False)
    _run_rounds(model, fmaps, tr, iters, advance)
    out = tr.traj.unsqueeze(0)
    return (out, tr.rounds) if return_rounds else out


def _check_queries(rgbs: torch.Tensor, queries: torch.Tensor) -> torch.Tensor:
    """Validates track_queries' inputs; returns the query frames (N,) as int64 on rgbs' device."""
    if not isinstance(rgbs, torch.Tensor) or rgbs.dim() != 5 or rgbs.shape[2] != 3:
        raise ValueError(f"rgbs must be (1, T, 3, H, W), got {tuple(getattr(rgbs, 'shape', ()))}")
    if rgbs.shape[0] != 1:
        raise ValueError(f"track_queries tracks one clip at a time (B == 1), got B = {rgbs.shape[0]}")
    T = rgbs.shape[1]
    if T < 1:
        raise ValueError("rgbs holds no frames")
    if not isinstance(queries, torch.Tensor) or queries.dim() != 3 or queries.shape[2] != 3:
        raise ValueError(f"queries must be (1, N, 3) as (t, x, y), got {tuple(getattr(queries, 'shape', ()))}")
    if queries.shape[0] != 1:
        raise ValueError(f"queries must have batch size 1 like rgbs, got {queries.shape[0]}")
    if queries.shape[1] < 1:
        raise ValueError("queries holds no query")
    q = queries[0].to(device=rgbs.device, dtype=torch.float64)
    t = q[:, 0]
    if not bool((t == torch.round(t)).all()):
        raise ValueError("query frames t must be integral")
    if not bool(((t >= 0) & (t <= T - 1)).all()):
        raise ValueError(f"query frames t must lie in 0..{T - 1}")
    if not bool(torch.isfinite(q[:, 1:]).all()):
        raise ValueError("query positions x, y must be finite")
    return t.long()


@torch.no_grad()
def track_queries(model, rgbs: torch.Tensor, queries: torch.Tensor, iters: int = 6, return_rounds: bool = False):
    """Tracks queries given at any frame, forward and backward in time (the TAP-Vid query format).

    rgbs (1, T, 3, H, W) float 0..255; queries (1, N, 3) as (t, x, y): an integral frame index t in 0..T-1 and a
    position in input pixels.  Returns trajs (1, T, N, 2) and vis (1, T, N) (and the round count when
    ``return_rounds``).  Frames t..T-1 of query n are the reference chain (chain_demo.py:40-83) run on rgbs[:, t:]
    from (x, y); frames 0..t-1 are the same chain run on the time-reversed clip (frames t, t-1, ..., 0), read back in
    forward order.  vis is sigmoid(vis_e) of the window that last wrote the frame.

    The clip is encoded once.  Every query is a forward track, and a backward track when t > 0; all tracks advance
    together, one refinement call per round, each reading its own window of the resident pyramid."""
    check_window(model)
    t = _check_queries(rgbs, queries)
    T = rgbs.shape[1]
    dev = rgbs.device
    xy = queries[0, :, 1:3].to(device=dev, dtype=torch.float32)
    back = (t > 0).nonzero().flatten()                                               # queries with a backward track
    tb = t[back]
    fmaps = _encode_clip(model, rgbs)
    tr = _Tracks(torch.cat([t, ~tb]), torch.cat([T - t, tb + 1]), torch.cat([xy, xy[back]]), T, want_vis=True)
    _run_rounds(model, fmaps, tr, iters)
    out = _merge_directions(tr, t, back, T, 0)
    return out + (tr.rounds,) if return_rounds else out


def _merge_directions(tr: _Tracks, t: torch.Tensor, back: torch.Tensor, T: int, c0: int):
    """trajs (1, T, N, 2) and vis (1, T, N) of N queries at frames t (N,) whose tracks are the columns c0 .. of tr:
    the N forward tracks, then the backward tracks of the queries ``back`` (those with t > 0).  Frame f of query n is
    step f - t of its forward track when f >= t, else step t - f of its backward track."""
    N = t.numel()
    dev = tr.traj.device
    f = torch.arange(T, device=dev).view(T, 1)
    bcol = torch.zeros(N, dtype=torch.long, device=dev)
    bcol[back] = c0 + N + torch.arange(back.numel(), device=dev)
    fwd = f >= t.view(1, N)
    step = torch.where(fwd, f - t.view(1, N), t.view(1, N) - f)                     # (T, N)
    col = torch.where(fwd, c0 + torch.arange(N, device=dev).view(1, N), bcol.view(1, N))
    return tr.traj[step, col].unsqueeze(0), tr.vis[step, col].unsqueeze(0)


def _batch_clip(rgbs, i: int) -> torch.Tensor:
    """Clip i of track_queries_batch, (T, 3, H, W) or (1, T, 3, H, W) -> a (T, 3, H, W) view with T >= 1."""
    if not isinstance(rgbs, torch.Tensor) or rgbs.dim() not in (4, 5) or rgbs.shape[-3] != 3 \
            or (rgbs.dim() == 5 and rgbs.shape[0] != 1):
        raise ValueError(f"clips[{i}] must be (T, 3, H, W) or (1, T, 3, H, W), got {tuple(getattr(rgbs, 'shape', ()))}")
    v = rgbs if rgbs.dim() == 4 else rgbs[0]
    if v.shape[0] < 1:
        raise ValueError(f"clips[{i}] holds no frames")
    return v


def _encode_batch(model, clips, chunk: int = 32, held=None, frames: Optional[int] = None) -> torch.Tensor:
    """The feature maps (1, F, 128, H8, W8) of all frames of ``clips`` ((T_i, 3, H, W) each) back to back, F = sum T_i.
    Frames are encoded once, ``chunk`` at a time across clip boundaries, so the encoder sees one full-chunk shape and one
    tail; each chunk goes to the model's device only when it is encoded.  The maps are written into one channels-last
    buffer as they come, so the batch's maps are never held twice.

    ``held`` (streaming): per clip, None or the feature maps (1, h_i, 128, H8, W8) of the frames before it, as
    ``_encode_clip(held=)`` takes them; the buffer then holds [held_0, clip_0, held_1, clip_1, ...], F = sum h_i + T_i,
    and T_i == 0 is allowed.  ``frames`` (>= F): the buffer's length, its last frames - F frames zero, so that a buffer
    whose contents vary keeps one shape."""
    dev = next(iter(model.parameters())).device
    nh = [0 if h is None else h.shape[1] for h in (held or [None] * len(clips))]
    ends = torch.tensor([c.shape[0] for c in clips]).cumsum(0).tolist()
    first = torch.tensor([0] + [h + c.shape[0] for h, c in zip(nh, clips)]).cumsum(0).tolist()  # clip i's held maps
    F = ends[-1]
    buf = None

    def alloc(h8, w8, dtype):
        return torch.empty(first[-1] if frames is None else frames, h8, w8, 128, dtype=dtype, device=dev)

    for t0 in range(0, F, chunk):
        t1 = min(F, t0 + chunk)
        parts, dst = [], []
        for i, (c, e) in enumerate(zip(clips, ends)):
            s = e - c.shape[0]                                                   # the clip holds frames s .. e-1
            if s < t1 and e > t0 and s < e:
                a = max(t0 - s, 0)
                parts.append(c[a:min(t1, e) - s].to(dev))
                dst.append(first[i] + nh[i] + a)
        f = model.encode(torch.cat(parts).unsqueeze(0))[0]                          # (k, 128, H8, W8)
        if buf is None:
            buf = alloc(f.shape[2], f.shape[3], f.dtype)
        k = 0
        for p, d in zip(parts, dst):
            buf[d:d + p.shape[0]].copy_(f[k:k + p.shape[0]].permute(0, 2, 3, 1))
            k += p.shape[0]
    for i, h in enumerate(held or []):
        if h is not None:
            if buf is None:
                buf = alloc(h.shape[3], h.shape[4], h.dtype)
            buf[first[i]:first[i] + nh[i]].copy_(h[0].permute(0, 2, 3, 1))
    if frames is not None:
        buf[first[-1]:].zero_()
    return buf.permute(0, 3, 1, 2).unsqueeze(0)


@torch.no_grad()
def track_queries_batch(model, clips, queries, iters: int = 6, return_rounds: bool = False):
    """``track_queries`` over many videos in one pass: every clip's tracks advance in the same rounds.

    ``clips`` is a sequence of videos, each (T_i, 3, H, W) or (1, T_i, 3, H, W), float 0..255 or uint8, on the host or
    the model's device (converted as ``Pips.encode`` converts them).  All share H x W; T_i may differ, T_i == 1 included.
    ``queries`` holds one (N_i, 3) or (1, N_i, 3) tensor of (t, x, y) per clip, t integral in 0..T_i-1.  Returns a list
    with one (trajs (1, T_i, N_i, 2), vis (1, T_i, N_i)) pair per clip -- the same bits as
    ``track_queries(model, clips[i][None], queries[i][None])`` -- and the number of rounds when ``return_rounds``.

    All frames are encoded once, in 32-frame chunks that run across clip boundaries, into one pyramid.  Every track
    reads its windows inside its own clip through a per-track clip table (pips_corr_gather_clips), so each round is one
    refinement call over the tracks of all clips, and the batch takes as many rounds as its longest clip's chain.  The
    device holds the feature maps and the pyramid of every frame of the batch, about 1.2 MiB per 256x256 frame at
    stride 8 with fp32 features: the caller bounds the batch."""
    views = _batch_views(model, clips, queries, "track_queries_batch")
    hw = tuple(views[0].shape[-2:])
    for i, v in enumerate(views):
        if tuple(v.shape[-2:]) != hw:
            raise ValueError(f"clips[{i}] frames are {tuple(v.shape[-2:])}, clips[0]'s are {hw}: one batch, one size")
    ts = _batch_query_frames(model, views, queries)
    fmaps = _encode_batch(model, views)
    first = torch.tensor([0] + [v.shape[0] for v in views]).cumsum(0).tolist()
    tr, cols = _batch_tracks(views, queries, ts, [[first[i], v.shape[0]] for i, v in enumerate(views)])
    _run_rounds(model, fmaps, tr, iters)
    outs = [_merge_directions(tr, t, back, v.shape[0], c0) for v, t, (c0, back) in zip(views, ts, cols)]
    return (outs, tr.rounds) if return_rounds else outs


def _batch_views(model, clips, queries, who: str):
    """The checks track_queries_batch and track_queries_mixed make before any work; returns the clips as
    (T_i, 3, H_i, W_i) views."""
    check_window(model)
    shard = getattr(model, "_shard", None)
    if shard is not None and shard[1] > 1:
        raise RuntimeError("pips_b200.chain: chained tracking does not cover particle-sharded models")
    if len(clips) != len(queries):
        raise ValueError(f"{len(clips)} clips but {len(queries)} query sets: one query set per clip")
    if len(clips) == 0:
        raise ValueError(f"empty batch: {who} needs at least one clip")
    return [_batch_clip(c, i) for i, c in enumerate(clips)]


def _batch_query_frames(model, views, queries):
    """Checks every clip's queries as track_queries does; returns each clip's query frames (N_i,) on the model's
    device."""
    dev = next(iter(model.parameters())).device
    ts = []
    for i, (v, q) in enumerate(zip(views, queries)):
        if isinstance(q, torch.Tensor) and q.dim() == 2:
            q = q.unsqueeze(0)
        try:
            ts.append(_check_queries(v.unsqueeze(0), q).to(dev))
        except ValueError as e:
            raise ValueError(f"queries[{i}]: {e}") from None
    return ts


def _batch_tracks(views, queries, ts, rows):
    """The _Tracks of a batch: each clip's forward tracks, then its backward tracks (queries with t > 0), clip after
    clip, every track of clip i carrying the clip table row rows[i].  Returns the tracks and, per clip, (its first
    column, its queries with a backward track) for _merge_directions."""
    dev = ts[0].device
    base0, length, xy, clip, cols = [], [], [], [], []
    c0 = 0
    for v, q, t, row in zip(views, queries, ts, rows):
        T, N = v.shape[0], t.numel()
        qxy = q.reshape(-1, 3)[:, 1:3].to(device=dev, dtype=torch.float32)
        back = (t > 0).nonzero().flatten()                                           # queries with a backward track
        tb = t[back]
        base0 += [t, ~tb]
        length += [T - t, tb + 1]
        xy += [qxy, qxy[back]]
        n = N + back.numel()
        clip.append(torch.tensor(row, dtype=torch.int32, device=dev).expand(n, len(row)))
        cols.append((c0, back))
        c0 += n
    tr = _Tracks(torch.cat(base0), torch.cat(length), torch.cat(xy), max(v.shape[0] for v in views), want_vis=True,
                 clip=torch.cat(clip).contiguous())
    return tr, cols


@torch.no_grad()
def track_queries_mixed(model, clips, queries, iters: int = 6, return_rounds: bool = False):
    """``track_queries_batch`` for clips of any frame sizes: every clip's tracks advance in the same rounds.

    ``clips`` and ``queries`` are as in track_queries_batch, except that each clip may have its own H x W; its feature
    map, (H // stride) x (W // stride), must be at least 8 x 8.  Returns a list with one (trajs (1, T_i, N_i, 2),
    vis (1, T_i, N_i)) pair per clip -- the same bits as ``track_queries(model, clips[i][None], queries[i][None])`` --
    and the number of rounds when ``return_rounds``.

    The clips are grouped by frame size.  Each group's frames are encoded once, in 32-frame chunks that run across its
    clips' boundaries, into that group's own pyramid.  Every track reads its windows inside its own clip of its own
    group's pyramid through a per-track table {first, count, group} (pips_corr_gather_groups), so each round is one
    refinement call over the tracks of all clips of all sizes, and the batch takes as many rounds as its longest clip's
    chain.  A batch with more than MAX_GROUPS sizes runs as successive sub-batches of at most MAX_GROUPS sizes, each
    with its own rounds.  The device holds the feature maps and the pyramids of every frame of a sub-batch: the caller
    bounds the batch."""
    views = _batch_views(model, clips, queries, "track_queries_mixed")
    stride = int(model.stride)
    for i, v in enumerate(views):
        h, w = v.shape[-2:]
        if h // stride < 8 or w // stride < 8:
            raise ValueError(f"clips[{i}] frames are {h}x{w}: the feature map at stride {stride} is "
                             f"{h // stride}x{w // stride}, under the 8x8 the 4-level pyramid needs")
    ts = _batch_query_frames(model, views, queries)
    sizes = list(dict.fromkeys(tuple(v.shape[-2:]) for v in views))                # in order of first appearance
    outs, rounds = [None] * len(views), 0
    for s0 in range(0, len(sizes), MAX_GROUPS):
        fmaps, order, rows = [], [], []
        for g, hw in enumerate(sizes[s0:s0 + MAX_GROUPS]):
            idx = [i for i, v in enumerate(views) if tuple(v.shape[-2:]) == hw]
            fmaps.append(_encode_batch(model, [views[i] for i in idx]))
            first = 0
            for i in idx:
                order.append(i)
                rows.append([first, views[i].shape[0], g])
                first += views[i].shape[0]
        tr, cols = _batch_tracks([views[i] for i in order], [queries[i] for i in order], [ts[i] for i in order], rows)
        _run_rounds(model, fmaps, tr, iters)
        for i, (c0, back) in zip(order, cols):
            outs[i] = _merge_directions(tr, ts[i], back, views[i].shape[0], c0)
        rounds += tr.rounds
        del fmaps, tr                                   # a sub-batch's maps go before the next one's are encoded
    return (outs, rounds) if return_rounds else outs
