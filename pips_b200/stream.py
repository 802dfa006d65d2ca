"""Tracking videos of any length in bounded device memory: frames streamed through the chained tracker in chunks.

``track_chain`` and ``track_queries`` (chain.py) hold the whole clip's feature maps and their pyramid on the device, so
their memory grows with the clip.  A chained track only ever reads the 8-frame window at its cursor, and once every
track's cursor is past a frame nothing reads that frame again.  ``TrackStream`` therefore encodes each chunk of frames
as it arrives, runs every track whose window has arrived (the round loop of chain.py over the held frames), and keeps
only the last 7 frames' feature maps for the next chunk: device memory depends on the chunk size, not on the length
of the video.  Trajectories go to the host as their frames become final.  Results are the same bits as
``track_queries`` on the whole clip: a frame is encoded alone, a track's outputs do not depend on the other tracks in
its call, and a window reads the same frames whatever buffer holds them.
"""
from __future__ import annotations

from typing import Iterable, Tuple

import torch

from .chain import S_WIN, _encode_clip, _run_rounds, _Tracks

# a track's length while the video has not ended: a runnable track's window has arrived, so nothing is truncated
_OPEN = 2 ** 62


def _as_queries(queries) -> torch.Tensor:
    """(N, 3) or (1, N, 3) queries (t, x, y) -> (N, 3) float64 on the host, validated."""
    if not isinstance(queries, torch.Tensor) or queries.dim() not in (2, 3) or queries.shape[-1] != 3 \
            or (queries.dim() == 3 and queries.shape[0] != 1):
        raise ValueError(f"queries must be (N, 3) or (1, N, 3) as (t, x, y), got {tuple(getattr(queries, 'shape', ()))}")
    q = queries.reshape(-1, 3).detach().to(device="cpu", dtype=torch.float64)
    if q.shape[0] < 1:
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
    chunk, and per-track state; it does not grow with the length of the video."""

    def __init__(self, model, queries, iters: int = 6):
        shard = getattr(model, "_shard", None)
        if shard is not None and shard[1] > 1:
            raise RuntimeError("pips_b200.stream: chained tracking does not cover particle-sharded models")
        q = _as_queries(queries)
        self.model, self.iters = model, iters
        self.device = next(iter(model.parameters())).device
        self.t = q[:, 0].long()
        base0 = self.t.to(self.device)
        self._tr = _Tracks(base0, torch.full_like(base0, _OPEN), q[:, 1:3].to(device=self.device, dtype=torch.float32),
                           0, want_vis=True, fill=float("nan"))
        self._tr.row0 = base0.clone()                # rows of traj / vis are frames p0, p0 + 1, ...
        self._p0 = 0                                 # first frame not yet returned
        self._frames = 0                             # frames received
        self._held = None                            # feature maps of the last <= 7 frames received
        self._hw = None
        self._finished = False

    @property
    def frames(self) -> int:
        """The number of frames pushed so far."""
        return self._frames

    @property
    def rounds(self) -> int:
        """The number of batched rounds run so far."""
        return self._tr.rounds

    @torch.no_grad()
    def push(self, chunk) -> Tuple[int, torch.Tensor, torch.Tensor]:
        if self._finished:
            raise ValueError("push after finish(): the stream has ended")
        clip = _as_clip(chunk)
        if self._hw is None:
            self._hw = tuple(clip.shape[-2:])
        elif tuple(clip.shape[-2:]) != self._hw:
            raise ValueError(f"chunk frames are {tuple(clip.shape[-2:])}, the stream's are {self._hw}")
        held = self._held
        f0 = self._frames - (0 if held is None else held.shape[1])
        self._held = None
        fmaps = _encode_clip(self.model, clip.to(self.device), held)                # frames f0 .. f0 + F - 1
        self._frames += clip.shape[1]
        return self._advance(fmaps, f0, ended=False)

    @torch.no_grad()
    def finish(self) -> Tuple[int, torch.Tensor, torch.Tensor]:
        if self._finished:
            raise ValueError("finish() called twice: the stream has ended")
        T = self._frames
        late = self.t > T - 1
        if bool(late.any()):
            raise ValueError(f"query frame {int(self.t[late][0])} never arrived: the video ended after {T} frames")
        self._finished = True
        self._tr.length = T - self._tr.base0
        fmaps, self._held = self._held, None
        return self._advance(fmaps, T - fmaps.shape[1], ended=True)

    def _advance(self, fmaps: torch.Tensor, f0: int, ended: bool) -> Tuple[int, torch.Tensor, torch.Tensor]:
        tr = self._tr
        grow = self._frames - self._p0 - tr.traj.shape[0]
        if grow > 0:
            n = tr.base0.numel()
            tr.traj = torch.cat([tr.traj, tr.traj.new_full((grow, n, 2), float("nan"))])
            tr.vis = torch.cat([tr.vis, tr.vis.new_full((grow, n), float("nan"))])
        _run_rounds(self.model, fmaps, tr, self.iters, f0=f0, ended=ended)
        if ended:
            last = self._frames
        else:
            # every track, started or not, still writes from frame base0 + cur on; after the rounds that is
            # at frame F - 6 or later, so the last 7 frames' feature maps are all the next chunk needs
            last = min(self._frames, int((tr.base0 + tr.cur).min()))
            self._held = fmaps[:, -(S_WIN - 1):].clone()
        k = last - self._p0
        out = (self._p0, tr.traj[:k].cpu(), tr.vis[:k].cpu())
        tr.traj, tr.vis = tr.traj[k:], tr.vis[k:]
        tr.row0 -= k
        self._p0 = last
        return out


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
