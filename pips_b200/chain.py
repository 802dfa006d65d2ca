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
negative frame offset (``~t``), so both directions share the pyramid and the rounds.
"""
from __future__ import annotations

from typing import Optional

import torch

S_WIN = 8


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


def _encode_clip(model, rgbs: torch.Tensor) -> torch.Tensor:
    """The whole clip's feature maps (1, T, 128, H8, W8), encoded once per frame in chunks of 32 frames."""
    T = rgbs.shape[1]
    fmaps = torch.cat([model.encode(rgbs[:, t0:t0 + 32]) for t0 in range(0, T, 32)], dim=1)   # (1,T,128,H8,W8)
    if not fmaps.is_contiguous() and not fmaps.reshape(T, *fmaps.shape[2:]).permute(0, 2, 3, 1).is_contiguous():
        fmaps = fmaps.contiguous()
    return fmaps


def _run_rounds(model, fmaps: torch.Tensor, base0: torch.Tensor, length: torch.Tensor, xy: torch.Tensor, iters: int,
                advance: Optional[int] = None, want_vis: bool = False):
    """The round loop shared by track_chain and track_queries: track k runs the reference chain from xy[k] (input
    pixels) over the length[k] frames of its direction, its first window read through frame_base base0[k] (t for a
    forward track from frame t, ~t for a backward one, see window_frame in csrc/corr_common.cuh).  A window that
    starts c frames further on is base0[k] + c in both directions (~(t - c) == ~t + c).  Every round is one
    refinement call over all tracks still inside their clip.  Returns traj (T, n, 2) indexed by frames from the
    track's start, vis (T, n) likewise -- sigmoid(vis_e) of the window that last wrote the frame; None unless
    ``want_vis`` -- and the round count."""
    T = fmaps.shape[1]
    n = base0.numel()
    dev = fmaps.device
    eng = model.engine
    stride = float(model.stride)
    thr = _threshold_table().to(dev)
    traj = torch.zeros(T, n, 2, dtype=torch.float32, device=dev)
    traj[0] = xy.float()
    vis = torch.zeros(T, n, dtype=torch.float32, device=dev) if want_vis else None
    cur = torch.zeros(n, dtype=torch.long, device=dev)
    feat: Optional[torch.Tensor] = None
    active = torch.arange(n, device=dev)
    rounds = 0
    while active.numel() > 0:
        na = active.numel()
        c = cur[active]
        start = traj[c, active]                                                      # (na, 2) current position
        coords = (start / stride).view(1, 1, na, 2).repeat(1, S_WIN, 1, 1)           # zero-velocity init, :453
        fi = None if feat is None else feat[:, active]
        preds, vis_e, ffeat = eng.refine(model, fmaps, coords, fi, iters, stride,
                                         frame_base=(base0[active] + c).view(1, na).to(torch.int32),
                                         reuse_pyramid=rounds > 0)                  # same clip every round
        if feat is None:
            feat = ffeat                                                             # outs[3], carried (chain_demo.py:57)
        xys = preds[-1][0]                                                           # (8, na, 2)
        lim = length[active]
        t_idx = c.view(1, na) + torch.arange(S_WIN, device=dev).view(S_WIN, 1)       # (8, na)
        ok = t_idx < lim.view(1, na)                                                 # S_local truncation, :61
        t_ok, cols = t_idx[ok], active.view(1, na).expand(S_WIN, na)[ok]
        traj[t_ok, cols] = xys[ok]
        v = torch.sigmoid(vis_e[0]) if want_vis or advance is None else None
        if want_vis:
            vis[t_ok, cols] = v[ok]
        si = pick_skip(v, thr) if advance is None else torch.full_like(c, int(advance))
        nxt = c + si
        cur[active] = nxt
        active = active[nxt < lim]
        rounds += 1
    return traj, vis, rounds


@torch.no_grad()
def track_chain(model, rgbs: torch.Tensor, xy0: torch.Tensor, iters: int = 6, return_rounds: bool = False,
                advance: Optional[int] = None):
    """rgbs (1, T, 3, H, W) float 0..255, xy0 (1, N, 2) start positions at frame 0 (input pixels).
    Returns trajs_e (1, T, N, 2).  Equivalent to chain_demo.py:run_model's per-particle loop.
    ``advance`` (2..7): every track moves on by that many frames per round instead of the visibility-driven
    choice -- a data-independent schedule (ceil((T-1)/advance) rounds) for throughput measurements (SURVEY.md 8d)."""
    if advance is not None and not 2 <= int(advance) <= S_WIN - 1:
        raise ValueError("advance must be in 2..7 (the reference's sweep never picks another frame, chain_demo.py:63-76)")
    B, T, C, H, W = rgbs.shape
    assert B == 1, "chained tracking follows the reference: one clip at a time"
    N = xy0.shape[1]
    dev = rgbs.device
    fmaps = _encode_clip(model, rgbs)
    traj, _, rounds = _run_rounds(model, fmaps, torch.zeros(N, dtype=torch.long, device=dev),
                                  torch.full((N,), T, dtype=torch.long, device=dev), xy0[0], iters, advance)
    out = traj.unsqueeze(0)
    return (out, rounds) if return_rounds else out


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
    t = _check_queries(rgbs, queries)
    T = rgbs.shape[1]
    N = t.numel()
    dev = rgbs.device
    xy = queries[0, :, 1:3].to(device=dev, dtype=torch.float32)
    back = (t > 0).nonzero().flatten()                                               # queries with a backward track
    tb = t[back]
    fmaps = _encode_clip(model, rgbs)
    traj, vis, rounds = _run_rounds(model, fmaps, torch.cat([t, ~tb]), torch.cat([T - t, tb + 1]),
                                    torch.cat([xy, xy[back]]), iters, want_vis=True)
    # frame f of query n: step f - t of its forward track when f >= t, else step t - f of its backward track
    f = torch.arange(T, device=dev).view(T, 1)
    bcol = torch.zeros(N, dtype=torch.long, device=dev)
    bcol[back] = N + torch.arange(back.numel(), device=dev)
    fwd = f >= t.view(1, N)
    step = torch.where(fwd, f - t.view(1, N), t.view(1, N) - f)                     # (T, N)
    col = torch.where(fwd, torch.arange(N, device=dev).view(1, N), bcol.view(1, N))
    out = (traj[step, col].unsqueeze(0), vis[step, col].unsqueeze(0))
    return out + (rounds,) if return_rounds else out
