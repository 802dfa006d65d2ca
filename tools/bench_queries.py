"""Queries at any frame of a long clip: pips_b200.chain.track_queries against what tracking them takes without it.

    python tools/bench_queries.py [--T 48] [--N 1024] [--reps 3] [--precision bf16x3]

Workload: one clip of T = 48 frames of 384 x 512 (smooth synthetic video, stride 8, 6 iterations), N = 1024 queries
(t, x, y) with t uniform in 0..T-1.  Both paths give every query its trajectory and visibility over the whole clip:
  - track_queries: the clip is encoded once; every query is a forward track, and a backward track when t > 0, and all
    tracks advance together, one refinement call per round.
  - per-frame slices: for every distinct t, track_chain on rgbs[:, t:] for the queries at t, and track_chain on the
    time-reversed rgbs[:, t::-1] when t > 0 -- each call encodes its slice again and runs its own rounds.
Wall time is a host clock around each path ending in a device synchronise (median of --reps runs after one warm-up);
the peak is torch.cuda.max_memory_allocated above what the clip itself holds.  The card's name, power limit and
maximum SM clock are read in the same run.  The last line is one JSON record of the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pips_oracle as po  # noqa: E402
from pips_b200 import Pips  # noqa: E402
from pips_b200.chain import track_chain, track_queries  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def per_slice(model, rgbs, queries, iters):
    """Every distinct query frame t: track_chain forward on the slice from t, and on the reversed slice to frame 0."""
    T = rgbs.shape[1]
    N = queries.shape[1]
    trajs = torch.zeros(1, T, N, 2, device=DEV)
    t_all = queries[0, :, 0].long()
    rounds = calls = frames = 0
    for t in torch.unique(t_all).tolist():
        idx = (t_all == t).nonzero().flatten()
        xy = queries[:, idx, 1:3]
        fwd, r = track_chain(model, rgbs[:, t:], xy, iters=iters, return_rounds=True)
        trajs[:, t:, idx] = fwd
        rounds, calls, frames = rounds + r, calls + 1, frames + T - t
        if t > 0:
            bwd, r = track_chain(model, rgbs[:, :t + 1].flip(1), xy, iters=iters, return_rounds=True)
            trajs[:, :t, idx] = bwd[:, 1:].flip(1)
            rounds, calls, frames = rounds + r, calls + 1, frames + t + 1
    return trajs, dict(rounds=rounds, chain_calls=calls, frames_encoded=frames)


def measure(fn, reps):
    fn()                                                      # warm-up: module loads, encoder plans, workspaces
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ts, out = [], None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, statistics.median(ts), (torch.cuda.max_memory_allocated() - base) / 2**20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=48)
    ap.add_argument("--N", type=int, default=1024)
    ap.add_argument("--H", type=int, default=384)
    ap.add_argument("--W", type=int, default=512)
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_queries: needs a CUDA device")
    sd = po.init_state_dict(seed=21, head_scale=0.05)
    model = Pips(S=8, stride=8, precision=a.precision).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    rgbs = po.smooth_video(1, a.T, a.H, a.W, seed=22).to(DEV)
    g = torch.Generator().manual_seed(23)
    t = torch.randint(0, a.T, (1, a.N, 1), generator=g).float()
    queries = torch.cat([t, po.random_queries(1, a.N, a.H, a.W, seed=24)], dim=2).to(DEV)
    name = card()

    (trajs, vis, rounds), t_new, m_new = measure(
        lambda: track_queries(model, rgbs, queries, iters=a.iters, return_rounds=True), a.reps)
    (trajs_old, stats), t_old, m_old = measure(lambda: per_slice(model, rgbs, queries, a.iters), a.reps)
    diff = (trajs - trajs_old).abs().max().item()
    distinct = int(torch.unique(queries[0, :, 0]).numel())
    print(f"card: {name}")
    print(f"workload: T={a.T} frames of {a.H}x{a.W}, N={a.N} queries at {distinct} distinct frames, stride 8, "
          f"{a.iters} iterations, {a.precision}")
    print(f"track_queries: {t_new * 1e3:.1f} ms, {rounds} rounds, {a.T} frames encoded, peak {m_new:.0f} MiB")
    print(f"per-frame slices: {t_old * 1e3:.1f} ms, {stats['rounds']} rounds in {stats['chain_calls']} track_chain calls, "
          f"{stats['frames_encoded']} frames encoded, peak {m_old:.0f} MiB")
    print(f"speed-up {t_old / t_new:.1f}x; max |trajs difference| {diff:.3g} px")
    print(json.dumps(dict(card=name, T=a.T, N=a.N, H=a.H, W=a.W, iters=a.iters, precision=a.precision,
                          distinct_t=distinct, queries_ms=round(t_new * 1e3, 2), queries_rounds=rounds,
                          queries_peak_mib=round(m_new), slices_ms=round(t_old * 1e3, 2), slices_rounds=stats["rounds"],
                          slices_calls=stats["chain_calls"], slices_frames_encoded=stats["frames_encoded"],
                          slices_peak_mib=round(m_old), max_traj_diff_px=diff)))


if __name__ == "__main__":
    main()
