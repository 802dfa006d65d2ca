"""Queries in videos of different frame sizes: pips_b200.chain.track_queries_mixed against one track_queries_batch per
frame size and against a loop of track_queries over the clips.

    python tools/bench_queries_mixed.py [--reps 3] [--precision bf16x3]

One seeded synthetic DAVIS-like workload: 30 clips of 34..104 frames, 20 queries each at random frames, every clip at a
frame size drawn from SIZES (square, landscape and portrait, as a dataset of user footage has them), stride 8,
6 iterations, the clips as uint8 on the host, as a dataset loader hands them over.  All three paths give every query
its trajectory and visibility over its whole clip:
  - track_queries_mixed: each size's frames are encoded once into that size's pyramid, and the tracks of all clips of
    all sizes advance in the same rounds, one refinement call per round;
  - per size: track_queries_batch on the clips of each size in turn, each batch with its own rounds;
  - loop: track_queries on each clip in turn (the clip moved to the device first), each with its own rounds.
Wall time is a host clock around each path ending in a device synchronise (median of --reps runs after one warm-up);
the peak is torch.cuda.max_memory_allocated above what was allocated before the path's first run, so it counts the
path's own pyramids.  The trajectories and visibilities of the three paths are compared; the differences must be 0.  The
card's name, power limit and maximum SM clock are read in the same run.  The last line is one JSON record of the numbers."""
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
from pips_b200.chain import track_queries, track_queries_batch, track_queries_mixed  # noqa: E402

DEV = "cuda:0"
SIZES = [(256, 256), (240, 320), (320, 240), (288, 512), (360, 640), (200, 360)]
WORKLOAD = dict(clips=30, frames=(34, 104), queries=20, seed=41)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def make_workload(w):
    """Host uint8 clips (T_i, 3, H_i, W_i) and (N_i, 3) queries (t, x, y) with t uniform in 0..T_i-1."""
    g = torch.Generator().manual_seed(w["seed"])
    clips, queries = [], []
    for i in range(w["clips"]):
        lo, hi = w["frames"]
        T = int(torch.randint(lo, hi + 1, (1,), generator=g))
        H, W = SIZES[int(torch.randint(0, len(SIZES), (1,), generator=g))]
        shift = (1, 1) if i % 2 == 0 else (-1, 1)                 # one pixel per frame keeps generation cheap
        clips.append(po.smooth_video(1, T, H, W, seed=w["seed"] * 1000 + i, shift=shift)[0].to(torch.uint8))
        n = w["queries"]
        t = torch.randint(0, T, (n, 1), generator=g).float()
        queries.append(torch.cat([t, po.random_queries(1, n, H, W, seed=w["seed"] * 1000 + 500 + i)[0]], dim=1))
    return clips, queries


def per_size(model, clips, queries, iters):
    outs, rounds = [None] * len(clips), 0
    for hw in dict.fromkeys(tuple(v.shape[-2:]) for v in clips):
        idx = [i for i, v in enumerate(clips) if tuple(v.shape[-2:]) == hw]
        o, r = track_queries_batch(model, [clips[i] for i in idx], [queries[i] for i in idx], iters=iters,
                                   return_rounds=True)
        for i, x in zip(idx, o):
            outs[i] = x
        rounds += r
    return outs, rounds


def loop(model, clips, queries, iters):
    outs, rounds = [], 0
    for v, q in zip(clips, queries):
        trajs, vis, r = track_queries(model, v.to(DEV).unsqueeze(0), q.to(DEV).unsqueeze(0), iters=iters,
                                      return_rounds=True)
        outs.append((trajs, vis))
        rounds += r
    return outs, rounds


def measure(model, fn, reps):
    """(last output, median seconds, peak MiB): the peak counts everything the path allocates, its pyramids included."""
    model.engine._pyr = None                                  # the previous path's cached pyramids
    model.engine._gpyr = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()                                                      # warm-up: module loads, encoder plans, workspaces
    ts, out = [], None
    for _ in range(reps):
        out = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, statistics.median(ts), (torch.cuda.max_memory_allocated() - base) / 2**20


def diff(outs, want):
    return (max((x[0] - y[0]).abs().max().item() for x, y in zip(outs, want)),
            max((x[1] - y[1]).abs().max().item() for x, y in zip(outs, want)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_queries_mixed: needs a CUDA device")
    sd = po.init_state_dict(seed=21, head_scale=0.05)
    model = Pips(S=8, stride=8, precision=a.precision).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    name = card()
    print(f"card: {name}")
    clips, queries = make_workload(WORKLOAD)
    frames = sum(v.shape[0] for v in clips)
    nq = sum(q.shape[0] for q in queries)
    sizes = len({tuple(v.shape[-2:]) for v in clips})
    (outs, r_mix), t_mix, m_mix = measure(
        model, lambda: track_queries_mixed(model, clips, queries, iters=a.iters, return_rounds=True), a.reps)
    (by_size, r_size), t_size, m_size = measure(model, lambda: per_size(model, clips, queries, a.iters), a.reps)
    (want, r_loop), t_loop, m_loop = measure(model, lambda: loop(model, clips, queries, a.iters), a.reps)
    dt_s, dv_s = diff(outs, by_size)
    dt_l, dv_l = diff(outs, want)
    print(f"{len(clips)} clips at {sizes} frame sizes, {frames} frames, {nq} queries, stride 8, {a.iters} iterations, "
          f"{a.precision}")
    print(f"  track_queries_mixed:            {t_mix * 1e3:.1f} ms, {r_mix} rounds, peak {m_mix:.0f} MiB")
    print(f"  track_queries_batch per size:   {t_size * 1e3:.1f} ms, {r_size} rounds, peak {m_size:.0f} MiB")
    print(f"  track_queries loop:             {t_loop * 1e3:.1f} ms, {r_loop} rounds, peak {m_loop:.0f} MiB")
    print(f"  speed-up {t_size / t_mix:.2f}x over per-size batches, {t_loop / t_mix:.2f}x over the loop; "
          f"max |trajs difference| {max(dt_s, dt_l):.3g} px, max |vis difference| {max(dv_s, dv_l):.3g}")
    print(json.dumps(dict(card=name, sizes=SIZES, clips=len(clips), frames=frames, queries=nq, iters=a.iters,
                          precision=a.precision, mixed_ms=round(t_mix * 1e3, 1), mixed_rounds=r_mix,
                          mixed_peak_mib=round(m_mix), per_size_ms=round(t_size * 1e3, 1), per_size_rounds=r_size,
                          per_size_peak_mib=round(m_size), loop_ms=round(t_loop * 1e3, 1), loop_rounds=r_loop,
                          loop_peak_mib=round(m_loop), max_traj_diff_px=max(dt_s, dt_l),
                          max_vis_diff=max(dv_s, dv_l))))


if __name__ == "__main__":
    main()
