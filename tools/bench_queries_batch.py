"""Queries in many videos at once: pips_b200.chain.track_queries_batch against a loop of track_queries over the clips.

    python tools/bench_queries_batch.py [--workload davis kinetics] [--reps 3] [--precision bf16x3]

Two seeded synthetic workloads at 256 x 256 (smooth synthetic video, stride 8, 6 iterations), the clips as uint8 on the
host, as a dataset loader hands them over:
  - davis: 30 clips of 34..104 frames, 20 queries each at random frames (DAVIS-like);
  - kinetics: 32 clips of 250 frames, 25 queries each at random frames (Kinetics-like).
Both paths give every query its trajectory and visibility over its whole clip:
  - track_queries_batch: all frames are encoded once in 32-frame chunks across clip boundaries, and the tracks of all
    clips advance in the same rounds, one refinement call per round;
  - loop: track_queries on each clip in turn (the clip moved to the device first), each with its own rounds.
Wall time is a host clock around each path ending in a device synchronise (median of --reps runs after one warm-up);
the peak is torch.cuda.max_memory_allocated above what was allocated before the path's first run, so it counts the
path's own pyramid.  The trajectories and visibilities of the two paths are compared; the difference must be 0.  The
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
from pips_b200.chain import track_queries, track_queries_batch  # noqa: E402

DEV = "cuda:0"
H = W = 256
WORKLOADS = {
    "davis": dict(clips=30, frames=(34, 104), queries=20, seed=31),
    "kinetics": dict(clips=32, frames=(250, 250), queries=25, seed=32),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def make_workload(w):
    """Host uint8 clips (T_i, 3, H, W) and (N_i, 3) queries (t, x, y) with t uniform in 0..T_i-1."""
    g = torch.Generator().manual_seed(w["seed"])
    clips, queries = [], []
    for i in range(w["clips"]):
        lo, hi = w["frames"]
        T = int(torch.randint(lo, hi + 1, (1,), generator=g))
        shift = (1, 1) if i % 2 == 0 else (-1, 1)                 # one pixel per frame keeps generation cheap
        clips.append(po.smooth_video(1, T, H, W, seed=w["seed"] * 1000 + i, shift=shift)[0].to(torch.uint8))
        n = w["queries"]
        t = torch.randint(0, T, (n, 1), generator=g).float()
        queries.append(torch.cat([t, po.random_queries(1, n, H, W, seed=w["seed"] * 1000 + 500 + i)[0]], dim=1))
    return clips, queries


def loop(model, clips, queries, iters):
    outs, rounds = [], 0
    for v, q in zip(clips, queries):
        trajs, vis, r = track_queries(model, v.to(DEV).unsqueeze(0), q.to(DEV).unsqueeze(0), iters=iters,
                                      return_rounds=True)
        outs.append((trajs, vis))
        rounds += r
    return outs, rounds


def measure(model, fn, reps):
    """(last output, median seconds, peak MiB): the peak counts everything the path allocates, its pyramid included."""
    model.engine._pyr = None                                  # the previous path's cached pyramid
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_queries_batch: needs a CUDA device")
    sd = po.init_state_dict(seed=21, head_scale=0.05)
    model = Pips(S=8, stride=8, precision=a.precision).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    name = card()
    print(f"card: {name}")
    records = []
    for wl in a.workload:
        clips, queries = make_workload(WORKLOADS[wl])
        frames = sum(v.shape[0] for v in clips)
        nq = sum(q.shape[0] for q in queries)
        (outs, r_batch), t_batch, m_batch = measure(
            model, lambda: track_queries_batch(model, clips, queries, iters=a.iters, return_rounds=True), a.reps)
        (want, r_loop), t_loop, m_loop = measure(model, lambda: loop(model, clips, queries, a.iters), a.reps)
        dt = max((x[0] - y[0]).abs().max().item() for x, y in zip(outs, want))
        dv = max((x[1] - y[1]).abs().max().item() for x, y in zip(outs, want))
        print(f"{wl}: {len(clips)} clips, {frames} frames of {H}x{W}, {nq} queries, stride 8, {a.iters} iterations, "
              f"{a.precision}")
        print(f"  track_queries_batch: {t_batch * 1e3:.1f} ms, {r_batch} rounds, peak {m_batch:.0f} MiB")
        print(f"  track_queries loop:  {t_loop * 1e3:.1f} ms, {r_loop} rounds, peak {m_loop:.0f} MiB")
        print(f"  speed-up {t_loop / t_batch:.2f}x; max |trajs difference| {dt:.3g} px, max |vis difference| {dv:.3g}")
        records.append(dict(workload=wl, clips=len(clips), frames=frames, queries=nq, batch_ms=round(t_batch * 1e3, 1),
                            batch_rounds=r_batch, batch_peak_mib=round(m_batch), loop_ms=round(t_loop * 1e3, 1),
                            loop_rounds=r_loop, loop_peak_mib=round(m_loop), max_traj_diff_px=dt, max_vis_diff=dv))
        del outs, want
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=name, H=H, W=W, iters=a.iters, precision=a.precision, workloads=records)))


if __name__ == "__main__":
    main()
