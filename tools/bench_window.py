"""Pips.forward at window lengths 8, 16 and 5 (the last shows the cost of padding 5 frames to 8).

    python tools/bench_window.py [--reps 10] [--out DIR]

384x512 frames, stride 8, 6 iterations, bf16x3, random seeded weights; B*S*N held at 8192 particle-frames, so each
window length refines the same number of (particle, frame) states per iteration.  Reports per S: the forward's time
(median over reps, CUDA events around calls that end in a device synchronise), particle-frame updates per second
(B*S*N*iters / time), and the per-iteration time of the token-mixing kernels (12 launches) next to the mixer's FC1 and
FC2 GEMMs, from RefineEngine.profile_iteration.  Prints the card's name and power limit with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import pips_oracle as po  # noqa: E402
from pips_b200 import Pips  # noqa: E402

PARTICLE_FRAMES = 8192
H, W, STRIDE, ITERS = 384, 512, 8, 6


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(S: int, reps: int) -> dict:
    dev = "cuda:0"
    N = PARTICLE_FRAMES // S
    m = Pips(S=S, stride=STRIDE, precision="bf16x3").to(dev).eval()
    m.load_state_dict(po.init_state_dict(seed=3, head_scale=0.05, S=S), strict=True)
    rgbs = po.smooth_video(1, S, H, W, seed=5).to(dev)
    xys = po.random_queries(1, N, H, W, seed=6).to(dev)
    with torch.no_grad():
        for _ in range(3):
            m(xys, rgbs, iters=ITERS)
        torch.cuda.synchronize()
        times = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            m(xys, rgbs, iters=ITERS)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        fmaps = m.encode(rgbs).float().contiguous()
        prof, _ = m.engine.profile_iteration(m, fmaps, xys[:, None].repeat(1, S, 1, 1) / STRIDE, float(STRIDE), reps=3)
    times.sort()
    ms = times[len(times) // 2]
    per_iter = {k: sorted(v)[len(v) // 2] * (len(v) // 3) for k, v in prof.items()}   # median launch x launches per iteration
    return dict(S=S, N=N, ms_forward=round(ms, 3), ms_min=round(times[0], 3), ms_max=round(times[-1], 3),
                particle_frame_updates_per_s=round(PARTICLE_FRAMES * ITERS / (ms * 1e-3), 1),
                ms_per_iter_tokenmix=round(per_iter["tokenmix"], 4), ms_per_iter_fc1=round(per_iter["gemm_fc1"], 4),
                ms_per_iter_fc2=round(per_iter["gemm_fc2"], 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_window.py measures on a CUDA device"
    res = dict(card=card(), frames=f"{H}x{W}", stride=STRIDE, iters=ITERS, precision="bf16x3",
               runs=[run(S, a.reps) for S in (8, 16, 5)])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_window.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
