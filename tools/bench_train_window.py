"""One training step (forward with is_train=True and ground truth, then the backward of the three losses) at window
lengths S = 4, 8, 12 and 16, at a train.py-like shape: B=2, N=768, 4 iterations, S x 384 x 512, stride 8 (48 x 64 maps).

    python tools/bench_train_window.py [--reps 5] [--B 2] [--S 4 8 12 16]

Per S it compares the correlation and the score-map loss on the torch paths (corr_path='torch', loss_path='torch': the
all-pairs volumes and the dense score maps under autograd) against corr_path='cuda' with loss_path='fused' (neither is
built).  The encoder is encoder_path='cuda' and the mixer mixer_path='torch' throughout, since the CUDA mixer trains S = 8
only; at S = 8 all four CUDA paths (mixer_path='cuda') are timed as well, for scale.  Median of --reps steps after one
warm-up, CUDA events; the peak is torch.cuda.max_memory_allocated over one more step, above what was allocated before
it (the model, its inputs).  The losses of the two configurations are printed side by side as a check that they compute
the same step.  Writes nothing; one JSON line per configuration follows the table."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pips_oracle as po  # noqa: E402
from pips_b200 import Pips  # noqa: E402

DEV = "cuda:0"
H, W, N, ITERS = 384, 512, 768, 4
CONFIGS = {  # name: (corr_path, loss_path, mixer_path)
    "torch": ("torch", "torch", "torch"),
    "cuda": ("cuda", "fused", "torch"),
    "all-cuda": ("cuda", "fused", "cuda"),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def inputs(B, S, seed=1):
    rgbs = po.smooth_video(B, S, H, W, seed=seed).to(DEV)
    xys = po.random_queries(B, N, H, W, seed=seed + 1).to(DEV)
    g = torch.Generator().manual_seed(seed + 2)
    tg = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, S, N, 2, generator=g) * 3.0, 1)).to(DEV)
    vg = (torch.rand(B, S, N, generator=g) > 0.1).float().to(DEV)
    va = torch.ones(B, S, N, device=DEV)
    return rgbs, xys, tg, vg, va


def run(S, name, batch, reps):
    corr, loss, mixer = CONFIGS[name]
    m = Pips(S=S, stride=8, loss_path=loss, corr_path=corr, mixer_path=mixer, encoder_path="cuda").to(DEV).train()
    m.load_state_dict(po.init_state_dict(seed=3, head_scale=0.05, S=S), strict=True)
    rgbs, xys, tg, vg, va = batch
    out = {}

    def step():
        m.zero_grad(set_to_none=True)
        _, _, _, losses = m(xys, rgbs, iters=ITERS, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
        sum(losses).backward()
        out["losses"] = [l.item() for l in losses]

    row = {"S": S, "config": name, "corr_path": corr, "loss_path": loss, "mixer_path": mixer, "encoder_path": "cuda",
           "B": rgbs.shape[0], "N": N, "iters": ITERS, "H": H, "W": W}
    try:
        step()                                                  # warm-up
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step()
        torch.cuda.synchronize()
        row.update(ms=statistics.median(ts), ms_min=min(ts), ms_max=max(ts),
                   peak_gib=(torch.cuda.max_memory_allocated() - base) / 2**30, losses=out["losses"])
    except torch.cuda.OutOfMemoryError:
        row.update(ms=None, peak_gib=None, error=f"out of memory in {torch.cuda.get_device_properties(0).total_memory / 2**30:.0f} GiB")
    del m
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--B", type=int, default=2)
    ap.add_argument("--S", type=int, nargs="+", default=[4, 8, 12, 16])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_window.py measures on the GPU; no CUDA device found")
    print(f"card: {card()}")
    print(f"training step, B={args.B}, N={N}, {ITERS} iterations, S x {H} x {W}, stride 8, encoder cuda; median of "
          f"{args.reps} steps")
    rows = []
    for S in args.S:
        batch = inputs(args.B, S)
        for name in ("torch", "cuda") + (("all-cuda",) if S == 8 else ()):
            r = run(S, name, batch, args.reps)
            rows.append(r)
            corr, loss, mixer = CONFIGS[name]
            label = f"S={S:2d} corr {corr:5s} loss {loss:5s} mixer {mixer:5s}"
            if r["ms"] is None:
                print(f"{label}: {r['error']}")
            else:
                print(f"{label}: {r['ms']:8.1f} ms (min {r['ms_min']:.1f}, max {r['ms_max']:.1f}), peak {r['peak_gib']:6.2f} "
                      f"GiB, losses {' '.join(f'{l:.6g}' for l in r['losses'])}")
        del batch
        torch.cuda.empty_cache()
    for r in rows:
        print(json.dumps(r))


if __name__ == "__main__":
    main()
