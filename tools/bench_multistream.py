"""Many live videos at once: pips_b200.stream.MultiStream against one TrackStream per video, fed the same ticks.

    python tools/bench_multistream.py [--videos 16] [--T 300] [--N 64] [--k 8] [--precision bf16x3]

Generated videos on the device (a periodic texture translated a few pixels per frame, as in tools/bench_stream.py):
--videos videos at the four SIZES in turn, --T frames each, --N queries each at random frames (a quarter of them added
live, at the video's pending frame or later), stride 8, 6 iterations.  One tick delivers --k frames to every running
video; a quarter of the videos start --k * 4 frames late and a quarter end early (after 3/4 of their frames), so
videos start and end mid-run.  Both arms take the same ticks: the MultiStream pushes one dict per tick; the TrackStream
arm pushes to each video's stream in turn (and finishes it in its last tick).  The two arms' trajectories and
visibilities are compared; the difference must be 0.

Time per tick is a host clock around each tick's pushes, ending in a device synchronise (frame generation is outside
it); the tool reports the median and the total.  Rounds are each arm's refinement rounds (the TrackStream arm's sum
over its streams).  The peak is torch.cuda.max_memory_allocated above what was allocated before the arm's run.  One
short run of both arms comes first as a warm-up (encoder plans, workspaces).  The card's name, power limit and maximum
SM clock are read in the same run.  The last line is one JSON record of the numbers."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_queries_mixed import card  # noqa: E402
from bench_stream import texture  # noqa: E402
from pips_b200 import Pips  # noqa: E402
from pips_b200.stream import MultiStream, TrackStream  # noqa: E402
from pips_b200.synthetic import random_queries  # noqa: E402

DEV = "cuda:0"
SIZES = [(256, 256), (240, 320), (320, 240), (288, 512)]


def workload(n_videos, T, N, k, seed=31):
    """Per video: its size, first tick, frame count, queries at open and live queries (tick, offset from the pending
    frame) with their (x, y), in the order they are added -- the order of their columns in a TrackStream."""
    g = torch.Generator().manual_seed(seed)
    vids = []
    for i in range(n_videos):
        H, W = SIZES[i % len(SIZES)]
        start = 4 if i % 4 == 1 else 0
        frames = T * 3 // 4 if i % 4 == 2 else T
        n_live = N // 4
        t = torch.randint(0, frames, (N - n_live, 1), generator=g).float()
        q = torch.cat([t, random_queries(1, N - n_live, H, W, seed=seed * 100 + i)[0]], dim=1)
        ticks = (frames + k - 1) // k
        live = sorted((int(torch.randint(1, max(2, ticks - 1), (1,), generator=g)),
                       int(torch.randint(0, 2 * k, (1,), generator=g))) for _ in range(n_live))   # in order of adding
        lxy = random_queries(1, n_live, H, W, seed=seed * 100 + 50 + i)[0]
        vids.append(dict(hw=(H, W), start=start, frames=frames, q=q, live=live, lxy=lxy,
                         tex=texture(H, W, seed=seed * 10 + i), shift=(1 + i % 3, 2 - i % 2)))
    return vids


def chunk(v, f0, f1):
    """Frames f0 .. f1-1 of video v: the texture translated by shift px per frame."""
    dy, dx = v["shift"]
    return torch.stack([torch.roll(v["tex"], (dy * f, dx * f), (-2, -1)) for f in range(f0, f1)])


def schedule(vids, k):
    """Per tick: {video: (f0, f1)} and the videos that end."""
    ticks, i = [], 0
    while True:
        ks, end = {}, set()
        for j, v in enumerate(vids):
            f0 = (i - v["start"]) * k
            if 0 <= f0 < v["frames"]:
                ks[j] = (f0, min(v["frames"], f0 + k))
                if ks[j][1] == v["frames"]:
                    end.add(j)
        if not ks and i > 0:
            return ticks
        ticks.append((ks, end))
        i += 1


def run_multi(model, vids, ticks, live, iters, pending_only=False):
    ms = MultiStream(model, iters=iters)
    ids, out, times, found = {}, {j: [] for j in range(len(vids))}, [], {}
    for i, (ks, end) in enumerate(ticks):
        for j in ks:
            if j not in ids:
                ids[j] = ms.open(vids[j]["q"])
        for j in ks:
            v = vids[j]
            sel = [n for n, (tick, _) in enumerate(v["live"]) if tick == i - v["start"]]
            if sel:
                if pending_only:
                    p = ms.pending(ids[j])
                    for n in sel:
                        found[(j, n)] = min(p + v["live"][n][1], v["frames"] - 1)
                else:
                    ms.add_queries(ids[j], live[j][sel])
        frames = {ids[j]: chunk(vids[j], *r) for j, r in ks.items()}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = ms.push(frames, end={ids[j] for j in end})
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        for j in ks:
            out[j].append(res[ids[j]])
    return found if pending_only else (out, times, ms.rounds)


def run_lone(model, vids, ticks, live, iters):
    streams, out, times = {}, {j: [] for j in range(len(vids))}, []
    rounds = 0
    for ks, end in ticks:
        for j in ks:
            if j not in streams:
                streams[j] = TrackStream(model, torch.cat([vids[j]["q"], live[j]]), iters=iters)
        frames = {j: chunk(vids[j], *r) for j, r in ks.items()}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for j, f in frames.items():
            out[j].append(streams[j].push(f))
            if j in end:
                out[j].append(streams[j].finish())
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    for s in streams.values():
        rounds += s.rounds
    return out, times, rounds


def concat(blocks, n):
    """The blocks of one video as (trajs, vis), the columns of live queries NaN before they were added."""
    tr = [torch.cat([b[1], b[1].new_full((b[1].shape[0], n - b[1].shape[1], 2), float("nan"))], 1) for b in blocks]
    vi = [torch.cat([b[2], b[2].new_full((b[2].shape[0], n - b[2].shape[1]), float("nan"))], 1) for b in blocks]
    return torch.cat(tr), torch.cat(vi)


def measure(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=16)
    ap.add_argument("--T", type=int, default=300)
    ap.add_argument("--N", type=int, default=64)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--precision", default="bf16x3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multistream: needs a CUDA device")
    from oracle import pips_oracle as po
    model = Pips(S=8, stride=8, precision=a.precision).to(DEV).eval()
    model.load_state_dict(po.init_state_dict(seed=21, head_scale=0.05), strict=True)
    name = card()
    print(f"card: {name}")

    def prepare(T):
        vids = workload(a.videos, T, a.N, a.k)
        ticks = schedule(vids, a.k)
        found = run_multi(model, vids, ticks, None, a.iters, pending_only=True)
        live = []
        for j, v in enumerate(vids):
            t = torch.tensor([[float(found[(j, n)])] for n in range(len(v["live"]))]).view(-1, 1)
            live.append(torch.cat([t, v["lxy"]], dim=1))
        return vids, ticks, live

    w = prepare(32)                                                  # warm-up of both arms
    run_multi(model, *w, a.iters)
    run_lone(model, *w, a.iters)
    vids, ticks, live = prepare(a.T)
    (m_out, m_times, m_rounds), m_peak = measure(lambda: run_multi(model, vids, ticks, live, a.iters))
    (l_out, l_times, l_rounds), l_peak = measure(lambda: run_lone(model, vids, ticks, live, a.iters))
    dt = dv = 0.0
    same = True
    for j, v in enumerate(vids):
        n = v["q"].shape[0] + live[j].shape[0]
        (mt, mv), (lt, lv) = concat(m_out[j], n), concat(l_out[j], n)
        same &= mt.shape == lt.shape and torch.equal(mt.view(torch.int32), lt.view(torch.int32)) \
            and torch.equal(mv.view(torch.int32), lv.view(torch.int32))
        dt = max(dt, (mt - lt).nan_to_num(0).abs().max().item())
        dv = max(dv, (mv - lv).nan_to_num(0).abs().max().item())
    frames = sum(v["frames"] for v in vids)
    queries = sum(v["q"].shape[0] + live[j].shape[0] for j, v in enumerate(vids))
    print(f"{a.videos} videos at {len(SIZES)} sizes, {frames} frames, {queries} queries ({sum(x.shape[0] for x in live)} "
          f"added live), {len(ticks)} ticks of {a.k} frames per video, stride 8, {a.iters} iterations, {a.precision}")
    for arm, ts, r, pk in (("MultiStream", m_times, m_rounds, m_peak), ("TrackStream per video", l_times, l_rounds,
                                                                        l_peak)):
        print(f"  {arm:22s} {statistics.median(ts) * 1e3:8.1f} ms per tick (median), {sum(ts):7.2f} s in all, "
              f"{r} rounds, peak {pk:.0f} MiB")
    print(f"  results identical: {same}; max |trajs difference| {dt:.3g} px, max |vis difference| {dv:.3g}")
    print(json.dumps(dict(card=name, videos=a.videos, sizes=SIZES, T=a.T, N=a.N, k=a.k, iters=a.iters,
                          precision=a.precision, ticks=len(ticks), frames=frames, queries=queries,
                          multi_ms_per_tick=round(statistics.median(m_times) * 1e3, 2),
                          multi_s=round(sum(m_times), 3), multi_rounds=m_rounds, multi_peak_mib=round(m_peak),
                          lone_ms_per_tick=round(statistics.median(l_times) * 1e3, 2),
                          lone_s=round(sum(l_times), 3), lone_rounds=l_rounds, lone_peak_mib=round(l_peak),
                          identical=bool(same), max_traj_diff_px=dt, max_vis_diff=dv)))
    if not same:
        raise SystemExit("bench_multistream: the two arms differ")


if __name__ == "__main__":
    main()
