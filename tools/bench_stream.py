"""Streamed tracking: pips_b200.stream.track_queries_stream against track_queries, and on a long video.

    python tools/bench_stream.py [--T 48] [--N 1024] [--chunk 32] [--long-T 3000] [--reps 3] [--precision bf16x3]

Two workloads, 384 x 512 frames, stride 8, 6 iterations, N = 1024 queries (t, x, y) with t uniform in 0..T-1:
  - cost of streaming: the bench_queries workload (T = 48, the clip resident on the device).  track_queries on the
    whole clip against track_queries_stream fed the same clip in chunks of --chunk frames, forward and then backward.
    The two must agree bit for bit; the maximum |difference| of trajectories and visibilities is reported.
  - long video: T = --long-T frames generated chunk by chunk on the device (a periodic texture translated 3 px and
    2 px per frame), streamed through track_queries_stream in chunks of --chunk frames.  Reported: time per frame of
    video (both passes), the peak device memory, and what track_queries would hold resident for the same clip, from
    the shapes: the clip as fp32, the feature maps, and their pyramid.
Wall time is a host clock around each call ending in a device synchronise (median of --reps runs after one warm-up for
the first workload, one run for the long video); peaks are torch.cuda.max_memory_allocated above what was allocated
before the call, the model's state and the resident clip included there.  The card's name, power limit and maximum SM
clock are read in the same run.  The last line is one JSON record of the numbers."""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_queries import card, measure  # noqa: E402
from pips_b200 import Pips, _lib  # noqa: E402
from pips_b200.chain import track_queries  # noqa: E402
from pips_b200.stream import track_queries_stream  # noqa: E402
from pips_b200.synthetic import random_queries  # noqa: E402

DEV = "cuda:0"
LATENT, LEVELS = 128, 4


def chunks(rgbs, k, reverse=False):
    clip = rgbs[0].flip(0) if reverse else rgbs[0]
    return (clip[i:i + k] for i in range(0, clip.shape[0], k))


def texture(H, W, seed):
    """(3, H, W) smooth noise on the device that tiles with period (H, W), values 0..255."""
    g = torch.Generator().manual_seed(seed)
    low = F.pad(torch.rand(1, 3, H // 16, W // 16, generator=g), (2, 2, 2, 2), mode="circular")
    big = F.interpolate(low, scale_factor=16, mode="bicubic", align_corners=False)[0, :, 32:32 + H, 32:32 + W]
    return (big.clamp(0, 1) * 255.0).round().to(DEV)


def generated(tex, T, k, reverse=False):
    """Frames 0..T-1 (or T-1..0) in chunks of k: frame f is the texture translated (3f, 2f) px."""
    for i in range(0, T, k):
        idx = torch.arange(i, min(T, i + k))
        idx = T - 1 - idx if reverse else idx
        yield torch.stack([torch.roll(tex, (2 * f, 3 * f), (-2, -1)) for f in idx.tolist()])


def resident_mib(T, H, W, stride, feat_bf16):
    """What track_queries holds for a T-frame clip besides the model: the clip as fp32, the feature maps and the pyramid
    (4 fp32 channels-last levels, plus a bf16 copy with feat_dtype='bf16')."""
    h, w = H // stride, W // stride
    fmaps = h * w * LATENT * 4
    pyr = 0
    for _ in range(LEVELS):
        pyr += h * w * LATENT * (4 + (2 if feat_bf16 else 0))
        h, w = h // 2, w // 2
    return T * (3 * H * W * 4 + fmaps + pyr) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=48)
    ap.add_argument("--long-T", type=int, default=3000)
    ap.add_argument("--N", type=int, default=1024)
    ap.add_argument("--H", type=int, default=384)
    ap.add_argument("--W", type=int, default=512)
    ap.add_argument("--chunk", type=int, default=32)
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream: needs a CUDA device")
    from oracle import pips_oracle as po      # the bench_queries workload: same weights, clip and queries
    sd = po.init_state_dict(seed=21, head_scale=0.05)
    model = Pips(S=8, stride=8, precision=a.precision).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    rgbs = po.smooth_video(1, a.T, a.H, a.W, seed=22).to(DEV)
    g = torch.Generator().manual_seed(23)
    t = torch.randint(0, a.T, (1, a.N, 1), generator=g).float()
    queries = torch.cat([t, po.random_queries(1, a.N, a.H, a.W, seed=24)], dim=2).to(DEV)
    name = card()

    (want_t, want_v), t_whole, m_whole = measure(lambda: track_queries(model, rgbs, queries, iters=a.iters), a.reps)
    (got_t, got_v), t_stream, m_stream = measure(
        lambda: track_queries_stream(model, chunks(rgbs, a.chunk), chunks(rgbs, a.chunk, True), queries, iters=a.iters),
        a.reps)
    diff = max((got_t - want_t.cpu()).abs().max().item(), (got_v - want_v.cpu()).abs().max().item())

    tex = texture(a.H, a.W, seed=25)
    g = torch.Generator().manual_seed(26)
    tl = torch.randint(0, a.long_T, (a.N, 1), generator=g).float()
    q_long = torch.cat([tl, random_queries(1, a.N, a.H, a.W, seed=27)[0]], dim=1)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    long_t, _ = track_queries_stream(model, generated(tex, a.long_T, a.chunk), generated(tex, a.long_T, a.chunk, True),
                                     q_long, iters=a.iters)
    torch.cuda.synchronize()
    t_long = time.perf_counter() - t0
    m_long = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    finite = bool(torch.isfinite(long_t).all())
    need = resident_mib(a.long_T, a.H, a.W, 8, model.engine.feat_dtype == _lib.FEAT_BF16)

    print(f"card: {name}")
    print(f"workload: {a.H}x{a.W}, N={a.N} queries at random frames, stride 8, {a.iters} iterations, {a.precision}, "
          f"chunks of {a.chunk} frames")
    print(f"T={a.T} resident clip: track_queries {t_whole * 1e3:.1f} ms, peak {m_whole:.0f} MiB; "
          f"track_queries_stream {t_stream * 1e3:.1f} ms, peak {m_stream:.0f} MiB; max |difference| {diff:.3g}")
    print(f"T={a.long_T} generated on the device: {t_long:.1f} s, {t_long / a.long_T * 1e3:.2f} ms per frame, "
          f"peak {m_long:.0f} MiB (track_queries would hold {need:.0f} MiB resident); trajectories finite: {finite}")
    print(json.dumps(dict(card=name, H=a.H, W=a.W, N=a.N, iters=a.iters, precision=a.precision, chunk=a.chunk,
                          T=a.T, queries_ms=round(t_whole * 1e3, 2), queries_peak_mib=round(m_whole),
                          stream_ms=round(t_stream * 1e3, 2), stream_peak_mib=round(m_stream), max_abs_diff=diff,
                          long_T=a.long_T, long_s=round(t_long, 2), long_ms_per_frame=round(t_long / a.long_T * 1e3, 3),
                          long_peak_mib=round(m_long), long_track_queries_resident_mib=round(need),
                          long_finite=finite)))


if __name__ == "__main__":
    main()
