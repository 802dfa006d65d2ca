"""K sweep of pips_gemm_tc at the FC1 output shape (M = 32768 token rows, N = 2048), bf16x3, automatic tile, for the
BIAS_GELU and BIAS epilogues:

    python tools/bench_gemm_ksweep.py [launches]

A persistent CTA (or cluster) runs `waves` tiles one after the other, each K/32 K-blocks of MMAs followed by the tile's
epilogue, so the time fits  t = waves * (a + b * K/32):  `a` is the fixed cost of a tile that the MMAs do not hide
(epilogue, pipeline refill), `b` the cost of one K-block.  The script prints each time and the least-squares a and b.
L2 is flushed before every launch; times are CUDA-event medians."""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pips_b200 import _lib as L
from bench_gemm import gpu_state

M, N = 32768, 2048
KS = [256, 512, 1024, 2048]


def main():
    launches = int(sys.argv[1]) if len(sys.argv) > 1 else 25
    lib = L.load()
    dev = "cuda:0"
    st = torch.cuda.current_stream().cuda_stream
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(launches):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts) // 2]

    name, plim, _, max_mhz = gpu_state()
    print(f"device {name}, power limit {plim:.0f} W, max SM clock {max_mhz} MHz, {launches} launches per median")
    # the automatic choice at this shape is the pair kernel: 256 x 256 tiles on clusters of two CTAs
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = (M // 256) * (N // 256)
    waves = -(-tiles // (sms // 2))
    torch.manual_seed(0)
    bias = torch.randn(N, device=dev)
    of = torch.empty(M, N, device=dev)
    oh = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
    ol = torch.empty_like(oh)
    for epi_name, epi in (("BIAS_GELU", L.EPI_BIAS_GELU), ("BIAS", L.EPI_BIAS)):
        us = []
        for K in KS:
            act = [torch.randn(M, K, device=dev).to(torch.bfloat16) for _ in range(2)]
            w = [(torch.randn(N, K, device=dev) / K ** 0.5).to(torch.bfloat16) for _ in range(2)]
            call = lambda: L.check(lib.pips_gemm_tc(L.ptr(act[0]), L.ptr(act[1]), K, M, L.ptr(w[0]), L.ptr(w[1]), K, N, M, N, K,
                                                    L.ptr(bias), epi, L.ptr(of), N, L.ptr(oh), L.ptr(ol), N, st))
            ms = timed(call)
            us.append(ms * 1e3)
            print(f"{epi_name:9s} M={M} N={N} K={K:5d} x3 {ms * 1e3:8.1f} us  issued {6.0 * M * N * K / ms / 1e9:6.1f} TFLOP/s  "
                  f"sm {gpu_state()[2]} MHz")
        kb = np.array(KS, dtype=np.float64) / 32
        per_kb, fixed = np.polyfit(kb, np.array(us), 1)
        print(f"{epi_name:9s} fit over {waves} waves: a = {fixed / waves:.2f} us per tile (fixed), b = {per_kb / waves:.3f} us "
              f"per K-block; at K=512 the fixed part is {fixed / (fixed + per_kb * 16):.2f} of the time")


if __name__ == "__main__":
    main()
