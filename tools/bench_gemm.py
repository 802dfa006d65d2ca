"""Micro-benchmark of pips_gemm_tc at the shapes of one BASELINE cfg-2 iteration (1024 particles x 4 clips x 8 frames =
32768 token rows), for both precision modes and every tile shape, with the bf16 torch.matmul (cuBLAS) of the same
M, N, K beside it as the ceiling this card reaches at these shapes.

    python tools/bench_gemm.py [launches]

L2 is flushed before every launch; times are CUDA-event medians.  "issued" counts the three MMAs per product of the
bf16x3 mode; "frac" is issued TFLOP/s over the 989 TFLOP/s dense-bf16 data-sheet rate of the H100 SXM (a rate the card
is not claimed to reach)."""
import os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pips_b200 import _lib as L

PEAK = 989.0
SHAPES = [("gemm_in", 32768, 512, 576, L.EPI_BIAS), ("fc1", 32768, 2048, 512, L.EPI_BIAS_GELU),
          ("fc2", 32768, 512, 2048, L.EPI_BIAS_RESID), ("head", 4096, 1040, 512, L.EPI_BIAS)]
TILES = ["", "pair", "256", "128", "64"]          # PIPS_B200_GEMM_TILE ("" = the choice pips_gemm_tc makes)


def gpu_state():
    """(name, power limit W, SM clock MHz, max SM clock MHz) of cuda:0, read now."""
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return (torch.cuda.get_device_name(), nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
                nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM), nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM))
    except Exception:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.split(",")
        return (torch.cuda.get_device_name(), *(float(v) for v in q[:3]))


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
    torch.manual_seed(0)
    for shape, M, N, K, epi in SHAPES:
        a = [torch.randn(M, K, device=dev).to(torch.bfloat16) for _ in range(2)]
        w = [(torch.randn(N, K, device=dev) / K ** 0.5).to(torch.bfloat16) for _ in range(2)]
        Ma, Na = (M + 255) // 256 * 256, (N + 255) // 256 * 256
        a = [torch.nn.functional.pad(t, (0, 0, 0, Ma - M)) for t in a]
        w = [torch.nn.functional.pad(t, (0, 0, 0, Na - N)) for t in w]
        bias = torch.randn(N, device=dev)
        of = torch.randn(M, N, device=dev)
        oh = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        ol = torch.empty_like(oh)
        useful = 2.0 * M * N * K
        ms_cublas = timed(lambda: torch.matmul(a[0][:M], w[0][:N].t()))
        for terms in (3, 1):
            for tile in TILES:
                os.environ["PIPS_B200_GEMM_TILE"] = tile
                x3 = terms == 3
                call = lambda: L.check(lib.pips_gemm_tc(L.ptr(a[0]), L.ptr(a[1]) if x3 else 0, K, Ma, L.ptr(w[0]),
                                                        L.ptr(w[1]) if x3 else 0, K, Na, M, N, K, L.ptr(bias), epi,
                                                        L.ptr(of), N, L.ptr(oh), L.ptr(ol) if x3 else 0, N, st))
                ms = timed(call)
                mhz = gpu_state()[2]
                issued = useful * terms / ms / 1e9
                print(f"{shape:8s} M={M} N={N} K={K} x{terms} tile={tile or 'auto':5s} {ms * 1e3:8.1f} us  "
                      f"useful {useful / ms / 1e9:6.1f} TFLOP/s  issued {issued:6.1f} TFLOP/s  frac {issued / PEAK:.3f}  "
                      f"sm {mhz} MHz")
        os.environ.pop("PIPS_B200_GEMM_TILE", None)
        print(f"{shape:8s} M={M} N={N} K={K} cuBLAS bf16 torch.matmul {ms_cublas * 1e3:8.1f} us  "
              f"{useful / ms_cublas / 1e9:6.1f} TFLOP/s  frac {useful / ms_cublas / 1e9 / PEAK:.3f}")


if __name__ == "__main__":
    main()
