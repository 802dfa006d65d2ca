"""Cost of evaluation with ground truth (test_on_flt.py:87, test_on_crohd.py:133): a forward with trajs_g / vis_g /
valids under torch.no_grad() on the dense torch path (loss_path='torch') and on the CUDA path (loss_path='cuda'),
beside the plain forward without ground truth, plus the score-map loss kernel (pips_scoremap_loss) alone.

    python tools/bench_losses.py [reps]

Times are medians after warm-up; peak memory is torch.cuda.max_memory_allocated over the warm-up and timed calls, above
what the model and inputs held before them (so the buffers a first call creates and keeps are counted).  The torch arm is
skipped when its dense footprint, computed from the shapes, exceeds DENSE_LIMIT; the bytes it would need are printed.
The kernel's share of peak is its issued bf16x3 rate (3 MMAs per product) over the 989 TFLOP/s dense-bf16 data-sheet
rate of the H100 SXM (a rate the card is not claimed to reach)."""
import os, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L
from tools.bench_gemm import gpu_state

PEAK = 989.0
HBM = 3.35e12
DENSE_LIMIT = 40 << 30
SHAPES = [("flt crop", 1, 256), ("cfg2", 4, 1024), ("cfg3", 4, 4096)]     # (name, B, N) at 8 x 384 x 512, stride 8
H, W, STRIDE, ITERS = 384, 512, 8, 6


def dense_bytes(B, N, H8, W8):
    """torch_path.forward_torch: the fcps list, its stack, and score_map_loss's permuted copy, one-hot and loss
    (5 x fcps), plus one iteration's all-pairs volumes."""
    fcps = 4 * B * 8 * ITERS * N * H8 * W8
    vols = 4 * B * 8 * N * sum((H8 >> l) * (W8 >> l) for l in range(4))
    return 5 * fcps + vols


def timed_call(fn, reps):
    """(median ms, peak MiB above what was allocated before the first call: graph plans and caches included)"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    ts.sort()
    return ts[len(ts) // 2] * 1e3, (torch.cuda.max_memory_allocated() - base) / 2**20


def kernel_time(B, N, H8, W8, reps):
    lib = L.load()
    dev = "cuda:0"
    P, S = H8 * W8, 8
    g = torch.Generator(device=dev).manual_seed(0)
    g_hi = (torch.randn(B * S, P, 128, device=dev, generator=g) * 0.1).to(torch.bfloat16)
    g_lo = (torch.randn(B * S, P, 128, device=dev, generator=g) * 1e-4).to(torch.bfloat16)
    ffeats = torch.randn(B * N, S, 128, device=dev, generator=g)
    target = torch.randint(-1, P, (B, S, N), device=dev, generator=g, dtype=torch.int32)
    n_split = lib.pips_scoremap_splits(H8, W8)
    neg = torch.empty(B * S * N, n_split, device=dev)
    pos = torch.empty(B * S * N, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    call = lambda: L.check(lib.pips_scoremap_loss(L.ptr(g_hi), L.ptr(g_lo), L.ptr(ffeats), B, S, N, H8, W8, L.ptr(target),
                                                  L.ptr(neg), L.ptr(pos), st), "pips_scoremap_loss")
    for _ in range(5):
        call()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); call(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], n_split


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    dev = "cuda:0"
    name, plim, _, max_mhz = gpu_state()
    print(f"device {name}, power limit {plim:.0f} W, max SM clock {max_mhz} MHz, medians of {reps} calls after warm-up")
    H8, W8 = H // STRIDE, W // STRIDE
    sd = po.init_state_dict(seed=1, head_scale=0.05)
    for shape, B, N in SHAPES:
        rgbs = po.smooth_video(B, 8, H, W, seed=31).to(dev)
        xys = po.random_queries(B, N, H, W, seed=32).to(dev)
        g = torch.Generator().manual_seed(33)
        tg = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 4.0, 1)).to(dev)
        vg = (torch.rand(B, 8, N, generator=g) > 0.2).float().to(dev)
        va = (torch.rand(B, 8, N, generator=g) > 0.1).float().to(dev)
        print(f"--- {shape}: B={B}, 8 x {H} x {W}, stride {STRIDE}, N={N}, {ITERS} iterations")
        for arm in ("plain", "cuda", "torch"):
            m = Pips(S=8, stride=STRIDE, loss_path="torch" if arm == "torch" else "cuda").to(dev).eval()
            m.load_state_dict(sd)
            if arm == "torch" and dense_bytes(B, N, H8, W8) > DENSE_LIMIT:
                print(f"  loss_path=torch  skipped: the dense path needs about {dense_bytes(B, N, H8, W8) / 2**30:.1f} GiB")
                continue
            kw = {} if arm == "plain" else dict(trajs_g=tg, vis_g=vg, valids=va)

            def fwd():
                with torch.no_grad():
                    return m(xys, rgbs, iters=ITERS, **kw)

            ms, peak = timed_call(fwd, reps)
            label = "no ground truth" if arm == "plain" else f"loss_path={arm}"
            print(f"  {label:16s} {ms:9.2f} ms per forward   peak {peak:8.0f} MiB")
            del m
            torch.cuda.empty_cache()
        ms, n_split = kernel_time(B, N, H8, W8, 25)
        flops = 2.0 * 3 * B * 8 * N * H8 * W8 * 128
        scores = B * 8 * N * H8 * W8
        byts = B * 8 * H8 * W8 * 128 * 4 + B * 8 * N * 128 * 4 + B * 8 * N * (n_split + 2) * 4
        frac = flops / (ms * 1e-3) / 1e12 / PEAK
        print(f"  pips_scoremap_loss alone: {ms * 1e3:8.1f} us per iteration, {scores / (ms * 1e-3) / 1e9:6.1f} G scores/s, "
              f"issued {flops / (ms * 1e-3) / 1e12:6.1f} TFLOP/s = {frac:.3f} of {PEAK:.0f}; "
              f"HBM bound {byts / HBM * 1e6:.1f} us, MMA bound {flops / (PEAK * 1e12) * 1e6:.1f} us")


if __name__ == "__main__":
    main()
