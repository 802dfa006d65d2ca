"""Cost of evaluation with ground truth (test_on_flt.py:87, test_on_crohd.py:133): a forward with trajs_g / vis_g /
valids under torch.no_grad() on the dense torch path (loss_path='torch') and on the CUDA path (loss_path='cuda'),
beside the plain forward without ground truth, plus the score-map loss kernel (pips_scoremap_loss) alone.

    python tools/bench_losses.py [reps]
    python tools/bench_losses.py grad [reps]

`grad` measures training with ground truth instead (train.py:82, gradients on), at train.py's per-GPU shape and at cfg 2:
the score-map loss's forward + backward given the ffeats and the pyramid (dense torch_path.score_map_loss against
torch_path.fused_score_map_loss), each backward kernel alone, and a whole training step (forward with is_train=True, then
the backward of the summed losses) with loss_path='torch' against loss_path='fused'.  A dense arm that runs out of memory
is reported as such.

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


GRAD_SHAPES = [("train.py per GPU", 4, 768, 4), ("cfg2", 4, 1024, 6)]     # (name, B, N, iters) at 8 x 384 x 512, stride 8


def event_ms(fn, reps):
    """median CUDA-event time of fn() in ms, after 3 warm-up calls"""
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def grad_kernel_times(B, N, I, H8, W8, reps):
    """pips_scoremap_grad_feats, pips_scoremap_grad_basis and pips_scoremap_basis_grad alone: (name, ms, flops)"""
    lib = L.load()
    dev = "cuda:0"
    S, P, C = 8, H8 * W8, 128
    g = torch.Generator(device=dev).manual_seed(0)
    g_hi = (torch.randn(B * S, P, C, device=dev, generator=g) * 0.1).to(torch.bfloat16)
    g_lo = (torch.randn(B * S, P, C, device=dev, generator=g) * 1e-4).to(torch.bfloat16)
    f = torch.randn(I, B * S, N, C, device=dev, generator=g)
    f_hi, f_lo = f.to(torch.bfloat16), (f - f.to(torch.bfloat16).float()).to(torch.bfloat16)
    target = torch.randint(-1, P, (B, S, N), device=dev, generator=g, dtype=torch.int32)
    coef = torch.tensor([1e-4, 1e-7], device=dev)
    df = torch.empty_like(f)
    dG = torch.empty(B * S, P, C, device=dev)
    dl = [torch.empty(B * S, H8 >> l, W8 >> l, C, device=dev) for l in range(4)]
    st = torch.cuda.current_stream().cuda_stream
    gemm_flops = 2.0 * 2 * 3 * I * B * S * N * P * C       # two bf16x3 GEMMs of M x N x K = (N or P) x P or N x 128 each
    runs = [
        ("pips_scoremap_grad_feats", lambda: L.check(lib.pips_scoremap_grad_feats(
            L.ptr(g_hi), L.ptr(g_lo), L.ptr(f), I, B, S, N, H8, W8, L.ptr(target), L.ptr(coef), L.ptr(df), st)), gemm_flops),
        ("pips_scoremap_grad_basis", lambda: L.check(lib.pips_scoremap_grad_basis(
            L.ptr(g_hi), L.ptr(g_lo), L.ptr(f_hi), L.ptr(f_lo), I, B, S, N, H8, W8, L.ptr(target), L.ptr(coef), L.ptr(dG),
            st)), gemm_flops),
        ("pips_scoremap_basis_grad", lambda: L.check(lib.pips_scoremap_basis_grad(
            L.ptr(dG), B * S, H8, W8, L.ptr_array(dl), st)), 0.0),
    ]
    return [(name, event_ms(fn, reps), flops) for name, fn, flops in runs]


def loss_arm(fused, fmaps, ffeats, tg, vg, va, reps):
    """score-map loss forward + backward given ffeats and fmaps (the pyramid is pooled inside, as in forward_torch)"""
    import torch.nn.functional as F
    from pips_b200 import torch_path

    def step():
        fm = fmaps.detach().requires_grad_(True)
        ff = [x.detach().requires_grad_(True) for x in ffeats]
        B, S = fm.shape[:2]
        pyr = [fm]
        for _ in range(3):
            p = F.avg_pool2d(pyr[-1].flatten(0, 1), 2, stride=2)
            pyr.append(p.reshape(B, S, *p.shape[1:]))
        if fused:
            loss = torch_path.fused_score_map_loss(ff, pyr, tg, vg, va)
        else:
            H8, W8 = fm.shape[-2:]
            fcps = []
            for x in ff:
                vols = [torch.matmul(x, p.flatten(3)).reshape(B, S, x.shape[2], *p.shape[-2:]) / (128 ** 0.5) for p in pyr]
                fcps.append(sum(F.interpolate(v.flatten(0, 1), (H8, W8), mode="bilinear", align_corners=True)
                                .reshape(B, S, x.shape[2], H8, W8) for v in vols))
            loss = torch_path.score_map_loss(torch.stack(fcps, dim=2), tg, vg, va)
        loss.backward()

    return timed_call(step, reps)


def train_arm(loss_path, sd, rgbs, xys, tg, vg, va, iters, reps):
    m = Pips(S=8, stride=STRIDE, loss_path=loss_path).to("cuda:0").train()
    m.load_state_dict(sd)

    def step():
        m.zero_grad(set_to_none=True)
        _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
        sum(losses).backward()

    try:
        return timed_call(step, reps)
    finally:
        del m


def run_or_oom(fn):
    try:
        return fn()
    except torch.cuda.OutOfMemoryError:
        return None
    finally:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def grad_main(reps):
    dev = "cuda:0"
    name, plim, _, max_mhz = gpu_state()
    print(f"device {name}, power limit {plim:.0f} W, max SM clock {max_mhz} MHz, medians of {reps} calls after warm-up")
    H8, W8 = H // STRIDE, W // STRIDE
    sd = po.init_state_dict(seed=1, head_scale=0.05)
    for shape, B, N, I in GRAD_SHAPES:
        print(f"--- {shape}: B={B}, 8 x {H} x {W}, stride {STRIDE}, N={N}, {I} iterations")
        g = torch.Generator(device=dev).manual_seed(7)
        fmaps = torch.randn(B, 8, 128, H8, W8, device=dev, generator=g)
        ffeats = [torch.randn(B, 8, N, 128, device=dev, generator=g) for _ in range(I)]
        tg = torch.rand(B, 8, N, 2, device=dev, generator=g) * torch.tensor([W8, H8], device=dev)
        vg = (torch.rand(B, 8, N, device=dev, generator=g) > 0.2).float()
        va = (torch.rand(B, 8, N, device=dev, generator=g) > 0.1).float()
        for arm in ("dense", "fused"):
            r = run_or_oom(lambda: loss_arm(arm == "fused", fmaps, ffeats, tg, vg, va, reps))
            print(f"  score-map loss fwd+bwd, {arm:5s}: " + ("out of memory" if r is None else
                  f"{r[0]:9.2f} ms   peak {r[1]:8.0f} MiB above the inputs"))
        del fmaps, ffeats
        for kname, ms, flops in grad_kernel_times(B, N, I, H8, W8, max(reps, 10)):
            rate = f", issued {flops / (ms * 1e-3) / 1e12:6.1f} TFLOP/s = {flops / (ms * 1e-3) / 1e12 / PEAK:.3f} of {PEAK:.0f}" \
                if flops else ""
            print(f"  {kname:26s} {ms * 1e3:9.1f} us{rate}")
        torch.cuda.empty_cache()
        rgbs = po.smooth_video(B, 8, H, W, seed=31).to(dev)
        xys = po.random_queries(B, N, H, W, seed=32).to(dev)
        gc = torch.Generator().manual_seed(33)
        tgi = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=gc) * 4.0, 1)).to(dev)
        vgi = (torch.rand(B, 8, N, generator=gc) > 0.2).float().to(dev)
        vai = (torch.rand(B, 8, N, generator=gc) > 0.1).float().to(dev)
        for lp in ("torch", "fused"):
            r = run_or_oom(lambda: train_arm(lp, sd, rgbs, xys, tgi, vgi, vai, I, reps))
            print(f"  training step, loss_path={lp:5s}: " + ("out of memory" if r is None else
                  f"{r[0]:9.2f} ms   peak {r[1]:8.0f} MiB"))
        del rgbs, xys
        torch.cuda.empty_cache()


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "grad":
        grad_main(int(sys.argv[2]) if len(sys.argv) > 2 else 3)
    else:
        main()
