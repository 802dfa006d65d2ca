"""Training-path timings on one GPU: the DeltaBlock mixer's forward + backward on the torch module against
torch_path.delta_block_cuda, each new backward kernel alone, and a whole training step (is_train=True, the backward of the
three losses) with loss_path='fused' and mixer_path 'torch' against 'cuda'.  The feature encoder likewise: its forward +
backward on the torch module (strict fp32, as forward_torch runs it) against torch_path.encoder_cuda at 32 and 128 frames
of 384 x 512, its backward kernels alone, and training steps with encoder_path 'torch' against 'cuda' (loss_path='fused',
mixer_path='cuda') at B=4 and at train.py's single-GPU default B=16 (N=768, 4 iterations).  The local correlation
likewise: its forward + backward over 4 iterations as forward_torch runs it (matmul volumes and grid_sample) against
torch_path.local_corr_cuda, its two backward kernels alone, and training steps with corr_path 'torch' against 'cuda'
(loss_path='fused', mixer and encoder 'cuda'), at B=4 and B=16.

    python tools/bench_train.py [--reps 5] [--skip-step] [--only mixer|encoder|corr]

Shapes: train.py's per-GPU shape (B=4, N=768, 4 iterations, 8 x 384 x 512, stride 8: R = 3072 tracks, M = 24576 mixer
rows) and BASELINE cfg 2 (N=1024, 6 iterations: M = 32768).  Medians of --reps timed runs after two warm-ups, CUDA
events; peaks from torch.cuda.max_memory_allocated.  Rates count useful FLOPs (2 M N K per GEMM); the share of 989
TFLOP/s (H100 SXM dense BF16) counts the three MMAs of every bf16x3 product."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pips_oracle as po  # noqa: E402
from pips_b200 import Pips, _lib as L, torch_path  # noqa: E402
from pips_b200.pips import DeltaBlock  # noqa: E402

DEV = "cuda:0"
PEAK = 989e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def peak_of(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**30


def delta_block(seed=3):
    sd = po.init_state_dict(seed=seed, head_scale=0.05)
    m = DeltaBlock().to(DEV)
    m.load_state_dict({k[len("delta_block."):]: v for k, v in sd.items() if k.startswith("delta_block.")})
    return m


def strict_fp32():
    """Strict fp32 for the torch module, the accuracy class of the bf16x3 kernels: cuDNN on (the token-mixing Conv1d
    layers), TF32 off for its convolutions and for matmul (off by default).  Returns the previous settings."""
    old = (torch.backends.cudnn.enabled, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.enabled = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return old


def bench_mixer(reps):
    m = delta_block()
    old = strict_fp32()
    try:
        _bench_mixer(m, reps)
    finally:
        torch.backends.cudnn.enabled, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _bench_mixer(m, reps):
    for R in (3072, 4096):
        x = torch.randn(R, 8, 519, device=DEV)
        dy = torch.randn(R, 8, 130, device=DEV)
        for name in ("torch", "cuda"):
            def step():
                m.zero_grad(set_to_none=True)
                xr = x.clone().requires_grad_(True)
                out = torch_path.delta_block_cuda(m, xr) if name == "cuda" else m(xr)
                (out * dy).sum().backward()
            try:
                ms = timed(step, reps)
                gib = peak_of(step)
                print(f"mixer fwd+bwd M={8 * R} {name:5s}: {ms:8.2f} ms, peak {gib:6.2f} GiB above inputs")
            except torch.cuda.OutOfMemoryError:
                print(f"mixer fwd+bwd M={8 * R} {name:5s}: out of memory")
            torch.cuda.empty_cache()


def split(v):
    hi = torch.empty(v.shape, dtype=torch.bfloat16, device=DEV)
    lo = torch.empty_like(hi)
    L.check(L.load().pips_split_bf16(L.ptr(v), L.ptr(hi), L.ptr(lo), v.numel(), torch.cuda.current_stream().cuda_stream))
    return hi, lo


def bench_kernels(reps):
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    M, R = 24576, 3072

    def report(name, ms, flop, mmas=3):
        print(f"{name:34s}: {ms * 1e3:8.1f} us, {flop / ms / 1e9:6.1f} TFLOP/s useful, {mmas * flop / (ms * 1e-3) / PEAK:.2f} of "
              f"989 TFLOP/s in issued MMAs" if flop else f"{name:34s}: {ms * 1e3:8.1f} us")

    for (Mv, N, K, what) in ((M, 512, 2048, "wgrad FC2 (512x2048)"), (M, 2048, 512, "wgrad FC1 (2048x512)"),
                             (M, 512, 576, "wgrad input (512x576)"), (R, 1040, 512, "wgrad head (1040x512)")):
        g, x = split(torch.randn(Mv, N, device=DEV)), split(torch.randn(Mv, K, device=DEV))
        dw = torch.empty(N, K, device=DEV)
        sc = torch.empty(max(1, lib.pips_wgrad_scratch_floats(Mv, N, K)), device=DEV)
        fn = lambda: L.check(lib.pips_wgrad(L.ptr(g[0]), L.ptr(g[1]), N, L.ptr(x[0]), L.ptr(x[1]), K, Mv, N, K, L.ptr(sc),
                                            L.ptr(dw), st))
        report(f"{what} M={Mv}", timed(fn, 20, 3), 2.0 * Mv * N * K)
    a, w = split(torch.randn(M, 512, device=DEV)), split(torch.randn(2048, 512, device=DEV) / 23)
    b = torch.randn(2048, device=DEV)
    hi, lo = torch.empty(M, 2048, dtype=torch.bfloat16, device=DEV), torch.empty(M, 2048, dtype=torch.bfloat16, device=DEV)
    pre = torch.empty(M, 2048, device=DEV)
    for epi, name in ((L.EPI_BIAS_GELU, "FC1 forward (BIAS_GELU)"), (L.EPI_BIAS_GELU_PRE, "FC1 recompute (BIAS_GELU_PRE)"),
                      (L.EPI_GELU_GRAD, "FC2 dgrad (GELU_GRAD)")):
        fn = lambda: L.check(lib.pips_gemm_tc_aux(L.ptr(a[0]), L.ptr(a[1]), 512, M, L.ptr(w[0]), L.ptr(w[1]), 512, 2048, M, 2048, 512,
                                                  L.ptr(b), epi, None, 0, L.ptr(hi), L.ptr(lo), 2048, L.ptr(pre), 2048, st))
        report(f"{name} M={M}", timed(fn, 20, 3), 2.0 * M * 2048 * 512)
    x = torch.randn(M, 512, device=DEV)
    dxb = torch.randn(M, 512, device=DEV)
    P = [torch.randn(n, device=DEV) for n in (512, 512, 256, 32, 256, 8, 512, 512)]
    sc = torch.empty(lib.pips_tokenmix_grad_scratch_floats(R), device=DEV)
    gr = torch.empty(2600, device=DEV)
    fn = lambda: L.check(lib.pips_tokenmix_grad(L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(dxb), R, *(L.ptr(p) for p in P), L.ptr(sc),
                                                L.ptr(gr), st))
    report(f"tokenmix_grad {R} sequences", timed(fn, 20, 3), 0)


def bench_step(reps):
    for label, B, N, iters in (("train.py shape", 4, 768, 4), ("cfg 2", 4, 1024, 6)):
        rgbs = po.smooth_video(B, 8, 384, 512, seed=1).to(DEV)
        xys = po.random_queries(B, N, 384, 512, seed=2).to(DEV)
        g = torch.Generator().manual_seed(3)
        tg = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 3.0, 1)).to(DEV)
        vg = torch.ones(B, 8, N, device=DEV)
        va = torch.ones(B, 8, N, device=DEV)
        for mixer in ("torch", "cuda"):
            m = Pips(S=8, stride=8, loss_path="fused", mixer_path=mixer).to(DEV).train()
            m.load_state_dict(po.init_state_dict(seed=3, head_scale=0.05))

            def step():
                m.zero_grad(set_to_none=True)
                _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
                sum(losses).backward()
            try:
                ms = timed(step, reps, warm=1)
                gib = peak_of(step)
                print(f"training step, {label} (B={B}, N={N}, {iters} iterations), mixer {mixer:5s}: {ms:8.1f} ms, "
                      f"peak {gib:6.2f} GiB")
            except torch.cuda.OutOfMemoryError:
                print(f"training step, {label} (B={B}, N={N}, {iters} iterations), mixer {mixer:5s}: does not fit in "
                      f"{torch.cuda.get_device_properties(0).total_memory / 2**30:.0f} GiB")
            del m
            torch.cuda.empty_cache()


ENC_LAYERS = [  # (name, Cin, Cout, R, stride, pad, input size at 384 x 512): the convolutions of BasicEncoder
    ("stem 4x1 over row pairs", 64, 64, 4, 1, 0, (195, 256)),
    ("layer1 3x3 64->64", 64, 64, 3, 1, 1, (192, 256)),
    ("layer2.0.conv1 3x3/2 64->96", 64, 96, 3, 2, 1, (192, 256)),
    ("layer2.0.downsample 1x1/2", 64, 96, 1, 2, 0, (192, 256)),
    ("layer2 3x3 96->96", 96, 96, 3, 1, 1, (96, 128)),
    ("layer3.0.conv1 3x3/2 96->128", 96, 128, 3, 2, 1, (96, 128)),
    ("layer3 3x3 128->128", 128, 128, 3, 1, 1, (48, 64)),
    ("layer4 3x3 128->128", 128, 128, 3, 1, 1, (24, 32)),
    ("head conv2 3x3 416->256", 416, 256, 3, 1, 1, (48, 64)),
    ("head conv3 1x1 256->128", 256, 128, 1, 1, 0, (48, 64)),
]


def bench_encoder_kernels(reps, frames=32):
    from pips_b200 import encoder_fast as E
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream

    def pair(N, H, W, C):
        p = E._Pair(N, H, W, C, DEV)
        v = torch.randn(N, H, W, p.Cp, device=DEV)
        L.check(lib.pips_split_bf16(L.ptr(v), L.ptr(p.hi), L.ptr(p.lo), v.numel(), st))
        return p

    N = frames
    for name, cin, cout, R, stride, pad, (H, W) in ENC_LAYERS:
        S = 1 if name.startswith("stem") else R
        Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - S) // stride + 1
        x, dy = pair(N, H, W, cin), pair(N, Ho, Wo, cout)
        K = R * S * x.Cp
        dw = torch.empty(cout, K, device=DEV)
        n = lib.pips_conv_wgrad_scratch_floats(N, Ho, Wo, cout, K)
        sc = torch.empty(max(n, 1), device=DEV)
        fn = lambda: L.check(lib.pips_conv_wgrad(L.ptr(dy.hi), L.ptr(dy.lo), dy.Cp, 1, L.ptr(x.hi), L.ptr(x.lo), N, H, W, x.Cp, cout,
                                                 R, S, stride, stride, pad, pad, L.ptr(sc), L.ptr(dw), st))
        ms = timed(fn, reps, 3)
        flop = 2.0 * N * Ho * Wo * cout * (7 * 7 * 3 if name.startswith("stem") else R * S * cin)
        print(f"conv_wgrad {name:30s} {N} frames: {ms * 1e3:8.1f} us, {flop / ms / 1e9:6.1f} TFLOP/s useful")
        del x, dy, dw, sc
    for C, (H, W), dil in ((64, (192, 256), None), (96, (96, 128), (192, 256)), (256, (48, 64), None)):
        y = torch.randn(N, H, W, C, device=DEV)
        stt = torch.rand(N, 2, C, device=DEV)
        g0 = torch.randn_like(y)
        Hd, Wd = dil or (H, W)
        out = E._Pair(N, Hd, Wd, C, DEV)
        sc = torch.empty(lib.pips_inorm_grad_scratch_floats(N, H * W, C), device=DEV)
        fn = lambda: L.check(lib.pips_inorm_grad(L.ptr(y), L.ptr(stt), None, None, 1, 0, L.ptr(g0), None, None, N, H, W, C, L.ptr(sc),
                                                 L.ptr(out.hi), L.ptr(out.lo), out.Cp, *(dil or (0, 0)), None, st))
        ms = timed(fn, reps, 3)
        print(f"inorm_grad {N}x{H}x{W}x{C}{' dilated' if dil else ''}: {ms * 1e3:8.1f} us")
    g = torch.randn(N, 48, 64, 416, device=DEV)
    for (Hs, Ws, C, off) in ((192, 256, 64, 0), (96, 128, 96, 64), (48, 64, 128, 160), (24, 32, 128, 288)):
        out = torch.empty(N, Hs, Ws, C, device=DEV)
        fn = lambda: L.check(lib.pips_resize_grad(L.ptr(g), 416, off, N, 48, 64, L.ptr(out), Hs, Ws, C, st))
        print(f"resize_grad {Hs}x{Ws}x{C} <- 48x64: {timed(fn, reps, 3) * 1e3:8.1f} us")


def bench_encoder(reps):
    from pips_b200.encoder import Encoder
    enc = Encoder(output_dim=128, stride=8).to(DEV)
    old = strict_fp32()
    try:
        for frames in (32, 128):
            rgbs = po.smooth_video(frames // 8, 8, 384, 512, seed=1).to(DEV).float()
            dfm = torch.randn(frames // 8, 8, 128, 48, 64, device=DEV)
            for name in ("torch", "cuda"):
                def step():
                    enc.zero_grad(set_to_none=True)
                    if name == "cuda":
                        f = torch_path.encoder_cuda(enc, rgbs)
                    else:
                        x = 2 * (rgbs / 255.0) - 1.0
                        f = enc(x.flatten(0, 1)).view(dfm.shape)
                    f.backward(dfm)
                try:
                    ms = timed(step, reps, warm=1)
                    gib = peak_of(step)
                    print(f"encoder fwd+bwd {frames} frames 384x512 {name:5s}: {ms:8.1f} ms, peak {gib:6.2f} GiB above inputs")
                except torch.cuda.OutOfMemoryError:
                    print(f"encoder fwd+bwd {frames} frames 384x512 {name:5s}: does not fit in "
                          f"{torch.cuda.get_device_properties(0).total_memory / 2**30:.0f} GiB")
                torch.cuda.empty_cache()
            del rgbs, dfm
    finally:
        torch.backends.cudnn.enabled, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def bench_encoder_step(reps):
    for B in (4, 16):
        N, iters = 768, 4
        rgbs = po.smooth_video(B, 8, 384, 512, seed=1).to(DEV)
        xys = po.random_queries(B, N, 384, 512, seed=2).to(DEV)
        g = torch.Generator().manual_seed(3)
        tg = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 3.0, 1)).to(DEV)
        vg = torch.ones(B, 8, N, device=DEV)
        va = torch.ones(B, 8, N, device=DEV)
        for encoder in ("torch", "cuda"):
            m = Pips(S=8, stride=8, loss_path="fused", mixer_path="cuda", encoder_path=encoder).to(DEV).train()
            m.load_state_dict(po.init_state_dict(seed=3, head_scale=0.05))

            def step():
                m.zero_grad(set_to_none=True)
                _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
                sum(losses).backward()
            label = f"training step B={B}, N={N}, {iters} iterations (mixer cuda, fused loss), encoder {encoder:5s}"
            try:
                ms = timed(step, reps, warm=1)
                gib = peak_of(step)
                print(f"{label}: {ms:8.1f} ms, peak {gib:6.2f} GiB")
            except torch.cuda.OutOfMemoryError:
                print(f"{label}: does not fit in {torch.cuda.get_device_properties(0).total_memory / 2**30:.0f} GiB")
            del m
            torch.cuda.empty_cache()
        del rgbs


def corr_inputs(B, N=768, H8=48, W8=64, seed=5):
    """4 iterations' ffeat rows (B*N, 8, 128) and coordinates (B, 8, N, 2), channels-last levels of an avg-pooled
    pyramid, and an upstream gradient per iteration: forward_torch's correlation inputs at 384 x 512, stride 8"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    fm = torch.randn(B * 8, H8, W8, 128, device=DEV, generator=g)
    levels = [fm]
    for _ in range(3):
        levels.append(torch.nn.functional.avg_pool2d(levels[-1].permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).contiguous())
    ff = [torch.randn(B * N, 8, 128, device=DEV, generator=g) for _ in range(4)]
    co = [torch.rand(B, 8, N, 2, device=DEV, generator=g) * torch.tensor([W8 - 1.0, H8 - 1.0], device=DEV) for _ in range(4)]
    dc = [torch.randn(B * N, 8, 196, device=DEV, generator=g) for _ in range(4)]
    return ff, levels, co, dc


def torch_corr(ff_rows, levels, coords):
    """forward_torch's correlation (nets/pips.py:355-398): matmul all-pairs volumes and grid_sample, (B*N, S, 196)"""
    B, S, N, _ = coords.shape
    ffeats = ff_rows.reshape(B, N, S, 128).permute(0, 2, 1, 3)
    offs = torch.linspace(-3, 3, 7, device=DEV)
    window = torch.stack(torch.meshgrid(offs, offs, indexing="ij"), dim=-1).view(1, 7, 7, 2)
    taps = []
    for i, lv in enumerate(levels):
        f = lv.reshape(B, S, *lv.shape[1:]).permute(0, 1, 4, 2, 3)          # (B,S,C,h,w), channels-last strides
        h, w = f.shape[-2:]
        v = torch.matmul(ffeats, f.flatten(3)).reshape(B, S, N, h, w) / torch.sqrt(torch.tensor(128.0))
        loc = coords.reshape(B * S * N, 1, 1, 2) / 2 ** i + window
        grid = torch.cat([2 * loc[..., :1] / (w - 1) - 1, 2 * loc[..., 1:] / (h - 1) - 1], dim=-1)
        taps.append(torch.nn.functional.grid_sample(v.reshape(B * S * N, 1, h, w), grid, align_corners=True).view(B, S, N, -1))
    return torch.cat(taps, dim=-1).permute(0, 2, 1, 3).reshape(B * N, S, -1)


def bench_corr(reps):
    """the correlation's forward + backward over 4 iterations, torch against local_corr_cuda, and each backward kernel"""
    old = strict_fp32()
    try:
        for B in (4, 16):
            ff, levels, co, dc = corr_inputs(B)
            for name in ("torch", "cuda"):
                def step():
                    lv = [l.requires_grad_(True) for l in levels]
                    fr = [f.requires_grad_(True) for f in ff]
                    loss = 0
                    for i in range(4):
                        out = torch_path.local_corr_cuda(fr[i], lv, co[i]) if name == "cuda" else torch_corr(fr[i], lv, co[i])
                        loss = loss + (out * dc[i]).sum()
                    loss.backward()
                    for t in lv + fr:
                        t.grad = None
                try:
                    ms = timed(step, reps)
                    gib = peak_of(step)
                    print(f"correlation fwd+bwd, 4 iterations, B={B}, N=768, 48x64 {name:5s}: {ms:8.2f} ms, peak "
                          f"{gib * 1024:7.0f} MiB above inputs")
                except torch.cuda.OutOfMemoryError:
                    print(f"correlation fwd+bwd, 4 iterations, B={B}, N=768, 48x64 {name:5s}: out of memory")
                torch.cuda.empty_cache()
            for t in levels + ff:
                t.requires_grad_(False)
            # each backward kernel alone; bytes it must move, from shapes
            lib = L.load()
            st = torch.cuda.current_stream().cuda_stream
            N, M = 768, B * 8 * 768
            lv_bytes = sum(l.numel() for l in levels) * 4
            dff = torch.empty(B * N, 8, 128, device=DEV)
            dls = [torch.empty_like(l) for l in levels]
            fn = lambda: L.check(lib.pips_corr_grad_feats(L.ptr_array(levels), B, 8, N, 48, 64, L.ptr(co[0]), L.ptr(dc[0]), 196,
                                                          L.ptr(dff), st))
            ms = timed(fn, 20, 3)
            # compulsory traffic: read every level pixel once, each unit's 196 dcorr and coordinates, write its dffeat row;
            # the footprint boxes move 4 x 64 px x 512 B per unit, mostly from L2 (neighbouring tracks share pixels)
            byt = lv_bytes + M * (196 * 4 + 8 + 512)
            print(f"corr_grad_feats B={B} (M={M}): {ms * 1e3:8.1f} us, {byt / 2**20:.0f} MiB compulsory, "
                  f"{byt / (ms * 1e-3) / 3.35e12:.2f} of 3.35 TB/s; footprint boxes {M * 4 * 64 * 512 / 2**30:.1f} GiB "
                  f"at {M * 4 * 64 * 512 / (ms * 1e-3) / 1e12:.1f} TB/s")
            fn = lambda: L.check(lib.pips_corr_grad_levels(B, 8, N, 48, 64, L.ptr(co[0]), L.ptr(ff[0]), L.ptr(dc[0]), 196,
                                                           L.ptr_array(dls), st))
            ms = timed(fn, 20, 3)
            # compulsory traffic: write every level pixel once, read each unit's ffeat row, 196 dcorr and coordinates once
            byt = lv_bytes + M * (512 + 196 * 4 + 8)
            print(f"corr_grad_levels B={B} (M={M}): {ms * 1e3:8.1f} us, {byt / 2**20:.0f} MiB compulsory, "
                  f"{byt / (ms * 1e-3) / 3.35e12:.2f} of 3.35 TB/s")
            del ff, levels, co, dc, dff, dls
            torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.enabled, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def bench_corr_step(reps):
    for B in (4, 16):
        N, iters = 768, 4
        rgbs = po.smooth_video(B, 8, 384, 512, seed=1).to(DEV)
        xys = po.random_queries(B, N, 384, 512, seed=2).to(DEV)
        g = torch.Generator().manual_seed(3)
        tg = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 3.0, 1)).to(DEV)
        vg = torch.ones(B, 8, N, device=DEV)
        va = torch.ones(B, 8, N, device=DEV)
        for corr in ("torch", "cuda"):
            m = Pips(S=8, stride=8, loss_path="fused", mixer_path="cuda", encoder_path="cuda", corr_path=corr).to(DEV).train()
            m.load_state_dict(po.init_state_dict(seed=3, head_scale=0.05))

            def step():
                m.zero_grad(set_to_none=True)
                _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
                sum(losses).backward()
            label = f"training step B={B}, N={N}, {iters} iterations (mixer, encoder cuda, fused loss), corr {corr:5s}"
            try:
                ms = timed(step, reps, warm=1)
                gib = peak_of(step)
                print(f"{label}: {ms:8.1f} ms, peak {gib:6.2f} GiB")
            except torch.cuda.OutOfMemoryError:
                print(f"{label}: does not fit in {torch.cuda.get_device_properties(0).total_memory / 2**30:.0f} GiB")
            del m
            torch.cuda.empty_cache()
        del rgbs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--only", choices=("mixer", "encoder", "corr"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py measures on the GPU; no CUDA device found")
    print(f"card: {card()}")
    if args.only in (None, "mixer"):
        bench_kernels(args.reps)
        bench_mixer(args.reps)
        if not args.skip_step:
            bench_step(args.reps)
    if args.only in (None, "encoder"):
        bench_encoder_kernels(args.reps)
        bench_encoder(args.reps)
        if not args.skip_step:
            bench_encoder_step(args.reps)
    if args.only in (None, "corr"):
        bench_corr(args.reps)
        if not args.skip_step:
            bench_corr_step(args.reps)


if __name__ == "__main__":
    main()
