"""Training with the fused score-map loss (Pips(loss_path='fused')): torch_path.fused_score_map_loss and its backward
kernels (csrc/scoremap_grad.cu) against autograd through the dense torch_path.score_map_loss in fp64, the training
step against loss_path='torch', determinism, memory and routing."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path

DEV = "cuda:0"


def _rel(a, b):
    """norm-wise relative error ||a - b|| / ||b|| (in fp64)"""
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-300)).item()


def _pyramid(fmaps):
    """the 4 levels of torch_path.forward_torch: avg_pool2d from fmaps (B,S,C,H8,W8)"""
    B, S = fmaps.shape[:2]
    pyr = [fmaps]
    for _ in range(3):
        f = F.avg_pool2d(pyr[-1].flatten(0, 1), 2, stride=2)
        pyr.append(f.reshape(B, S, *f.shape[1:]))
    return pyr


def _dense_loss(ffeats, pyr, tg, vg, va):
    """the score maps of forward_torch (nets/pips.py:384-398, :504-511) and score_map_loss over them"""
    B, S, N, _ = ffeats[0].shape
    H8, W8 = pyr[0].shape[-2:]
    fcps = []
    for ff in ffeats:
        vols = [torch.matmul(ff, f.flatten(3)).reshape(B, S, N, *f.shape[-2:]) / (128 ** 0.5) for f in pyr]
        fcps.append(sum(F.interpolate(v.flatten(0, 1), (H8, W8), mode="bilinear", align_corners=True).reshape(B, S, N, H8, W8)
                        for v in vols))
    return torch_path.score_map_loss(torch.stack(fcps, dim=2), tg, vg, va)


def _problem(H8, W8, N, I, B=1, seed=0):
    """fmaps (B,S,128,H8,W8), I ffeats (B,S,N,128) and ground truth in feature pixels with rows dropped for each reason
    and targets on the map edges"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    S = 8
    fmaps = torch.randn(B, S, 128, H8, W8, device=DEV, generator=g, dtype=torch.float64)
    ffeats = [torch.randn(B, S, N, 128, device=DEV, generator=g, dtype=torch.float64) * 0.7 for _ in range(I)]
    tg = torch.rand(B, S, N, 2, device=DEV, generator=g, dtype=torch.float64) * torch.tensor([W8 + 2.0, H8 + 2.0], device=DEV) - 1.0
    vg = (torch.rand(B, S, N, device=DEV, generator=g) > 0.2).float()
    va = (torch.rand(B, S, N, device=DEV, generator=g) > 0.1).float()
    edges = [(0, 0), (W8 - 1, 0), (0, H8 - 1), (W8 - 1, H8 - 1), (W8 // 2, 0), (0, H8 // 2)]
    for s in range(S):
        if N > 1:
            tg[0, s, s % N] = torch.tensor(edges[s % len(edges)], dtype=torch.float64)
        else:
            tg[0, s, 0] = torch.tensor(edges[s % len(edges)], dtype=torch.float64)
            vg[0, s, 0] = va[0, s, 0] = 1.0
    if N > 3:
        tg[0, 0, 1] = torch.tensor([W8 - 0.5, 1.0])                 # rounds to W8: out of bounds
        tg[0, 1, 2] = torch.tensor([2.0, -0.6])                     # rounds to -1: out of bounds
        vg[0, 2, 3] = 0.0
        va[0, 3, 3] = 0.0
    return fmaps, ffeats, tg.float(), vg, va                        # fp32 positions: both paths round the same values


def _grads(dtype, fmaps, ffeats, tg, vg, va, fused):
    fm = fmaps.detach().to(dtype).requires_grad_(True)
    ff = [f.detach().to(dtype).requires_grad_(True) for f in ffeats]
    pyr = _pyramid(fm)
    if fused:
        loss = torch_path.fused_score_map_loss(ff, pyr, tg.float(), vg, va)
    else:
        loss = _dense_loss(ff, pyr, tg.to(dtype), vg.to(dtype), va.to(dtype))
    loss.backward()
    return loss.detach(), [f.grad for f in ff], fm.grad


CASES = [  # (H8, W8, N, I)
    (16, 16, 1, 1),
    (16, 16, 100, 4),
    (45, 80, 300, 6),          # odd levels: 45 -> 22 -> 11 -> 5, 80 -> 40 -> 20 -> 10
    (45, 80, 1, 4),
    (48, 64, 100, 6),
    (48, 64, 300, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("H8,W8,N,I", CASES)
def test_gradients_match_fp64(H8, W8, N, I):
    prob = _problem(H8, W8, N, I, seed=H8 * 1000 + N + I)
    l64, df64, dm64 = _grads(torch.float64, *prob, fused=False)
    l32, df32, dm32 = _grads(torch.float32, *prob, fused=False)
    lf, dff, dmf = _grads(torch.float32, *prob, fused=True)
    assert lf.dim() == 0 and lf.dtype == torch.float32
    e_loss, e_loss32 = abs(lf.item() - l64.item()) / abs(l64.item()), abs(l32.item() - l64.item()) / abs(l64.item())
    e_df = max(_rel(a, b) for a, b in zip(dff, df64))
    e_df32 = max(_rel(a, b) for a, b in zip(df32, df64))
    e_dm, e_dm32 = _rel(dmf, dm64), _rel(dm32, dm64)
    print(f"{H8}x{W8} N={N} I={I}: fused vs fp64: loss {e_loss:.2e}, dF {e_df:.2e}, dfmaps {e_dm:.2e} | "
          f"dense fp32 vs fp64: loss {e_loss32:.2e}, dF {e_df32:.2e}, dfmaps {e_dm32:.2e}")
    assert e_loss <= 1e-5
    assert e_df <= 1e-4 and e_dm <= 1e-4


@pytest.mark.gpu
def test_all_rows_dropped_gives_zero_loss_and_gradients():
    fmaps, ffeats, tg, vg, va = _problem(16, 16, 100, 3, seed=3)
    loss, dfs, dm = _grads(torch.float32, fmaps, ffeats, tg, torch.zeros_like(vg), va, fused=True)
    print(f"all rows dropped: loss {loss.item()}, max |dF| {max(d.abs().max().item() for d in dfs)}, max |dfmaps| {dm.abs().max().item()}")
    assert loss.item() == 0.0
    assert all(torch.equal(d, torch.zeros_like(d)) for d in dfs) and torch.equal(dm, torch.zeros_like(dm))


@pytest.mark.gpu
def test_backward_is_deterministic():
    prob = _problem(48, 64, 300, 4, B=2, seed=11)
    a = _grads(torch.float32, *prob, fused=True)
    b = _grads(torch.float32, *prob, fused=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert all(torch.equal(x, y) for x, y in zip(a[1], b[1]))


def _train_model(loss_path, seed=3):
    sd = po.init_state_dict(seed=seed, head_scale=0.05)
    m = Pips(S=8, stride=8, loss_path=loss_path).to(DEV).train()
    m.load_state_dict(sd, strict=True)
    return m


def _train_inputs(B=2, N=64, H=128, W=128, seed=5):
    rgbs = po.smooth_video(B, 8, H, W, seed=100 + seed).to(DEV)
    xys = po.random_queries(B, N, H, W, seed=200 + seed).to(DEV)
    g = torch.Generator().manual_seed(400 + seed)
    tg = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 3.0, 1)).to(DEV)
    vg = (torch.rand(B, 8, N, generator=g) > 0.2).float().to(DEV)
    va = (torch.rand(B, 8, N, generator=g) > 0.1).float().to(DEV)
    return rgbs, xys, tg, vg, va


def _train_step(m, rgbs, xys, tg, vg, va, iters=4):
    """train.py:82-95: a forward with is_train=True and gradients on, then the backward of the summed losses"""
    m.zero_grad(set_to_none=True)
    _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    sum(losses).backward()
    return [l.detach() for l in losses], {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


@pytest.mark.gpu
def test_training_step_matches_torch_path(monkeypatch):
    # fnet's backward runs outside the strict-fp32 forward context, in cuDNN's default TF32 math, where a 1e-5 change of
    # its input gradient flips roundings at the 1e-3 level: strict, deterministic fp32 here, so the comparison measures
    # the score-map loss's gradients
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    inputs = _train_inputs()
    lt, gt = _train_step(_train_model("torch"), *inputs)
    lf, gf = _train_step(_train_model("fused"), *inputs)
    rel_l = [abs(a.item() - b.item()) / abs(b.item()) for a, b in zip(lf, lt)]
    assert gt.keys() == gf.keys() and len(gt) > 0
    total = torch.cat([g.flatten() for g in gt.values()]).double().norm().item()
    rel_all = _rel(torch.cat([gf[n].flatten() for n in gt]), torch.cat([gt[n].flatten() for n in gt]))
    # Some biases have an exact gradient of 0: the following normalisation removes them (the token-mixing FC2 biases add
    # one constant to all 512 channels of a token before a LayerNorm; fnet's conv biases feed an InstanceNorm).  Their
    # .grad is rounding noise, ~1e-7 of the whole gradient's norm on either path, so they are compared to that norm.
    zero = {n for n in gt if gt[n].double().norm().item() <= 1e-5 * total}
    assert all(n.endswith("bias") for n in zero), zero
    rel_g = {n: _rel(gf[n], gt[n]) for n in gt if n not in zero}
    noise = max([(gf[n] - gt[n]).double().norm().item() / total for n in zero], default=0.0)
    worst = max(rel_g, key=rel_g.get)
    print(f"losses fused {[l.item() for l in lf]} vs torch {[l.item() for l in lt]}: relative {rel_l}; all gradients "
          f"{rel_all:.2e}; {len(rel_g)} parameter gradients, worst {worst} {rel_g[worst]:.2e}; {len(zero)} zero-gradient "
          f"biases, difference {noise:.2e} of the gradient's norm")
    assert max(rel_l) <= 1e-5
    assert rel_all <= 1e-4 and rel_g[worst] <= 1e-4 and noise <= 1e-6


@pytest.mark.gpu
def test_memory_at_train_shape():
    """train.py's per-GPU shape: B=4, N=768, I=4, 8 x 384 x 512, stride 8 (48 x 64 maps)."""
    B, S, N, I, H8, W8 = 4, 8, 768, 4, 48, 64
    prob = _problem(H8, W8, N, I, B=B, seed=9)
    fmaps, ffeats, tg, vg, va = prob
    fmaps = fmaps.float()
    ffeats = [f.float() for f in ffeats]
    del prob
    peaks = {}
    for name in ("fused", "dense"):
        fm = fmaps.clone().requires_grad_(True)
        ff = [f.clone().requires_grad_(True) for f in ffeats]
        pyr = _pyramid(fm)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        if name == "fused":
            loss = torch_path.fused_score_map_loss(ff, pyr, tg.float(), vg, va)
        else:
            loss = _dense_loss(ff, pyr, tg.float(), vg, va)
        loss.backward()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del fm, ff, pyr, loss
        torch.cuda.empty_cache()
    one_map = 4 * B * S * I * N * H8 * W8
    print(f"score-map loss forward + backward at B={B}, N={N}, I={I}, {H8}x{W8}: peak above inputs: fused "
          f"{peaks['fused'] / 2**20:.0f} MiB, dense {peaks['dense'] / 2**20:.0f} MiB "
          f"(one (B,S,I,N,H8,W8) fp32 tensor is {one_map / 2**20:.0f} MiB)")
    assert peaks["fused"] <= 512 * 2**20


@pytest.mark.gpu
def test_routing_under_fused(monkeypatch):
    rgbs, xys, tg, vg, va = _train_inputs(B=1, N=16, seed=8)
    calls, dense = [], []
    real_fwd, real_loss = torch_path.forward_torch, torch_path.score_map_loss

    def spy_fwd(*a, **k):
        calls.append(1)
        return real_fwd(*a, **k)

    def spy_loss(*a, **k):
        dense.append(1)
        return real_loss(*a, **k)

    monkeypatch.setattr(torch_path, "forward_torch", spy_fwd)
    monkeypatch.setattr(torch_path, "score_map_loss", spy_loss)
    monkeypatch.setenv("PIPS_B200_LOSSES", "fused")
    m = Pips(S=8, stride=8).to(DEV).eval()
    m.load_state_dict(po.init_state_dict(seed=3, head_scale=0.05))
    assert m.loss_path == "fused"
    with torch.no_grad():
        _, _, _, losses = m(xys, rgbs, iters=2, trajs_g=tg, vis_g=vg, valids=va)
    assert calls == [] and dense == [] and losses[2].dim() == 0           # the CUDA path, as under 'cuda'
    _, _, _, losses = m(xys, rgbs, iters=2, trajs_g=tg, vis_g=vg, valids=va)
    assert calls == [1] and dense == [] and losses[2].requires_grad      # gradients on: fused loss on the torch path
    with torch.no_grad():
        m(xys, rgbs, iters=2, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert calls == [1, 1] and dense == []


def test_cpu_tensors_keep_the_dense_loss_under_fused(monkeypatch):
    from tests.golden.make_golden import LOSS_CASE, case_inputs, loss_targets
    c = LOSS_CASE
    dense = []
    real_loss = torch_path.score_map_loss

    def spy_loss(*a, **k):
        dense.append(1)
        return real_loss(*a, **k)

    monkeypatch.setattr(torch_path, "score_map_loss", spy_loss)
    m = Pips(S=8, stride=8, loss_path="fused").train()
    m.load_state_dict(po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"]))
    rgbs, xys, _ = case_inputs(c)
    tg, vg, va = loss_targets(c, xys)
    _, _, _, losses = m(xys[:1, :3], rgbs[:1], iters=1, trajs_g=tg[:1, :, :3], vis_g=vg[:1, :, :3], valids=va[:1, :, :3],
                        is_train=True)
    assert dense == [1]
    sum(losses).backward()
    assert m.delta_block.to_delta[0].weight.grad is not None
    with pytest.raises(RuntimeError):
        torch_path.fused_score_map_loss([torch.zeros(1, 8, 2, 128)], [torch.zeros(1, 8, 128, 16 >> l, 16 >> l) for l in range(4)],
                                        torch.zeros(1, 8, 2, 2), torch.ones(1, 8, 2), torch.ones(1, 8, 2))


def test_scoremap_grad_entry_points_validate_arguments_without_gpu():
    lib = L.load()
    p = C.c_void_p(256)
    q = C.c_void_p(264)                                                   # 8-byte aligned only
    feats = lib.pips_scoremap_grad_feats
    assert feats(None, p, p, 4, 1, 8, 4, 16, 16, p, p, p, None) != 0
    assert b"pips_scoremap_grad_feats: null pointer" in lib.pips_last_error()
    assert feats(p, p, p, 4, 1, 8, 4, 16, 16, p, None, p, None) != 0                 # no coefficients
    assert feats(p, p, p, 4, 1, 7, 4, 16, 16, p, p, p, None) != 0                    # S != 8
    assert b"S must be 8" in lib.pips_last_error()
    assert feats(p, p, p, 0, 1, 8, 4, 16, 16, p, p, p, None) != 0                    # no iterations
    assert feats(p, p, p, 4, 1, 8, 0, 16, 16, p, p, p, None) != 0                    # no particles
    assert b"empty problem" in lib.pips_last_error()
    assert feats(q, p, p, 4, 1, 8, 4, 16, 16, p, p, p, None) != 0                    # misaligned G
    assert b"16-byte aligned" in lib.pips_last_error()
    assert feats(p, p, p, 4, 1, 8, 4, 16, 16, p, p, q, None) != 0                    # misaligned output
    assert b"16-byte aligned" in lib.pips_last_error()

    basis = lib.pips_scoremap_grad_basis
    assert basis(p, p, None, p, 4, 1, 8, 4, 16, 16, p, p, p, None) != 0
    assert b"pips_scoremap_grad_basis: null pointer" in lib.pips_last_error()
    assert basis(p, p, p, p, 4, 1, 9, 4, 16, 16, p, p, p, None) != 0                 # S != 8
    assert b"S must be 8" in lib.pips_last_error()
    assert basis(p, p, p, p, 4, 1, 8, 4, 0, 16, p, p, p, None) != 0                  # empty map
    assert b"empty problem" in lib.pips_last_error()
    assert basis(q, p, p, p, 4, 1, 8, 4, 16, 16, p, p, p, None) != 0                 # misaligned G
    assert b"16-byte aligned" in lib.pips_last_error()

    adj = lib.pips_scoremap_basis_grad
    lv = (C.c_void_p * 4)(256, 256, 256, 256)
    assert adj(None, 8, 16, 16, lv, None) != 0
    assert b"pips_scoremap_basis_grad: null pointer" in lib.pips_last_error()
    assert adj(p, 0, 16, 16, lv, None) != 0
    assert b"empty problem" in lib.pips_last_error()
    assert adj(p, 8, 4, 16, lv, None) != 0                                          # too small for 4 levels
    assert b"too small" in lib.pips_last_error()
    assert adj(q, 8, 16, 16, lv, None) != 0                                         # misaligned dG
    assert b"16-byte aligned" in lib.pips_last_error()
    lv_null = (C.c_void_p * 4)(256, 256, None, 256)
    assert adj(p, 8, 16, 16, lv_null, None) != 0
    assert b"null pyramid level" in lib.pips_last_error()
