"""Training the DeltaBlock mixer on the sm_90a kernels (Pips(mixer_path='cuda'), torch_path.delta_block_cuda): the
weight-gradient GEMM, the pre-activation GEMM epilogues and the fused LayerNorm / token-mixing backward against fp64,
the whole mixer's forward and backward against fp64 autograd of the DeltaBlock module, determinism, a training step
against mixer_path='torch', memory, routing, and argument validation without a GPU.  Errors are norm-wise relative
errors against fp64 (``_rel``); bf16x3 products carry about 2^-17 relative error each."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path
from pips_b200.pips import DeltaBlock

DEV = "cuda:0"


def _rel(a, b):
    """norm-wise relative error ||a - b|| / ||b|| (in fp64)"""
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-300)).item()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _split(v, rows=None):
    """(hi, lo) bf16 of the fp32 matrix v, in buffers of `rows` rows (default: v's)"""
    v = v.float().contiguous()
    rows = rows or v.shape[0]
    hi = torch.full((rows, v.shape[1]), float("nan"), dtype=torch.bfloat16, device=DEV)
    lo = hi.clone()
    L.check(L.load().pips_split_bf16(L.ptr(v), L.ptr(hi), L.ptr(lo), v.numel(), _st()), "pips_split_bf16")
    return hi, lo


def _wgrad(g, x):
    lib = L.load()
    M, N = g.shape
    K = x.shape[1]
    gp, xp = _split(g), _split(x)
    dw = torch.full((N, K), float("nan"), device=DEV)
    n = lib.pips_wgrad_scratch_floats(M, N, K)
    scratch = torch.full((max(n, 1),), float("nan"), device=DEV)
    L.check(lib.pips_wgrad(L.ptr(gp[0]), L.ptr(gp[1]), N, L.ptr(xp[0]), L.ptr(xp[1]), K, M, N, K, L.ptr(scratch), L.ptr(dw),
                           _st()), "pips_wgrad")
    return dw


WGRAD_SHAPES = [  # (M, N, K): FC2 (dx^T h), FC1 (dh^T y), input layer, head over pooled rows; M not a multiple of a tile
    (8 * 3072, 512, 2048),
    (8 * 3071, 2048, 512),
    (8 * 37, 512, 576),
    (3072, 1040, 512),
    (37, 1040, 512),
    (8, 512, 576),
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", WGRAD_SHAPES)
def test_wgrad_matches_fp64(M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    G = torch.randn(M, N, device=DEV, generator=g)
    X = torch.randn(M, K, device=DEV, generator=g) + 0.5
    dw = _wgrad(G, X)
    ref = G.double().t() @ X.double()
    e, e32 = _rel(dw, ref), _rel(G.t() @ X, ref)
    print(f"wgrad M={M} N={N} K={K}: {e:.2e} (fp32 torch {e32:.2e})")
    assert torch.isfinite(dw).all()
    assert e <= 1e-4
    assert torch.equal(dw, _wgrad(G, X))                                  # the same bits on a second run


@pytest.mark.gpu
@pytest.mark.parametrize("M,N", [(8 * 3071, 2048), (37, 1040), (300, 512)])
def test_colsum_matches_fp64(M, N):
    lib = L.load()
    G = torch.randn(M, N, device=DEV) + 0.25
    out = torch.empty(N, device=DEV)
    n = lib.pips_colsum_scratch_floats(M, N)
    scratch = torch.empty(max(n, 1), device=DEV)
    L.check(lib.pips_colsum(L.ptr(G), None, None, N, M, N, L.ptr(scratch), L.ptr(out), _st()), "pips_colsum")
    hi, lo = _split(G)
    out2 = torch.empty(N, device=DEV)
    L.check(lib.pips_colsum(None, L.ptr(hi), L.ptr(lo), N, M, N, L.ptr(scratch), L.ptr(out2), _st()), "pips_colsum")
    ref = G.double().sum(0)
    print(f"colsum M={M} N={N}: fp32 {_rel(out, ref):.2e}, (hi, lo) {_rel(out2, ref):.2e}")
    assert _rel(out, ref) <= 1e-5 and _rel(out2, ref) <= 1e-4


def _gelu_grad64(x):
    return 0.5 * torch.erfc(-x / math.sqrt(2.0)) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [8 * 37, 2048 + 8])
def test_pre_activation_epilogues_match_fp64(M):
    lib = L.load()
    N, K = 2048, 512
    g = torch.Generator(device=DEV).manual_seed(M)
    A = torch.randn(M, K, device=DEV, generator=g)
    W = torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)
    b = torch.randn(N, device=DEV, generator=g)
    b[::7] += 9.0                                                         # pre-activations in both GELU tails, |x| > 6
    b[3::7] -= 9.0
    ap, wp = _split(A, 256 * ((M + 255) // 256)), _split(W)
    hi = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    lo = hi.clone()
    pre = torch.full((M, N), float("nan"), device=DEV)
    L.check(lib.pips_gemm_tc_aux(L.ptr(ap[0]), L.ptr(ap[1]), K, ap[0].shape[0], L.ptr(wp[0]), L.ptr(wp[1]), K, N, M, N, K,
                                 L.ptr(b), L.EPI_BIAS_GELU_PRE, None, 0, L.ptr(hi), L.ptr(lo), N, L.ptr(pre), N, _st()),
            "pips_gemm_tc_aux")
    h64 = A.double() @ W.double().t() + b.double()
    gelu64 = F.gelu(h64)
    e_pre, e_gelu = _rel(pre, h64), _rel(hi.double() + lo.double(), gelu64)
    tails = h64.abs() > 6
    e_tail = _rel((hi.double() + lo.double())[tails], gelu64[tails])
    # GELU_GRAD: (A W^T + b) * gelu'(pre), with the pre-activation just written
    dh_hi = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    dh_lo = dh_hi.clone()
    L.check(lib.pips_gemm_tc_aux(L.ptr(ap[0]), L.ptr(ap[1]), K, ap[0].shape[0], L.ptr(wp[0]), L.ptr(wp[1]), K, N, M, N, K,
                                 L.ptr(b), L.EPI_GELU_GRAD, None, 0, L.ptr(dh_hi), L.ptr(dh_lo), N, L.ptr(pre), N, _st()),
            "pips_gemm_tc_aux")
    dref = h64 * _gelu_grad64(pre.double())
    e_grad = _rel(dh_hi.double() + dh_lo.double(), dref)
    e_gtail = _rel((dh_hi.double() + dh_lo.double())[tails], dref[tails])
    print(f"M={M}: pre {e_pre:.2e}, gelu {e_gelu:.2e} (tails {e_tail:.2e}), gelu' product {e_grad:.2e} (tails {e_gtail:.2e}); "
          f"{int(tails.sum())} tail elements")
    assert tails.sum() > 1000
    assert max(e_pre, e_gelu, e_tail, e_grad, e_gtail) <= 1e-4


def _tok_params(seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = {"ln1_w": 1 + 0.2 * torch.randn(512, generator=g, device=DEV), "ln1_b": 0.1 * torch.randn(512, generator=g, device=DEV),
         "tok_w1": torch.randn(32, 8, generator=g, device=DEV) / math.sqrt(8), "tok_b1": 0.3 * torch.randn(32, generator=g, device=DEV),
         "tok_w2": torch.randn(8, 32, generator=g, device=DEV) / math.sqrt(32), "tok_b2": 0.1 * torch.randn(8, generator=g, device=DEV),
         "ln2_w": 1 + 0.2 * torch.randn(512, generator=g, device=DEV), "ln2_b": 0.1 * torch.randn(512, generator=g, device=DEV)}
    return {k: v.contiguous() for k, v in P.items()}


def _tok_block64(x, P):
    """the token-mixing PreNormResidual and the LayerNorm of the channel-mixing one, in fp64: (x_mid, LN2(x_mid))"""
    u = F.layer_norm(x, (512,), P["ln1_w"], P["ln1_b"])
    h = F.gelu(torch.einsum("js,rsc->rjc", P["tok_w1"], u) + P["tok_b1"][None, :, None])
    x_mid = torch.einsum("sj,rjc->rsc", P["tok_w2"], h) + P["tok_b2"][None, :, None] + x
    return x_mid, F.layer_norm(x_mid, (512,), P["ln2_w"], P["ln2_b"])


@pytest.mark.gpu
@pytest.mark.parametrize("seqs", [1, 37, 700])
def test_tokenmix_grad_matches_fp64(seqs):
    lib = L.load()
    g = torch.Generator(device=DEV).manual_seed(seqs)
    P = _tok_params(seqs)
    x = torch.randn(seqs, 8, 512, generator=g, device=DEV) * 2 + 0.5
    dy = torch.randn(seqs, 8, 512, generator=g, device=DEV)
    dxo = torch.randn(seqs, 8, 512, generator=g, device=DEV)
    P64 = {k: v.double().requires_grad_(True) for k, v in P.items()}
    x64 = x.double().requires_grad_(True)
    x_mid, y = _tok_block64(x64, P64)
    ((y * dy.double()).sum() + (x_mid * dxo.double()).sum()).backward()
    xm = x_mid.detach().float().contiguous()
    dx = dxo.clone()
    scratch = torch.empty(lib.pips_tokenmix_grad_scratch_floats(seqs), device=DEV)
    grads = torch.full((2600,), float("nan"), device=DEV)
    L.check(lib.pips_tokenmix_grad(L.ptr(x), L.ptr(xm), L.ptr(dy), L.ptr(dx), seqs,
                                   *(L.ptr(P[k]) for k in ("ln1_w", "ln1_b", "tok_w1", "tok_b1", "tok_w2", "tok_b2", "ln2_w", "ln2_b")),
                                   L.ptr(scratch), L.ptr(grads), _st()), "pips_tokenmix_grad")
    errs = {"dx": _rel(dx, x64.grad)}
    off = 0
    for k in ("ln1_w", "ln1_b", "tok_w1", "tok_b1", "tok_w2", "tok_b2", "ln2_w", "ln2_b"):
        n = P[k].numel()
        ref = P64[k].grad.reshape(-1)
        errs[k] = _rel(grads[off:off + n], ref)             # dxo reaches x_mid directly: no gradient here is 0
        off += n
    print(f"tokenmix backward, {seqs} sequences: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert max(errs.values()) <= 1e-4


def _delta_block(seed, head_scale, dtype=torch.float32):
    sd = po.init_state_dict(seed=seed, head_scale=head_scale)
    m = DeltaBlock().to(DEV, dtype)
    m.load_state_dict({k[len("delta_block."):]: v for k, v in sd.items() if k.startswith("delta_block.")})
    return m


def _mixer_input(R, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(R, 8, 519, generator=g, device=DEV)


def _fwd_bwd(m, x, cuda, dy):
    m.zero_grad(set_to_none=True)
    xr = x.clone().requires_grad_(True)
    out = torch_path.delta_block_cuda(m, xr) if cuda else m(xr)
    (out * dy).sum().backward()
    return out.detach(), xr.grad, {n: p.grad.detach().clone() for n, p in m.named_parameters()}


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 37, 3072])
@pytest.mark.parametrize("head_scale", [0.05, 1.0])
def test_delta_block_cuda_matches_fp64_autograd(R, head_scale):
    m = _delta_block(3, head_scale)
    m64 = _delta_block(3, head_scale, torch.float64)
    x = _mixer_input(R, R)
    dy = torch.randn(R, 8, 130, device=DEV, generator=torch.Generator(device=DEV).manual_seed(R + 1))
    o64, dx64, g64 = _fwd_bwd(m64, x.double(), False, dy.double())
    oc, dxc, gc = _fwd_bwd(m, x, True, dy)
    assert len(gc) == 150
    total = torch.cat([g.flatten() for g in g64.values()]).norm().item()
    zero = {n for n in g64 if g64[n].norm().item() <= 1e-6 * total}
    assert all(n.endswith("0.fn.3.bias") for n in zero), zero
    e = {n: _rel(gc[n], g64[n]) for n in g64 if n not in zero}
    worst = max(e, key=e.get)
    noise = max([(gc[n].double() - g64[n]).norm().item() / total for n in zero], default=0.0)
    e_out, e_dx = _rel(oc, o64), _rel(dxc, dx64)
    e_all = _rel(torch.cat([gc[n].flatten() for n in g64]), torch.cat([g64[n].flatten() for n in g64]))
    msg = ""
    if R <= 37:
        o32, dx32, g32 = _fwd_bwd(m, x, False, dy)
        msg = (f" | fp32 torch: out {_rel(o32, o64):.2e}, dx {_rel(dx32, dx64):.2e}, all gradients "
               f"{_rel(torch.cat([g32[n].flatten() for n in g64]), torch.cat([g64[n].flatten() for n in g64])):.2e}")
    print(f"R={R} head x{head_scale}: out {e_out:.2e}, dx {e_dx:.2e}, all gradients {e_all:.2e}, worst {worst} {e[worst]:.2e}, "
          f"{len(zero)} zero-gradient biases {noise:.2e} of the norm{msg}")
    assert e_out <= 1e-3 and e_dx <= 1e-3 and e[worst] <= 1e-3 and noise <= 1e-5


@pytest.mark.gpu
def test_delta_block_cuda_is_deterministic():
    m = _delta_block(4, 0.05)
    x = _mixer_input(3000, 9)
    dy = torch.randn(3000, 8, 130, device=DEV)
    a, b = _fwd_bwd(m, x, True, dy), _fwd_bwd(m, x, True, dy)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(a[2][n], b[2][n]) for n in a[2])


def _train_model(mixer_path, seed=3):
    m = Pips(S=8, stride=8, loss_path="fused", mixer_path=mixer_path).to(DEV).train()
    m.load_state_dict(po.init_state_dict(seed=seed, head_scale=0.05), strict=True)
    return m


def _train_inputs(B=2, N=64, H=128, W=128, seed=5):
    rgbs = po.smooth_video(B, 8, H, W, seed=100 + seed).to(DEV)
    xys = po.random_queries(B, N, H, W, seed=200 + seed).to(DEV)
    g = torch.Generator().manual_seed(400 + seed)
    tg = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 3.0, 1)).to(DEV)
    vg = (torch.rand(B, 8, N, generator=g) > 0.2).float().to(DEV)
    va = (torch.rand(B, 8, N, generator=g) > 0.1).float().to(DEV)
    return rgbs, xys, tg, vg, va


def _train_step(m, rgbs, xys, tg, vg, va, iters):
    m.zero_grad(set_to_none=True)
    _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    sum(losses).backward()
    return [l.detach() for l in losses], {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [1, 3])
def test_training_step_matches_torch_mixer(monkeypatch, iters):
    # strict fp32 and deterministic cuDNN, as in test_losses_grad_gpu.py: the comparison then measures the mixer
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    inputs = _train_inputs()
    lt, gt = _train_step(_train_model("torch"), *inputs, iters=iters)
    lc, gc = _train_step(_train_model("cuda"), *inputs, iters=iters)
    rel_l = [abs(a.item() - b.item()) / abs(b.item()) for a, b in zip(lc, lt)]
    assert gt.keys() == gc.keys() and len(gt) > 0
    total = torch.cat([g.flatten() for g in gt.values()]).double().norm().item()
    rel_all = _rel(torch.cat([gc[n].flatten() for n in gt]), torch.cat([gt[n].flatten() for n in gt]))
    # Biases with an exact gradient of 0 (a following normalisation removes them: the token-mixing FC2 biases, fnet's conv
    # biases) are compared to the whole norm.  Every other gradient is compared to its own norm: at iters=1 the mixer's
    # are small against fnet's, but the kernels' errors are relative to each gradient.
    zero = {n for n in gt if n.endswith("bias") and gt[n].double().norm().item() <= 1e-5 * total}
    rel_g = {n: _rel(gc[n], gt[n]) for n in gt if n not in zero}
    noise = max([(gc[n] - gt[n]).double().norm().item() / total for n in zero], default=0.0)
    worst = max(rel_g, key=rel_g.get)
    print(f"iters={iters}: losses cuda {[l.item() for l in lc]} vs torch {[l.item() for l in lt]}: relative {rel_l}; all "
          f"gradients {rel_all:.2e}; {len(rel_g)} parameter gradients, worst {worst} {rel_g[worst]:.2e}; {len(zero)} "
          f"zero-gradient biases, difference {noise:.2e} of the gradient's norm")
    assert max(rel_l) <= 1e-3
    assert rel_all <= 1e-3 and rel_g[worst] <= 1e-3 and noise <= 1e-5


@pytest.mark.gpu
def test_memory_at_train_shape():
    """train.py's per-GPU shape: B=4, N=768 -> R = 3072 sequences, M = 24576 mixer rows."""
    R = 3072
    x = _mixer_input(R, 1)
    dy = torch.randn(R, 8, 130, device=DEV)
    peaks, held = {}, {}
    for name in ("cuda", "torch"):
        m = _delta_block(3, 0.05)
        xr = x.clone().requires_grad_(True)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = torch_path.delta_block_cuda(m, xr) if name == "cuda" else m(xr)
        torch.cuda.synchronize()
        held[name] = torch.cuda.memory_allocated() - base             # kept from the forward until the backward
        (out * dy).sum().backward()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del m, xr, out
    # What a call keeps between forward and backward -- a training step holds one such set per iteration: the residual
    # stream at 13 block boundaries, the (hi, lo) input rows, the output, and the packs the backward reads (fc1_w, fc1_w^T
    # and fc2_w^T as (hi, lo) bf16 per block, 12 MiB each, plus the small ones), and 32 MiB of slack.  The fp32 weight
    # copies (~100 MiB) and the forward-only packs (~52 MiB) do not fit in it.
    M = 8 * R
    budget = 13 * M * 512 * 4 + M * 576 * 4 + R * 1040 * 4 + 12 * 12 * 2**20 + 8 * 2**20 + 32 * 2**20
    print(f"DeltaBlock forward + backward at M = {M}: peak above inputs: cuda {peaks['cuda'] / 2**30:.2f} GiB, "
          f"torch {peaks['torch'] / 2**30:.2f} GiB; held from forward to backward: cuda {held['cuda'] / 2**20:.0f} MiB "
          f"(budget {budget / 2**20:.0f} MiB), torch {held['torch'] / 2**20:.0f} MiB")
    assert peaks["cuda"] <= 2.5 * 2**30
    assert held["cuda"] <= budget


@pytest.mark.gpu
def test_routing(monkeypatch):
    rgbs, xys, tg, vg, va = _train_inputs(B=1, N=16, seed=8)
    calls = []
    real = torch_path.delta_block_cuda

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(torch_path, "delta_block_cuda", spy)
    m = _train_model(None)
    assert m.mixer_path == "torch"
    mod_calls = []
    h = m.delta_block.register_forward_hook(lambda *a: mod_calls.append(1))
    m(xys, rgbs, iters=2, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert calls == [] and mod_calls == [1, 1]                       # the default keeps the torch module
    h.remove()
    monkeypatch.setenv("PIPS_B200_MIXER", "cuda")
    m = _train_model(None)
    assert m.mixer_path == "cuda"
    _, _, _, losses = m(xys, rgbs, iters=2, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert calls == [1, 1] and losses[0].requires_grad
    # no gradients: the path runs and keeps nothing but its output; with gradients a call keeps the block boundaries
    mod, x = m.delta_block, _mixer_input(64, 2)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        out = torch_path.delta_block_cuda(mod, x)
    torch.cuda.synchronize()
    kept_no_grad = torch.cuda.memory_allocated() - base
    assert out.grad_fn is None and out.shape == (64, 8, 130)
    del out
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    out = torch_path.delta_block_cuda(mod, x)
    torch.cuda.synchronize()
    kept_grad = torch.cuda.memory_allocated() - base
    print(f"kept after a call: no_grad {kept_no_grad} B (output {64 * 1040 * 4} B), with gradients {kept_grad / 2**20:.1f} MiB")
    assert kept_no_grad <= 64 * 1040 * 4 + 4096
    assert kept_grad >= 13 * 512 * 512 * 4 and out.grad_fn is not None
    del out
    assert _train_model("torch").mixer_path == "torch"               # the argument wins over the environment


def test_routing_without_gpu(monkeypatch):
    with pytest.raises(ValueError):
        Pips(S=8, stride=8, mixer_path="fast")
    monkeypatch.setenv("PIPS_B200_MIXER", "bogus")
    with pytest.raises(ValueError):
        Pips(S=8, stride=8)
    # CPU tensors keep the torch module
    from tests.golden.make_golden import LOSS_CASE, case_inputs, loss_targets
    c = LOSS_CASE
    m = Pips(S=8, stride=8, mixer_path="cuda").train()
    m.load_state_dict(po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"]))
    calls = []
    m.delta_block.register_forward_hook(lambda *a: calls.append(1))
    rgbs, xys, _ = case_inputs(c)
    tg, vg, va = loss_targets(c, xys)
    _, _, _, losses = m(xys[:1, :3], rgbs[:1], iters=1, trajs_g=tg[:1, :, :3], vis_g=vg[:1, :, :3], valids=va[:1, :, :3],
                        is_train=True)
    assert calls == [1]
    sum(losses).backward()
    assert m.delta_block.to_delta[0].weight.grad is not None
    with pytest.raises(RuntimeError):
        torch_path.delta_block_cuda(m.delta_block, torch.zeros(2, 8, 519))


def test_mixer_grad_entry_points_validate_arguments_without_gpu():
    lib = L.load()
    p = C.c_void_p(256)
    q = C.c_void_p(264)                                                   # 8-byte aligned only
    wg = lib.pips_wgrad
    assert wg(None, p, 512, p, p, 512, 100, 512, 512, p, p, None) != 0
    assert b"pips_wgrad: null pointer" in lib.pips_last_error()
    assert wg(p, p, 512, p, p, 512, 0, 512, 512, p, p, None) != 0
    assert b"empty problem" in lib.pips_last_error()
    assert wg(p, p, 1036, p, p, 512, 100, 1036, 512, p, p, None) != 0     # N not a multiple of 8
    assert b"multiples of 8" in lib.pips_last_error()
    assert wg(p, p, 256, p, p, 512, 100, 512, 512, p, p, None) != 0      # ldg < N
    assert wg(q, p, 512, p, p, 512, 100, 512, 512, p, p, None) != 0      # misaligned G
    assert b"16-byte aligned" in lib.pips_last_error()
    assert wg(p, p, 512, p, p, 512, 5000, 512, 512, None, p, None) != 0  # several splits, no scratch
    assert b"scratch" in lib.pips_last_error()
    assert lib.pips_wgrad_scratch_floats(2048, 512, 512) == 0
    assert lib.pips_wgrad_scratch_floats(2049, 512, 512) == 2 * 512 * 512

    cs = lib.pips_colsum
    assert cs(None, None, None, 512, 10, 512, None, p, None) != 0
    assert b"pips_colsum: null pointer" in lib.pips_last_error()
    assert cs(p, None, None, 100, 10, 512, None, p, None) != 0          # ld < N
    assert cs(p, None, None, 512, 1000, 512, None, p, None) != 0        # several splits, no scratch
    assert b"scratch" in lib.pips_last_error()
    assert lib.pips_colsum_scratch_floats(256, 10) == 0 and lib.pips_colsum_scratch_floats(257, 10) == 20

    tg = lib.pips_tokenmix_grad
    args = [p] * 4 + [4] + [p] * 10
    bad = list(args)
    bad[1] = None
    assert tg(*bad, None) != 0 and b"pips_tokenmix_grad: null pointer" in lib.pips_last_error()
    bad = list(args)
    bad[4] = 0
    assert tg(*bad, None) != 0 and b"no sequences" in lib.pips_last_error()
    bad = list(args)
    bad[3] = q
    assert tg(*bad, None) != 0 and b"16-byte aligned" in lib.pips_last_error()

    lp = lib.pips_ln_pool_grad
    assert lp(p, None, 4, p, p, p, p, p, None) != 0 and b"pips_ln_pool_grad: null pointer" in lib.pips_last_error()
    assert lp(p, p, 0, p, p, p, p, p, None) != 0 and b"no sequences" in lib.pips_last_error()
    assert lp(p, q, 4, p, p, p, p, p, None) != 0 and b"16-byte aligned" in lib.pips_last_error()

    ga = lib.pips_gemm_tc_aux
    assert ga(p, p, 512, 256, p, p, 512, 2048, 256, 2048, 512, p, L.EPI_GELU_GRAD, None, 0, p, p, 2048, None, 0, None) != 0
    assert b"aux" in lib.pips_last_error()
    assert ga(p, None, 512, 256, p, None, 512, 2048, 256, 2048, 512, p, L.EPI_BIAS_GELU_PRE, None, 0, p, p, 2048, p, 2048,
              None) != 0
    assert b"bf16x3 only" in lib.pips_last_error()
    assert lib.pips_gemm_tc(p, p, 512, 256, p, p, 512, 2048, 256, 2048, 512, p, L.EPI_GELU_GRAD, None, 0, p, p, 2048, None) != 0


@pytest.mark.gpu
def test_delta_block_cuda_rejects_bad_inputs():
    m = _delta_block(3, 0.05)
    with pytest.raises(ValueError):
        torch_path.delta_block_cuda(m, torch.zeros(2, 7, 519, device=DEV))          # S != 8
    with pytest.raises(ValueError):
        torch_path.delta_block_cuda(m, torch.zeros(2, 8, 520, device=DEV))
    with pytest.raises(ValueError):
        torch_path.delta_block_cuda(m, torch.zeros(2, 8, 519, device=DEV, dtype=torch.float64))


@pytest.mark.gpu
def test_data_parallel_replica_on_one_gpu():
    """A replica made by torch.nn.parallel.replicate (what nn.DataParallel runs, train.py:254) lists no parameters: its
    broadcast copies are plain attributes.  delta_block_cuda finds them by name, and the gradients flow back through the
    broadcast to the original parameters, with the bits of a direct call."""
    m = _delta_block(3, 0.05)
    replica = torch.nn.parallel.replicate(m, [0])[0]
    print(f"replica lists {len(list(replica.parameters()))} parameters")
    x = _mixer_input(37, 5)
    dy = torch.randn(37, 8, 130, device=DEV)
    m.zero_grad(set_to_none=True)
    out_r = torch_path.delta_block_cuda(replica, x)
    (out_r * dy).sum().backward()
    via_replica = {n: p.grad for n, p in m.named_parameters()}
    _, _, direct = _fwd_bwd(m, x, True, dy)
    assert all(via_replica[n] is not None for n in direct), [n for n in direct if via_replica[n] is None]
    assert all(torch.equal(via_replica[n], direct[n]) for n in direct)
    assert torch.equal(out_r.detach(), torch_path.delta_block_cuda(m, x).detach())


@pytest.mark.gpu
def test_data_parallel_matches_one_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    m = _delta_block(3, 0.05)

    class Wrap(torch.nn.Module):
        def __init__(self, mod):
            super().__init__()
            self.mod = mod

        def forward(self, x):
            return torch_path.delta_block_cuda(self.mod, x)

    x = _mixer_input(64, 3)
    dy = torch.randn(64, 8, 130, device=DEV)
    w = Wrap(m)
    w.zero_grad()
    (w(x) * dy).sum().backward()
    one = {n: p.grad.clone() for n, p in m.named_parameters()}
    w.zero_grad()
    (torch.nn.DataParallel(w, device_ids=[0, 1])(x) * dy).sum().backward()
    e = max(_rel(p.grad, one[n]) for n, p in m.named_parameters() if one[n].norm() > 0)
    print(f"DataParallel over 2 GPUs vs one: worst gradient {e:.2e}")
    assert e <= 1e-5
