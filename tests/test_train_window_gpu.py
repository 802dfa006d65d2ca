"""Training at window lengths 2 to 16 on the sm_90a kernels: the correlation gradients (pips_corr_grad_*_window) per
element against fp64, the fused score-map loss and its gradients (pips_scoremap_loss_window, pips_scoremap_grad_*_window)
against fp64 autograd of the dense loss, the _window entry points' bits at S = 8, determinism, a whole training step of
Pips(S=S, loss_path='fused', corr_path='cuda', encoder_path='cuda', mixer_path='torch') against fp64 autograd pinned to
the CUDA forward's own decisions, and the routing of such a step.

The error measures and bounds are those of the S = 8 tests: tests/test_corr_grad_gpu.py (units of 2^-24 * sum|terms|),
tests/test_losses_grad_gpu.py (norm-wise, against fp64) and tests/test_train_step_gpu.py (max|err| / max|ref| within
max(2 x strict fp32's error, a floor))."""
import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path
from tests.test_corr_grad_gpu import C_FEATS, _bound_levels, _sample, _units
from tests.test_encoder_grad_gpu import BF16X3_BOUND, _cuda_masks
from tests.test_loop_kernels_gpu import _special_coords
from tests.test_losses_grad_gpu import _dense_loss, _pyramid, _rel
from tests.test_mixer_grad_gpu import MIX_FLOOR
from tests.test_train_step_gpu import _copies, _model_step, _reference_grads

DEV = "cuda:0"


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.view(torch.int32)


# ------------------------------------------------------------------------------------------------ correlation gradients
# tests/test_corr_grad_gpu.py's helpers with the window length S as a parameter

def _levels(B, S, H, W, seed):
    """the 4 channels-last levels (B*S, H>>l, W>>l, 128) of an avg-pooled pyramid, fp32"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    lv = [torch.randn(B * S, 128, H, W, device=DEV, generator=g)]
    for _ in range(3):
        lv.append(F.avg_pool2d(lv[-1], 2, stride=2))
    return [t.permute(0, 2, 3, 1).contiguous() for t in lv]


def _coords(B, S, N, H, W, seed):
    """random positions over and around the map, then _special_coords' edge cases, the diverged tracks and NaN"""
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(B, S, N, 2, generator=g) * torch.tensor([W + 4.0, H + 4.0]) - 2.0
    pts, far = _special_coords(H, W)
    far = torch.cat([far, torch.tensor([[float("nan"), 3.0], [2.0, float("nan")], [float("nan"), float("nan")]])])
    flat = c.view(-1, 2)
    k = min(len(pts), flat.shape[0] - len(far))
    flat[:k] = pts[:k]
    flat[-len(far):] = far
    return c.to(DEV)


def _diverged(coords):
    """(B*N, S) rows whose every footprint lies off the map: non-finite or 1e9-far coordinates"""
    S = coords.shape[1]
    d = ~torch.isfinite(coords).all(-1) | (coords.abs() >= 1e9).any(-1)
    return d.permute(0, 2, 1).reshape(-1, S)


def _grads(levels, coords, ff_rows, dcorr, window=True, ld=196):
    """both backward entry points (the _window ones, or the S = 8 ones) into NaN-filled outputs: (dffeat_rows, [dlevel])"""
    lib = L.load()
    B, S, N, _ = coords.shape
    H, W = levels[0].shape[1:3]
    sfx = "_window" if window else ""
    dff = torch.full((B * N, S, 128), float("nan"), device=DEV)
    dls = [torch.full_like(lv, float("nan")) for lv in levels]
    L.check(getattr(lib, "pips_corr_grad_feats" + sfx)(L.ptr_array(levels), B, S, N, H, W, L.ptr(coords), L.ptr(dcorr), ld,
                                                       L.ptr(dff), _st()), "pips_corr_grad_feats" + sfx)
    L.check(getattr(lib, "pips_corr_grad_levels" + sfx)(B, S, N, H, W, L.ptr(coords), L.ptr(ff_rows), L.ptr(dcorr), ld,
                                                        L.ptr_array(dls), _st()), "pips_corr_grad_levels" + sfx)
    torch.cuda.synchronize()
    return dff, dls


def _ref_corr(ff_rows, levels, coords, ones=False):
    """fp64 forward_torch correlation (all-pairs volumes / sqrt(128) sampled at the 49 taps of each level, grid_sample's
    arithmetic written out by _sample), the position clamped to [-8, size + 8] (NaN to -8) as the kernels clamp it"""
    B, S, N, _ = coords.shape
    q = ff_rows.reshape(B, N, S, 128).permute(0, 2, 1, 3)
    a = torch.arange(7, dtype=torch.float64, device=DEV) - 3
    out = []
    for l, lv in enumerate(levels):
        h, w = lv.shape[1:3]
        vol = torch.matmul(q, lv.reshape(B, S, h * w, 128).transpose(-1, -2)) / 128 ** 0.5          # (B,S,N,h*w)
        c = coords.double() / 2 ** l
        c = torch.where(torch.isnan(c), torch.full_like(c, -8.0), c)
        cx = c[..., 0].clamp(-8, w + 8).reshape(-1, 1, 1)
        cy = c[..., 1].clamp(-8, h + 8).reshape(-1, 1, 1)
        x = (cx + a.view(1, 7, 1)).expand(-1, 7, 7).reshape(-1, 49)
        y = (cy + a.view(1, 1, 7)).expand(-1, 7, 7).reshape(-1, 49)
        out.append(_sample(vol.reshape(-1, h, w), x, y, ones).view(B, S, N, 49))
    return torch.cat(out, -1).permute(0, 2, 1, 3).reshape(B * N, S, 196)


def _ref_grads(levels, coords, ff_rows, dcorr):
    """fp64 autograd of _ref_corr: ([dffeat, dlevel_0..3], [their sum|terms|])"""
    def grads(ff, lv, dc, ones=False):
        ff = ff.double().requires_grad_(True)
        lv = [t.double().requires_grad_(True) for t in lv]
        return list(torch.autograd.grad(_ref_corr(ff, lv, coords, ones), [ff, *lv], dc.double()))
    ref = grads(ff_rows, levels, dcorr)
    absd = [t.abs() for t in levels]
    mag = [a + b for a, b in zip(grads(ff_rows.abs(), absd, dcorr.abs()), grads(ff_rows.abs(), absd, dcorr.abs(), ones=True))]
    return ref, mag


def _corr_problem(B, S, N, H, W, seed):
    levels = _levels(B, S, H, W, seed=seed)
    coords = _coords(B, S, N, H, W, seed=seed + 1)
    g = torch.Generator(device=DEV).manual_seed(seed + 2)
    ff = torch.randn(B * N, S, 128, device=DEV, generator=g)
    dc = torch.randn(B * N, S, 196, device=DEV, generator=g)
    return levels, coords, ff, dc


@pytest.mark.gpu
@pytest.mark.parametrize("S", [2, 5, 9, 12, 16])
@pytest.mark.parametrize("H,W", [(9, 40), (45, 12)])
def test_corr_backward_matches_fp64(S, H, W):
    """N = 37, B = 2.  Level 3 is one pixel high (9x40: 1x5) or one pixel wide (45x12: 5x1), and the odd sizes drop a
    row or column at several levels.  Coordinates on every level's edges, off the map on either side of the kernels'
    +-8 px clamp, diverged and NaN."""
    B, N = 2, 37
    levels, coords, ff, dc = _corr_problem(B, S, N, H, W, seed=100 * S + H)
    dff, dls = _grads(levels, coords, ff, dc)
    ref, mag = _ref_grads(levels, coords, ff, dc)
    for t in [dff] + dls:
        assert not torch.isnan(t).any(), "NaN left in an output"
    r_f = _units(dff, ref[0], mag[0])
    r_l = [_units(d, r, m) for d, r, m in zip(dls, ref[1:], mag[1:])]
    for d, m in zip(dls, mag[1:]):
        assert (d[m == 0] == 0).all(), "a pixel no footprint touches is not exactly 0"
    assert (dff[_diverged(coords)] == 0).all(), "a diverged track's dffeat is not exactly 0"
    print(f"S={S} {H}x{W}: dffeat {r_f:.3g} (bound {C_FEATS}), dlevel {' '.join(f'{r:.3g}' for r in r_l)} "
          f"(bound {_bound_levels(N)}) units of U sum|terms|")
    assert r_f <= C_FEATS
    assert max(r_l) <= _bound_levels(N)


@pytest.mark.gpu
def test_corr_window_entry_points_have_the_s8_bits():
    levels, coords, ff, dc = _corr_problem(2, 8, 300, 45, 80, seed=7)
    a, b = _grads(levels, coords, ff, dc, window=False), _grads(levels, coords, ff, dc, window=True)
    assert torch.equal(_bits(a[0]), _bits(b[0]))
    assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a[1], b[1]))


@pytest.mark.gpu
def test_corr_backward_at_s12_is_deterministic_and_autograd_uses_the_kernels():
    B, S, N = 2, 12, 300
    levels, coords, ff, dc = _corr_problem(B, S, N, 45, 80, seed=9)
    a, b = _grads(levels, coords, ff, dc), _grads(levels, coords, ff, dc)
    assert torch.equal(_bits(a[0]), _bits(b[0])) and all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a[1], b[1]))
    # through autograd, with the gradient of a column slice of a 519-wide mixer input (row stride 519)
    ffr = ff.clone().requires_grad_(True)
    lvr = [t.clone().requires_grad_(True) for t in levels]
    x = torch.cat([ffr.detach(), torch_path.local_corr_cuda(ffr, lvr, coords), torch.zeros(B * N, S, 195, device=DEV)], 2)
    gx = torch.zeros_like(x)
    gx[..., 128:324] = dc
    x.backward(gx)
    assert torch.equal(_bits(ffr.grad), _bits(a[0]))
    assert all(torch.equal(_bits(t.grad), _bits(d)) for t, d in zip(lvr, a[1]))


# ------------------------------------------------------------------------------------------------ score-map loss

def _loss_problem(S, H8, W8, N, I, B=1, seed=0):
    """tests/test_losses_grad_gpu.py's _problem at S frames: fmaps (B,S,128,H8,W8), I ffeats (B,S,N,128) and ground
    truth in feature pixels with rows dropped for each reason (out of bounds, not visible, not valid) and targets on the
    map edges"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    fmaps = torch.randn(B, S, 128, H8, W8, device=DEV, generator=g, dtype=torch.float64)
    ffeats = [torch.randn(B, S, N, 128, device=DEV, generator=g, dtype=torch.float64) * 0.7 for _ in range(I)]
    tg = torch.rand(B, S, N, 2, device=DEV, generator=g, dtype=torch.float64) * torch.tensor([W8 + 2.0, H8 + 2.0], device=DEV) - 1.0
    vg = (torch.rand(B, S, N, device=DEV, generator=g) > 0.2).float()
    va = (torch.rand(B, S, N, device=DEV, generator=g) > 0.1).float()
    edges = [(0, 0), (W8 - 1, 0), (0, H8 - 1), (W8 - 1, H8 - 1), (W8 // 2, 0), (0, H8 // 2)]
    for s in range(S):
        tg[0, s, s % N] = torch.tensor(edges[s % len(edges)], dtype=torch.float64)
    tg[0, 0, 1] = torch.tensor([W8 - 0.5, 1.0])                     # rounds to W8: out of bounds
    tg[0, 1, 2] = torch.tensor([2.0, -0.6])                         # rounds to -1: out of bounds
    vg[0, S - 1, 3] = 0.0
    va[0, S - 2, 3] = 0.0
    return fmaps, ffeats, tg.float(), vg, va


def _loss_grads(dtype, fmaps, ffeats, tg, vg, va, fused):
    fm = fmaps.detach().to(dtype).requires_grad_(True)
    ff = [f.detach().to(dtype).requires_grad_(True) for f in ffeats]
    pyr = [lv.detach().requires_grad_(True) for lv in _pyramid(fm)]     # gradients of every level, not only fmaps'
    if fused:
        loss = torch_path.fused_score_map_loss(ff, pyr, tg.float(), vg, va)
    else:
        loss = _dense_loss(ff, pyr, tg.to(dtype), vg.to(dtype), va.to(dtype))
    loss.backward()
    return loss.detach(), [f.grad for f in ff], [lv.grad for lv in pyr]


@pytest.mark.gpu
@pytest.mark.parametrize("S", [2, 5, 12, 16])
@pytest.mark.parametrize("H8,W8,N,I", [(45, 80, 37, 3), (16, 16, 100, 2)])
def test_fused_loss_gradients_match_fp64(S, H8, W8, N, I):
    """the loss, its gradient in every iteration's ffeats and in each of the 4 levels against fp64 autograd of the
    dense score_map_loss; bounds of tests/test_losses_grad_gpu.py"""
    prob = _loss_problem(S, H8, W8, N, I, B=2, seed=S * 1000 + H8 + N)
    l64, df64, dl64 = _loss_grads(torch.float64, *prob, fused=False)
    l32, df32, dl32 = _loss_grads(torch.float32, *prob, fused=False)
    lf, dff, dlf = _loss_grads(torch.float32, *prob, fused=True)
    assert lf.dim() == 0 and lf.dtype == torch.float32
    e_loss, e_loss32 = abs(lf.item() - l64.item()) / abs(l64.item()), abs(l32.item() - l64.item()) / abs(l64.item())
    e_df = max(_rel(a, b) for a, b in zip(dff, df64))
    e_df32 = max(_rel(a, b) for a, b in zip(df32, df64))
    e_dl = [_rel(a, b) for a, b in zip(dlf, dl64)]
    e_dl32 = [_rel(a, b) for a, b in zip(dl32, dl64)]
    print(f"S={S} {H8}x{W8} N={N} I={I}: fused vs fp64: loss {e_loss:.2e}, dF {e_df:.2e}, dlevels "
          f"{' '.join(f'{e:.2e}' for e in e_dl)} | dense fp32 vs fp64: loss {e_loss32:.2e}, dF {e_df32:.2e}, dlevels "
          f"{' '.join(f'{e:.2e}' for e in e_dl32)}")
    assert e_loss <= 1e-5
    assert e_df <= 1e-4 and max(e_dl) <= 1e-4


def _scoremap_grads(prob, window):
    """pips_scoremap_grad_feats / _basis (or their _window siblings) on one problem, called directly into NaN-filled
    outputs, with the operands _FusedScoreMapLoss builds: (dF, dG)"""
    lib = L.load()
    fmaps, ffeats, tg, vg, va = prob
    B, S, N, C = ffeats[0].shape
    H8, W8 = fmaps.shape[-2:]
    P, I = H8 * W8, len(ffeats)
    sfx = "_window" if window else ""
    lvls = [lv.float().permute(0, 1, 3, 4, 2).contiguous() for lv in _pyramid(fmaps.float())]
    g_hi = torch.empty(B * S, P, C, dtype=torch.bfloat16, device=DEV)
    g_lo = torch.empty_like(g_hi)
    L.check(lib.pips_scoremap_basis(L.ptr_array(lvls), B * S, H8, W8, L.ptr(g_hi), L.ptr(g_lo), _st()), "pips_scoremap_basis")
    target = torch_path.score_map_targets(tg, vg, va, H8, W8)
    coef = torch.tensor([0.37, 1.3e-4], device=DEV)
    F_ = torch.stack([f.float() for f in ffeats]).contiguous()
    f_hi = torch.empty(F_.shape, dtype=torch.bfloat16, device=DEV)
    f_lo = torch.empty_like(f_hi)
    L.check(lib.pips_split_bf16(L.ptr(F_), L.ptr(f_hi), L.ptr(f_lo), F_.numel(), _st()), "pips_split_bf16")
    dF = torch.full_like(F_, float("nan"))
    dG = torch.full((B * S, P, C), float("nan"), device=DEV)
    L.check(getattr(lib, "pips_scoremap_grad_feats" + sfx)(L.ptr(g_hi), L.ptr(g_lo), L.ptr(F_), I, B, S, N, H8, W8,
                                                           L.ptr(target), L.ptr(coef), L.ptr(dF), _st()), "grad_feats")
    L.check(getattr(lib, "pips_scoremap_grad_basis" + sfx)(L.ptr(g_hi), L.ptr(g_lo), L.ptr(f_hi), L.ptr(f_lo), I, B, S, N,
                                                           H8, W8, L.ptr(target), L.ptr(coef), L.ptr(dG), _st()),
            "grad_basis")
    torch.cuda.synchronize()
    return dF, dG


@pytest.mark.gpu
def test_scoremap_window_entry_points_have_the_s8_bits():
    prob = _loss_problem(8, 45, 80, 300, 3, B=2, seed=21)
    a, b = _scoremap_grads(prob, window=False), _scoremap_grads(prob, window=True)
    assert not torch.isnan(a[0]).any() and not torch.isnan(a[1]).any()
    assert torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(_bits(a[1]), _bits(b[1]))


@pytest.mark.gpu
def test_fused_loss_at_s12_is_deterministic():
    prob = _loss_problem(12, 48, 64, 300, 4, B=2, seed=11)
    a = _loss_grads(torch.float32, *prob, fused=True)
    b = _loss_grads(torch.float32, *prob, fused=True)
    assert torch.equal(_bits(a[0]), _bits(b[0]))
    assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a[1] + a[2], b[1] + b[2]))
    c, d = _scoremap_grads(prob, window=True), _scoremap_grads(prob, window=True)
    assert torch.equal(_bits(c[0]), _bits(d[0])) and torch.equal(_bits(c[1]), _bits(d[1]))


# ------------------------------------------------------------------------------------------------ a whole training step

def _model(S, stride=8, head_scale=0.05, seed=3, **paths):
    kw = dict(loss_path="fused", corr_path="cuda", encoder_path="cuda", mixer_path="torch")
    kw.update(paths)
    m = Pips(S=S, stride=stride, **kw).to(DEV).train()
    m.load_state_dict(po.init_state_dict(seed=seed, head_scale=head_scale, S=S), strict=True)
    return m


def _inputs(B, S, N, H, W, seed):
    """tests/test_train_step_gpu.py's _inputs at S frames: queries on the frame's edges and corners as well as inside,
    two tracks whose ground truth leaves the feature map, one track never visible, about 10% of the valids zero"""
    rgbs = po.smooth_video(B, S, H, W, seed=100 + seed)
    xys = po.random_queries(B, N, H, W, seed=200 + seed)
    edge = torch.tensor([[0.0, 0.0], [W - 1.0, 0.0], [0.0, H - 1.0], [W - 1.0, H - 1.0],
                         [W / 2 + 0.3, 0.0], [W / 2 - 0.7, H - 1.0], [0.0, H / 2 + 0.4], [W - 1.0, H / 2 - 0.2]])
    k = min(len(edge), N // 2)
    xys[:, :k] = edge[:k]
    g = torch.Generator().manual_seed(400 + seed)
    tg = xys[:, None] + torch.cumsum(torch.randn(B, S, N, 2, generator=g) * 3.0, 1)
    tg[:, S // 2:, k, 0] = -20.0                    # left of the map
    tg[:, S - 1:, k + 1, 1] = H + 20.0              # below it
    vg = (torch.rand(B, S, N, generator=g) > 0.2).float()
    vg[0, :, k + 2] = 0
    va = (torch.rand(B, S, N, generator=g) > 0.1).float()
    return tuple(t.to(DEV) for t in (rgbs, xys, tg, vg, va))


def _spied_step(monkeypatch, m, inputs, iters):
    """one step with a spy on each CUDA node: (losses, gradients, per-iteration coordinates, call counts)"""
    calls = {"encoder_cuda": 0, "local_corr_cuda": 0, "delta_block_cuda": 0, "fused_score_map_loss": 0}
    coords = []
    real = {n: getattr(torch_path, n) for n in calls}

    def spy(name):
        def f(*a, **k):
            calls[name] += 1
            if name == "local_corr_cuda":
                coords.append(a[2].detach().clone())
            return real[name](*a, **k)
        return f

    with monkeypatch.context() as mp:
        for n in calls:
            mp.setattr(torch_path, n, spy(n))
        losses, grads = _model_step(m, *inputs, iters)
    return losses, grads, coords, calls


# (S, B, N, H, W, iters): odd pyramid levels 17x25 -> 8x12 -> 4x6 -> 2x3; N not a multiple of 8
STEP_CASES = [(4, 2, 37, 136, 200, 3), (12, 1, 37, 136, 200, 3), (16, 1, 24, 64, 96, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("S,B,N,H,W,iters", STEP_CASES)
def test_training_step_matches_fp64(monkeypatch, S, B, N, H, W, iters):
    """Losses and every parameter gradient of one step with the encoder, the correlation and the loss on CUDA and the
    torch mixer, against fp64 autograd of tests/test_train_step_gpu.py's _reference_step under the CUDA forward's ReLU
    decisions and coordinates: max|err| / max|ref| per tensor within max(2 x strict fp32's error under the same
    decisions, iters x MIX_FLOOR, plus BF16X3_BOUND for fnet tensors).  64x96 at S = 16: level 3 is 1x1."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    model = _model(S)
    inputs = _inputs(B, S, N, H, W, seed=H + N + S)
    lc, gc, coords, calls = _spied_step(monkeypatch, model, inputs, iters)
    assert calls == {"encoder_cuda": 1, "local_corr_cuda": iters, "delta_block_cuda": 0, "fused_score_map_loss": 1}
    masks = _cuda_masks(model.fnet, inputs[0])
    l64, g64, _ = _reference_grads(_copies(model, torch.float64), inputs, iters, masks=masks, coords=coords)
    l32, g32, _ = _reference_grads(_copies(model, torch.float32), inputs, iters, masks=masks, coords=coords)

    assert set(gc) == set(g64) and len(gc) == len(list(model.parameters()))
    total = torch.cat([t.flatten() for t in g64.values()]).norm().item()
    fnet_zero = [n for n in g64 if n.startswith("fnet.") and n.endswith("bias") and n != "fnet.conv3.bias"]
    tok_zero = [n for n in g64 if n.endswith("0.fn.3.bias")]
    assert len(fnet_zero) == 21 and len(tok_zero) == 12
    for n in fnet_zero:                        # before an InstanceNorm: exactly zero
        assert (gc[n] == 0).all(), n
    noise = max((gc[n].double() - g64[n]).norm().item() / total for n in tok_zero)
    assert noise <= 1e-5, f"token-mixing FC2 biases differ by {noise:.2e} of the gradients' norm"

    def err(a, b):
        return ((a.double() - b).abs().max() / b.abs().max().clamp(min=1e-300)).item()

    cases = {f"loss{i}": (lc[i], l32[i], l64[i]) for i in range(3)}
    cases.update({n: (gc[n], g32[n], g64[n]) for n in g64 if n not in fnet_zero and n not in tok_zero})
    e = {n: (err(c, r), err(t, r)) for n, (c, t, r) in cases.items()}
    floor = {n: (BF16X3_BOUND if n.startswith("fnet.") else 0.0) + iters * MIX_FLOOR for n in e}
    ratio = {n: ec / max(2 * et, floor[n]) for n, (ec, et) in e.items()}
    worst = max(ratio, key=ratio.get)
    top = sorted(ratio, key=ratio.get, reverse=True)[:4]
    print(f"\nS={S} B={B} N={N} {H}x{W} iters={iters}: worst {worst} ratio {ratio[worst]:.3f} (cuda {e[worst][0]:.2e}, "
          f"fp32 {e[worst][1]:.2e}); losses " + " ".join(f"{ratio[f'loss{i}']:.3f}" for i in range(3))
          + "; next " + ", ".join(f"{n} {ratio[n]:.3f}" for n in top[1:]))
    assert ratio[worst] <= 1.0, f"{worst}: {ratio[worst]:.3f} of its bound"


@pytest.mark.gpu
def test_training_step_routing_at_s12(monkeypatch):
    """At S = 12 with the fused loss and the CUDA correlation, neither direction builds an all-pairs volume (no matmul,
    no grid_sample) or a dense score map (no interpolate, no score_map_loss): local_corr_cuda runs once per iteration"""
    S, iters = 12, 3
    model = _model(S)
    rgbs, xys, tg, vg, va = _inputs(1, S, 16, 128, 128, seed=8)
    calls = {"grid_sample": 0, "matmul": 0, "interpolate": 0, "score_map_loss": 0, "local_corr_cuda": 0,
             "fused_score_map_loss": 0}
    real = {"grid_sample": F.grid_sample, "matmul": torch.matmul, "interpolate": F.interpolate,
            "score_map_loss": torch_path.score_map_loss, "local_corr_cuda": torch_path.local_corr_cuda,
            "fused_score_map_loss": torch_path.fused_score_map_loss}

    def spy(name):
        def f(*a, **k):
            calls[name] += 1
            return real[name](*a, **k)
        return f

    monkeypatch.setattr(F, "grid_sample", spy("grid_sample"))
    monkeypatch.setattr(F, "interpolate", spy("interpolate"))
    monkeypatch.setattr(torch, "matmul", spy("matmul"))
    for n in ("score_map_loss", "local_corr_cuda", "fused_score_map_loss"):
        monkeypatch.setattr(torch_path, n, spy(n))
    _, _, _, losses = model(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    sum(losses).backward()
    assert calls == {"grid_sample": 0, "matmul": 0, "interpolate": 0, "score_map_loss": 0, "local_corr_cuda": iters,
                     "fused_score_map_loss": 1}, calls
    assert all(torch.isfinite(l) for l in losses)
    assert model.fnet.conv1.weight.grad.abs().sum() > 0 and model.delta_block.to_delta[0].weight.grad.abs().sum() > 0
