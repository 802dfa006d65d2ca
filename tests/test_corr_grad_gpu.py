"""Training the local correlation on the sm_90a kernels (Pips(corr_path='cuda'), torch_path.local_corr_cuda): the
forward against pips_corr_gather and fp64, the two backward kernels (csrc/corr_grad.cu) against fp64 autograd of the
reference formulation, crowded frames, coverage of the outputs, determinism, a training step against corr_path='torch',
memory and routing.

Errors are in units of U * sum|terms| (U = 2^-24), sum|terms| being the same fp64 computation on absolute values plus
the |terms| of all four corners of every tap unweighted: the fp32 fractional position of a tap rounds for -1 < x < 0,
which moves a bilinear weight by up to U (tests/test_loop_kernels_gpu.py's _corr_ref does the same).  A sum of n fp32
terms in a fixed order is off by at most (n - 1) U sum|terms|, so each bound is the longest summation chain of its
output plus the weight's few roundings."""
import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path
from tests.test_loop_kernels_gpu import C_CORR, _corr_ref, _special_coords

DEV = "cuda:0"
U = 2.0 ** -24
S = 8
C_FEATS = 4 * 64 + 8            # dffeat: 4 levels x 64 footprint pixels accumulated per channel, A's 4 terms and scale


def _bound_levels(n_per_frame):
    return n_per_frame + 8      # dlevel: one term per unit of the frame, in ascending n, A's 4 terms and scale


def _st():
    return torch.cuda.current_stream().cuda_stream


def _levels(B, H, W, seed):
    """the 4 channels-last levels (B*S, H>>l, W>>l, 128) of an avg-pooled pyramid, fp32"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    lv = [torch.randn(B * S, 128, H, W, device=DEV, generator=g)]
    for _ in range(3):
        lv.append(F.avg_pool2d(lv[-1], 2, stride=2))
    return [t.permute(0, 2, 3, 1).contiguous() for t in lv]


def _coords(B, N, H, W, seed, special=True):
    """random positions over and around the map, then _special_coords' edge cases, the diverged tracks and NaN"""
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(B, S, N, 2, generator=g) * torch.tensor([W + 4.0, H + 4.0]) - 2.0
    if special:
        pts, far = _special_coords(H, W)
        far = torch.cat([far, torch.tensor([[float("nan"), 3.0], [2.0, float("nan")], [float("nan"), float("nan")]])])
        flat = c.view(-1, 2)
        k = min(len(pts), flat.shape[0] - len(far))
        flat[:k] = pts[:k]
        flat[-len(far):] = far
    return c.to(DEV)


def _diverged(coords):
    """(B*N, S) rows whose every footprint lies off the map: non-finite or 1e9-far coordinates"""
    d = ~torch.isfinite(coords).all(-1) | (coords.abs() >= 1e9).any(-1)
    return d.permute(0, 2, 1).reshape(-1, S)


def _grads(levels, coords, ff_rows, dcorr, ld=196):
    """both backward entry points into NaN-filled outputs: (dffeat_rows, [dlevel_l])"""
    lib = L.load()
    B, _, N, _ = coords.shape
    H, W = levels[0].shape[1:3]
    dff = torch.full((B * N, S, 128), float("nan"), device=DEV)
    dls = [torch.full_like(lv, float("nan")) for lv in levels]
    L.check(lib.pips_corr_grad_feats(L.ptr_array(levels), B, S, N, H, W, L.ptr(coords), L.ptr(dcorr), ld, L.ptr(dff), _st()),
            "pips_corr_grad_feats")
    L.check(lib.pips_corr_grad_levels(B, S, N, H, W, L.ptr(coords), L.ptr(ff_rows), L.ptr(dcorr), ld, L.ptr_array(dls), _st()),
            "pips_corr_grad_levels")
    torch.cuda.synchronize()
    return dff, dls


def _sample(vol, x, y, ones):
    """bilinear samples of vol (R, h, w) at (x, y) (R, K), zero outside the map: grid_sample's align_corners=True
    arithmetic written out, so that a level one pixel wide stays defined (grid_sample divides by size - 1 = 0 there).
    ones: every corner weighted 1."""
    R, h, w = vol.shape
    x0, y0 = torch.floor(x), torch.floor(y)
    fx, fy = x - x0, y - y0
    flat = vol.reshape(R, h * w)
    out = 0
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        wt = 1.0 if ones else (fx if dx else 1 - fx) * (fy if dy else 1 - fy)
        xi, yi = x0 + dx, y0 + dy
        inside = ((xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)).double()
        idx = (yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1)).long()
        out = out + wt * inside * torch.gather(flat, 1, idx)
    return out


def _ref_corr(ff_rows, levels, coords, ones=False):
    """fp64 forward_torch correlation (nets/pips.py:355-398): all-pairs volumes / sqrt(128) sampled at the 49 taps of
    each level, channel l*49 + a*7 + b at x = cx/2^l + a - 3, y = cy/2^l + b - 3 -> (B*N, S, 196).  The position is
    clamped to [-8, size + 8] (NaN to -8) first, as the kernels clamp it; past 8 px off the map every tap is zero
    either way."""
    B, _, N, _ = coords.shape
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
        out = _ref_corr(ff, lv, coords, ones)
        return list(torch.autograd.grad(out, [ff, *lv], dc.double()))
    ref = grads(ff_rows, levels, dcorr)
    absd = [t.abs() for t in levels]
    mag = [a + b for a, b in zip(grads(ff_rows.abs(), absd, dcorr.abs()), grads(ff_rows.abs(), absd, dcorr.abs(), ones=True))]
    return ref, mag


def _units(got, ref, mag):
    return ((got.double() - ref).abs() / (U * mag).clamp(min=1e-300)).max().item()


def _check_grads(levels, coords, ff, dc, dff, dls, n_per_frame, label):
    ref, mag = _ref_grads(levels, coords, ff, dc)
    for t in [dff] + dls:
        assert not torch.isnan(t).any(), f"{label}: NaN left in an output"
    r_f = _units(dff, ref[0], mag[0])
    r_l = [_units(d, r, m) for d, r, m in zip(dls, ref[1:], mag[1:])]
    for d, m in zip(dls, mag[1:]):
        assert (d[m == 0] == 0).all(), f"{label}: a pixel no footprint touches is not exactly 0"
    assert (dff[_diverged(coords)] == 0).all(), f"{label}: a diverged track's dffeat is not exactly 0"
    print(f"{label}: dffeat {r_f:.3g} (bound {C_FEATS}), dlevel {' '.join(f'{r:.3g}' for r in r_l)} "
          f"(bound {_bound_levels(n_per_frame)}) units of U sum|terms|")
    assert r_f <= C_FEATS
    assert max(r_l) <= _bound_levels(n_per_frame)


# ------------------------------------------------------------------------------------------------ 1. forward

@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(8, 8), (45, 80)])
def test_forward_is_corr_gather(H, W):
    B, N = 2, 12
    levels = _levels(B, H, W, seed=1)
    coords = _coords(B, N, H, W, seed=2)
    ff = torch.randn(B * N, S, 128, device=DEV)
    got = torch_path.local_corr_cuda(ff, levels, coords)
    x = torch.full((B * N * S, 576), float("nan"), device=DEV)
    times = torch.linspace(0, S, S, device=DEV)
    L.check(L.load().pips_corr_gather(L.ptr_array(levels), L.FEAT_F32, B, S, N, H, W, L.ptr(coords), L.ptr(ff), L.ptr(times),
                                      None, 0, None, None, L.ptr(x), 576, _st()), "pips_corr_gather")
    assert torch.equal(got.reshape(-1, 196).view(torch.int32), x[:, 128:324].view(torch.int32))
    fidx = (torch.arange(B).view(B, 1, 1) * S + torch.arange(S).view(1, S, 1)).expand(B, S, N)
    q = ff.reshape(B, N, S, 128).permute(0, 2, 1, 3).double().cpu()
    far = torch.nan_to_num(coords.cpu(), nan=-1e9)       # NaN is clamped as far off the map as -1e9: all taps 0
    ref, mag = _corr_ref([t.cpu().double() for t in levels], fidx, far, q)
    r = ((got.reshape(-1, 196).double().cpu() - ref).abs() / (U * mag + 1e-300)).max().item()
    print(f"local_corr_cuda {H}x{W}: {r:.3g} units (bound {C_CORR})")
    assert r <= C_CORR


# ------------------------------------------------------------------------------------------------ 2.-4. backward

@pytest.mark.gpu
@pytest.mark.parametrize("N", [12, 300])
@pytest.mark.parametrize("H,W", [(8, 8), (9, 40), (15, 8), (45, 80)])
def test_backward_matches_fp64(H, W, N):
    B = 2
    levels = _levels(B, H, W, seed=3)
    coords = _coords(B, N, H, W, seed=4)
    g = torch.Generator(device=DEV).manual_seed(5)
    ff = torch.randn(B * N, S, 128, device=DEV, generator=g)
    dc = torch.randn(B * N, S, 196, device=DEV, generator=g)
    dff, dls = _grads(levels, coords, ff, dc)
    _check_grads(levels, coords, ff, dc, dff, dls, N, f"corr backward {H}x{W} N={N}")


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["point", "tile corner"])
def test_backward_crowded_frame(where):
    """all 1024 tracks of every frame at one position; on a tile corner every footprint straddles 4 tiles of level 0"""
    B, N, H, W = 1, 1024, 40, 48
    levels = _levels(B, H, W, seed=6)
    pos = torch.tensor([17.3, 21.6]) if where == "point" else torch.tensor([19.0, 27.0])   # origin (16, 24) at level 0
    coords = pos.expand(B, S, N, 2).contiguous().to(DEV)
    g = torch.Generator(device=DEV).manual_seed(7)
    ff = torch.randn(B * N, S, 128, device=DEV, generator=g)
    dc = torch.randn(B * N, S, 196, device=DEV, generator=g)
    dff, dls = _grads(levels, coords, ff, dc)
    _check_grads(levels, coords, ff, dc, dff, dls, N, f"corr backward, crowded at a {where}")


@pytest.mark.gpu
def test_backward_is_deterministic_and_autograd_uses_the_kernels():
    B, N, H, W = 2, 300, 45, 80
    levels = _levels(B, H, W, seed=8)
    coords = _coords(B, N, H, W, seed=9)
    g = torch.Generator(device=DEV).manual_seed(10)
    ff = torch.randn(B * N, S, 128, device=DEV, generator=g)
    dc = torch.randn(B * N, S, 196, device=DEV, generator=g)
    a, b = _grads(levels, coords, ff, dc), _grads(levels, coords, ff, dc)
    bits = lambda t: t.view(torch.int32)
    assert torch.equal(bits(a[0]), bits(b[0])) and all(torch.equal(bits(x), bits(y)) for x, y in zip(a[1], b[1]))
    # through autograd, with the gradient of a column slice of a 519-wide mixer input (row stride 519)
    ffr = ff.clone().requires_grad_(True)
    lvr = [t.clone().requires_grad_(True) for t in levels]
    x = torch.cat([ffr.detach(), torch_path.local_corr_cuda(ffr, lvr, coords), torch.zeros(B * N, S, 195, device=DEV)], 2)
    gx = torch.zeros_like(x)
    gx[..., 128:324] = dc
    x.backward(gx)
    assert torch.equal(bits(ffr.grad), bits(a[0]))
    assert all(torch.equal(bits(t.grad), bits(d)) for t, d in zip(lvr, a[1]))


# ------------------------------------------------------------------------------------------------ 6. training step

def _train_model(corr_path, seed=3):
    m = Pips(S=8, stride=8, loss_path="fused", mixer_path="torch", encoder_path="torch", corr_path=corr_path).to(DEV).train()
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


def _train_step(m, rgbs, xys, tg, vg, va, iters=4):
    m.zero_grad(set_to_none=True)
    _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    sum(losses).backward()
    return [l.detach() for l in losses], {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-300)).item()


@pytest.mark.gpu
def test_training_step_matches_torch_path(monkeypatch):
    # strict, deterministic fp32 as in test_losses_grad_gpu.py: the comparison then measures the correlation alone
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    inputs = _train_inputs()
    lt, gt = _train_step(_train_model("torch"), *inputs)
    lc, gc = _train_step(_train_model("cuda"), *inputs)
    rel_l = [abs(a.item() - b.item()) / abs(b.item()) for a, b in zip(lc, lt)]
    assert gt.keys() == gc.keys() and len(gt) > 0
    assert gc["fnet.conv1.weight"].abs().sum() > 0 and gc["fnet.layer4.1.conv2.weight"].abs().sum() > 0
    total = torch.cat([g.flatten() for g in gt.values()]).double().norm().item()
    rel_all = _rel(torch.cat([gc[n].flatten() for n in gt]), torch.cat([gt[n].flatten() for n in gt]))
    # biases with an exact gradient of 0 (before a LayerNorm or an InstanceNorm) are compared to the whole norm
    zero = {n for n in gt if gt[n].double().norm().item() <= 1e-5 * total}
    assert all(n.endswith("bias") for n in zero), zero
    rel_g = {n: _rel(gc[n], gt[n]) for n in gt if n not in zero}
    noise = max([(gc[n] - gt[n]).double().norm().item() / total for n in zero], default=0.0)
    worst = max(rel_g, key=rel_g.get)
    print(f"losses corr cuda {[l.item() for l in lc]} vs torch {[l.item() for l in lt]}: relative {rel_l}; all gradients "
          f"{rel_all:.2e}; worst {worst} {rel_g[worst]:.2e}; zero-gradient biases {noise:.2e} of the norm")
    assert max(rel_l) <= 1e-5
    assert rel_all <= 1e-4 and rel_g[worst] <= 1e-4 and noise <= 1e-6


# ------------------------------------------------------------------------------------------------ 7. memory

def _torch_corr(ff_rows, levels, coords):
    """forward_torch's formulation: matmul all-pairs volumes, grid_sample of the 49 taps"""
    B, _, N, _ = coords.shape
    ffeats = ff_rows.reshape(B, N, S, 128).permute(0, 2, 1, 3)
    offs = torch.linspace(-3, 3, 7, device=DEV)
    window = torch.stack(torch.meshgrid(offs, offs, indexing="ij"), dim=-1).view(1, 7, 7, 2)
    taps = []
    for i, lv in enumerate(levels):
        f = lv.reshape(B, S, *lv.shape[1:]).permute(0, 1, 4, 2, 3)
        h, w = f.shape[-2:]
        v = torch.matmul(ffeats, f.flatten(3)).reshape(B, S, N, h, w) / 128 ** 0.5
        loc = coords.reshape(B * S * N, 1, 1, 2) / 2 ** i + window
        grid = torch.cat([2 * loc[..., :1] / (w - 1) - 1, 2 * loc[..., 1:] / (h - 1) - 1], dim=-1)
        taps.append(F.grid_sample(v.reshape(B * S * N, 1, h, w), grid, align_corners=True).view(B, S, N, -1))
    return torch.cat(taps, dim=-1).permute(0, 2, 1, 3).reshape(B * N, S, -1)


@pytest.mark.gpu
def test_memory_at_train_shape():
    """train.py's per-GPU shape: B=4, N=768, 4 iterations, 48 x 64 maps"""
    B, N, I, H, W = 4, 768, 4, 48, 64
    levels = _levels(B, H, W, seed=11)
    g = torch.Generator(device=DEV).manual_seed(12)
    ffs = [torch.randn(B * N, S, 128, device=DEV, generator=g) for _ in range(I)]
    cos = [_coords(B, N, H, W, seed=13 + i, special=False) for i in range(I)]
    dcs = [torch.randn(B * N, S, 196, device=DEV, generator=g) for _ in range(I)]
    peaks = {}
    for name, fn in (("cuda", torch_path.local_corr_cuda), ("torch", _torch_corr)):
        lv = [t.clone().requires_grad_(True) for t in levels]
        ff = [f.clone().requires_grad_(True) for f in ffs]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        loss = sum((fn(ff[i], lv, cos[i]) * dcs[i]).sum() for i in range(I))
        loss.backward()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del lv, ff, loss
        torch.cuda.empty_cache()
    vol = 4 * B * S * N * sum((H >> l) * (W >> l) for l in range(4))
    print(f"correlation forward + backward over {I} iterations at B={B}, N={N}, {H}x{W}: peak above inputs cuda "
          f"{peaks['cuda'] / 2**20:.0f} MiB, torch {peaks['torch'] / 2**20:.0f} MiB (one iteration's volumes: "
          f"{vol / 2**20:.0f} MiB)")
    assert peaks["cuda"] <= 256 * 2**20


# ------------------------------------------------------------------------------------------------ 8. routing

@pytest.mark.gpu
def test_routing(monkeypatch):
    rgbs, xys, tg, vg, va = _train_inputs(B=1, N=16, seed=8)
    calls = {"grid_sample": 0, "matmul": 0, "local_corr_cuda": 0}
    real = {"grid_sample": F.grid_sample, "matmul": torch.matmul, "local_corr_cuda": torch_path.local_corr_cuda}

    def spy(name):
        def f(*a, **k):
            calls[name] += 1
            return real[name](*a, **k)
        return f

    monkeypatch.setattr(F, "grid_sample", spy("grid_sample"))
    monkeypatch.setattr(torch, "matmul", spy("matmul"))
    monkeypatch.setattr(torch_path, "local_corr_cuda", spy("local_corr_cuda"))

    def run(m, iters=2):
        for k in calls:
            calls[k] = 0
        _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
        sum(losses).backward()
        return dict(calls)

    sd = po.init_state_dict(seed=3, head_scale=0.05)
    m = Pips(S=8, stride=8, loss_path="fused", corr_path="cuda").to(DEV).train()
    m.load_state_dict(sd)
    assert run(m) == {"grid_sample": 0, "matmul": 0, "local_corr_cuda": 2}      # no all-pairs volume at all
    m = Pips(S=8, stride=8, corr_path="cuda").to(DEV).train()                   # dense score maps: volumes, no grid_sample
    m.load_state_dict(sd)
    assert run(m) == {"grid_sample": 0, "matmul": 8, "local_corr_cuda": 2}
    monkeypatch.setenv("PIPS_B200_CORR", "cuda")
    m = Pips(S=8, stride=8, loss_path="fused").to(DEV).train()
    m.load_state_dict(sd)
    assert m.corr_path == "cuda" and run(m)["local_corr_cuda"] == 2
    monkeypatch.delenv("PIPS_B200_CORR")
    m = Pips(S=8, stride=8, loss_path="fused").to(DEV).train()
    m.load_state_dict(sd)
    assert m.corr_path == "torch" and run(m) == {"grid_sample": 8, "matmul": 8, "local_corr_cuda": 0}


@pytest.mark.gpu
def test_channels_last_levels_are_free_after_encoder_cuda():
    """avg_pool2d keeps encoder_cuda's channels-last strides: forward_torch's permute(...).contiguous() copies nothing"""
    m = Pips(S=8, stride=8).to(DEV)
    rgbs = po.smooth_video(1, 8, 128, 128, seed=1).to(DEV)
    fmaps = torch_path.encoder_cuda(m.fnet, rgbs)
    pyr = [fmaps]
    for _ in range(3):
        f = F.avg_pool2d(pyr[-1].flatten(0, 1), 2, stride=2)
        pyr.append(f.reshape(1, 8, *f.shape[1:]))
    for lv in pyr:
        assert lv.permute(0, 1, 3, 4, 2).contiguous().data_ptr() == lv.data_ptr()
