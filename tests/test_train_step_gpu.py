"""A whole training step with all four CUDA autograd nodes at once (Pips(loss_path='fused', mixer_path='cuda',
encoder_path='cuda', corr_path='cuda'): encoder_cuda, local_corr_cuda, delta_block_cuda, fused_score_map_loss) against
fp64 autograd of a teacher-forced restatement of forward_torch's training path.

The step is smooth except at two kinds of decision: the encoder's ReLUs and the bilinear cells (and zero padding) that
the detached coordinates of every iteration select.  Pinned to the CUDA forward's own choices -- the ReLU masks of
tests/test_encoder_grad_gpu.py's _cuda_masks and the coordinates forward_torch hands local_corr_cuda -- the step is a
smooth function of the parameters, and its fp64 gradient is the exact target.  There the fnet gradient has four sources
that autograd sums before _EncoderFn.backward runs: the initial feature's sample_clamped, the corr node's level
gradients, the fused loss's level gradients and the avg_pool2d chain between the levels; level 0 is encoder_cuda's own
channels-last output.  Each gradient and loss is compared as max|err| / max|ref| against max(2 x strict fp32's error
under the same decisions, a floor derived from the bounds of the per-node tests)."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path
from tests.test_encoder_grad_gpu import BF16X3_BOUND, _cuda_masks, _masked_forward
from tests.test_mixer_grad_gpu import MIX_FLOOR

DEV = "cuda:0"
MODULES = ("fnet", "delta_block", "norm", "ffeat_updater", "vis_predictor")


def _reference_step(fnet, delta_block, norm, ffeat_updater, vis_predictor, rgbs, xys, trajs_g, vis_g, valids, iters,
                    masks=None, coords=None):
    """forward_torch's training path (is_train=True, corr_path='torch', dense score maps) in torch ops, for modules and
    inputs of any dtype.  masks: the encoder's ReLU decisions (_cuda_masks' order) to evaluate it under instead of its
    own; coords: the (B, S, N, 2) coordinates to start every iteration from instead of the detached result of the last.
    Returns the three losses and the coordinates each iteration started from."""
    dtype = next(fnet.parameters()).dtype
    B, N, _ = xys.shape
    _, S, C, H, W = rgbs.shape
    stride = fnet.stride
    H8, W8 = H // stride, W // stride
    r = 3
    dev = rgbs.device
    xys, trajs_g, vis_g, valids = (t.to(dtype) for t in (xys, trajs_g, vis_g, valids))

    x = (2 * (rgbs.to(dtype) / 255.0) - 1.0).reshape(B * S, C, H, W)
    fmaps = (fnet(x) if masks is None else _masked_forward(fnet, x, masks)).reshape(B, S, -1, H8, W8)
    c = (xys.clone() / float(stride)).reshape(B, 1, N, 2).repeat(1, S, 1, 1)
    pyramid = [fmaps]
    for _ in range(3):
        f = F.avg_pool2d(pyramid[-1].flatten(0, 1), 2, stride=2)
        pyramid.append(f.reshape(B, S, *f.shape[1:]))
    ffeat = torch_path.sample_clamped(fmaps[:, 0], c[:, 0, :, 0], c[:, 0, :, 1])
    ffeats = ffeat.unsqueeze(1).repeat(1, S, 1, 1)

    offs = torch.linspace(-r, r, 2 * r + 1, device=dev, dtype=dtype)
    window = torch.stack(torch.meshgrid(offs, offs, indexing="ij"), dim=-1).view(1, 2 * r + 1, 2 * r + 1, 2)
    # the model's fp32 constants (nets/pips.py:519, :397): in fp64, the exact sqrt(128) is 1.7e-8 off the model's
    times = torch.linspace(0, S, S, device=dev).to(dtype).reshape(1, S, 1)
    scale = torch.sqrt(torch.tensor(float(fmaps.shape[2]))).to(dtype)
    preds, fcps, used = [], [], []
    for i in range(iters):
        c = c.detach() if coords is None else coords[i].to(dtype)
        used.append(c)
        feats_ = ffeats.permute(0, 2, 1, 3).reshape(B * N, S, -1)
        vols = [torch.matmul(ffeats, f.flatten(3)).reshape(B, S, N, *f.shape[-2:]) / scale for f in pyramid]
        fcps.append(sum(F.interpolate(v.flatten(0, 1), (H8, W8), mode="bilinear", align_corners=True).reshape(B, S, N, H8, W8)
                        for v in vols))
        taps = []
        for l, v in enumerate(vols):
            h, w = v.shape[-2:]
            loc = c.reshape(B * S * N, 1, 1, 2) / 2 ** l + window
            if h > 1 and w > 1:
                grid = torch.cat([2 * loc[..., :1] / (w - 1) - 1, 2 * loc[..., 1:] / (h - 1) - 1], dim=-1)
                taps.append(F.grid_sample(v.reshape(B * S * N, 1, h, w), grid, align_corners=True).view(B, S, N, -1))
            else:
                grid = torch.cat([(2 * loc[..., :1] + 1) / w - 1, (2 * loc[..., 1:] + 1) / h - 1], dim=-1)
                taps.append(F.grid_sample(v.reshape(B * S * N, 1, h, w), grid, align_corners=False).view(B, S, N, -1))
        fcorr = torch.cat(taps, dim=-1).permute(0, 2, 1, 3).reshape(B * N, S, -1)
        flow = (c - c[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        flow = torch.cat([flow, times.expand(B * N, -1, -1)], dim=2)
        x_mix = torch.cat([feats_, fcorr, torch_path.motion_embedding(flow)], dim=2)
        delta = delta_block(x_mix)
        dfeat = delta[:, :, 2:].reshape(B * N * S, -1)
        feats_ = ffeat_updater(norm(dfeat)) + feats_.reshape(B * N * S, -1)
        ffeats = feats_.reshape(B, N, S, -1).permute(0, 2, 1, 3)
        c = c + delta[:, :, :2].reshape(B, N, S, 2).permute(0, 2, 1, 3)
        preds.append(c * stride)
    vis_e = vis_predictor(ffeats.reshape(B * S * N, -1)).reshape(B, S, N)
    losses = (torch_path.sequence_loss(preds, trajs_g, vis_g, valids, 0.8),
              torch_path.balanced_ce_loss(vis_e, vis_g, valids)[0],
              torch_path.score_map_loss(torch.stack(fcps, dim=2), trajs_g / float(stride), vis_g, valids))
    return losses, used


def _copies(model, dtype):
    mods = [copy.deepcopy(getattr(model, n)).to(dtype) for n in MODULES]
    mods[0].mode = "plain"
    return mods


def _reference_grads(mods, inputs, iters, masks=None, coords=None):
    """_reference_step and sum(losses).backward() -> (losses, {model parameter name: gradient}, coordinates)"""
    for m in mods:
        m.zero_grad(set_to_none=True)
    losses, used = _reference_step(*mods, *inputs, iters, masks=masks, coords=coords)
    sum(losses).backward()
    grads = {f"{p}.{n}": t.grad.detach() for p, m in zip(MODULES, mods) for n, t in m.named_parameters() if t.grad is not None}
    return [l.detach() for l in losses], grads, [u.detach() for u in used]


def _model_step(m, rgbs, xys, tg, vg, va, iters):
    m.zero_grad(set_to_none=True)
    _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    sum(losses).backward()
    return [l.detach() for l in losses], {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


def _inputs(B, N, H, W, seed, dev):
    """rgbs, xys, trajs_g, vis_g, valids: queries on the four frame edges and corners as well as inside, two tracks whose
    ground truth leaves the feature map (the score-map target drops those rows), one track never visible, about 10% of
    the valids zero"""
    rgbs = po.smooth_video(B, 8, H, W, seed=100 + seed)
    xys = po.random_queries(B, N, H, W, seed=200 + seed)
    edge = torch.tensor([[0.0, 0.0], [W - 1.0, 0.0], [0.0, H - 1.0], [W - 1.0, H - 1.0],
                         [W / 2 + 0.3, 0.0], [W / 2 - 0.7, H - 1.0], [0.0, H / 2 + 0.4], [W - 1.0, H / 2 - 0.2]])
    k = min(len(edge), N // 2)
    xys[:, :k] = edge[:k]
    g = torch.Generator().manual_seed(400 + seed)
    tg = xys[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 3.0, 1)
    tg[:, 3:, k, 0] = -20.0                         # left of the map
    tg[:, 5:, k + 1, 1] = H + 20.0                  # below it
    vg = (torch.rand(B, 8, N, generator=g) > 0.2).float()
    vg[0, :, k + 2] = 0
    va = (torch.rand(B, 8, N, generator=g) > 0.1).float()
    return tuple(t.to(dev) for t in (rgbs, xys, tg, vg, va))


# ------------------------------------------------------------------------------------------- the reference, on the CPU

def test_reference_step_is_forward_torch():
    """The restatement has the bits of Pips' training path on the CPU (forward_torch with the torch correlation and
    the dense score maps), free-running and pinned to its own coordinates: the three losses and every gradient.  At
    64x96 level 3 is one pixel: forward_torch's grid_sample with align_corners=True divided by zero there and every
    loss was NaN."""
    B, N, H, W, iters = 1, 8, 64, 96, 2
    model = Pips(S=8, stride=8).train()
    model.load_state_dict(po.init_state_dict(seed=3, head_scale=0.05), strict=True)
    inputs = _inputs(B, N, H, W, seed=1, dev="cpu")
    lm, gm = _model_step(model, *inputs, iters)
    assert all(torch.isfinite(l) for l in lm)
    mods = _copies(model, torch.float32)
    lr, gr, used = _reference_grads(mods, inputs, iters)
    lp, gp, _ = _reference_grads(mods, inputs, iters, coords=used)
    assert len(used) == iters
    assert set(gr) == set(gm) == set(gp) and len(gm) == len(list(model.parameters()))
    for name, losses, grads in (("free-running", lr, gr), ("pinned", lp, gp)):
        assert all(torch.equal(a, b) for a, b in zip(losses, lm)), f"{name}: losses {losses} against {lm}"
        diff = [n for n in gm if not torch.equal(grads[n], gm[n])]
        assert not diff, f"{name}: gradients differ in {diff[:5]}"


# ------------------------------------------------------------------------------------------- the composed step on H100

def _cuda_model(stride, head_scale, seed=3):
    m = Pips(S=8, stride=stride, loss_path="fused", mixer_path="cuda", encoder_path="cuda", corr_path="cuda").to(DEV).train()
    m.load_state_dict(po.init_state_dict(seed=seed, head_scale=head_scale), strict=True)
    return m


def _spied_step(monkeypatch, m, inputs, iters):
    """one CUDA step with a spy on each of the four nodes: (losses, gradients, per-iteration coordinates, call counts)"""
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


def _free_relu_decisions(fnet64, rgbs):
    """every ReLU decision of the free-running fp64 Encoder, in _cuda_masks' order"""
    B, S, C, H, W = rgbs.shape
    got, real = [], F.relu

    def relu(v, *a, **k):
        got.append(v > 0)
        return real(v, *a, **k)

    with torch.no_grad(), pytest.MonkeyPatch.context() as mp:
        mp.setattr(F, "relu", relu)
        fnet64((2 * (rgbs.double() / 255.0) - 1.0).reshape(B * S, C, H, W))
    return got


def _cells(coords, levels=4):
    """the bilinear cell floor(c / 2^l) of every iteration, frame, track and level: (I, B, S, N, L, 2)"""
    return torch.stack([torch.stack([torch.floor(c.double() / 2 ** l) for l in range(levels)], -2) for c in coords])


# (B, N, H, W, stride, iters, head_scale).  The worst ratio to the bound measured on an H100 80GB HBM3 (700 W) follows
# each case; at each of these worst tensors the bound is the floor.
STEP_CASES = [
    # odd levels 17x25 -> 8x12 -> 4x6 -> 2x3 (floors in avg_pool2d); N not a multiple of 8; 74 mixer rows in 256-row tiles
    (2, 37, 136, 200, 8, 4, 0.05),       # 0.17, fnet.conv1.weight
    (2, 37, 136, 200, 8, 4, 1.0),        # 0.17, fnet.conv1.weight; tracks pushed beyond the frame: zero padding,
                                         # out-of-map taps in the corr gradient
    (1, 768, 384, 512, 8, 4, 0.05),      # 0.74, fnet.conv1.weight; one train.py sample: N=768, I=4, 384x512 crop
    (1, 16, 64, 64, 8, 2, 0.05),         # 0.29, a token-mixing FC1 bias; the smallest map corr_path='cuda' takes: 8x8
                                         # level 0, 1x1 level 3
    (1, 24, 96, 128, 4, 3, 0.05),        # 0.68, vis_predictor.0.bias; stride 4, the demo model's
]


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,H,W,stride,iters,head_scale", STEP_CASES)
def test_composed_step_matches_fp64(monkeypatch, B, N, H, W, stride, iters, head_scale):
    """Losses and every parameter gradient of one step on the four CUDA nodes against fp64 autograd of _reference_step
    under the CUDA forward's ReLU decisions and coordinates, per tensor max|err| / max|ref| within max(2 x strict fp32's
    error under the same decisions, floor).  The floors are the per-node tests' bounds along the longest chain: every
    iteration's mixer carries the feature state (iters x MIX_FLOOR), and an fnet gradient adds the encoder's own
    (BF16X3_BOUND).  The free-running fp64 step's errors are printed, not bounded: a ReLU or a cell decided the other way
    moves a gradient by far more than rounding.  Worst ratio per case, measured on an H100 80GB HBM3 (700 W): see
    DESIGN.md section 7."""
    model = _cuda_model(stride, head_scale)
    inputs = _inputs(B, N, H, W, seed=H + N, dev=DEV)
    check_pinned_step(monkeypatch, model, inputs, iters, f"B={B} N={N} {H}x{W}/{stride} iters={iters} head x{head_scale}")


def check_pinned_step(monkeypatch, model, inputs, iters, label):
    """test_composed_step_matches_fp64's check of one step of a CUDA-path model (the four nodes, or the three other
    than delta_block_cuda where model.mixer_path == 'torch') on inputs (rgbs, xys, trajs_g, vis_g, valids); asserts
    its bound and returns the step's (losses, {parameter name: gradient})"""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    rgbs = inputs[0]
    lc, gc, coords, calls = _spied_step(monkeypatch, model, inputs, iters)
    mix = iters if model.mixer_path == "cuda" else 0
    assert calls == {"encoder_cuda": 1, "local_corr_cuda": iters, "delta_block_cuda": mix, "fused_score_map_loss": 1}
    masks = _cuda_masks(model.fnet, rgbs)
    m64, m32 = _copies(model, torch.float64), _copies(model, torch.float32)
    l64, g64, _ = _reference_grads(m64, inputs, iters, masks=masks, coords=coords)
    l32, g32, _ = _reference_grads(m32, inputs, iters, masks=masks, coords=coords)
    lu, gu, cu = _reference_grads(m64, inputs, iters)
    relu_diff = sum((m != f).sum().item() for m, f in zip(masks, _free_relu_decisions(m64[0], rgbs)))
    cell_diff = (_cells(coords) != _cells(cu)).any(-1).sum().item()

    assert set(gc) == set(g64)
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

    cases = {f"loss{i}": (lc[i], l32[i], l64[i], lu[i]) for i in range(3)}
    cases.update({n: (gc[n], g32[n], g64[n], gu[n]) for n in g64 if n not in fnet_zero and n not in tok_zero})
    e = {n: (err(c, r), err(t, r), err(c, u)) for n, (c, t, r, u) in cases.items()}
    floor = {n: (BF16X3_BOUND if n.startswith("fnet.") else 0.0) + iters * MIX_FLOOR for n in e}
    ratio = {n: ec / max(2 * et, floor[n]) for n, (ec, et, _) in e.items()}
    worst = max(ratio, key=ratio.get)
    top = sorted(ratio, key=ratio.get, reverse=True)[:4]
    print(f"\n{label}: worst {worst} ratio {ratio[worst]:.3f}; "
          f"cuda / fp32 / cuda vs free-running fp64: {e[worst][0]:.2e} / {e[worst][1]:.2e} / {e[worst][2]:.2e}; "
          f"{relu_diff} ReLU decisions and {cell_diff} sample cells differ from the free-running fp64 step; losses "
          + " ".join(f"{ratio[f'loss{i}']:.3f}" for i in range(3)) + "; next " + ", ".join(f"{n} {ratio[n]:.3f}" for n in top[1:])
          + f"; worst free-running fp64 {max(v[2] for v in e.values()):.2e}")
    assert ratio[worst] <= 1.0, f"{worst}: {ratio[worst]:.3f} of its bound"
    return lc, gc


# ------------------------------------------------------------------------------------------- three checks of the step

SMALL = (2, 37, 136, 200, 8, 2)                   # B, N, H, W, stride, iters


def _small():
    B, N, H, W, stride, iters = SMALL
    return _cuda_model(stride, 0.05), _inputs(B, N, H, W, seed=9, dev=DEV), iters


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.gpu
def test_composed_step_is_deterministic():
    """Each node claims no atomics: so must the sum of their gradients"""
    model, inputs, iters = _small()
    la, ga = _model_step(model, *inputs, iters)
    lb, gb = _model_step(model, *inputs, iters)
    assert set(ga) == set(gb) and len(ga) == len(list(model.parameters()))
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(la, lb))
    assert all(torch.equal(_bits(ga[n]), _bits(gb[n])) for n in ga), [n for n in ga if not torch.equal(ga[n], gb[n])][:5]


LEVEL_KERNELS = ("pips_corr_grad_levels", "pips_scoremap_grad_basis", "pips_scoremap_basis_grad", "pips_conv_wgrad",
                 "pips_inorm_grad")
FEAT_KERNELS = ("pips_corr_grad_feats", "pips_scoremap_grad_feats")


@pytest.mark.gpu
def test_frozen_encoder(monkeypatch):
    """With the encoder frozen no fnet parameter gets a gradient, every other gradient keeps the bits of the trained
    encoder's step, and neither the level-gradient branches of the corr node and the fused loss nor the encoder's
    backward launch a kernel."""
    model, inputs, iters = _small()
    lib = L.load()
    counts = dict.fromkeys(LEVEL_KERNELS + FEAT_KERNELS, 0)

    def counted(name):
        real = getattr(lib, name)

        def f(*a):
            counts[name] += 1
            return real(*a)
        return f

    for n in counts:
        monkeypatch.setattr(lib, n, counted(n))
    lf, gf = _model_step(model, *inputs, iters)
    assert all(counts[n] > 0 for n in counts), counts
    counts.update(dict.fromkeys(counts, 0))
    model.fnet.requires_grad_(False)
    lz, gz = _model_step(model, *inputs, iters)
    assert not [n for n in gz if n.startswith("fnet.")]
    assert set(gz) == {n for n in gf if not n.startswith("fnet.")}
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(lz, lf))
    assert all(torch.equal(_bits(gz[n]), _bits(gf[n])) for n in gz), [n for n in gz if not torch.equal(gz[n], gf[n])][:5]
    assert all(counts[n] == 0 for n in LEVEL_KERNELS), counts
    # the first iteration's ffeats come from the frozen encoder alone: no gradient for them, so one corr call fewer
    assert counts["pips_corr_grad_feats"] == iters - 1 and counts["pips_scoremap_grad_feats"] == 1, counts


@pytest.mark.gpu
def test_replica_of_the_whole_model():
    """A replica of the whole Pips from torch.nn.parallel.replicate (what nn.DataParallel runs) gives the direct call's
    bits on one GPU, through its broadcast copies back to the parameters."""
    model, inputs, iters = _small()
    ld, gd = _model_step(model, *inputs, iters)
    rgbs, xys, tg, vg, va = inputs
    model.zero_grad(set_to_none=True)
    replica = torch.nn.parallel.replicate(model, [0])[0]
    assert len(list(replica.parameters())) == 0
    _, _, _, losses = replica(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    sum(losses).backward()
    assert all(torch.equal(_bits(a.detach()), _bits(b)) for a, b in zip(losses, ld))
    assert all(p.grad is not None and torch.equal(_bits(p.grad), _bits(gd[n])) for n, p in model.named_parameters())
