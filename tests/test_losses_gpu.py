"""Evaluation with ground truth on the CUDA path (Pips(loss_path='cuda')): the fused score-map loss kernel
(csrc/scoremap_loss.cu) against the reference's recorded losses, the dense torch path and dense score maps."""
import os

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path
from pips_b200.engine import Pyramid
from tests.golden.make_golden import LOSS_CASE, case_inputs, loss_targets

DEV = "cuda:0"
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_outputs.npz"))
STRICT = dict(precision="fp32", fnet_mode="plain")


def _model(c=LOSS_CASE, **kw):
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    m = Pips(S=8, stride=c["stride"], **kw).to(DEV).eval()
    m.load_state_dict(sd, strict=True)
    return m


def _loss_case():
    c = LOSS_CASE
    rgbs, xys, _ = case_inputs(c)
    tg, vg, va = loss_targets(c, xys)
    return c, rgbs.to(DEV), xys.to(DEV), tg.to(DEV), vg.to(DEV), va.to(DEV)


def _gt_call(m, c, rgbs, xys, tg, vg, va, iters=None):
    with torch.no_grad():
        return m(xys, rgbs, iters=iters or c["iters"], trajs_g=tg, vis_g=vg, valids=va)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["strict", "default"])
def test_losses_match_reference(mode):
    c, rgbs, xys, tg, vg, va = _loss_case()
    m = _model(loss_path="cuda", **(STRICT if mode == "strict" else {}))
    preds, preds2, vis_e, losses = _gt_call(m, c, rgbs, xys, tg, vg, va)
    assert len(preds2) == c["iters"] + 4
    assert all(l.dim() == 0 and l.dtype == torch.float32 and l.is_cuda for l in losses)
    got = np.array([float(l) for l in losses])
    ref = GOLD["loss_s8/losses"]
    err = np.abs(got - ref) / np.maximum(1.0, np.abs(ref))
    print(f"losses [{mode}]: got {got}, reference {ref}, scaled |err| {err}")
    assert (err <= (5e-4 if mode == "strict" else 2e-3)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [True, False])
def test_tracking_is_unaffected_by_losses(graph):
    c, rgbs, xys, tg, vg, va = _loss_case()
    m = _model(loss_path="cuda")
    m.engine.use_graph = graph
    preds, _, vis_e, losses = _gt_call(m, c, rgbs, xys, tg, vg, va)
    with torch.no_grad():
        p0, _, v0, l0 = m(xys, rgbs, iters=c["iters"])
    assert l0 is None and losses is not None
    assert torch.equal(torch.stack(preds), torch.stack(p0)) and torch.equal(vis_e, v0)


def _realistic(seed=21, B=1, H=384, W=512, N=256):
    c = dict(B=B, H=H, W=W, N=N, stride=8, iters=6, head_scale=0.05, seed=seed)
    rgbs = po.smooth_video(B, 8, H, W, seed=100 + seed)
    xys = po.random_queries(B, N, H, W, seed=200 + seed)
    g = torch.Generator().manual_seed(400 + seed)
    tg = xys[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 4.0, 1)
    vg = (torch.rand(B, 8, N, generator=g) > 0.2).float()
    va = (torch.rand(B, 8, N, generator=g) > 0.1).float()
    return c, rgbs.to(DEV), xys.to(DEV), tg.to(DEV), vg.to(DEV), va.to(DEV)


@pytest.mark.gpu
def test_losses_match_dense_torch_path_at_eval_shape():
    """The test_on_flt crop: B=1, 8 x 384 x 512, stride 8, N=256, 6 iterations, strict mode, both paths on this GPU."""
    c, rgbs, xys, tg, vg, va = _realistic()
    m = _model(c, loss_path="cuda", **STRICT)
    _, _, _, lc = _gt_call(m, c, rgbs, xys, tg, vg, va)
    m.loss_path = "torch"
    _, _, _, lt = _gt_call(m, c, rgbs, xys, tg, vg, va)
    lc, lt = [float(x) for x in lc], [float(x) for x in lt]
    rel = [abs(a - b) / max(abs(b), 1e-12) for a, b in zip(lc, lt)]
    print(f"cuda {lc} vs dense torch {lt}: relative differences {rel}")
    assert rel[2] <= 1e-4
    assert rel[0] <= 1e-4 and rel[1] <= 1e-3


def _dense_terms(scores, target):
    """Per-row (pos, neg) of the balanced CE, in fp64, from dense scores (rows, P) and targets (rows,)."""
    s = scores.double()
    sp = torch.nn.functional.softplus(s)
    keep = target >= 0
    t = target.clamp(min=0).long()
    at_t = s.gather(1, t[:, None])[:, 0]
    pos = torch.where(keep, torch.nn.functional.softplus(-at_t), torch.zeros_like(at_t))
    neg = torch.where(keep, sp.sum(1) - sp.gather(1, t[:, None])[:, 0], torch.zeros_like(at_t))
    return pos, neg


@pytest.mark.gpu
@pytest.mark.parametrize("H8,W8", [(16, 16), (45, 80), (96, 128)])
@pytest.mark.parametrize("N", [9, 200])
def test_kernel_rows_match_dense_score_maps(H8, W8, N):
    lib = L.load()
    B, S = 1, 8
    P = H8 * W8
    g = torch.Generator(device=DEV).manual_seed(H8 * 1000 + N)
    fmaps = torch.randn(B * S, 128, H8, W8, device=DEV, generator=g)
    pyr = Pyramid(B * S, H8, W8, L.FEAT_F32, DEV)
    st = torch.cuda.current_stream().cuda_stream
    pyr.build(fmaps, st)
    ffeats = torch.randn(B * N, S, 128, device=DEV, generator=g) * 4.0
    target = torch.randint(0, P, (B, S, N), device=DEV, generator=g, dtype=torch.int32)
    target[0, :, 0] = -1                                           # rows the loss ignores
    target[0, 1::2, 1] = 0                                         # first and last pixel
    target[0, 0::2, 1] = P - 1
    n_split = lib.pips_scoremap_splits(H8, W8)
    g_hi = torch.empty(B * S, P, 128, dtype=torch.bfloat16, device=DEV)
    g_lo = torch.empty_like(g_hi)
    neg = torch.full((B * S * N, n_split), float("nan"), device=DEV)
    pos = torch.full((B * S * N,), float("nan"), device=DEV)
    L.check(lib.pips_scoremap_basis(pyr.f32_ptrs, B * S, H8, W8, L.ptr(g_hi), L.ptr(g_lo), st), "basis")
    L.check(lib.pips_scoremap_loss(L.ptr(g_hi), L.ptr(g_lo), L.ptr(ffeats), B, S, N, H8, W8, L.ptr(target), L.ptr(neg),
                                   L.ptr(pos), st), "loss")
    # dense reference: pips_heatmap over every particle (fp32 CUDA cores), softplus in fp64
    sel = torch.arange(N, dtype=torch.int32, device=DEV)
    dense = torch.empty(B * S, N, H8, W8, device=DEV)
    scratch = torch.empty(lib.pips_heatmap_scratch_floats(B * S, N, H8, W8), device=DEV)
    L.check(lib.pips_heatmap(L.ptr_array(pyr.f32), L.FEAT_F32, B, S, N, H8, W8, L.ptr(ffeats), L.ptr(sel), None, N,
                             L.ptr(scratch), L.ptr(dense), N * P, st), "heatmap")
    torch.cuda.synchronize()
    rp, rn = _dense_terms(dense.reshape(B * S * N, P), target.reshape(-1))
    assert not torch.isnan(neg).any() and not torch.isnan(pos).any()      # every row and split written
    got_neg = neg.double().sum(1)
    rel = ((got_neg - rn).abs() / rn.abs().clamp(min=1e-30))[target.reshape(-1) >= 0].max().item()
    abs_pos = (pos.double() - rp).abs().max().item()
    print(f"{H8}x{W8} N={N} n_split={n_split}: neg max rel err {rel:.2e}, pos max abs err {abs_pos:.2e}")
    assert rel <= 1e-4 and abs_pos <= 1e-3
    ign = target.reshape(-1) < 0
    assert (neg[ign] == 0).all() and (pos[ign] == 0).all()


@pytest.mark.gpu
def test_chunking_graphs_and_repeats_are_bit_identical():
    c, rgbs, xys, tg, vg, va = _loss_case()
    ref = _gt_call(_model(loss_path="cuda"), c, rgbs, xys, tg, vg, va)[3]
    again_model = _model(loss_path="cuda")
    a = _gt_call(again_model, c, rgbs, xys, tg, vg, va)[3]
    b = _gt_call(again_model, c, rgbs, xys, tg, vg, va)[3]
    chunked = _gt_call(_model(loss_path="cuda", max_seqs=8), c, rgbs, xys, tg, vg, va)[3]   # 4 particles per chunk
    eager_model = _model(loss_path="cuda")
    eager_model.engine.use_graph = False
    eager = _gt_call(eager_model, c, rgbs, xys, tg, vg, va)[3]
    for other in (a, b, chunked, eager):
        assert torch.equal(ref[2], other[2]), (ref, other)
        assert torch.equal(ref[0], other[0]) and torch.equal(ref[1], other[1])


@pytest.mark.gpu
def test_reference_edge_semantics():
    # .5 positions round half to even, out-of-bounds targets are dropped: the kernel's targets reproduce
    # torch_path.score_map_loss on arbitrary score maps
    B, S, N, I, H8, W8 = 1, 8, 6, 2, 8, 12
    g = torch.Generator(device=DEV).manual_seed(5)
    tg = torch.tensor([[0.5, 0.5], [1.5, 2.5], [10.5, 6.5], [11.5, 3.0], [-0.5, 7.4], [3.0, 7.5]], device=DEV)
    tg = tg[None, None].repeat(B, S, 1, 1)
    vis = torch.ones(B, S, N, device=DEV)
    val = torch.ones(B, S, N, device=DEV)
    val[0, 3, 2] = 0
    vis[0, 4, 1] = 0
    t = torch_path.score_map_targets(tg, vis, val, H8, W8)
    assert t[0, 0].tolist() == [0, 2 * W8 + 2, 6 * W8 + 10, -1, 7 * W8 + 0, -1]      # 11.5 -> 12, 7.5 -> 8: outside
    assert t[0, 3, 2] == -1 and t[0, 4, 1] == -1
    fcps = torch.randn(B, S, I, N, H8, W8, device=DEV, generator=g, dtype=torch.float64) * 3
    want = torch_path.score_map_loss(fcps, tg.double(), vis, val)
    rows = fcps.permute(0, 1, 3, 2, 4, 5).reshape(B * S * N * I, H8 * W8)
    pos, neg = _dense_terms(rows, t.reshape(-1).repeat_interleave(I))
    k = (t >= 0).sum().item() * I
    got = pos.sum() / (1e-6 + k) + neg.sum() / (1e-6 + k * (H8 * W8 - 1))
    assert abs(got.item() - want.item()) < 1e-6 * max(1.0, abs(want.item()))

    # no visible target at all: the score-map loss is exactly 0, as in the reference
    c, rgbs, xys, tgc, vgc, vac = _loss_case()
    losses = _gt_call(_model(loss_path="cuda"), c, rgbs, xys, tgc, torch.zeros_like(vgc), vac)[3]
    assert losses[2].item() == 0.0
    # every target outside the map: dropped, loss 0 as well
    losses = _gt_call(_model(loss_path="cuda"), c, rgbs, xys, tgc + 1e4, vgc, vac)[3]
    assert losses[2].item() == 0.0


@pytest.mark.gpu
def test_routing(monkeypatch):
    c, rgbs, xys, tg, vg, va = _loss_case()
    calls = []
    real = torch_path.forward_torch

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(torch_path, "forward_torch", spy)
    monkeypatch.delenv("PIPS_B200_LOSSES", raising=False)
    _gt_call(_model(), c, rgbs, xys, tg, vg, va)                  # default: the dense path
    assert len(calls) == 1
    m = _model(loss_path="cuda")
    _gt_call(m, c, rgbs, xys, tg, vg, va)
    assert len(calls) == 1                                         # the CUDA path
    m(xys, rgbs, iters=1, trajs_g=tg, vis_g=vg, valids=va)        # grad enabled
    assert len(calls) == 2
    with torch.no_grad():
        m(xys, rgbs, iters=1, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert len(calls) == 3
    monkeypatch.setenv("PIPS_B200_LOSSES", "cuda")
    _gt_call(_model(), c, rgbs, xys, tg, vg, va)
    assert len(calls) == 3
    with pytest.raises(ValueError):
        Pips(S=8, stride=8, loss_path="cudnn")


@pytest.mark.gpu
def test_memory_at_cfg3():
    """B=4, 8 x 384 x 512, N=4096: the dense score maps alone would be 4*8*6*4096*48*64*4 B = 9.7 GB."""
    c, rgbs, xys, tg, vg, va = _realistic(seed=22, B=4, N=4096)
    peaks = {}
    for name in ("plain", "gt"):
        m = _model(c, loss_path="cuda")
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with torch.no_grad():
            if name == "gt":
                m(xys, rgbs, iters=6, trajs_g=tg, vis_g=vg, valids=va)
            else:
                m(xys, rgbs, iters=6)
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del m
    extra = peaks["gt"] - peaks["plain"]
    print(f"peak: plain {peaks['plain'] / 2**20:.0f} MiB, with losses {peaks['gt'] / 2**20:.0f} MiB (+{extra / 2**20:.0f} MiB)")
    assert extra <= 512 * 2**20


def test_scoremap_entry_points_validate_arguments_without_gpu():
    import ctypes as C
    lib = L.load()
    assert lib.pips_scoremap_splits(48, 64) == 6 and lib.pips_scoremap_splits(16, 16) == 1 and lib.pips_scoremap_splits(0, 4) == 0
    p = C.c_void_p(256)
    assert lib.pips_scoremap_loss(None, p, p, 1, 8, 4, 16, 16, p, p, p, None) != 0
    assert b"pips_scoremap_loss: null pointer" in lib.pips_last_error()
    assert lib.pips_scoremap_loss(p, p, p, 1, 7, 4, 16, 16, p, p, p, None) != 0               # S != 8
    assert lib.pips_scoremap_loss(p, p, p, 1, 8, 0, 16, 16, p, p, p, None) != 0               # no particles
    assert lib.pips_scoremap_loss(C.c_void_p(264), p, p, 1, 8, 4, 16, 16, p, p, p, None) != 0 # misaligned G
    assert b"16-byte aligned" in lib.pips_last_error()
    assert lib.pips_scoremap_basis(None, 8, 16, 16, p, p, None) != 0
    lv = (C.c_void_p * 4)(256, 256, 256, 256)
    assert lib.pips_scoremap_basis(lv, 8, 4, 16, p, p, None) != 0                              # too small for 4 levels
    assert b"too small" in lib.pips_last_error()
    assert lib.pips_scoremap_basis(lv, 0, 16, 16, p, p, None) != 0
