"""Sparse score maps (SURVEY.md section 8f-3, pips_heatmap) against the reference's recorded fcps and the
dense torch path."""
import os

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from pips_b200 import Pips
from tests.golden.make_golden import FCP_SEL, LOSS_CASE, case_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_outputs.npz"))


def _model(**kw):
    c = LOSS_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    m = Pips(S=8, stride=c["stride"], **kw).to(DEV).eval()
    m.load_state_dict(sd, strict=True)
    return m


@pytest.mark.parametrize("mode", ["strict", "default", "bf16feat"])
def test_score_maps_match_reference(mode):
    kw = {"strict": dict(precision="fp32", fnet_mode="plain"), "default": {}, "bf16feat": dict(feat_dtype="bf16")}[mode]
    tol = {"strict": 5e-4, "default": 5e-3, "bf16feat": 0.5}[mode]
    c = LOSS_CASE
    m = _model(**kw)
    rgbs, xys, _ = case_inputs(c)
    fcps, preds, vis_e = m.score_maps(xys.to(DEV), rgbs.to(DEV), FCP_SEL, iters=c["iters"])
    ref = GOLD["loss_s8/fcps_sel"]
    assert tuple(fcps.shape) == ref.shape
    err = np.abs(fcps.cpu().numpy() - ref).max()
    print(f"score maps [{mode}]: max err {err:.3e} (|fcps| max {np.abs(ref).max():.1f})")
    assert err < tol
    # the run that produced them is the ordinary forward
    assert np.abs(torch.stack(preds).cpu().numpy() - GOLD["loss_s8/preds"]).max() < (1e-3 if mode != "bf16feat" else 5e-2)


def test_score_maps_equal_dense_torch_path_selection():
    """fcps[:, :, :, sel] of the dense, differentiable path (the one the losses consume) == the sparse kernel."""
    from pips_b200 import torch_path
    c = LOSS_CASE
    m = _model(precision="fp32", fnet_mode="plain")
    rgbs, xys, _ = case_inputs(c)
    rgbs, xys = rgbs.to(DEV), xys.to(DEV)
    seen = {}
    real = torch_path.score_map_loss

    def spy(fcps, *a, **k):
        seen["fcps"] = fcps.detach()
        return real(fcps, *a, **k)

    from tests.golden.make_golden import loss_targets
    tg, vg, va = loss_targets(c, xys.cpu())
    torch_path.score_map_loss = spy
    try:
        with torch.no_grad():
            m(xys, rgbs, iters=c["iters"], trajs_g=tg.to(DEV), vis_g=vg.to(DEV), valids=va.to(DEV))
    finally:
        torch_path.score_map_loss = real
    sel = [8, 0, 3, 3]                                          # unsorted, repeated
    fcps, _, _ = m.score_maps(xys, rgbs, sel, iters=c["iters"])
    err = (fcps - seen["fcps"][:, :, :, sel]).abs().max().item()
    print("sparse vs dense torch path: max err", err, "of |fcps| max", seen["fcps"].abs().max().item())
    assert err < 2e-3                     # |fcps| ~ 50; the two runs' ffeats differ by fp32 summation order


def test_score_maps_chunking_is_transparent():
    c = LOSS_CASE
    rgbs, xys, _ = case_inputs(c)
    rgbs, xys = rgbs.to(DEV), xys.to(DEV)
    sel = [7, 1, 4]
    a, pa, _ = _model().score_maps(xys, rgbs, sel, iters=2)
    b, pb, _ = _model(max_seqs=8).score_maps(xys, rgbs, sel, iters=2)        # 2 batches x 4 particles per chunk
    assert torch.equal(a, b)
    assert torch.equal(torch.stack(pa), torch.stack(pb))


def test_heatmap_rejects_bad_arguments():
    from pips_b200 import _lib as L
    lib = L.load()
    assert lib.pips_heatmap(None, 0, 1, 8, 4, 16, 16, None, None, None, 1, None, None, 0, None) != 0
    assert b"pips_heatmap" in lib.pips_last_error()
    m = _model()
    c = LOSS_CASE
    rgbs, xys, _ = case_inputs(c)
    with pytest.raises(AssertionError):
        m.score_maps(xys.to(DEV), rgbs.to(DEV), [c["N"]], iters=1)
