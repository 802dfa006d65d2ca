"""Models of window lengths 2..16 on the CUDA path: end to end against the unmodified reference's outputs
(tests/golden/reference_window.npz).  The kernels themselves are checked per element at these window lengths by
test_loop_kernels_gpu.py, test_tc_exact_gpu.py and test_scoremap_exact_gpu.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L
from tests.golden.make_golden_window import CASES, FCP_SEL, LOSS_CASE, case_inputs, loss_targets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_window.npz"))
TOL = {"fp32": 1e-3, "bf16x3": 1e-3, "bf16": 0.25}          # as tests/test_parity_gpu.py


def _model(c, **kw):
    m = Pips(S=c["S"], stride=c["stride"], **kw).to(DEV).eval()
    m.load_state_dict(po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"], S=c["S"]), strict=True)
    return m


def _run(m, c):
    rgbs, xys, extra = case_inputs(c)
    extra = {k: v.to(DEV) for k, v in extra.items()}
    with torch.no_grad():
        preds, _, vis_e, ffeat, _ = m(xys.to(DEV), rgbs.to(DEV), iters=c["iters"], return_feat=True, **extra)
    return torch.stack(preds).cpu(), vis_e.cpu(), ffeat.cpu()


@pytest.mark.parametrize("precision", ["bf16x3", "fp32", "bf16"])
@pytest.mark.parametrize("name", list(CASES))
def test_forward_matches_reference(name, precision):
    c = CASES[name]
    preds, vis_e, _ = _run(_model(c, precision=precision), c)
    err = np.abs(preds.numpy() - GOLD[name + "/preds"]).max()
    print(f"{name} {precision}: max |err| {err:.3e} px")
    assert err < TOL[precision]
    assert np.abs(vis_e.numpy() - GOLD[name + "/vis_e"]).max() < (5e-3 if precision != "bf16" else 0.5)


def test_simt_token_mixing_matches_reference():
    """PIPS_B200_TOKENMIX=simt is read once per process: every case in a child process."""
    code = ("import sys, numpy as np, torch; sys.path.insert(0, %r)\n"
            "from tests.test_window_gpu import CASES, GOLD, _model, _run\n"
            "for name, c in CASES.items():\n"
            "    preds, vis_e, _ = _run(_model(c), c)\n"
            "    err = np.abs(preds.numpy() - GOLD[name + '/preds']).max()\n"
            "    verr = np.abs(vis_e.numpy() - GOLD[name + '/vis_e']).max()\n"
            "    print(name, err, verr)\n"
            "    assert err < 1e-3 and verr < 5e-3, (name, err, verr)\n" % ROOT)
    env = dict(os.environ, PIPS_B200_TOKENMIX="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    print(r.stdout)
    assert r.returncode == 0, r.stderr[-3000:]


@pytest.mark.parametrize("name", ["s5_st4", "s16_st8"])
def test_graph_replay_and_split_problem_are_bit_identical(name):
    c = CASES[name]
    m = _model(c)
    ref = _run(m, c)
    again = _run(m, c)                                       # replay of the captured graph
    m.engine.use_graph = False
    eager = _run(m, c)
    m.engine.max_seqs = 4                                    # 4 * 8 // S tracks per call
    split = _run(m, c)
    for a, b, e, s in zip(ref, again, eager, split):
        assert torch.equal(a, b) and torch.equal(a, e) and torch.equal(a, s)


def test_score_maps_and_losses_match_reference():
    c = LOSS_CASE
    m = _model(c, loss_path="cuda")
    rgbs, xys, _ = case_inputs(c)
    trajs_g, vis_g, valids = (t.to(DEV) for t in loss_targets(c, xys))
    with torch.no_grad():
        preds, _, vis_e, losses = m(xys.to(DEV), rgbs.to(DEV), iters=c["iters"], trajs_g=trajs_g, vis_g=vis_g, valids=valids)
    assert np.abs(torch.stack(preds).cpu().numpy() - GOLD["loss/preds"]).max() < 1e-3
    got = [float(l) for l in losses]
    rel = [abs(a - b) / abs(b) for a, b in zip(got, GOLD["loss/losses"])]
    print("losses", got, "reference", GOLD["loss/losses"], "relative", rel)
    assert rel[0] <= 1e-3 and rel[1] <= 1e-3 and rel[2] <= 1e-4
    fcps, _, _ = m.score_maps(xys.to(DEV), rgbs.to(DEV), FCP_SEL, iters=c["iters"])
    err = np.abs(fcps.cpu().numpy() - GOLD["loss/fcps_sel"]).max()
    scale = np.abs(GOLD["loss/fcps_sel"]).max()
    print(f"fcps max |err| {err:.3e} (max |fcp| {scale:.3e})")
    assert err <= 1e-3 * max(1.0, scale)


def test_pack_round_trip_at_s16(tmp_path):
    from pips_b200 import pack
    c = CASES["s16_st8"]
    m = _model(c)
    ref = _run(m, c)
    path = str(tmp_path / "s16.pack")
    pack.save_pack(m, path)
    m2 = _model(c)
    assert pack.load_pack(m2, path)
    assert m2.engine.weights(m2).S == 16
    for a, b in zip(ref, _run(m2, c)):
        assert torch.equal(a, b)
    m8 = Pips(S=8, stride=8).to(DEV).eval()
    m8.load_state_dict(po.init_state_dict(seed=1, S=8), strict=True)
    p8 = str(tmp_path / "s8.pack")
    pack.save_pack(m8, p8)
    assert not pack.load_pack(m2, p8)                        # another model's pack: refused by the fingerprint
    with pytest.raises(L.PipsCudaError, match="S=8"):
        pack.load_pack(m2, p8, expect_fingerprint=pack.read_manifest(p8)["fingerprint"])


def test_refusals():
    c = CASES["s12_st8"]
    m = _model(c)
    rgbs, xys, _ = case_inputs(c)
    with pytest.raises(L.PipsCudaError, match="S=12"):
        m(xys.to(DEV), rgbs[:, :8].to(DEV))                  # the clip's frame count is not the model's S
    for S in (1, 17):
        ms = Pips(S=S, stride=8).to(DEV).eval()
        with pytest.raises(L.PipsCudaError, match="2 <= S <= 16"):
            ms(xys.to(DEV), po.smooth_video(1, S, 64, 64).to(DEV))
    mc = _model(c, mixer_path="cuda")
    trajs_g, vis_g, valids = (t.to(DEV) for t in loss_targets(c, xys))
    with pytest.raises(ValueError, match="S=12"):
        mc(xys.to(DEV), rgbs.to(DEV), trajs_g=trajs_g, vis_g=vis_g, valids=valids, is_train=True)
    m._shard = (0, 2, None)                                  # a particle-sharded model: refused before any collective
    with pytest.raises(ValueError, match="S=12"):
        m(xys.to(DEV), rgbs.to(DEV))
    m._shard = None
