"""Models of window lengths 2..16 on the CUDA path: end to end against the unmodified reference's outputs
(tests/golden/reference_window.npz), and the token-mixing kernels against fp64."""
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


# ------------------------------------------------------------------------------------------------ kernels vs fp64

def _tokenmix_ref(x, p, S):
    """nets/pips.py:117 + the LayerNorm of :118 in fp64: x (R, S, 512) -> (x + tokenmix, LN2(x + tokenmix))."""
    ln = lambda v, w, b: torch.nn.functional.layer_norm(v, (512,), w, b, 1e-5)
    y = ln(x, p["ln1_w"], p["ln1_b"])
    h = torch.nn.functional.gelu(torch.einsum("rsc,js->rjc", y, p["w1"]) + p["b1"][None, :, None])
    z = torch.einsum("rjc,sj->rsc", h, p["w2"]) + p["b2"][None, :, None]
    xn = x + z
    return xn, ln(xn, p["ln2_w"], p["ln2_b"])


@pytest.mark.parametrize("S", [2, 5, 8, 9, 16])
@pytest.mark.parametrize("path", ["tc", "f32"])
def test_tokenmix_against_fp64(S, path):
    lib = L.load()
    g = torch.Generator().manual_seed(S)
    R = 37
    p = {"ln1_w": 1 + 0.1 * torch.randn(512, generator=g), "ln1_b": 0.1 * torch.randn(512, generator=g),
         "w1": torch.randn(4 * S, S, generator=g) / S ** 0.5, "b1": 0.1 * torch.randn(4 * S, generator=g),
         "w2": torch.randn(S, 4 * S, generator=g) / (2 * S ** 0.5), "b2": 0.1 * torch.randn(S, generator=g),
         "ln2_w": 1 + 0.1 * torch.randn(512, generator=g), "ln2_b": 0.1 * torch.randn(512, generator=g)}
    x = torch.randn(R, S, 512, generator=g) * 2 + 0.5
    xn_ref, y_ref = _tokenmix_ref(x.double(), {k: v.double() for k, v in p.items()}, S)
    pd = {k: v.to(DEV).contiguous() for k, v in p.items()}
    rows = R * S
    xd = torch.full((rows + 40, 512), float("nan"), device=DEV)          # rows after the last track: NaN, untouched
    xd[:rows] = x.reshape(rows, 512).to(DEV)
    args = [pd[k].data_ptr() for k in ("ln1_w", "ln1_b", "w1", "b1", "w2", "b2", "ln2_w", "ln2_b")]
    if path == "tc":
        hi = torch.full((rows + 40, 512), float("nan"), dtype=torch.bfloat16, device=DEV)
        lo = torch.full_like(hi, float("nan"))
        L.check(lib.pips_tokenmix_tc_s(xd.data_ptr(), R, S, *args, hi.data_ptr(), lo.data_ptr(), None))
        y = hi.float() + lo.float()
    else:
        y = torch.full((rows + 40, 512), float("nan"), device=DEV)
        L.check(lib.pips_tokenmix_s(xd.data_ptr(), R, S, *args, None, None, y.data_ptr(), None))
    torch.cuda.synchronize()
    assert torch.isnan(xd[rows:]).all() and torch.isnan(y[rows:]).all()
    ex = (xd[:rows].cpu().double() - xn_ref.reshape(rows, 512)).abs().max().item()
    ey = (y[:rows].cpu().double() - y_ref.reshape(rows, 512)).abs().max().item()
    print(f"S={S} {path}: residual max |err| {ex:.2e}, LN2 output max |err| {ey:.2e}")
    assert ex < 1e-4 and ey < (2e-4 if path == "tc" else 1e-4)


@pytest.mark.parametrize("S", [5, 16])
def test_ln_pool_against_fp64(S):
    lib = L.load()
    g = torch.Generator().manual_seed(100 + S)
    R = 29
    x = torch.randn(R * S, 512, generator=g) * 3 - 1
    w, b = 1 + 0.1 * torch.randn(512, generator=g), 0.1 * torch.randn(512, generator=g)
    ref = torch.nn.functional.layer_norm(x.double(), (512,), w.double(), b.double(), 1e-5).reshape(R, S, 512).mean(1)
    xd = torch.full((R * S + 16, 512), float("nan"), device=DEV)
    xd[:R * S] = x.to(DEV)
    out = torch.full((R + 3, 512), float("nan"), device=DEV)
    wd, bd = w.to(DEV), b.to(DEV)
    L.check(lib.pips_ln_pool_s(xd.data_ptr(), R, S, wd.data_ptr(), bd.data_ptr(), None, None, out.data_ptr(), None))
    torch.cuda.synchronize()
    assert torch.isnan(out[R:]).all()
    err = (out[:R].cpu().double() - ref).abs().max().item()
    print(f"S={S}: ln_pool max |err| {err:.2e}")
    assert err < 1e-5
