"""End-to-end parity of pips_b200.Pips.forward (CUDA) against the reference's recorded outputs
(tests/golden) and the CPU oracle, through the public module API."""
import os

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from pips_b200 import Pips
from tests.golden.make_golden import CASES, case_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_outputs.npz"))

# tolerance in input pixels on trajs (BASELINE.json north_star: 1e-3 max-abs)
TOL = {"fp32": 1e-3, "bf16x3": 1e-3, "bf16": 0.25}


def _run(name, precision, feat="fp32"):
    c = CASES[name]
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    model = Pips(S=8, stride=c["stride"], precision=precision, feat_dtype=feat).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    rgbs, xys, extra = case_inputs(c)
    extra = {k: v.to(DEV) for k, v in extra.items()}
    with torch.no_grad():
        out = model(xys.to(DEV), rgbs.to(DEV), iters=c["iters"], return_feat=True, **extra)
    torch.cuda.synchronize()
    return c, out


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_forward_matches_reference_golden(name, precision):
    c, (preds, preds2, vis_e, ffeat, losses) = _run(name, precision)
    assert losses is None and len(preds) == c["iters"] and len(preds2) == c["iters"] + 4
    got = torch.stack(preds).cpu().numpy()
    ref = GOLD[name + "/preds"]
    err = np.abs(got - ref).reshape(c["iters"], -1).max(1)
    print(f"{name} {precision}: per-iter max|d trajs| px = {err}")
    tol = TOL[precision] * (5 if c["head_scale"] >= 1.0 else 1)
    assert err.max() < tol, err
    # initial features come straight from fnet (3xTF32 split convolutions by default: fmaps within ~2e-4)
    assert np.abs(ffeat.cpu().numpy() - GOLD[name + "/ffeat"]).max() < 5e-4
    vtol = 5e-3 if precision != "bf16" else 0.5
    assert np.abs(vis_e.cpu().numpy() - GOLD[name + "/vis_e"]).max() < vtol
    assert torch.equal(preds2[0], preds2[1]) and torch.equal(preds2[-1], preds[-1])


def test_bf16_features_are_close():
    c, (preds, _, _, _, _) = _run("tiny_s8", "bf16x3", feat="bf16")
    err = np.abs(torch.stack(preds).cpu().numpy() - GOLD["tiny_s8/preds"]).max()
    print("bf16 features, bf16x3 mixer: max err px", err)
    assert err < 5e-2


def test_teacher_forced_single_iteration_vs_oracle():
    """One iteration from identical state, larger N than the golden cases, oracle live on CPU."""
    c = dict(B=2, H=128, W=160, N=300, stride=8, iters=1, head_scale=0.05, seed=9, oob=True, warm=True)
    sd = po.init_state_dict(seed=9, head_scale=0.05)
    rgbs, xys, extra = case_inputs(c)
    with torch.no_grad():
        ref = po.forward(sd, xys, rgbs, iters=1, stride=8, return_feat=True, **extra)
    model = Pips(S=8, stride=8).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    with torch.no_grad():
        got = model(xys.to(DEV), rgbs.to(DEV), iters=1, return_feat=True, **{k: v.to(DEV) for k, v in extra.items()})
    err = (got[0][0].cpu() - ref[0][0]).abs().max().item()
    print("teacher-forced 1 iter, N=300: max err px", err)
    assert err < 1e-3
    assert (got[2].cpu() - ref[2]).abs().max() < 5e-3


def test_strict_fp32_fnet_mode():
    c = CASES["tiny_s8"]
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    model = Pips(S=8, stride=c["stride"], precision="fp32", fnet_mode="plain").to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    rgbs, xys, _ = case_inputs(c)
    with torch.no_grad():
        preds, _, _, ffeat, _ = model(xys.to(DEV), rgbs.to(DEV), iters=c["iters"], return_feat=True)
    assert np.abs(ffeat.cpu().numpy() - GOLD["tiny_s8/ffeat"]).max() < 1e-4
    assert np.abs(torch.stack(preds).cpu().numpy() - GOLD["tiny_s8/preds"]).max() < 1e-4


@pytest.mark.parametrize("H,W,stride", [(128, 160, 8), (184, 360, 8), (96, 128, 4),
                                        (100, 130, 8), (90, 122, 4)])      # last two: sizes no stage divides evenly
def test_fnet_modes_agree(H, W, stride):
    """'fast' (channels-last, fused element-wise kernels, 3xTF32 convs) and 'x3' against strict-fp32 cuDNN."""
    sd = po.init_state_dict(seed=3)
    rgbs = po.smooth_video(1, 8, H, W, seed=77).to(DEV)
    outs = {}
    for mode in ("plain", "x3", "fast", "tc"):
        model = Pips(S=8, stride=stride, fnet_mode=mode).to(DEV).eval()
        model.load_state_dict(sd, strict=True)
        with torch.no_grad():
            outs[mode] = model.encode(rgbs).contiguous()
        assert outs[mode].shape == (1, 8, 128, H // stride, W // stride)
    scale = outs["plain"].abs().max().item()
    for mode in ("x3", "fast", "tc"):
        err = (outs[mode] - outs["plain"]).abs().max().item()
        print(f"fnet {mode} vs plain: max|err| {err:.3e} (|fmaps| max {scale:.2f})")
        assert err < 1e-3
    with torch.no_grad():
        ref = po.fnet(sd, (2 * (rgbs.cpu() / 255.0) - 1.0).reshape(8, 3, H, W), stride)
    err = (outs["fast"].cpu().reshape(8, 128, H // stride, W // stride) - ref).abs().max().item()
    print(f"fnet fast vs CPU oracle: max|err| {err:.3e}")
    assert err < 1e-3


def test_graph_replay_equals_eager():
    c = CASES["rect_s4_oob"]
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    rgbs, xys, _ = case_inputs(c)
    outs = []
    for use_graph in (True, False):
        model = Pips(S=8, stride=c["stride"]).to(DEV).eval()
        model.engine.use_graph = use_graph
        model.load_state_dict(sd, strict=True)
        with torch.no_grad():
            for _ in range(2):                      # second call replays the captured graph
                out = model(xys.to(DEV), rgbs.to(DEV), iters=3)
        outs.append((torch.stack(out[0]).cpu(), out[2].cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_particle_chunking_is_transparent():
    c = CASES["rect_s4_oob"]
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    rgbs, xys, _ = case_inputs(c)
    outs = []
    for max_seqs in (32768, 2 * 7):               # second: chunks of 7 particles
        model = Pips(S=8, stride=c["stride"], max_seqs=max_seqs).to(DEV).eval()
        model.load_state_dict(sd, strict=True)
        with torch.no_grad():
            outs.append(torch.stack(model(xys.to(DEV), rgbs.to(DEV), iters=3)[0]).cpu())
    assert torch.equal(outs[0], outs[1])


def test_cpu_inputs_fail_loudly():
    model = Pips(S=8, stride=8).eval()
    with pytest.raises(RuntimeError, match="CUDA-only"):
        model(torch.zeros(1, 4, 2), torch.zeros(1, 8, 3, 64, 64), iters=1)


def test_demo_configuration_matches_oracle():
    """BASELINE configs[0]: 8 x 360x640, N = 256 (16x16 grid as demo.py:32-36), iters = 6, B = 1, stride 4 --
    the reference's own CPU-runnable case; the oracle runs live on the host (local-correlation formulation)."""
    H, W, N_ = 360, 640, 16
    sd = po.init_state_dict(seed=21, head_scale=0.05)
    rgbs = po.smooth_video(1, 8, H, W, seed=22)
    gy, gx = torch.meshgrid(torch.arange(N_).float(), torch.arange(N_).float(), indexing="ij")
    xy = torch.stack([8 + gx.reshape(1, -1) / float(N_ - 1) * (W - 16), 8 + gy.reshape(1, -1) / float(N_ - 1) * (H - 16)], dim=-1)
    with torch.no_grad():
        ref = po.forward(sd, xy, rgbs, iters=6, stride=4)
    model = Pips(S=8, stride=4).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    with torch.no_grad():
        preds, preds2, vis_e, _ = model(xy.to(DEV), rgbs.to(DEV), iters=6)
    err = (preds[-1].cpu() - ref[0][-1]).abs().max().item()
    print(f"demo configuration (360x640, N=256, stride 4, iters 6): max err {err:.2e} px")
    assert err < 1e-3
    assert (vis_e.cpu() - ref[2]).abs().max() < 5e-3
    assert len(preds2) == 10


def test_peer_slab_exchange_world1():
    """The peer-slab result path (update kernel storing into the slab, scatter, flag barrier, slab reuse) with a
    single rank: same kernels as the multi-GPU run (tools/check_sharded.py covers 2+ GPUs), bit-exact results."""
    import torch.distributed as dist
    from pips_b200 import sharding
    c = CASES["rect_s4_oob"]
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    model = Pips(S=8, stride=c["stride"]).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    rgbs, xys, _ = case_inputs(c)
    rgbs, xys = rgbs.to(DEV), xys.to(DEV)
    created = not dist.is_initialized()
    if created:
        dist.init_process_group("gloo", init_method="tcp://127.0.0.1:29533", rank=0, world_size=1)
    try:
        with torch.no_grad():
            fmaps = model.encode(rgbs)
            coords = (xys / c["stride"]).reshape(xys.shape[0], 1, -1, 2).repeat(1, 8, 1, 1)
            ref = model.engine.refine(model, fmaps.float(), coords, None, c["iters"], float(c["stride"]))
            model._shard = (0, 1, None)
            for _ in range(3):                               # the slab is reused: barriers fence it
                got = sharding.refine_sharded_p2p(model, fmaps.float(), coords, None, c["iters"], float(c["stride"]))
                for a, b in zip(ref, got):
                    assert torch.equal(a, b)
            # the frame-sharded encoder's exchange through its own slab (scatter between two barriers), twice (reuse)
            for _ in range(2):
                assert torch.equal(sharding.encode_sharded(model, rgbs).contiguous(), fmaps.contiguous())
            big = coords.repeat(1, 1, 40, 1)                 # more particles: the slab grows (collective re-allocation)
            ref2 = model.engine.refine(model, fmaps.float(), big, None, 2, float(c["stride"]))
            got2 = sharding.refine_sharded_p2p(model, fmaps.float(), big, None, 2, float(c["stride"]))
            assert all(torch.equal(a, b) for a, b in zip(ref2, got2))
        model.close_peer_slabs()
    finally:
        model._shard = None
        if created:
            dist.destroy_process_group()
