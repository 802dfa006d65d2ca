"""Chained long-video tracking (chain_demo.py:40-83): threshold sweep logic on CPU, oracle vs the reference's
recorded chain, and the batched CUDA implementation vs the same recording (GPU)."""
import os

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from pips_b200.chain import _threshold_table, pick_skip
from tests.golden.make_golden import CHAIN_CASE, chain_inputs

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_outputs.npz"))


def _gold_skips():
    a = GOLD["chain/skips"]
    n = CHAIN_CASE["N"]
    lens, flat, out, k = a[:n], a[n:], [], 0
    for L in lens:
        out.append(list(flat[k:k + L]))
        k += L
    return out


def _loop_skip(vis):                      # literal chain_demo.py:63-76
    thr, si = 0.9, 7
    while True:
        if vis[si] > thr:
            return si
        si -= 1
        if si == 1:
            thr -= 0.02
            si = 7


def test_pick_skip_equals_reference_loop():
    torch.manual_seed(0)
    vis = torch.sigmoid(torch.randn(8, 500) * 2)
    vis[:, 0] = 0.05                      # needs many sweeps
    vis[:, 1] = torch.tensor([0.99, 0.99, 0.91, 0.2, 0.2, 0.2, 0.2, 0.95])
    vis[:, 2] = 0.9                       # exactly at the first threshold: not '>' in fp32
    got = pick_skip(vis, _threshold_table())
    ref = torch.tensor([_loop_skip(vis[:, n]) for n in range(vis.shape[1])])
    assert torch.equal(got.cpu(), ref)
    assert int(got.min()) >= 2 and int(got.max()) <= 7


def test_oracle_chain_matches_reference_recording():
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    rgbs, xy0 = chain_inputs(c)

    def window(xys, seq, feat_init):
        with torch.no_grad():
            o = po.forward(sd, xys, seq, iters=c["iters"], stride=c["stride"], feat_init=feat_init, return_feat=True)
        return o[0], o[2], o[3]

    trajs, skips = po.chain_track(window, rgbs, xy0, iters=c["iters"])
    assert skips == _gold_skips()
    assert np.abs(trajs.numpy() - GOLD["chain/trajs"]).max() < 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_batched_chain_matches_reference_recording(precision):
    from pips_b200 import Pips
    from pips_b200.chain import track_chain
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    model = Pips(S=8, stride=c["stride"], precision=precision).to("cuda:0").eval()
    model.load_state_dict(sd, strict=True)
    rgbs, xy0 = chain_inputs(c)
    trajs, rounds = track_chain(model, rgbs.to("cuda:0"), xy0.to("cuda:0"), iters=c["iters"], return_rounds=True)
    assert trajs.shape == (1, c["T"], c["N"], 2)
    err = np.abs(trajs.cpu().numpy() - GOLD["chain/trajs"]).max()
    print(f"chain {precision}: {rounds} batched rounds (reference: {sum(len(h) for h in _gold_skips())} model calls), max err {err:.2e} px")
    assert rounds == max(len(h) for h in _gold_skips())
    assert err < 2e-3


def test_batched_chain_host_logic_on_cpu():
    """pips_b200.chain.track_chain with the CUDA engine replaced by the oracle (one 8-frame window per track, selected
    through ``frame_base`` exactly as pips_corr_gather does: frame min(base + s, T-1)): the batching, the per-track
    frame offsets, the truncation at the end of the clip, the carried feature and the threshold sweep reproduce the
    reference's per-particle loop (same skips, same trajectories) -- no GPU involved."""
    from pips_b200.chain import track_chain
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    rgbs, xy0 = chain_inputs(c)
    T = rgbs.shape[1]
    log = []

    class Engine:
        def refine(self, module, fmaps, coords, feat_init, iters, stride, frame_base=None, reuse_pyramid=False):
            B, _, na, _ = coords.shape
            assert B == 1 and fmaps.shape[1] == T and frame_base.shape == (1, na) and frame_base.dtype == torch.int32
            preds = torch.zeros(iters, 1, 8, na, 2)
            vis = torch.zeros(1, 8, na)
            ffeat = torch.zeros(1, na, 128)
            for n in range(na):
                idx = (int(frame_base[0, n]) + torch.arange(8)).clamp(max=T - 1)
                fi = None if feat_init is None else feat_init[:, n:n + 1]
                with torch.no_grad():
                    o = po.forward(sd, coords[:, 0, n:n + 1] * stride, torch.zeros(1, 8, 3, c["H"], c["W"]), iters=iters,
                                   stride=int(stride), fmaps=fmaps[:, idx], feat_init=fi, return_feat=True)
                preds[:, :, :, n] = torch.stack(o[0])[:, :, :, 0]
                vis[:, :, n] = o[2][:, :, 0]
                ffeat[:, n] = o[3][:, 0]
            log.append(frame_base[0].tolist())
            return preds, vis, ffeat

    class Model:
        stride = c["stride"]
        engine = Engine()

        def encode(self, clip):
            Bc, Tc = clip.shape[:2]
            x = 2 * (clip / 255.0) - 1.0
            with torch.no_grad():
                f = po.fnet(sd, x.reshape(Bc * Tc, 3, c["H"], c["W"]), c["stride"])
            return f.reshape(Bc, Tc, 128, c["H"] // c["stride"], c["W"] // c["stride"])

    trajs, rounds = track_chain(Model(), rgbs, xy0, iters=c["iters"], return_rounds=True)
    gold = _gold_skips()
    assert rounds == max(len(h) for h in gold)
    # window starts seen by the engine == cumulative skips of the reference, per surviving track
    starts = [[0] + list(np.cumsum(h)[:-1]) for h in gold]
    for r, bases in enumerate(log):
        assert bases == [s[r] for s in starts if len(s) > r]
    err = np.abs(trajs.numpy() - GOLD["chain/trajs"]).max()
    print("batched chain host logic (oracle windows) vs reference recording: max err px", err)
    assert err < 1e-3


def test_fixed_advance_schedule_is_data_independent():
    """advance=7: ceil((T-1)/7) rounds, every track in every round, window starts 0, 7, 14, ..."""
    from pips_b200.chain import track_chain
    T, N = 30, 6
    seen = []

    class Engine:
        def refine(self, module, fmaps, coords, feat_init, iters, stride, frame_base=None, reuse_pyramid=False):
            na = coords.shape[2]
            seen.append(frame_base[0].tolist())
            preds = (coords * stride).unsqueeze(0).repeat(iters, 1, 1, 1, 1) + 1.0
            return preds, torch.full((1, 8, na), -10.0), torch.zeros(1, na, 128)      # "invisible": the sweep would lower thr

    class Model:
        stride = 4
        engine = Engine()

        def encode(self, clip):
            return torch.zeros(clip.shape[0], clip.shape[1], 128, 4, 4)

    trajs, rounds = track_chain(Model(), torch.zeros(1, T, 3, 16, 16), torch.rand(1, N, 2) * 16, iters=2, return_rounds=True,
                                advance=7)
    assert rounds == 5 and seen == [[7 * r] * N for r in range(5)]
    assert trajs.shape == (1, T, N, 2) and bool(torch.isfinite(trajs).all())
    with pytest.raises(ValueError):
        track_chain(Model(), torch.zeros(1, T, 3, 16, 16), torch.rand(1, N, 2), advance=1)
