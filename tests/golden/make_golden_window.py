"""Golden vectors for models of window lengths other than 8, from the UNMODIFIED reference.

    python tests/golden/make_golden_window.py          # needs the reference checkout (see make_golden.py)

The reference's Pips takes the window length S as its constructor argument (train.py, test_on_flt.py); its token
mixing is Conv1d(S, 4S) -> GELU -> Conv1d(4S, S), its head Linear(512, 130 S) and its time channel linspace(0, S, S).
Weights come from ``oracle.pips_oracle.init_state_dict(S=...)``, loaded with ``strict=True``.  Inputs are regenerated
from seeds by the tests (``case_inputs``), so only outputs are stored in reference_window.npz.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")

from oracle import pips_oracle as po  # noqa: E402

CASES = {
    # name: dict(S, B, H, W, N, stride, iters, head_scale, seed, oob, warm)
    "s2_st8": dict(S=2, B=2, H=128, W=160, N=12, stride=8, iters=3, head_scale=0.05, seed=21, oob=True, warm=False),
    "s5_st4": dict(S=5, B=1, H=64, W=96, N=10, stride=4, iters=3, head_scale=0.05, seed=22, oob=True, warm=False),
    "s5_warm": dict(S=5, B=1, H=128, W=160, N=9, stride=8, iters=2, head_scale=0.05, seed=23, oob=False, warm=True),
    "s12_st8": dict(S=12, B=1, H=128, W=160, N=11, stride=8, iters=3, head_scale=0.05, seed=24, oob=True, warm=False),
    "s16_st4": dict(S=16, B=1, H=64, W=96, N=9, stride=4, iters=3, head_scale=0.05, seed=25, oob=True, warm=False),
    "s16_st8": dict(S=16, B=2, H=128, W=160, N=7, stride=8, iters=3, head_scale=0.05, seed=26, oob=False, warm=True),
}

LOSS_CASE = dict(S=12, B=2, H=128, W=160, N=9, stride=8, iters=3, head_scale=0.05, seed=27, oob=False, warm=False)
FCP_SEL = [0, 4, 7]          # particles whose dense score maps (nets/pips.py:504-511) are recorded for LOSS_CASE


def case_inputs(c):
    """Shared with tests/: deterministic inputs for a golden case."""
    S = c["S"]
    rgbs = po.smooth_video(c["B"], S, c["H"], c["W"], seed=100 + c["seed"])
    xys = po.random_queries(c["B"], c["N"], c["H"], c["W"], seed=200 + c["seed"])
    if c["oob"]:
        xys[:, 0] = torch.tensor([0.0, 0.0])
        xys[:, 1] = torch.tensor([c["W"] - 1.0, c["H"] - 1.0])
        xys[:, 2] = torch.tensor([-5.5, 17.25])
        xys[:, 3] = torch.tensor([c["W"] + 3.0, c["H"] + 6.5])
    extra = {}
    if c["warm"]:
        g = torch.Generator().manual_seed(300 + c["seed"])
        drift = torch.cumsum(torch.randn(c["B"], S, c["N"], 2, generator=g) * 1.5, 1)
        extra["coords_init"] = xys[:, None] + drift - drift[:, :1]
        extra["feat_init"] = torch.randn(c["B"], c["N"], 128, generator=g) * 0.5
    return rgbs, xys, extra


def loss_targets(c, xys):
    g = torch.Generator().manual_seed(400 + c["seed"])
    S = c["S"]
    trajs_g = xys[:, None] + torch.cumsum(torch.randn(c["B"], S, c["N"], 2, generator=g), 1)
    vis_g = (torch.rand(c["B"], S, c["N"], generator=g) > 0.3).float()
    valids = (torch.rand(c["B"], S, c["N"], generator=g) > 0.1).float()
    return trajs_g, vis_g, valids


def main():
    torch.Tensor.cuda = lambda self, *a, **k: self
    import nets.pips as ref_mod
    from nets.pips import Pips  # the reference, unmodified

    torch.set_num_threads(8)
    out = {}
    for name, c in CASES.items():
        sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"], S=c["S"])
        model = Pips(S=c["S"], stride=c["stride"]).eval()
        model.load_state_dict(sd, strict=True)
        rgbs, xys, extra = case_inputs(c)
        with torch.no_grad():
            preds, preds2, vis_e, ffeat, losses = model(xys, rgbs, iters=c["iters"], return_feat=True, **extra)
        assert losses is None and len(preds2) == c["iters"] + 4
        out[name + "/preds"] = torch.stack(preds).numpy()
        out[name + "/vis_e"] = vis_e.numpy()
        out[name + "/ffeat"] = ffeat.numpy()
        print(name, "mean |d| from init", float((preds[-1] - xys[:, None]).abs().mean()))
    c = LOSS_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"], S=c["S"])
    model = Pips(S=c["S"], stride=c["stride"]).eval()
    model.load_state_dict(sd, strict=True)
    rgbs, xys, _ = case_inputs(c)
    trajs_g, vis_g, valids = loss_targets(c, xys)
    seen, real_loss = {}, ref_mod.score_map_loss

    def spy(fcps, *a, **k):                      # fcps is only visible as this loss's argument (nets/pips.py:603)
        seen["fcps"] = fcps.detach().clone()
        return real_loss(fcps, *a, **k)

    ref_mod.score_map_loss = spy
    try:
        with torch.no_grad():
            preds, _, vis_e, losses = model(xys, rgbs, iters=c["iters"], trajs_g=trajs_g, vis_g=vis_g, valids=valids)
    finally:
        ref_mod.score_map_loss = real_loss
    out["loss/fcps_sel"] = seen["fcps"][:, :, :, FCP_SEL].numpy()      # (B,S,I,3,H8,W8)
    out["loss/preds"] = torch.stack(preds).numpy()
    out["loss/vis_e"] = vis_e.numpy()
    out["loss/losses"] = np.array([float(l) for l in losses], dtype=np.float64)
    print("loss", out["loss/losses"])
    np.savez_compressed(os.path.join(HERE, "reference_window.npz"), **out)
    print("wrote", os.path.join(HERE, "reference_window.npz"))


if __name__ == "__main__":
    main()
