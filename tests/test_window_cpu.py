"""Models of window lengths other than 8 without a GPU: the oracle against the unmodified reference's outputs
(tests/golden/reference_window.npz, written by tests/golden/make_golden_window.py) in both correlation formulations,
and the refusals of what stays S = 8 (chained tracking, streaming)."""
import os

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from pips_b200 import Pips
from tests.golden.make_golden_window import CASES, LOSS_CASE, case_inputs

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_window.npz"))


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("allpairs", [True, False])
def test_oracle_matches_reference_at_any_window(name, allpairs):
    c = CASES[name]
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"], S=c["S"])
    rgbs, xys, extra = case_inputs(c)
    with torch.no_grad():
        preds, _, vis_e, ffeat, _ = po.forward(sd, xys, rgbs, iters=c["iters"], stride=c["stride"], allpairs=allpairs,
                                               return_feat=True, **extra)
    got = torch.stack(preds).numpy()
    assert got.shape == GOLD[name + "/preds"].shape == (c["iters"], c["B"], c["S"], c["N"], 2)
    assert np.abs(got - GOLD[name + "/preds"]).max() < 1e-3
    assert np.abs(ffeat.numpy() - GOLD[name + "/ffeat"]).max() < 1e-5
    assert np.abs(vis_e.numpy() - GOLD[name + "/vis_e"]).max() < 2e-3


def test_loss_golden_is_finite_and_shaped():
    c = LOSS_CASE
    assert GOLD["loss/fcps_sel"].shape == (c["B"], c["S"], c["iters"], 3, c["H"] // c["stride"], c["W"] // c["stride"])
    assert np.isfinite(GOLD["loss/losses"]).all() and GOLD["loss/losses"].shape == (3,)


def test_modules_follow_the_window_length():
    for S in (2, 5, 16):
        m = Pips(S=S, stride=8)
        spec = dict(po.state_dict_spec(S))
        assert all(tuple(v.shape) == spec[k] for k, v in m.state_dict().items())
        m.load_state_dict(po.init_state_dict(1, S=S), strict=True)


def test_chaining_and_streams_refuse_other_windows():
    from pips_b200 import chain, stream
    m = Pips(S=12, stride=8).eval()
    rgbs = torch.zeros(1, 20, 3, 64, 64)
    q = torch.tensor([[[0.0, 10.0, 10.0]]])
    for call in (lambda: chain.track_chain(m, rgbs, q[:, :, 1:]), lambda: chain.track_queries(m, rgbs, q),
                 lambda: chain.track_queries_batch(m, [rgbs[0]], [q[0]]),
                 lambda: chain.track_queries_mixed(m, [rgbs[0]], [q[0]]),
                 lambda: stream.TrackStream(m, q), lambda: stream.MultiStream(m)):
        with pytest.raises(ValueError, match="S=12"):
            call()
