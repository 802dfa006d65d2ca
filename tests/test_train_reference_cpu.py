"""The training gradients against the unmodified reference (tests/golden/reference_train.npz, made by
tests/golden/make_golden_train.py): each of the three losses' gradient in every parameter, per tensor digest (max|g|,
16 seeded elements, 4 seeded +-1 projections), from the reference's Pips.train() in fp64 ('ref64'), and the losses and
per-tensor digest error of the reference as shipped in fp32 ('ref32').

* tests/test_train_step_gpu.py's _reference_step -- the fp64 target of every GPU training test -- in fp64 on the CPU,
  within REF64_BOUND of ref64 per loss and per tensor.
* Pips.train() (forward_torch, fp32, CPU) within max(2 x ref32's own error on the same digest, FP32_FLOOR) of ref64,
  with ref32's losses within LOSS32_BOUND.

An error is digest_error: the largest |difference| over a tensor's digest entries in units of ref64's max|g| (the
projections in units of sqrt(numel) max|g|); a structurally zero tensor (exactly 0 in exact arithmetic) counts against
the 2-norm of the loss's whole gradient instead.  Which parameters a loss reaches at all must match as well.  None of
this needs a GPU."""
import functools

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po
from pips_b200 import Pips
from tests.golden import make_golden_train as mg
from tests.test_train_step_gpu import MODULES, _copies, _reference_step

GOLDEN = mg.FILE
# Measured on the CPU (x86-64, torch 2.11): the restatement's worst error is 1e-14 (s2_st8), Pips.train()'s worst ratio
# to its bound 0.55 (s16_st8, fnet.conv3.bias under the visibility loss)
REF64_BOUND = 1e-12
FP32_FLOOR = 1e-5
LOSS32_BOUND = 1e-6                     # 8 fp32 ulps


@functools.lru_cache(maxsize=None)
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def gold_record(case):
    """ref64's record of a case"""
    g = golden()
    return {k: g[f"{case}/ref64/{k}"] for k in ("losses", "has", "gnorm") + mg.DIGEST}


def ref32_errors(case):
    """ref32's own error against ref64, keyed as errors() keys its result"""
    g, names = golden(), [str(n) for n in golden()["names"]]
    l64, l32, err, has = (g[f"{case}/{k}"] for k in ("ref64/losses", "ref32/losses", "ref32/err", "ref64/has"))
    e = {}
    for i, l in enumerate(mg.LOSSES):
        e[(l, "loss")] = abs(l32[i] - l64[i]) / abs(l64[i])
        e.update({(l, n): err[i, j] for j, n in enumerate(names) if has[i, j]})
    return e


def case_model(c, dev="cpu", **paths):
    m = Pips(S=c["S"], stride=c["stride"], **paths).to(dev).train()
    m.load_state_dict(po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"], S=c["S"]), strict=True)
    return m


def case_inputs(c, dev="cpu"):
    return tuple(t.to(dev) for t in mg.case_inputs(c))


def record(losses, named_params, c):
    """make_golden_train's record of a step: losses and each loss's gradient digest, in the golden's parameter order"""
    names = [str(n) for n in golden()["names"]]
    params = dict(named_params)
    assert set(params) == set(names)
    grads = mg.loss_grads(losses, [params[n] for n in names])
    return mg.digest_step(losses, names, grads, c["seed"])


def restatement_record(c, dtype, dev="cpu"):
    """_reference_step (free-running) on copies of the case's model in dtype"""
    mods = _copies(case_model(c, dev), dtype)
    losses, _ = _reference_step(*mods, *case_inputs(c, dev), c["iters"])
    return record(losses, [(f"{p}.{n}", t) for p, m in zip(MODULES, mods) for n, t in m.named_parameters()], c)


def model_record(m, c, dev="cpu"):
    """one Pips training step (is_train=True) on the case's inputs"""
    rgbs, xys, tg, vg, va = case_inputs(c, dev)
    _, _, _, losses = m(xys, rgbs, iters=c["iters"], trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    return record(losses, m.named_parameters(), c)


def errors(rec, gold, S):
    """{(loss, parameter or 'loss'): digest_error of rec against gold}; the reached parameters must agree"""
    names = [str(n) for n in golden()["names"]]
    assert (rec["has"] == gold["has"]).all(), \
        [(mg.LOSSES[i], names[j]) for i, j in zip(*np.nonzero(rec["has"] != gold["has"]))][:5]
    sizes = {n: int(np.prod(shape)) for n, shape in po.state_dict_spec(S)}
    e = {}
    for i, l in enumerate(mg.LOSSES):
        e[(l, "loss")] = abs(rec["losses"][i] - gold["losses"][i]) / abs(gold["losses"][i])
        for j, n in enumerate(names):
            if gold["has"][i, j]:
                e[(l, n)] = mg.digest_error(mg.entry(rec, i, j), mg.entry(gold, i, j), sizes[n],
                                            mg.error_scale(gold, i, j, n))
    return e


CASES = list(mg.CASES)


def test_generator_helpers_regenerate_the_recorded_inputs():
    """case_inputs and digest are the generator's: every case's queries and the digest of its frames come back exactly"""
    g = golden()
    assert [str(n) for n in g["names"]] == [n for n, _ in case_model(mg.CASES["s8_st8"]).named_parameters()]
    for name, c in mg.CASES.items():
        rgbs, xys, _, _, _ = mg.case_inputs(c)
        assert np.array_equal(xys.numpy(), g[f"{name}/xys"]), name
        got = mg.digest([rgbs], mg.digest_seed(c["seed"], "rgbs"))
        for k, v in zip(mg.DIGEST, got):
            assert np.array_equal(v[0], g[f"{name}/rgbs/{k}"]), (name, k)


def _worst(e, bound):
    r = {k: v / bound[k] for k, v in e.items()}
    w = max(r, key=r.get)
    return w, r[w]


@pytest.mark.parametrize("case", CASES)
def test_reference_step_matches_the_reference_in_fp64(case):
    """The fp64 restatement every GPU training test compares with is the reference's own fp64 step: each loss and each
    loss's gradient digest in every parameter within REF64_BOUND of ref64"""
    c = mg.CASES[case]
    e = errors(restatement_record(c, torch.float64), gold_record(case), c["S"])
    w, r = _worst(e, dict.fromkeys(e, REF64_BOUND))
    print(f"{case}: restatement vs ref64 worst {w} {e[w]:.2e}, ratio {r:.3g}")
    assert r <= 1.0, f"{w}: {e[w]:.3e} > {REF64_BOUND}"


@pytest.mark.parametrize("case", CASES)
def test_training_path_matches_the_reference(case):
    """Pips.train() on the CPU (forward_torch in fp32) has ref32's losses to a few ulps, and each loss's gradient digest
    in every parameter within max(2 x ref32's own error, FP32_FLOOR) of ref64"""
    c = mg.CASES[case]
    rec = model_record(case_model(c), c)
    # the same fp32 losses as the reference as shipped: bit for bit at the thread count the golden was made with, a few
    # ulps apart at others, whose parallel reductions sum in another order
    l32 = golden()[f"{case}/ref32/losses"]
    assert (np.abs(rec["losses"] - l32) <= LOSS32_BOUND * np.abs(l32)).all(), (rec["losses"], l32)
    e, e32 = errors(rec, gold_record(case), c["S"]), ref32_errors(case)
    assert set(e) == set(e32)
    w, r = _worst(e, {k: max(2 * e32[k], FP32_FLOOR) for k in e})
    print(f"{case}: Pips.train() vs ref64 worst {w} ratio {r:.3f} (error {e[w]:.2e}, ref32's {e32[w]:.2e})")
    assert r <= 1.0, f"{w}: {r:.3f} of its bound"
