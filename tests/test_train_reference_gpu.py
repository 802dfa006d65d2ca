"""The training gradients on the device against the unmodified reference (tests/golden/reference_train.npz, see
tests/test_train_reference_cpu.py).

* tests/test_train_step_gpu.py's _reference_step in fp64 on the device (cuDNN and cuBLAS in fp64), the target every GPU
  training test compares with, within the CPU bound (REF64_BOUND) of the reference's own fp64 step.
* At each golden case, the CUDA training step against that restatement pinned to the CUDA forward's ReLU decisions and
  coordinates, with tests/test_train_step_gpu.py's check and bounds: at S = 8 all four CUDA nodes (encoder,
  correlation, DeltaBlock mixer, fused score-map loss), at other window lengths all but the mixer.  Its free-running
  distance to the golden is printed, not bounded: the encoder's ReLU decisions differ from the fp64 reference's."""
import numpy as np
import pytest
import torch

from tests.golden import make_golden_train as mg
from tests.test_train_reference_cpu import (CASES, REF64_BOUND, case_inputs, case_model, errors, gold_record, golden,
                                            restatement_record)
from tests.test_train_step_gpu import check_pinned_step

DEV = "cuda:0"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_reference_step_on_the_device_matches_the_reference(monkeypatch, case):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    c = mg.CASES[case]
    e = errors(restatement_record(c, torch.float64, dev=DEV), gold_record(case), c["S"])
    w = max(e, key=e.get)
    print(f"{case}: device restatement vs ref64 worst {w} {e[w]:.2e}, ratio {e[w] / REF64_BOUND:.3g}")
    assert e[w] <= REF64_BOUND, f"{w}: {e[w]:.3e} > {REF64_BOUND}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_cuda_step_at_the_golden_cases(monkeypatch, case):
    c = mg.CASES[case]
    model = case_model(c, DEV, loss_path="fused", corr_path="cuda", encoder_path="cuda",
                       mixer_path="cuda" if c["S"] == 8 else "torch")
    _, grads = check_pinned_step(monkeypatch, model, case_inputs(c, DEV), c["iters"], case)
    # free-running: the summed loss's gradient against the sum of the golden's per-loss digests (samples and
    # projections are linear), in units of the largest per-loss max|g|
    g64 = gold_record(case)
    worst, at = 0.0, None
    for j, n in enumerate(str(n) for n in golden()["names"]):
        if mg.structurally_zero(n):
            continue
        _, smp, prj = mg.digest([grads[n]], mg.digest_seed(c["seed"], n))
        scale = g64["max"][:, j].max()
        e = max(np.abs(smp[0] - g64["samples"][:, j].sum(0)).max(),
                np.abs(prj[0] - g64["proj"][:, j].sum(0)).max() / np.sqrt(grads[n].numel())) / scale
        if e > worst:
            worst, at = e, n
    print(f"{case}: free-running CUDA step vs ref64 (not bounded): worst {at} {worst:.2e}")
