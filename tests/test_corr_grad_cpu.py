"""Host-only checks of the local correlation's CUDA path: Pips(corr_path=...), the torch formulation that CPU tensors
keep under corr_path='cuda', and argument validation of pips_corr_grad_feats / pips_corr_grad_levels, none of which
needs a GPU."""
import pytest
import torch

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path
from tests.golden.make_golden import LOSS_CASE, case_inputs, loss_targets


def test_corr_path_argument_without_gpu(monkeypatch):
    with pytest.raises(ValueError, match="'torch'.*'cuda'"):
        Pips(S=8, stride=8, corr_path="fused")
    monkeypatch.setenv("PIPS_B200_CORR", "cuda")
    assert Pips(S=8, stride=8).corr_path == "cuda"
    assert Pips(S=8, stride=8, corr_path="torch").corr_path == "torch"
    monkeypatch.delenv("PIPS_B200_CORR")
    assert Pips(S=8, stride=8).corr_path == "torch"
    with pytest.raises(RuntimeError, match="CUDA kernels only"):
        torch_path.local_corr_cuda(torch.zeros(4, 8, 128), [torch.zeros(8, 8 >> l, 8 >> l, 128) for l in range(4)],
                                   torch.zeros(1, 8, 4, 2))


def _train_step(corr_path):
    c = LOSS_CASE
    m = Pips(S=8, stride=c["stride"], corr_path=corr_path).train()
    m.load_state_dict(po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"]), strict=True)
    rgbs, xys, _ = case_inputs(c)
    trajs_g, vis_g, valids = loss_targets(c, xys)
    preds, _, vis_e, losses = m(xys[:1, :3], rgbs[:1], iters=2, trajs_g=trajs_g[:1, :, :3], vis_g=vis_g[:1, :, :3],
                                valids=valids[:1, :, :3], is_train=True)
    sum(losses).backward()
    return torch.stack(preds), vis_e, losses, {n: p.grad for n, p in m.named_parameters() if p.grad is not None}


def test_cpu_tensors_keep_the_torch_formulation_under_cuda():
    pt, vt, lt, gt = _train_step("torch")
    pc, vc, lc, gc = _train_step("cuda")
    assert torch.equal(pt, pc) and torch.equal(vt, vc)
    assert all(torch.equal(a, b) for a, b in zip(lt, lc))
    assert gt.keys() == gc.keys() and len(gt) > 0
    assert all(torch.equal(gt[n], gc[n]) for n in gt)


def _ptrs(*addrs):
    """a C array of raw addresses: the checks run before any device access"""
    import ctypes as C
    return (C.c_void_p * len(addrs))(*addrs)


def test_corr_grad_entry_points_validate_arguments_without_gpu():
    lib = L.load()
    lv = _ptrs(16, 16, 16, 16)
    # pips_corr_grad_feats(lvl, B, S, N, H, W, coords, dcorr, ld_dcorr, dffeat_rows, stream)
    ok = [lv, 2, 8, 12, 8, 8, 16, 16, 196, 16, None]
    bad = {0: (None, b"null pointer"), 6: (None, b"null pointer"), 7: (None, b"null pointer"), 9: (None, b"null pointer"),
           2: (4, b"S must be 8"), 1: (0, b"empty problem"), 3: (0, b"empty problem"),
           4: (7, b"level-0 map must be at least 8x8"), 5: (7, b"level-0 map must be at least 8x8"),
           8: (195, b"ld_dcorr must be >= 196"), 6 + 100: (12, b"aligned"), 9 + 100: (24, b"aligned")}
    for i, (v, msg) in bad.items():
        args = list(ok)
        args[i % 100] = v
        assert lib.pips_corr_grad_feats(*args) != 0, (i, v)
        err = lib.pips_last_error()
        assert err.startswith(b"pips_corr_grad_feats: ") and msg in err, (i, v, err)
    args = list(ok)
    args[0] = _ptrs(16, 16, 24, 16)                       # a misaligned level
    assert lib.pips_corr_grad_feats(*args) != 0 and b"aligned" in lib.pips_last_error()
    args[0] = _ptrs(16, 16, None, 16)
    assert lib.pips_corr_grad_feats(*args) != 0 and b"null level pointer" in lib.pips_last_error()
    # pips_corr_grad_levels(B, S, N, H, W, coords, ffeat_rows, dcorr, ld_dcorr, dlvl, stream)
    ok = [2, 8, 12, 8, 8, 16, 16, 16, 196, lv, None]
    bad = {5: (None, b"null pointer"), 6: (None, b"null pointer"), 7: (None, b"null pointer"), 9: (None, b"null pointer"),
           1: (7, b"S must be 8"), 0: (0, b"empty problem"), 2: (-1, b"empty problem"),
           3: (4, b"level-0 map must be at least 8x8"), 4: (4, b"level-0 map must be at least 8x8"),
           8: (100, b"ld_dcorr must be >= 196"), 5 + 100: (20, b"aligned"), 6 + 100: (20, b"aligned"),
           7 + 100: (18, b"aligned")}
    for i, (v, msg) in bad.items():
        args = list(ok)
        args[i % 100] = v
        assert lib.pips_corr_grad_levels(*args) != 0, (i, v)
        err = lib.pips_last_error()
        assert err.startswith(b"pips_corr_grad_levels: ") and msg in err, (i, v, err)
    args = list(ok)
    args[9] = _ptrs(16, 40, 16, 16)
    assert lib.pips_corr_grad_levels(*args) != 0 and b"aligned" in lib.pips_last_error()
