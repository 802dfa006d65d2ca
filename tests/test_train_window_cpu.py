"""Host-only checks of training at window lengths 2 to 16: the _window entry points of the correlation and score-map
gradient kernels refuse other lengths before any launch, their S = 8 siblings keep refusing S != 8, and
torch_path.local_corr_cuda refuses a window outside 2..16 before it touches a tensor.  None of this needs a GPU."""
import ctypes as C

import pytest
import torch

from pips_b200 import _lib as L, torch_path


def _calls(lib):
    """the four gradient entry points of each family, called with S and otherwise valid-looking arguments"""
    p = C.c_void_p(256)
    lv = (C.c_void_p * 4)(256, 256, 256, 256)
    return {
        "pips_corr_grad_feats": lambda name, S: getattr(lib, name)(lv, 1, S, 4, 16, 16, p, p, 196, p, None),
        "pips_corr_grad_levels": lambda name, S: getattr(lib, name)(1, S, 4, 16, 16, p, p, p, 196, lv, None),
        "pips_scoremap_grad_feats": lambda name, S: getattr(lib, name)(p, p, p, 2, 1, S, 4, 16, 16, p, p, p, None),
        "pips_scoremap_grad_basis": lambda name, S: getattr(lib, name)(p, p, p, p, 2, 1, S, 4, 16, 16, p, p, p, None),
    }


def test_window_gradient_entry_points_reject_other_lengths_without_gpu():
    lib = L.load()
    for base, call in _calls(lib).items():
        who = base + "_window"
        for S in (1, 17):
            assert call(who, S) != 0, (who, S)
            assert lib.pips_last_error() == f"{who}: S must be in 2..16".encode(), (who, S, lib.pips_last_error())


def test_s8_gradient_entry_points_still_take_s8_only():
    lib = L.load()
    for base, call in _calls(lib).items():
        for S in (7, 9):
            assert call(base, S) != 0, (base, S)
            err = lib.pips_last_error()
            assert err.startswith(f"{base}: ".encode()) and b"S must be 8" in err, (base, S, err)
            if base.startswith("pips_scoremap"):
                assert f"({base}_window takes 2..16)".encode() in err, (base, S, err)


def test_window_entry_points_pass_the_window_check_at_every_length():
    """2 <= S <= 16 gets past the window check: a later check (ld, map size, alignment) is the one that refuses"""
    lib = L.load()
    p = C.c_void_p(256)
    lv = (C.c_void_p * 4)(256, 256, 256, 256)
    for S in range(2, 17):
        assert lib.pips_corr_grad_feats_window(lv, 1, S, 4, 16, 16, p, p, 195, p, None) != 0
        assert lib.pips_last_error() == b"pips_corr_grad_feats_window: ld_dcorr must be >= 196", S
        assert lib.pips_corr_grad_levels_window(1, S, 4, 7, 16, p, p, p, 196, lv, None) != 0
        assert lib.pips_last_error() == b"pips_corr_grad_levels_window: level-0 map must be at least 8x8", S
        assert lib.pips_scoremap_grad_feats_window(p, p, p, 2, 1, S, 4, 16, 16, p, p, C.c_void_p(264), None) != 0
        assert b"16-byte aligned" in lib.pips_last_error(), S
        assert lib.pips_scoremap_grad_basis_window(p, p, p, p, 2, 1, S, 4, 16, 16, p, p, C.c_void_p(264), None) != 0
        assert b"16-byte aligned" in lib.pips_last_error(), S


@pytest.mark.parametrize("S", [1, 17])
def test_local_corr_cuda_rejects_other_lengths(S):
    B, N, H, W = 1, 4, 16, 16
    levels = [torch.zeros(B * S, H >> l, W >> l, 128) for l in range(4)]
    with pytest.raises(ValueError, match=r"2 <= S <= 16"):
        torch_path.local_corr_cuda(torch.zeros(B * N, S, 128), levels, torch.zeros(B, S, N, 2))


def test_local_corr_cuda_takes_other_lengths_as_far_as_the_device():
    """a valid window length on CPU tensors reaches the CUDA-only refusal, as S = 8 does"""
    for S in (2, 12, 16):
        levels = [torch.zeros(S, 16 >> l, 16 >> l, 128) for l in range(4)]
        with pytest.raises(RuntimeError, match="CUDA kernels only"):
            torch_path.local_corr_cuda(torch.zeros(4, S, 128), levels, torch.zeros(1, S, 4, 2))
