"""Host-only checks of the encoder's backward: argument validation of its entry points and of Pips(encoder_path=...),
none of which needs a GPU."""
import pytest
import torch

from pips_b200 import Pips, _lib as L, torch_path
from pips_b200.encoder import Encoder


def test_encoder_grad_entry_points_validate_arguments_without_gpu():
    lib = L.load()
    # pips_conv_wgrad(dy_hi, dy_lo, ldy, dy_step, x_hi, x_lo, N, H, W, Cp, Cout, R, S, sy, sx, py, px, scratch, dw, stream)
    ok = (16, 16, 64, 1, 16, 16, 2, 8, 8, 64, 64, 3, 3, 1, 1, 1, 1, 0, 16, None)
    assert lib.pips_conv_wgrad(0, *ok[1:]) != 0 and b"null pointer" in lib.pips_last_error()
    bad = {9: (96, b"Cp must be a positive multiple of 64"), 2: (60, b"ldy must be >= Cout"),
           3: (2, b"dy_step must be 1, or 2 for a stride-2"), 11: (9, b"unsupported filter geometry"),
           13: (3, b"unsupported filter geometry")}
    for i, (v, msg) in bad.items():
        args = list(ok)
        args[i] = v
        assert lib.pips_conv_wgrad(*args) != 0 and msg in lib.pips_last_error(), (i, v, lib.pips_last_error())
    args = list(ok)
    args[0] = 8                                                 # not 16-byte aligned
    assert lib.pips_conv_wgrad(*args) != 0 and b"aligned" in lib.pips_last_error()
    args = list(ok)
    args[6], args[7], args[8] = 512, 192, 256                   # many tiles: the partial sums need scratch
    assert lib.pips_conv_wgrad(*args) != 0 and b"scratch" in lib.pips_last_error()
    assert lib.pips_conv_wgrad_scratch_floats(512, 192, 256, 64, 576) == 205 * 64 * 576    # ceil(1024 / 5 blocks) chunks
    assert lib.pips_conv_wgrad_scratch_floats(1, 4, 4, 64, 576) == 0
    assert lib.pips_conv_wgrad_scratch_floats(0, 4, 4, 64, 576) == 0
    # pips_inorm_grad(y, stats, r, stats_r, relu_main, relu_out, g0, g1, g2, N, H, W, C, scratch, hi, lo, ld, dh, dw, g_out, st)
    ok = [16, 16, None, None, 1, 0, 16, None, None, 2, 8, 8, 64, 16, 16, 16, 64, 0, 0, None, None]
    assert lib.pips_inorm_grad(*ok[:6], None, *ok[7:]) != 0 and b"null pointer" in lib.pips_last_error()
    for i, (v, msg) in {12: (62, b"bad shape (C % 4 == 0"), 16: (60, b"pair_ld must be >= C"), 17: (20, b"dilated grid must be"),
                        3: (16, b"stats_r without r")}.items():
        args = list(ok)
        args[i] = v
        if i == 17:
            args[18] = 16
        assert lib.pips_inorm_grad(*args) != 0 and msg in lib.pips_last_error(), (i, v, lib.pips_last_error())
    args = list(ok)
    args[2] = 16                                                # a residual without the output ReLU
    assert lib.pips_inorm_grad(*args) != 0 and b"relu_out" in lib.pips_last_error()
    assert lib.pips_inorm_grad_scratch_floats(2, 64 * 64, 64) == 2 * 16 * 2 * 64 * 2 + 2 * 2 * 64
    # pips_resize_grad(g, ldg, c_off, N, Ho, Wo, out, Hs, Ws, C, stream)
    assert lib.pips_resize_grad(None, 416, 0, 1, 8, 8, 16, 4, 4, 64, None) != 0 and b"null pointer" in lib.pips_last_error()
    assert lib.pips_resize_grad(16, 416, 380, 1, 8, 8, 16, 4, 4, 64, None) != 0 and b"bad shape" in lib.pips_last_error()
    assert lib.pips_resize_grad(16, 416, 2, 1, 8, 8, 16, 4, 4, 64, None) != 0 and b"bad shape" in lib.pips_last_error()


def test_encoder_path_argument_without_gpu(monkeypatch):
    with pytest.raises(ValueError, match="'torch'.*'cuda'"):
        Pips(S=8, stride=8, encoder_path="fused")
    monkeypatch.setenv("PIPS_B200_ENCODER", "cuda")
    assert Pips(S=8, stride=8).encoder_path == "cuda"
    assert Pips(S=8, stride=8, encoder_path="torch").encoder_path == "torch"
    monkeypatch.delenv("PIPS_B200_ENCODER")
    assert Pips(S=8, stride=8).encoder_path == "torch"
    with pytest.raises(RuntimeError, match="CUDA kernels only"):
        torch_path.encoder_cuda(Encoder(), torch.zeros(1, 1, 3, 64, 64))
    assert len(torch_path.ENCODER_PARAMS) == 44
    assert [n for n, _ in Encoder().named_parameters()] == list(torch_path.ENCODER_PARAMS)
