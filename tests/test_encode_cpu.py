"""pips_encode without a GPU: its argument checks and messages, the workspace size as a formula of the shapes, the launch
count, and the declarations in include/pips_b200.h and _lib._SIGNATURES."""
import json
import os
import re
import subprocess
import sys

import pytest

from pips_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _up(b):
    return (b + 255) // 256 * 256


def _half(v):
    return (v - 1) // 2 + 1


def workspace_bytes(N, H, W, stride):
    """The regions of one pips_encode call, each rounded up to 256 bytes: stem operand pair, 2 block outputs and their 2
    pairs, the pair between two convolutions, the convolution output, the downsample output, the partial statistics,
    2 statistics buffers, the concatenation pair."""
    if stride not in (4, 8) or not 1 <= N <= 65535 or H < stride or W < stride or H * W > 2 ** 26:
        return 0
    lib = L.load()
    sh, sw = _half(H), _half(W)
    H8, W8 = H // stride, W // stride
    levels, h, w = [], sh, sw
    for i, c in enumerate((64, 96, 128, 128)):
        if i:
            h, w = _half(h), _half(w)
        levels.append((h, w, c))

    def rows(h, w, R, st, pad, layer1):
        ho, wo = (h + 2 * pad - R) // st + 1, (w + 2 * pad - R) // st + 1
        c = max(lib.pips_conv_tc_chunks(h, w, R, R, st, st, pad, pad), max(1, min(64, ho * wo // 256)))
        return max(c, lib.pips_conv_rows_chunks(h, w)) if layer1 else c

    x = pair = N * sh * sw * 64
    d = 0
    part = lib.pips_conv_tc_chunks(sh + 3, sw, 4, 1, 1, 1, 0, 0) * 64
    prev = (sh, sw)
    for l, (h, w, c) in enumerate(levels):
        n = N * h * w
        x, pair = max(x, n * c), max(pair, n * ((c + 63) // 64 * 64))
        if l:
            d = max(d, n * c)
        r = max(rows(*prev, 3, 2 if l else 1, 1, l == 0), rows(*prev, 1, 2, 0, False) if l else 0, rows(h, w, 3, 1, 1, l == 0))
        part = max(part, r * c)
        prev = (h, w)
    part = max(part, rows(H8, W8, 3, 1, 1, False) * 256)
    head = N * H8 * W8 * 256
    unf = N * (sh + 3) * sw * 64 * 2
    sizes = ([unf] * 2 + [x * 4] * 2 + [pair * 2] * 4 + [max(pair, head) * 2] * 2 + [max(x, head) * 4, d * 4, N * part * 12]
             + [N * 2 * 256 * 4] * 2 + [N * H8 * W8 * 448 * 2] * 2)
    return sum(_up(s) for s in sizes)


@pytest.mark.parametrize("N,H,W,stride", [
    (1, 8, 8, 8), (1, 4, 4, 4), (1, 100, 136, 8), (1, 100, 136, 4), (3, 101, 137, 8), (2, 127, 161, 4), (1, 128, 160, 8),
    (32, 384, 512, 8), (1, 720, 1280, 4), (32, 720, 1280, 8), (5, 9, 1000, 8), (1, 1000, 9, 4), (65535, 8, 8, 8)])
def test_workspace_bytes_formula(N, H, W, stride):
    lib = L.load()
    got = lib.pips_encode_workspace_bytes(N, H, W, stride)
    assert got == workspace_bytes(N, H, W, stride) and got > 0 and got % 256 == 0


@pytest.mark.parametrize("N,H,W,stride", [(1, 64, 64, 2), (1, 64, 64, 16), (0, 64, 64, 8), (65536, 8, 8, 8), (-1, 64, 64, 8),
                                          (1, 7, 64, 8), (1, 64, 3, 4), (1, 0, 0, 8), (1, 8193, 8193, 8)])
def test_workspace_bytes_refuses_bad_shapes(N, H, W, stride):
    lib = L.load()
    assert lib.pips_encode_workspace_bytes(N, H, W, stride) == 0
    assert lib.pips_encode_launches(N, H, W, stride) == 0


def _launches(W, rows=True, fused=True):
    """stem 3 + its apply; per ResBlock 2 convolutions with statistics (+ the downsample's) and 2 applies; 4 resizes;
    the head's convolution with statistics, its apply and conv3"""
    def conv(layer1):
        if layer1 and rows and _half(W) / (((_half(W) + 255) // 256) * 256) >= 0.75:
            return 2
        return 2 if fused else 3
    n = 4
    for b in range(8):
        n += conv(b < 2) * 2 + 2 + (conv(False) if b in (2, 4, 6) else 0)
    return n + 4 + conv(False) + 2


@pytest.mark.parametrize("rows,stats", [(None, None), ("0", None), (None, "0"), ("0", "0")])
def test_launch_count(monkeypatch, rows, stats):
    for name, v in (("PIPS_B200_CONV_ROWS", rows), ("PIPS_B200_CONV_STATS", stats)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, v)
    lib = L.load()
    for N, H, W, stride in [(1, 384, 512, 8), (8, 360, 640, 8), (2, 100, 136, 4), (1, 720, 1280, 4)]:
        assert lib.pips_encode_launches(N, H, W, stride) == _launches(W, rows is None, stats is None), (N, H, W, stride)
    if rows is None and stats is None:
        assert lib.pips_encode_launches(1, 384, 512, 8) == 66


_REFUSALS = r"""
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from pips_b200 import _lib as L
lib = L.load()
FAKE = 1 << 40                                        # 256-byte aligned, never dereferenced: every call below is refused

def weights(skip=None):
    w = L.EncoderWeights()
    for i, (name, _) in enumerate(L.EncoderWeights._fields_):
        f = getattr(w, name)
        f.w_hi = f.w_lo = f.b = FAKE + 4096 * i
        if name == skip:
            f.w_lo = None
    return w

N, H, W, s = 2, 100, 136, 8
need = lib.pips_encode_workspace_bytes(N, H, W, s)
keep_bad = (C.c_void_p * 9)(*([FAKE] * 8 + [0]))
keep_odd = (C.c_void_p * 9)(*([FAKE] * 4 + [FAKE + 8] + [FAKE] * 4))
cases = {
    "weights": (None, FAKE, 0, N, H, W, s, FAKE, need, FAKE, None),
    "filter": (C.byref(weights("layer3_0_downsample_0")), FAKE, 0, N, H, W, s, FAKE, need, FAKE, None),
    "rgb": (C.byref(weights()), None, 0, N, H, W, s, FAKE, need, FAKE, None),
    "fmaps": (C.byref(weights()), FAKE, 0, N, H, W, s, FAKE, need, None, None),
    "dtype": (C.byref(weights()), FAKE, 2, N, H, W, s, FAKE, need, FAKE, None),
    "stride": (C.byref(weights()), FAKE, 0, N, H, W, 2, FAKE, need, FAKE, None),
    "frames": (C.byref(weights()), FAKE, 0, 0, H, W, s, FAKE, need, FAKE, None),
    "small": (C.byref(weights()), FAKE, 0, N, 7, W, s, FAKE, need, FAKE, None),
    "workspace": (C.byref(weights()), FAKE, 0, N, H, W, s, None, need, FAKE, None),
    "short": (C.byref(weights()), FAKE, 0, N, H, W, s, FAKE, need - 1, FAKE, None),
    "ws_align": (C.byref(weights()), FAKE, 0, N, H, W, s, FAKE + 128, need, FAKE, None),
    "rgb_align": (C.byref(weights()), FAKE + 2, 0, N, H, W, s, FAKE, need, FAKE, None),
    "fmaps_align": (C.byref(weights()), FAKE, 0, N, H, W, s, FAKE, need, FAKE + 4, None),
    "keep_null": (C.byref(weights()), FAKE, 0, N, H, W, s, FAKE, need, FAKE, keep_bad),
    "keep_align": (C.byref(weights()), FAKE, 1, N, H, W, s, FAKE, need, FAKE, keep_odd),
}
out = {}
for k, a in cases.items():
    rc = lib.pips_encode(*a, None)
    out[k] = [rc, lib.pips_last_error().decode()]
print(json.dumps(out))
"""

_MESSAGES = {
    "weights": "null pointer (weights, rgb or fmaps_nhwc)",
    "filter": "null filter pointer in convolution 12 of pips_encoder_weights",
    "rgb": "null pointer (weights, rgb or fmaps_nhwc)",
    "fmaps": "null pointer (weights, rgb or fmaps_nhwc)",
    "dtype": "dtype must be 0 (fp32) or 1 (bf16)",
    "stride": "stride must be 4 or 8 (got 2)",
    "frames": "need 1 <= N <= 65535 frames (got 0)",
    "small": "a 7x136 frame is too small",
    "workspace": "null workspace",
    "short": "workspace too small: {} bytes given, {} needed",
    "ws_align": "workspace must be 256-byte aligned",
    "rgb_align": "rgb is not aligned to its element size",
    "fmaps_align": "fmaps_nhwc must be 16-byte aligned",
    "keep_null": "keep[8] is null or not 16-byte aligned",
    "keep_align": "keep[4] is null or not 16-byte aligned",
}


def test_encode_refuses_bad_arguments_before_any_launch():
    """Run with no visible CUDA device: a call that got past its checks would fail in its first launch with a CUDA
    error, so each message below also shows that the call stopped before launching anything."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _REFUSALS, ROOT], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0, r.stderr
    got = json.loads(r.stdout.strip().splitlines()[-1])
    need = L.load().pips_encode_workspace_bytes(2, 100, 136, 8)
    assert set(got) == set(_MESSAGES)
    for k, msg in _MESSAGES.items():
        rc, err = got[k]
        expect = "pips_encode: " + (msg.format(need - 1, need) if k == "short" else msg)
        assert rc != 0 and err.startswith(expect), (k, err)


def test_encode_is_declared():
    hdr = open(os.path.join(ROOT, "include", "pips_b200.h")).read()
    for name in ("pips_encode", "pips_encode_workspace_bytes", "pips_encode_launches"):
        assert re.search(r"^(?:int|size_t)\s+%s\s*\(" % name, hdr, flags=re.M), name
        assert name in L._SIGNATURES
    assert L._SIGNATURES["pips_encode_workspace_bytes"][0] is L.C.c_size_t
    assert re.search(r"#define PIPS_B200_ABI_VERSION 4\b", hdr) and L.ABI_VERSION == 4
    # pips_encoder_weights: the pack's fnet.* names with '.' -> '_', in module order, three pointers each
    body = re.search(r"typedef struct pips_encoder_weights \{(.*?)\} pips_encoder_weights;", hdr, flags=re.S).group(1)
    fields = re.findall(r"\b(conv\d|layer\d_\d_\w+?)\b(?=[,;])", body)
    assert fields == [n.replace(".", "_") for n in L.ENCODER_CONVS]
    assert [f for f, _ in L.EncoderWeights._fields_] == fields
    assert [f for f, _ in L.ConvWeights._fields_] == ["w_hi", "w_lo", "b"]
    assert L.C.sizeof(L.EncoderWeights) == 22 * 3 * L.C.sizeof(L.C.c_void_p)


def test_encoder_convs_match_the_module():
    from pips_b200 import encoder_fast as E
    from pips_b200.encoder import Encoder
    assert tuple(n for n, _ in E.packed_convs(Encoder())) == L.ENCODER_CONVS
    assert E.keep_shapes(2, 100, 136) == [(2, 50, 68, 64)] * 3 + [(2, 25, 34, 96)] * 2 + [(2, 13, 17, 128)] * 2 \
        + [(2, 7, 9, 128)] * 2
