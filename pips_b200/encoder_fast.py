"""Channels-last inference path of the feature encoder.

Same arithmetic as ``Encoder.forward`` in 'x3' mode (cuDNN TF32 tensor-core convolutions over
[hi | lo | hi] split operands => fp32-class accuracy), but every activation stays NHWC and the
element-wise work between two convolutions -- InstanceNorm, ReLU, residual add, TF32 split, bilinear
resize into the 416-channel concat -- runs in three fused kernels of libpips_b200
(csrc/encoder_ops.cu) instead of ~14 eager passes per convolution.  The result is returned
channels-last, which is already the layout of pyramid level 0.

Reference semantics: BasicEncoder.forward nets/pips.py:247-281, ResidualBlock.forward :173-181.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.nn.functional as F

from . import _lib as L
from .encoder import Encoder, _tf32_hi


LAUNCHES = [0]          # kernels of libpips_b200 launched by the last fnet_tc / fnet_fast call (bench accounting)


def _st() -> int:
    return torch.cuda.current_stream().cuda_stream


def _w3(conv: torch.nn.Conv2d, pad_in_to: int = 0) -> torch.Tensor:
    """[w_hi | w_hi | w_lo] along the input channels, channels-last, cached per weight version."""
    w = conv.weight
    key = (w.data_ptr(), w._version, pad_in_to)
    if getattr(conv, "_w3cl_key", None) != key:
        wd = w.detach().float()
        if pad_in_to and wd.shape[1] < pad_in_to:
            wd = F.pad(wd, (0, 0, 0, 0, 0, pad_in_to - wd.shape[1]))
        hi = _tf32_hi(wd)
        conv._w3cl = torch.cat([hi, hi, wd - hi], dim=1).contiguous(memory_format=torch.channels_last)
        conv._w3cl_key = key
    return conv._w3cl


def _conv(x3_nhwc: torch.Tensor, conv: torch.nn.Conv2d, pad_in_to: int = 0, bias: bool = False) -> torch.Tensor:
    """x3_nhwc (N,H,W,3C) -> conv output as an (N,Ho,Wo,Cout) contiguous NHWC tensor.
    ``bias=False`` for every convolution that feeds an InstanceNorm: a per-channel constant is removed again by
    the normalisation (mean shifts by the same constant, variance unchanged), so adding it would only cost a
    full element-wise pass; the result differs from the reference's by fp32 rounding only."""
    y = F.conv2d(x3_nhwc.permute(0, 3, 1, 2), _w3(conv, pad_in_to), conv.bias if bias else None, conv.stride, conv.padding)
    y = y.permute(0, 2, 3, 1)
    return y if y.is_contiguous() else y.contiguous()


class _Ops:
    def __init__(self, device):
        self.lib = L.load()
        self.dev = device

    def stats(self, y: torch.Tensor) -> torch.Tensor:
        N, H, W, C = y.shape
        hw = H * W
        # partial sums per image: by image size only (never by N: a rank's share of a frame-sharded batch must give
        # the bits of the whole batch); 64 chunks keep even an 8-frame clip at 512 CTAs
        chunks = max(1, min(64, hw // 256))
        partial = torch.empty(N, chunks, 3, C, dtype=torch.float32, device=self.dev)
        st = torch.empty(N, 2, C, dtype=torch.float32, device=self.dev)
        L.check(self.lib.pips_inorm_stats(L.ptr(y), N, hw, C, L.ptr(partial), chunks, L.ptr(st), _st()), "pips_inorm_stats")
        LAUNCHES[0] += 2
        return st

    def apply(self, y, stats, r=None, stats_r=None, relu_main=True, relu_out=False, plain=False, split=True):
        N, H, W, C = y.shape
        out_p = torch.empty_like(y) if plain else None
        out_s = torch.empty(N, H, W, 3 * C, dtype=torch.float32, device=self.dev) if split else None
        L.check(self.lib.pips_inorm_apply(L.ptr(y), L.ptr(stats), L.ptr(r), L.ptr(stats_r), int(relu_main), int(relu_out),
                                          L.ptr(out_p), L.ptr(out_s), 3 * C, N, H * W, C, _st()), "pips_inorm_apply")
        LAUNCHES[0] += 1
        return out_p, out_s

    def resize_into(self, src, dst3, c_off, ctot):
        N, Hs, Ws, C = src.shape
        _, Ho, Wo, _ = dst3.shape
        L.check(self.lib.pips_resize_split3(L.ptr(src), N, Hs, Ws, C, L.ptr(dst3), Ho, Wo, ctot, c_off, _st()),
                "pips_resize_split3")


def fnet_fast(enc: Encoder, x: torch.Tensor) -> torch.Tensor:
    """x (N,3,H,W) fp32 in [-1,1] on CUDA -> feature maps (N, H//stride, W//stride, 128) NHWC fp32.
    Requires torch.backends.cudnn.allow_tf32 = True (set by Pips.encode)."""
    assert x.is_cuda and x.dtype == torch.float32
    ops = _Ops(x.device)
    N, _, H, W = x.shape
    H8, W8 = H // enc.stride, W // enc.stride

    # stem: 3 -> 64, 7x7 / 2.  Input channels padded 3 -> 4 per split block (cuDNN NHWC kernels want C % 4 == 0).
    xh = _tf32_hi(x)
    z = torch.zeros(N, 1, H, W, dtype=torch.float32, device=x.device)
    x12 = torch.cat([xh, z, x - xh, z, xh, z], dim=1).permute(0, 2, 3, 1).contiguous()
    y = _conv(x12, enc.conv1, pad_in_to=4)
    X, X3 = ops.apply(y, ops.stats(y), relu_main=True, plain=True, split=True)

    ctot = 64 + 96 + 128 + 128
    cat3 = torch.empty(N, H8, W8, 3 * ctot, dtype=torch.float32, device=x.device)
    c_off = 0
    for i in range(1, 5):
        for blk in getattr(enc, f"layer{i}"):
            y1 = _conv(X3, blk.conv1)
            _, A3 = ops.apply(y1, ops.stats(y1), relu_main=True)
            y2 = _conv(A3, blk.conv2)
            s2 = ops.stats(y2)
            if blk.downsample is not None:
                d = _conv(X3, blk.downsample[0])
                X, X3 = ops.apply(y2, s2, r=d, stats_r=ops.stats(d), relu_main=True, relu_out=True, plain=True)
            else:
                X, X3 = ops.apply(y2, s2, r=X, relu_main=True, relu_out=True, plain=True)
        ops.resize_into(X, cat3, c_off, ctot)
        c_off += X.shape[-1]

    y = _conv(cat3, enc.conv2)
    _, A3 = ops.apply(y, ops.stats(y), relu_main=True)
    return _conv(A3, enc.conv3, bias=True)


# --------------------------------------------------------------------------------------------------------------
# 'tc' path: every 3x3 / 1x1 convolution on the wgmma implicit-GEMM kernel (csrc/conv_tc.cu), bf16x3 operands
# --------------------------------------------------------------------------------------------------------------

def _pad64(c: int) -> int:
    return (c + 63) // 64 * 64


def pack_conv_weight(w: torch.Tensor):
    """(Cout, Cin, R, S) -> ((BN, R*S*Cp) bf16 hi, lo) with k = (r*S + s)*Cp + ci, the filter layout of pips_conv_tc."""
    lib = L.load()
    cout, cin, R, S = w.shape
    cp = _pad64(cin)
    bn = 64 if cout <= 64 else (128 if cout <= 128 else 256)
    packed = torch.zeros(bn, R, S, cp, dtype=torch.float32, device=w.device)
    packed[:cout, :, :, :cin] = w.detach().float().permute(0, 2, 3, 1)
    packed = packed.reshape(bn, R * S * cp).contiguous()
    hi = torch.empty_like(packed, dtype=torch.bfloat16)
    lo = torch.empty_like(packed, dtype=torch.bfloat16)
    L.check(lib.pips_split_bf16(L.ptr(packed), L.ptr(hi), L.ptr(lo), packed.numel(), _st()), "pips_split_bf16")
    return hi, lo


def _packed_weight(conv: torch.nn.Conv2d):
    """pack_conv_weight of conv.weight, cached per weight version."""
    w = conv.weight
    key = (w.data_ptr(), w._version)
    if getattr(conv, "_wtc_key", None) != key:
        conv._wtc = pack_conv_weight(w)
        conv._wtc_key = key
    return conv._wtc


class _Pair:
    """bf16 (hi, lo) channels-last activation (N, H, W, Cp); the producing kernel (pips_inorm_apply_pair, pips_resize_pair,
    pips_stem_pack) writes the padding channels [C, Cp) as zero itself, so no fill pass is needed."""

    def __init__(self, N, H, W, C, device):
        self.shape, self.C, self.Cp = (N, H, W), C, _pad64(C)
        self.hi = torch.empty(N, H, W, self.Cp, dtype=torch.bfloat16, device=device)
        self.lo = torch.empty(N, H, W, self.Cp, dtype=torch.bfloat16, device=device)


def conv_tc(x: _Pair, conv: torch.nn.Conv2d, bias: bool = False, stats: bool = False, w=None):
    """-> output (N,Ho,Wo,Cout) fp32; with ``stats`` also the InstanceNorm statistics (N,2,Cout) of the output, from
    partial sums the convolution's epilogue accumulates (no separate pass over the output).  ``w``: the (hi, lo) filter
    pack to use instead of the module's cached one."""
    lib = L.load()
    N, H, W = x.shape
    cout, cin, R, S = conv.weight.shape
    assert cin == x.C and conv.stride[0] == conv.stride[1] and conv.padding[0] == conv.padding[1]
    st, pad = conv.stride[0], conv.padding[0]
    Ho, Wo = (H + 2 * pad - R) // st + 1, (W + 2 * pad - S) // st + 1
    w_hi, w_lo = _packed_weight(conv) if w is None else w
    dev = x.hi.device
    out = torch.empty(N, Ho, Wo, cout, dtype=torch.float32, device=dev)
    b = conv.bias.detach().float().contiguous() if bias and conv.bias is not None else None
    if not stats:
        L.check(lib.pips_conv_tc(L.ptr(x.hi), L.ptr(x.lo), N, H, W, x.Cp, L.ptr(w_hi), L.ptr(w_lo), cout, R, S, st, pad,
                                 L.ptr(b), L.ptr(out), _st()), "pips_conv_tc")
        LAUNCHES[0] += 1
        return out
    chunks = lib.pips_conv_tc_chunks(H, W, R, S, st, st, pad, pad)
    partial = torch.empty(N, chunks, 3, cout, dtype=torch.float32, device=dev)
    stt = torch.empty(N, 2, cout, dtype=torch.float32, device=dev)
    L.check(lib.pips_conv_tc_stats(L.ptr(x.hi), L.ptr(x.lo), N, H, W, x.Cp, L.ptr(w_hi), L.ptr(w_lo), cout, R, S, st, st, pad, pad,
                                   L.ptr(b), L.ptr(out), L.ptr(partial), _st()), "pips_conv_tc_stats")
    L.check(lib.pips_inorm_finalize(L.ptr(partial), N, chunks, Ho * Wo, cout, L.ptr(stt), _st()), "pips_inorm_finalize")
    LAUNCHES[0] += 2
    return out, stt


def conv_rows_ok(x: _Pair, conv: torch.nn.Conv2d) -> bool:
    """The row-ring kernel (csrc/conv_rows.cu) covers BasicEncoder's layer1 convolutions: 3x3, stride 1, pad 1, 64 -> 64."""
    W = x.shape[2]
    # a CTA pair covers 256 pixels of a row: widths that fill less than 3/4 of the last pair (e.g. 320 = 256 + 64) are
    # faster on the tap-by-tap kernel (measured: 8 x 180 x 320 maps, 136 vs 121 + 25 us)
    fill = W / float(((W + 255) // 256) * 256)
    return (x.C == 64 and x.Cp == 64 and tuple(conv.weight.shape) == (64, 64, 3, 3) and conv.stride == (1, 1)
            and conv.padding == (1, 1) and fill >= 0.75 and os.environ.get("PIPS_B200_CONV_ROWS", "1") != "0")


def conv_rows(x: _Pair, conv: torch.nn.Conv2d, w=None):
    """-> (out (N,H,W,64) fp32, InstanceNorm statistics (N,2,64) of out): the statistics come from partial sums the
    convolution's epilogue accumulates, so no separate pass reads the output."""
    lib = L.load()
    N, H, W = x.shape
    w_hi, w_lo = _packed_weight(conv) if w is None else w
    dev = x.hi.device
    out = torch.empty(N, H, W, 64, dtype=torch.float32, device=dev)
    chunks = lib.pips_conv_rows_chunks(H, W)
    partial = torch.empty(N, chunks, 3, 64, dtype=torch.float32, device=dev)
    st = torch.empty(N, 2, 64, dtype=torch.float32, device=dev)
    L.check(lib.pips_conv_rows(L.ptr(x.hi), L.ptr(x.lo), N, H, W, L.ptr(w_hi), L.ptr(w_lo), L.ptr(out), L.ptr(partial), _st()),
            "pips_conv_rows")
    L.check(lib.pips_inorm_finalize(L.ptr(partial), N, chunks, H * W, 64, L.ptr(st), _st()), "pips_inorm_finalize")
    LAUNCHES[0] += 2
    return out, st


def _conv_stats(ops: _Ops, x: _Pair, conv: torch.nn.Conv2d, w=None):
    """Convolution feeding an InstanceNorm: (output, statistics)."""
    if conv_rows_ok(x, conv):
        return conv_rows(x, conv, w)
    if os.environ.get("PIPS_B200_CONV_STATS", "1") == "0":      # separate statistics pass (round 1), for A/B
        y = conv_tc(x, conv, w=w)
        return y, ops.stats(y)
    return conv_tc(x, conv, stats=True, w=w)


def _apply_pair(ops: _Ops, y, stats, r=None, stats_r=None, relu_main=True, relu_out=False, plain=False):
    N, H, W, C = y.shape
    out_p = torch.empty_like(y) if plain else None
    pair = _Pair(N, H, W, C, y.device)
    L.check(ops.lib.pips_inorm_apply_pair(L.ptr(y), L.ptr(stats), L.ptr(r), L.ptr(stats_r), int(relu_main), int(relu_out),
                                          L.ptr(out_p), L.ptr(pair.hi), L.ptr(pair.lo), pair.Cp, N, H * W, C, _st()),
            "pips_inorm_apply_pair")
    LAUNCHES[0] += 1
    return out_p, pair


def pack_stem_weight(w: torch.Tensor):
    """7x7x3 stem (Cout,3,7,7) -> (64, 4*64) bf16 (hi, lo) for the 4x1 convolution over pips_stem_pack's row-pair pixels:
    tap d (row pair) major, then [filter row 2d: k = s*3 + colour, 21 of 32 | filter row 2d+1: same; row 7 does not exist: 0]."""
    lib = L.load()
    cout = w.shape[0]
    rows = torch.zeros(64, 8, 32, dtype=torch.float32, device=w.device)                    # [co][filter row r][s*3+ci]
    rows[:cout, :7, :21] = w.detach().float().permute(0, 2, 3, 1).reshape(cout, 7, 21)
    packed = rows.reshape(64, 4 * 64).contiguous()                                          # (r = 2d, 2d+1) -> 64 channels of tap d
    hi = torch.empty_like(packed, dtype=torch.bfloat16)
    lo = torch.empty_like(packed, dtype=torch.bfloat16)
    L.check(lib.pips_split_bf16(L.ptr(packed), L.ptr(hi), L.ptr(lo), packed.numel(), _st()), "pips_split_bf16")
    return hi, lo


def _packed_stem_weight(conv: torch.nn.Conv2d):
    """pack_stem_weight of conv.weight, cached per weight version."""
    w = conv.weight
    key = (w.data_ptr(), w._version)
    if getattr(conv, "_wstem_key", None) != key:
        conv._wstem = pack_stem_weight(w)
        conv._wstem_key = key
    return conv._wstem


# ---- weight-pack hooks (pips_b200/pack.py): enumerate, export and adopt the packed filters ------------------

def packed_convs(enc: Encoder):
    """(dotted name, module) of every convolution the 'tc' path packs, in module order."""
    return [(n, m) for n, m in enc.named_modules() if isinstance(m, torch.nn.Conv2d)]


def packed_filter(enc: Encoder, name: str, conv: torch.nn.Conv2d):
    return _packed_stem_weight(conv) if conv is enc.conv1 else _packed_weight(conv)


def adopt_filter(enc: Encoder, name: str, conv: torch.nn.Conv2d, hi: torch.Tensor, lo: torch.Tensor) -> None:
    """Install an already packed (hi, lo) filter as the cache entry of ``conv``'s current weight version."""
    w = conv.weight
    key = (w.data_ptr(), w._version)
    if conv is enc.conv1:
        expect = (64, 4 * 64)
    else:
        cout, cin, R, S = w.shape
        bn = 64 if cout <= 64 else (128 if cout <= 128 else 256)
        expect = (bn, R * S * _pad64(cin))
    if tuple(hi.shape) != expect or tuple(lo.shape) != expect or hi.dtype != torch.bfloat16 or hi.device != w.device:
        raise L.PipsCudaError(f"pips_b200: packed filter {name} has shape {tuple(hi.shape)}, expected {expect}")
    if conv is enc.conv1:                                   # validated: only now does it become the cache entry
        conv._wstem, conv._wstem_key = (hi, lo), key
    else:
        conv._wtc, conv._wtc_key = (hi, lo), key


def fnet_tc(enc: Encoder, rgb: torch.Tensor) -> torch.Tensor:
    """rgb (N,3,H,W) fp32 or bf16 with values 0..255 (NOT normalised) -> feature maps (N,H/stride,W/stride,128) NHWC.
    The whole encoder on libpips_b200: the 7x7/2 stem as a 4x1 stride-1 wgmma convolution over the unfolded,
    normalised image (pips_stem_pack: row pairs x 7 column taps x 3 colours per pixel), residual stages and head on pips_conv_tc, element-wise stages fused."""
    assert rgb.is_cuda and rgb.dtype in (torch.float32, torch.bfloat16)
    from .engine import nvtx_range
    with nvtx_range("pips/fnet"):
        return _fnet_tc(enc, rgb)


def stem_tc(rgb: torch.Tensor, w):
    """The stem's convolution as fnet_tc runs it: rgb (N,3,H,W) contiguous, 0..255, and the pack_stem_weight pack w ->
    (the pips_stem_pack operand, the (N,Ho,Wo,64) output before its InstanceNorm, that InstanceNorm's statistics).
    The backward of torch_path.encoder_cuda recomputes the stem through this same function."""
    lib = L.load()
    N, _, H, W = rgb.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    unf = _Pair(N, Ho + 3, Wo, 64, rgb.device)                   # row pairs (2j-3, 2j-2) x 7 column taps x 3 colours
    L.check(lib.pips_stem_pack(L.ptr(rgb), 0 if rgb.dtype == torch.float32 else 1, N, H, W, L.ptr(unf.hi), L.ptr(unf.lo), _st()),
            "pips_stem_pack")
    w_hi, w_lo = w
    y = torch.empty(N, Ho, Wo, 64, dtype=torch.float32, device=rgb.device)
    chunks = lib.pips_conv_tc_chunks(Ho + 3, Wo, 4, 1, 1, 1, 0, 0)
    partial = torch.empty(N, chunks, 3, 64, dtype=torch.float32, device=rgb.device)
    s_stem = torch.empty(N, 2, 64, dtype=torch.float32, device=rgb.device)
    L.check(lib.pips_conv_tc_stats(L.ptr(unf.hi), L.ptr(unf.lo), N, Ho + 3, Wo, 64, L.ptr(w_hi), L.ptr(w_lo), 64, 4, 1, 1, 1, 0, 0,
                                   None, L.ptr(y), L.ptr(partial), _st()), "pips_conv_tc_stats")
    L.check(lib.pips_inorm_finalize(L.ptr(partial), N, chunks, Ho * Wo, 64, L.ptr(s_stem), _st()), "pips_inorm_finalize")
    LAUNCHES[0] += 3                                   # stem_pack + stem conv + statistics finalize
    return unf, y, s_stem


def encoder_weights(enc: Encoder, packs=None):
    """-> (pips_encoder_weights of ``enc``, the tensors it points into).  ``packs``: {conv module: (hi, lo)} filter packs
    to use instead of the modules' caches (which are then neither read nor written)."""
    w = L.EncoderWeights()
    hold = []
    convs = dict(packed_convs(enc))
    for name in L.ENCODER_CONVS:
        conv = convs[name]
        hi, lo = packed_filter(enc, name, conv) if packs is None else packs[conv]
        b = None if conv.bias is None else conv.bias.detach().float().contiguous()
        f = getattr(w, name.replace(".", "_"))
        f.w_hi, f.w_lo, f.b = L.ptr(hi), L.ptr(lo), L.ptr(b)
        hold += [hi, lo, b]
    return w, hold


def keep_shapes(N: int, H: int, W: int):
    """Shapes of the 9 block boundaries pips_encode can keep: the stem output, then every ResBlock output (NHWC)."""
    h, w = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = [(N, h, w, 64)]
    for i, c in enumerate((64, 96, 128, 128)):
        if i:
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        out += [(N, h, w, c)] * 2
    return out


def _fnet_tc(enc: Encoder, rgb: torch.Tensor, packs=None, keep=None) -> torch.Tensor:
    """The whole encoder as one pips_encode call, its workspace from torch's caching allocator.
    ``packs``: {conv module: (hi, lo)} filter packs to use instead of the modules' caches (torch_path.encoder_cuda);
    ``keep``: a list that receives the block boundaries -- the stem output and every ResBlock output, fp32."""
    lib = L.load()
    rgb = rgb.contiguous()
    N, _, H, W = rgb.shape
    dev = rgb.device
    w, hold = encoder_weights(enc, packs)
    nbytes = lib.pips_encode_workspace_bytes(N, H, W, enc.stride)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    out = torch.empty(N, H // enc.stride, W // enc.stride, 128, dtype=torch.float32, device=dev)
    kept = [torch.empty(s, dtype=torch.float32, device=dev) for s in keep_shapes(N, H, W)] if keep is not None else None
    L.check(lib.pips_encode(C.byref(w), L.ptr(rgb), 0 if rgb.dtype == torch.float32 else 1, N, H, W, enc.stride, L.ptr(ws),
                            nbytes, L.ptr(out), None if kept is None else L.ptr_array(kept), _st()), "pips_encode")
    LAUNCHES[0] = lib.pips_encode_launches(N, H, W, enc.stride)
    if keep is not None:
        keep.extend(kept)
    return out


# ---- the whole encoder as one CUDA graph per input shape ---------------------------------------------------
# pips_encode launches 66 kernels per call (pips_encode_launches); for few frames (the demo clip, a rank's share of a
# frame-sharded batch, chained windows) the kernels are microseconds long and the encoder is launch-bound when enqueued
# one by one.

class _FnetGraph:
    def __init__(self, enc: Encoder, shape, dtype, dev):
        self.x = torch.zeros(shape, dtype=dtype, device=dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            fnet_tc(enc, self.x)                          # packs the filters, sets function attributes
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = fnet_tc(enc, self.x)
        self.launches = LAUNCHES[0]

    def run(self, x: torch.Tensor) -> torch.Tensor:
        self.x.copy_(x)
        self.graph.replay()
        LAUNCHES[0] = self.launches
        return self.out.clone()                           # the static output is overwritten by the next replay


def fnet_tc_graphed(enc: Encoder, rgb: torch.Tensor) -> torch.Tensor:
    """fnet_tc replayed from a CUDA graph captured per (shape, dtype, parameter versions); two plans are kept."""
    key = (tuple(rgb.shape), rgb.dtype, str(rgb.device), tuple((p.data_ptr(), p._version) for p in enc.parameters()))
    plans = enc.__dict__.setdefault("_fnet_plans", {})
    plan = plans.get(key)
    if plan is None:
        while len(plans) >= 2:                            # each plan owns every activation of one encoder pass
            plans.pop(next(iter(plans)))
        plan = plans[key] = _FnetGraph(enc, rgb.shape, rgb.dtype, rgb.device)
    else:
        plans[key] = plans.pop(key)                       # LRU order
    return plan.run(rgb)
