"""Per-kernel parity of the feature encoder's CUDA entry points (csrc/encoder_ops.cu, conv_tc.cu, conv_rows.cu, the
weight split of abi.cu) against fp64 torch references on the host.

Output buffers are poisoned with NaN before every call, so a test sees exactly which elements a kernel wrote: K padding
must come out as exact zero and channels outside a call's slice must stay NaN.  Layouts, zero padding and the hi/lo
split identities are compared bit for bit; sums get a tolerance relative to fp64 and print the measured error."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import _lib as L

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 1e-5                                    # InstanceNorm2d eps
BF16_NAN = 0x7FC0                             # bit pattern torch.full(..., nan, dtype=bfloat16) writes
PARTIAL_ROWS = 3                              # rows per (image, chunk) of the partial statistics: (mean, M2, count)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32).cpu()


def _split_bf16(t):
    """The (hi, lo) pair the kernels write: hi = rn_bf16(v), lo = rn_bf16(v - hi)."""
    hi = t.to(torch.bfloat16)
    return hi, (t - hi.float()).to(torch.bfloat16)


def _tf32_hi(t):
    return (t.contiguous().view(torch.int32) & -8192).view(torch.float32)       # 0xffffe000: TF32 truncation


def _pad64(c):
    return (c + 63) // 64 * 64


def _ref_stats(y):
    """fp64 (mean, rstd) per (image, channel) of y (N, ..., C)."""
    yd = y.double().reshape(y.shape[0], -1, y.shape[-1])
    mean = yd.mean(1)
    var = yd.var(1, unbiased=False)
    return mean, 1.0 / torch.sqrt(var + EPS), var.sqrt()


def _stats_err(st, y):
    """(mean error relative to |mean| + std, rstd relative error) of kernel statistics st (N, 2, C) against fp64."""
    mean, rstd, std = _ref_stats(y.cpu())
    st = st.double().cpu()
    e_mean = ((st[:, 0] - mean).abs() / (mean.abs() + std + 1e-30)).max().item()
    e_rstd = ((st[:, 1] - rstd).abs() / rstd).max().item()
    return e_mean, e_rstd


# ------------------------------------------------------------------------------------------------ 1. stem unfolding

def _stem_unfold_ref(rgb):
    """(N,3,H,W) 0..255 -> (N, Ho+3, Wo, 64) fp32: pixel (j, ox) holds rows 2j-3 (channels 0..31) and 2j-2 (32..63),
    channel s*3 + colour of a row = 2*(rgb/255)-1 at column 2*ox + s - 3, zero outside the image and for s*3 + c >= 21."""
    v = 2.0 * (rgb.float() / 255.0) - 1.0
    N, _, H, W = v.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    J = Ho + 3
    vp = torch.zeros(N, 3, 2 * J + 2, 2 * Wo + 8)
    vp[:, :, 3:3 + H, 3:3 + W] = v
    out = torch.zeros(N, J, Wo, 64)
    for half in range(2):
        rows = vp[:, :, half:half + 2 * J:2]                                     # input row 2j - 3 + half
        for s in range(7):
            cols = rows[:, :, :, s:s + 2 * Wo:2]                                  # input column 2*ox + s - 3
            out[..., half * 32 + s * 3:half * 32 + s * 3 + 3] = cols.permute(0, 2, 3, 1)
    return out


def _stem_pack(rgb_dev):
    lib = L.load()
    N, _, H, W = rgb_dev.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    hi, lo = _nan(N, Ho + 3, Wo, 64, dtype=torch.bfloat16), _nan(N, Ho + 3, Wo, 64, dtype=torch.bfloat16)
    L.check(lib.pips_stem_pack(L.ptr(rgb_dev), 0 if rgb_dev.dtype == torch.float32 else 1, N, H, W, L.ptr(hi), L.ptr(lo), _st()),
            "pips_stem_pack")
    return hi, lo


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("H,W", [(1, 1), (7, 9), (23, 37), (360, 640)])
def test_stem_pack_bit_exact(dtype, H, W):
    torch.manual_seed(31)
    rgb = (torch.rand(3, 3, H, W) * 255.0).to(dtype)          # not integers: the division and the split must round alike
    hi, lo = _stem_pack(rgb.to(DEV))
    torch.cuda.synchronize()
    r_hi, r_lo = _split_bf16(_stem_unfold_ref(rgb))
    assert hi.shape == r_hi.shape
    assert torch.equal(_bits(hi), _bits(r_hi)), "hi differs (layout, normalisation or zero padding)"
    assert torch.equal(_bits(lo), _bits(r_lo)), "lo differs"


# ------------------------------------------------------------------------------------------------ 2. stem / anisotropic convolution

def _stem_conv(rgb_dev, conv):
    """pips_stem_pack -> pips_conv_tc_stats (4x1, stride 1, no padding) -> pips_inorm_finalize, as fnet_tc runs the stem."""
    from pips_b200.encoder_fast import _packed_stem_weight
    lib = L.load()
    N, _, H, W = rgb_dev.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    hi, lo = _stem_pack(rgb_dev)
    w_hi, w_lo = _packed_stem_weight(conv)
    chunks = lib.pips_conv_tc_chunks(Ho + 3, Wo, 4, 1, 1, 1, 0, 0)
    out = _nan(N, Ho, Wo, 64)
    partial = _nan(N, chunks, PARTIAL_ROWS, 64)
    st = _nan(N, 2, 64)
    L.check(lib.pips_conv_tc_stats(L.ptr(hi), L.ptr(lo), N, Ho + 3, Wo, 64, L.ptr(w_hi), L.ptr(w_lo), 64, 4, 1, 1, 1, 0, 0, None,
                                   L.ptr(out), L.ptr(partial), _st()), "pips_conv_tc_stats")
    L.check(lib.pips_inorm_finalize(L.ptr(partial), N, chunks, Ho * Wo, 64, L.ptr(st), _st()), "pips_inorm_finalize")
    torch.cuda.synchronize()
    return out, st


def _stem_module(seed=0):
    conv = torch.nn.Conv2d(3, 64, 7, stride=2, padding=3).to(DEV)
    with torch.no_grad():
        conv.weight.copy_(po.init_state_dict(seed)["fnet.conv1.weight"])
    return conv


@pytest.mark.parametrize("N,H,W", [(2, 64, 80), (1, 45, 67), (3, 23, 37)])
def test_stem_conv(N, H, W):
    torch.manual_seed(37)
    conv = _stem_module()
    rgb = torch.randint(0, 256, (N, 3, H, W)).float()
    out, st = _stem_conv(rgb.to(DEV), conv)
    x = (2.0 * (rgb / 255.0) - 1.0).double()
    ref = F.conv2d(x, conv.weight.detach().double().cpu(), None, stride=2, padding=3).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    err = (out.cpu().double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    e_mean, e_rstd = _stats_err(st, ref)
    s_mean, s_rstd = _stats_err(st, out)
    print(f"stem {N}x{H}x{W}: max err {err:.2e} (|out| max {scale:.2f}); stats vs fp64 conv: mean {e_mean:.2e}, rstd {e_rstd:.2e}; "
          f"vs own output: mean {s_mean:.2e}, rstd {s_rstd:.2e}")
    assert err < 3e-4 * max(1.0, scale)
    assert e_mean < 1e-4 and e_rstd < 1e-4             # bounded by the convolution's own error
    assert s_mean < 1e-6 and s_rstd < 1e-5             # the statistics of what the kernel wrote


@pytest.mark.parametrize("stats", [False, True])
def test_conv_tc_aniso(stats):
    """A generic anisotropic geometry: 3x1 filter, stride (2, 1), padding (1, 0)."""
    from pips_b200.encoder_fast import _Pair, _packed_weight
    lib = L.load()
    torch.manual_seed(41)
    N, H, W, cin, cout = 2, 37, 45, 64, 96
    conv = torch.nn.Conv2d(cin, cout, (3, 1)).to(DEV)
    x = torch.randn(N, H, W, cin, device=DEV)
    pair = _Pair(N, H, W, cin, DEV)
    pair.hi.copy_(x.to(torch.bfloat16))
    pair.lo.copy_((x - pair.hi.float()).to(torch.bfloat16))
    w_hi, w_lo = _packed_weight(conv)
    Ho, Wo = (H + 2 - 3) // 2 + 1, W
    out = _nan(N, Ho, Wo, cout)
    if stats:
        chunks = lib.pips_conv_tc_chunks(H, W, 3, 1, 2, 1, 1, 0)
        partial = _nan(N, chunks, PARTIAL_ROWS, cout)
        st = _nan(N, 2, cout)
        L.check(lib.pips_conv_tc_stats(L.ptr(pair.hi), L.ptr(pair.lo), N, H, W, 64, L.ptr(w_hi), L.ptr(w_lo), cout, 3, 1, 2, 1, 1, 0,
                                       None, L.ptr(out), L.ptr(partial), _st()), "pips_conv_tc_stats")
        L.check(lib.pips_inorm_finalize(L.ptr(partial), N, chunks, Ho * Wo, cout, L.ptr(st), _st()), "pips_inorm_finalize")
    else:
        L.check(lib.pips_conv_tc_aniso(L.ptr(pair.hi), L.ptr(pair.lo), N, H, W, 64, L.ptr(w_hi), L.ptr(w_lo), cout, 3, 1, 2, 1, 1, 0,
                                       None, L.ptr(out), _st()), "pips_conv_tc_aniso")
    torch.cuda.synchronize()
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), conv.weight.double(), None, stride=(2, 1), padding=(1, 0)).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    err = (out.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"conv_tc 3x1 s(2,1) p(1,0): max err {err:.2e} (|out| max {scale:.2f})")
    assert err < 3e-4 * max(1.0, scale)
    if stats:
        s_mean, s_rstd = _stats_err(st, out)
        print(f"  statistics vs own output: mean {s_mean:.2e}, rstd {s_rstd:.2e}")
        assert s_mean < 1e-6 and s_rstd < 1e-5


# ------------------------------------------------------------------------------------------------ 3./4. statistics

def _inorm_stats(y, chunks):
    lib = L.load()
    N, HW, C = y.shape
    partial = _nan(N, chunks, PARTIAL_ROWS, C)
    st = _nan(N, 2, C)
    L.check(lib.pips_inorm_stats(L.ptr(y), N, HW, C, L.ptr(partial), chunks, L.ptr(st), _st()), "pips_inorm_stats")
    torch.cuda.synchronize()
    return st


@pytest.mark.parametrize("C", [4, 64, 96, 128, 256, 1024])
def test_inorm_stats_random(C):
    """Every HW / chunk count combination, including one pixel, chunks that do not divide HW and empty chunks."""
    torch.manual_seed(43)
    hws = [1, 255, 256 * 3 + 17] + ([192 * 256] if C <= 256 else [256 * 8 + 17])
    worst = [0.0, 0.0]
    for hw in hws:
        mean = torch.rand(C) * 2 - 1
        std = torch.rand(C) * 1.5 + 0.5
        y = (torch.randn(2, hw, C) * std + mean).to(DEV)
        for chunks in sorted({1, 64, hw + 3} if hw <= 4096 else {1, 64}):
            e_mean, e_rstd = _stats_err(_inorm_stats(y, chunks), y)
            worst = [max(worst[0], e_mean), max(worst[1], e_rstd)]
            # a chunk of one thread per channel (C = 1024) sums up to ~2000 pixels in sequence: the mean's rounding
            # walks like sqrt(n) fp32 ulps
            assert e_mean < 4e-6 and e_rstd < 1e-5, (hw, chunks, e_mean, e_rstd)
    print(f"inorm_stats C={C}: mean err {worst[0]:.2e} (relative to |mean| + std), rstd rel err {worst[1]:.2e}")


def _hard_channels(N, HW, C, seed):
    """Channels that cancel in (sum, sum of squares): constant, and mean/std of 1e2 and 1e3."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(N, 1, C, generator=g) * 4 - 2
    noise = torch.randn(N, HW, C, generator=g)
    kind = torch.arange(C) % 3
    ratio = torch.tensor([0.0, 1e2, 1e3])[kind]
    std = torch.where(kind == 0, torch.zeros(C), base.abs().clamp_min(0.5) / ratio.clamp_min(1.0))
    return base + noise * std, kind


@pytest.mark.parametrize("HW,C,chunks", [(192 * 256, 64, 64), (360 * 640, 64, 64), (24 * 32, 256, 3), (4097, 96, 1)])
def test_inorm_stats_flat_channels(HW, C, chunks):
    y, kind = _hard_channels(2, HW, C, seed=HW + C)
    st = _inorm_stats(y.to(DEV), chunks).double().cpu()
    mean, rstd, std = _ref_stats(y)
    e_rstd = ((st[:, 1] - rstd).abs() / rstd)
    e_mean = ((st[:, 0] - mean).abs() / (mean.abs() + std))
    e_const = (st[:, 1, kind == 0] * math.sqrt(EPS) - 1).abs().max().item()
    print(f"inorm_stats flat HW={HW} C={C} chunks={chunks}: constant channels rstd rel err {e_const:.2e}; "
          f"mean/std 1e2: rstd {e_rstd[:, kind == 1].max().item():.2e}; 1e3: rstd {e_rstd[:, kind == 2].max().item():.2e}; "
          f"mean {e_mean.max().item():.2e}")
    assert e_const < 1e-6
    assert e_rstd.max().item() < 1e-5
    assert e_mean.max().item() < 1e-6


def _flat_pair(N, H, W, C, seed):
    """A constant activation (per channel) with a one-pixel border of other values, as a bf16 (hi, lo) pair."""
    from pips_b200.encoder_fast import _Pair
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(1, 1, 1, C, generator=g) + 0.5).expand(N, H, W, C).clone()
    border = torch.rand(N, H, W, C, generator=g) * 3
    x[:, 0], x[:, -1], x[:, :, 0], x[:, :, -1] = border[:, 0], border[:, -1], border[:, :, 0], border[:, :, -1]
    pair = _Pair(N, H, W, C, DEV)
    pair.hi.zero_()
    pair.lo.zero_()
    hi, lo = _split_bf16(x)
    pair.hi[..., :C] = hi.to(DEV)
    pair.lo[..., :C] = lo.to(DEV)
    return pair


@pytest.mark.parametrize("producer,N,H,W,cin,cout,k,stride", [
    ("conv_tc", 2, 96, 128, 64, 64, 3, 1),
    ("conv_tc", 1, 90, 160, 128, 128, 3, 2),
    ("conv_tc", 2, 48, 64, 128, 256, 1, 2),
    ("conv_tc", 1, 24, 32, 416, 256, 3, 1),          # the head convolution over the concat
    ("conv_rows", 2, 96, 256, 64, 64, 3, 1),
    ("conv_rows", 1, 180, 640, 64, 64, 3, 1),
])
def test_conv_stats_flat_input(producer, N, H, W, cin, cout, k, stride):
    """Epilogue statistics of a convolution over a flat input: every interior output pixel is the same value, so the
    mean is large against the spread the border leaves."""
    from pips_b200.encoder_fast import conv_rows, conv_tc
    torch.manual_seed(47)
    conv = torch.nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2).to(DEV)
    pair = _flat_pair(N, H, W, cin, seed=H * W + cin)
    out, st = conv_rows(pair, conv) if producer == "conv_rows" else conv_tc(pair, conv, stats=True)
    torch.cuda.synchronize()
    mean, rstd, std = _ref_stats(out.cpu())
    e_mean, e_rstd = _stats_err(st, out)
    ratio = (mean.abs() / std.clamp_min(1e-30)).median().item()
    print(f"{producer} flat {N}x{H}x{W} {cin}->{cout} k{k} s{stride}: median |mean|/std {ratio:.1e}; "
          f"mean err {e_mean:.2e}, rstd rel err {e_rstd:.2e}")
    assert e_mean < 1e-6 and e_rstd < 1e-5


@pytest.mark.parametrize("H,W,value", [(720, 1280, 255.0), (384, 512, 255.0), (384, 512, 0.0), (384, 512, 128.0)])
def test_stem_stats_flat_frame(H, W, value):
    """The stem over a uniform frame: the only spread is the zero padding at the border."""
    conv = _stem_module()
    out, st = _stem_conv(torch.full((1, 3, H, W), value, device=DEV), conv)
    e_mean, e_rstd = _stats_err(st, out)
    print(f"stem statistics, uniform {value:g} {H}x{W}: mean err {e_mean:.2e}, rstd rel err {e_rstd:.2e}")
    assert e_mean < 1e-6 and e_rstd < 1e-5


# ------------------------------------------------------------------------------------------------ 5. normalise / apply

def _apply_ref(y, sy, r, sr, relu_main, relu_out):
    N, HW, C = y.shape
    v = y.double()
    if sy is not None:
        v = (v - sy[:, 0].double().unsqueeze(1)) * sy[:, 1].double().unsqueeze(1)
    if relu_main:
        v = v.clamp_min(0)
    if r is not None:
        w = r.double()
        if sr is not None:
            w = (w - sr[:, 0].double().unsqueeze(1)) * sr[:, 1].double().unsqueeze(1)
        v = v + w
    if relu_out:
        v = v.clamp_min(0)
    return v


@pytest.mark.parametrize("C", [64, 96, 128])
def test_inorm_apply(C):
    lib = L.load()
    torch.manual_seed(53)
    N, HW = 2, 301
    y = (torch.randn(N, HW, C) * 2 + 0.5).to(DEV)
    r = torch.randn(N, HW, C).to(DEV)
    sy = torch.stack([torch.randn(N, C) * 0.5, torch.rand(N, C) + 0.3], 1).to(DEV).contiguous()
    sr = torch.stack([torch.randn(N, C) * 0.5, torch.rand(N, C) + 0.3], 1).to(DEV).contiguous()
    split_ld, pair_ld = 3 * C + 8, _pad64(C)
    worst = 0.0
    for relu_main in (0, 1):
        for relu_out in (0, 1):
            for res in ("none", "raw", "norm"):
                for norm_y in (True, False):
                    rr = None if res == "none" else r
                    srr = sr if res == "norm" else None
                    syy = sy if norm_y else None
                    ref = _apply_ref(y.cpu(), None if syy is None else syy.cpu(), None if rr is None else rr.cpu(),
                                     None if srr is None else srr.cpu(), relu_main, relu_out)
                    plain, split = _nan(N, HW, C), _nan(N, HW, split_ld)
                    L.check(lib.pips_inorm_apply(L.ptr(y), L.ptr(syy), L.ptr(rr), L.ptr(srr), relu_main, relu_out, L.ptr(plain),
                                                 L.ptr(split), split_ld, N, HW, C, _st()), "pips_inorm_apply")
                    plain2, hi, lo = _nan(N, HW, C), _nan(N, HW, pair_ld, dtype=torch.bfloat16), _nan(N, HW, pair_ld, dtype=torch.bfloat16)
                    L.check(lib.pips_inorm_apply_pair(L.ptr(y), L.ptr(syy), L.ptr(rr), L.ptr(srr), relu_main, relu_out, L.ptr(plain2),
                                                      L.ptr(hi), L.ptr(lo), pair_ld, N, HW, C, _st()), "pips_inorm_apply_pair")
                    torch.cuda.synchronize()
                    what = f"relu_main={relu_main} relu_out={relu_out} residual={res} stats_y={'set' if norm_y else 'NULL'}"
                    p = plain.cpu()
                    err = ((p.double() - ref).abs() / ref.abs().clamp_min(1.0)).max().item()
                    worst = max(worst, err)
                    assert err < 2e-6, (what, err)
                    assert torch.equal(_bits(plain2), _bits(plain)), what
                    # [hi | lo | hi] TF32 split at row stride split_ld; the columns past 3C are not the kernel's
                    h = _tf32_hi(p)
                    s = split.cpu()
                    assert torch.equal(_bits(s[..., :C]), _bits(h)), what
                    assert torch.equal(_bits(s[..., C:2 * C]), _bits(p - h)), what
                    assert torch.equal(_bits(s[..., 2 * C:3 * C]), _bits(h)), what
                    assert torch.isnan(s[..., 3 * C:]).all(), what
                    # bf16 pair: the split of the plain output, K padding [C, pair_ld) exact zero
                    r_hi, r_lo = _split_bf16(p)
                    assert torch.equal(_bits(hi[..., :C]), _bits(r_hi)), what
                    assert torch.equal(_bits(lo[..., :C]), _bits(r_lo)), what
                    assert (_bits(hi[..., C:]) == 0).all() and (_bits(lo[..., C:]) == 0).all(), what
    print(f"inorm_apply C={C}: max err {worst:.2e} relative to max(1, |ref|) over 24 combinations")


# ------------------------------------------------------------------------------------------------ 6. resize into the concat

def _resize_ref(src, Ho, Wo):
    return F.interpolate(src.permute(0, 3, 1, 2).double(), (Ho, Wo), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)


def _resize_tol(src, Hs, Ws):
    # the sampling positions sh * oy, sw * ox are formed in fp32: each may move by an ulp of Hs (Ws), which moves the sample
    # by that fraction of the difference of two neighbours (<= 2 max|src|); plus the fp32 rounding of the blend
    return 2 ** -22 * (Hs + Ws + 4) * src.abs().max().item()


RESIZE_SHAPES = [
    (48, 64, 12, 16),       # down: H/2 -> H/8
    (6, 8, 12, 16),         # up: H/16 -> H/8
    (6, 8, 24, 32),         # up: H/16 -> H/4
    (12, 16, 12, 16),       # identity
    (9, 13, 1, 7),          # Ho == 1: scale 0 along y
    (9, 13, 5, 1),          # Wo == 1
    (1, 13, 6, 9),          # Hs == 1
    (50, 65, 12, 16), (25, 33, 12, 16), (13, 17, 12, 16), (7, 9, 12, 16),       # 100 x 130 at stride 8
    (45, 61, 22, 30), (12, 16, 22, 30),                                          # 90 x 122 at stride 4
]


@pytest.mark.parametrize("Hs,Ws,Ho,Wo", RESIZE_SHAPES)
def test_resize_split3(Hs, Ws, Ho, Wo):
    lib = L.load()
    torch.manual_seed(59)
    N, C, Ctot, c_off = 2, 96, 416, 64
    src = (torch.randn(N, Hs, Ws, C) * 3).to(DEV)
    dst = _nan(N, Ho, Wo, 3 * Ctot)
    L.check(lib.pips_resize_split3(L.ptr(src), N, Hs, Ws, C, L.ptr(dst), Ho, Wo, Ctot, c_off, _st()), "pips_resize_split3")
    torch.cuda.synchronize()
    d = dst.cpu()
    blocks = [d[..., b * Ctot + c_off:b * Ctot + c_off + C] for b in range(3)]
    mask = torch.ones(3 * Ctot, dtype=torch.bool)
    for b in range(3):
        mask[b * Ctot + c_off:b * Ctot + c_off + C] = False
    assert torch.isnan(d[..., mask]).all(), "a write outside the call's three slices"
    hi, lo = blocks[0], blocks[1]
    assert torch.equal(_bits(blocks[2]), _bits(hi))
    v = hi + lo                                                   # exact: lo holds the bits TF32 truncation removed
    assert torch.equal(_bits(_tf32_hi(v)), _bits(hi)) and torch.equal(_bits(v - hi), _bits(lo))
    ref = _resize_ref(src.cpu(), Ho, Wo)
    err = (v.double() - ref).abs().max().item()
    tol = _resize_tol(src, Hs, Ws)
    print(f"resize_split3 {Hs}x{Ws} -> {Ho}x{Wo}: max err {err:.2e} (tol {tol:.2e})")
    assert err <= tol


@pytest.mark.parametrize("Hs,Ws,Ho,Wo", RESIZE_SHAPES)
def test_resize_pair(Hs, Ws, Ho, Wo):
    lib = L.load()
    torch.manual_seed(61)
    N, C, Ctot, c_off = 2, 128, 448, 160
    src = (torch.randn(N, Hs, Ws, C) * 3).to(DEV)
    hi, lo = _nan(N, Ho, Wo, Ctot, dtype=torch.bfloat16), _nan(N, Ho, Wo, Ctot, dtype=torch.bfloat16)
    L.check(lib.pips_resize_pair(L.ptr(src), N, Hs, Ws, C, L.ptr(hi), L.ptr(lo), Ho, Wo, Ctot, c_off, _st()), "pips_resize_pair")
    torch.cuda.synchronize()
    bh, bl = _bits(hi), _bits(lo)
    for b in (bh, bl):                       # 160 channels remain after the slice: no padding is written
        assert (b[..., :c_off] == BF16_NAN).all() and (b[..., c_off + C:] == BF16_NAN).all()
    h, l = hi[..., c_off:c_off + C].float().cpu(), lo[..., c_off:c_off + C].float().cpu()
    ref = _resize_ref(src.cpu(), Ho, Wo)
    # hi = rn_bf16(v): lo is within half an ulp of hi, and hi + lo is v to 2^-17
    assert ((l.abs() <= h.abs() * 2 ** -8 + 1e-38)).all()
    err = ((h.double() + l.double()) - ref).abs().max().item()
    tol = _resize_tol(src, Hs, Ws) + 2 ** -17 * ref.abs().max().item()
    print(f"resize_pair {Hs}x{Ws} -> {Ho}x{Wo}: max err {err:.2e} (tol {tol:.2e})")
    assert err <= tol


@pytest.mark.parametrize("H8,W8", [(12, 16), (11, 15)])
def test_resize_pair_concat(H8, W8):
    """The four stage outputs of BasicEncoder into the 416-channel concat (row stride 448): every channel written, the
    K padding [416, 448) exact zero, and a slice that is not the last leaves the channels after it alone."""
    lib = L.load()
    torch.manual_seed(67)
    N, Ctot = 2, 448
    hi, lo = _nan(N, H8, W8, Ctot, dtype=torch.bfloat16), _nan(N, H8, W8, Ctot, dtype=torch.bfloat16)
    srcs = []
    c_off = 0
    for C, f in ((64, 4), (96, 2), (128, 1), (128, 0.5)):
        Hs, Ws = max(1, int(H8 * f)), max(1, int(W8 * f))
        src = torch.randn(N, Hs, Ws, C).to(DEV)
        srcs.append(src)
        L.check(lib.pips_resize_pair(L.ptr(src), N, Hs, Ws, C, L.ptr(hi), L.ptr(lo), H8, W8, Ctot, c_off, _st()), "pips_resize_pair")
        torch.cuda.synchronize()
        c_off += C
        if c_off < 416:
            assert (_bits(hi)[..., c_off:] == BF16_NAN).all() and (_bits(lo)[..., c_off:] == BF16_NAN).all(), c_off
    assert not torch.isnan(hi.float()).any() and not torch.isnan(lo.float()).any()
    assert (_bits(hi)[..., 416:] == 0).all() and (_bits(lo)[..., 416:] == 0).all()
    ref = torch.cat([_resize_ref(s.cpu(), H8, W8) for s in srcs], -1)
    err = ((hi[..., :416].double() + lo[..., :416].double()).cpu() - ref).abs().max().item()
    tol = max(_resize_tol(s, s.shape[1], s.shape[2]) for s in srcs) + 2 ** -17 * ref.abs().max().item()
    print(f"resize_pair concat {H8}x{W8}: max err {err:.2e} (tol {tol:.2e})")
    assert err <= tol


# ------------------------------------------------------------------------------------------------ 7. weight split

def _special_values():
    f = torch.tensor
    specials = f([0.0, -0.0, float("inf"), -float("inf"), float("nan"),
                  1e-40, -3e-39, 1.4e-45, -1.4e-45, 1.1754942e-38,               # subnormals, the largest one
                  3.3961e38, -3.3961e38, 3.4028235e38, 3.39e38,                   # round to +-Inf in bf16 / stay finite
                  1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -8 + 2 ** -20],   # ties to even, just above a tie
                 dtype=torch.float32)
    mags = torch.cat([torch.randn(64) * 10.0 ** e for e in range(-38, 38, 4)])
    return torch.cat([specials, mags.float()])


@pytest.mark.parametrize("n", [1, 255, 257, 10 ** 6 + 3])
def test_split_bf16(n):
    lib = L.load()
    torch.manual_seed(71)
    sp = _special_values()
    t = torch.randn(n) * torch.exp(torch.randn(n) * 8)
    k = min(n, sp.numel())
    t[torch.randperm(n)[:k]] = sp[:k] if n >= sp.numel() else sp[torch.randperm(sp.numel())[:k]]
    td = t.to(DEV)
    hi, lo = _nan(n, dtype=torch.bfloat16), _nan(n, dtype=torch.bfloat16)
    L.check(lib.pips_split_bf16(L.ptr(td), L.ptr(hi), L.ptr(lo), n, _st()), "pips_split_bf16")
    hi2, lo2 = _nan(n, dtype=torch.bfloat16), _nan(n, dtype=torch.bfloat16)
    L.check(lib.pips_split_bf16(L.ptr(td), L.ptr(hi2), None, n, _st()), "pips_split_bf16")
    torch.cuda.synchronize()
    r_hi = t.to(torch.bfloat16)
    r_lo = (t - r_hi.float()).to(torch.bfloat16)
    for got, ref in ((hi, r_hi), (lo, r_lo), (hi2, r_hi)):
        nan = torch.isnan(ref.float())
        assert torch.equal(torch.isnan(got.float().cpu()), nan)
        assert torch.equal(_bits(got)[~nan], _bits(ref)[~nan])
    assert (_bits(lo2) == BF16_NAN).all(), "lo = NULL must leave the lo buffer alone"


# ------------------------------------------------------------------------------------------------ 8. per-image independence

def _encoder(stride=8):
    from pips_b200 import Pips
    model = Pips(S=8, stride=stride).to(DEV).eval()
    model.load_state_dict(po.init_state_dict(seed=3), strict=True)
    return model


@pytest.mark.parametrize("H,W", [(384, 512), (100, 130)])
def test_fnet_tc_frames_are_independent(H, W):
    """Every kernel of the 'tc' encoder works per image: encoding any subset of the frames gives the same bits
    (sharding.encode_sharded relies on it)."""
    from pips_b200.encoder_fast import fnet_tc, fnet_tc_graphed
    model = _encoder()
    rgb = po.smooth_video(1, 8, H, W, seed=5)[0].to(DEV)
    rgb[2] = 255.0                                                  # one flat frame among textured ones
    with torch.no_grad():
        full = fnet_tc(model.fnet, rgb)
        for a, b in ((0, 1), (4, 5), (2, 5), (3, 8)):
            part = fnet_tc(model.fnet, rgb[a:b].contiguous())
            assert torch.equal(part, full[a:b]), (a, b)
        if H == 384:
            for a, b in ((0, 8), (1, 4), (0, 8)):
                assert torch.equal(fnet_tc_graphed(model.fnet, rgb[a:b].contiguous()), full[a:b]), ("graphed", a, b)


def test_conv_tc_partials_are_per_image():
    """The partial statistics rows of a 5-image batch are the single-image rows, bit for bit."""
    from pips_b200.encoder_fast import _Pair, _packed_weight
    lib = L.load()
    torch.manual_seed(73)
    N, H, W, cin, cout = 5, 45, 80, 64, 128
    conv = torch.nn.Conv2d(cin, cout, 3, stride=2, padding=1).to(DEV)
    x = torch.randn(N, H, W, cin, device=DEV) + 3.0
    pair = _Pair(N, H, W, cin, DEV)
    pair.hi.copy_(x.to(torch.bfloat16))
    pair.lo.copy_((x - pair.hi.float()).to(torch.bfloat16))
    w_hi, w_lo = _packed_weight(conv)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    chunks = lib.pips_conv_tc_chunks(H, W, 3, 3, 2, 2, 1, 1)

    def run(hi, lo, n):
        out, partial = _nan(n, Ho, Wo, cout), _nan(n, chunks, PARTIAL_ROWS, cout)
        L.check(lib.pips_conv_tc_stats(L.ptr(hi), L.ptr(lo), n, H, W, 64, L.ptr(w_hi), L.ptr(w_lo), cout, 3, 3, 2, 2, 1, 1, None,
                                       L.ptr(out), L.ptr(partial), _st()), "pips_conv_tc_stats")
        return out, partial

    out, partial = run(pair.hi, pair.lo, N)
    for i in range(N):
        o1, p1 = run(pair.hi[i:i + 1].contiguous(), pair.lo[i:i + 1].contiguous(), 1)
        torch.cuda.synchronize()
        assert torch.equal(_bits(o1), _bits(out[i:i + 1])), i
        assert torch.equal(_bits(p1), _bits(partial[i:i + 1])), i
    assert not torch.isnan(partial).any()


# ------------------------------------------------------------------------------------------------ 9. flat frames end to end

def _flat_clip(H, W):
    clip = torch.zeros(8, 3, H, W)
    clip[1] = 255.0
    clip[2] = 128.0
    clip[3] = torch.tensor([200.0, 30.0, 90.0]).view(3, 1, 1)
    clip[4] = 40.0
    clip[4, :, H // 3, W // 5] = 255.0                                          # one bright pixel
    clip[5] = torch.linspace(0, 255, W).round().view(1, 1, W)                   # horizontal ramp
    tex = po.smooth_video(1, 2, H, W, seed=9)[0]
    clip[6] = 90.0
    clip[6, :, :, W // 2:] = tex[0, :, :, W // 2:]                              # half flat, half textured
    clip[7] = tex[1]
    return clip


def _oracle(sd, rgb, stride, dtype):
    x = (2 * (rgb.to(DEV, dtype) / 255.0) - 1.0)
    sdd = {k: v.to(DEV, dtype) for k, v in sd.items()}
    with torch.no_grad(), torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        return torch.cat([po.fnet(sdd, x[i:i + 1], stride) for i in range(x.shape[0])]).double()


@pytest.mark.parametrize("H,W,frames", [(384, 512, slice(0, 8)), (720, 1280, slice(1, 2))])
def test_fnet_flat_frames(H, W, frames):
    """'tc' and 'fast' against the fp64 oracle on flat frames (black, white, grey, one colour, one bright pixel, a ramp,
    half flat): 1e-3 absolute, or 5x the fp32 oracle's own error where that is larger."""
    from pips_b200 import Pips
    sd = po.init_state_dict(seed=3)
    clip = _flat_clip(H, W)[frames]
    ref = _oracle(sd, clip, 8, torch.float64)
    e32 = (_oracle(sd, clip, 8, torch.float32) - ref).abs().flatten(1).amax(1).cpu()
    bound = torch.where(e32 > 1e-3, 5 * e32, torch.full_like(e32, 1e-3))
    for mode in ("tc", "fast"):
        model = Pips(S=8, stride=8, fnet_mode=mode).to(DEV).eval()
        model.load_state_dict(sd, strict=True)
        with torch.no_grad():
            f = model.encode(clip.unsqueeze(0).to(DEV))[0].double()
        err = (f - ref).abs().flatten(1).amax(1).cpu()
        print(f"fnet {mode} {H}x{W} flat frames: max|err| per frame {[f'{e:.1e}' for e in err.tolist()]}; "
              f"fp32 oracle {[f'{e:.1e}' for e in e32.tolist()]}")
        assert (err <= bound).all(), (mode, err.tolist(), bound.tolist())
        del model
