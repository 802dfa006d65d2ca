"""Per-kernel parity of the refinement loop's CUDA entry points (csrc/pyramid.cu, corr_gather.cu, heatmap.cu,
mixer_simt.cu, tokenmix_tc.cu, peer.cu and the mixer / iteration operators of abi.cu) against fp64 torch references on
the host.

The references restate the reference model's algorithm, not the kernels': the all-pairs correlation volume sampled with
grid_sample(align_corners=True), F.interpolate(align_corners=True) for the score maps, the oracle's mixer with the
weights in float64.  A bf16 pyramid is compared in fp64 on its bf16-rounded values.

Output buffers are poisoned with NaN before every call, so a test sees exactly which elements a kernel wrote.  Layouts,
copies and hi/lo splits are compared bit for bit.  Sums are compared per element against a bound c * 2^-24 * sum|terms|
computed in fp64 (the size of what was added up), and every test prints its measured error as a multiple of that unit.
The constants c are the largest ratio measured on an H100 80GB HBM3 with a margin of about 2-4x."""
import ctypes as C
import math
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import _lib as L
from pips_b200 import engine, torch_path

DEV = "cuda:0"
U = 2.0 ** -24                                # fp32 unit roundoff
S = 8
TD = "delta_block.to_delta"

# Bounds, in units of U * sum|terms| unless stated otherwise.
C_INIT = 8.0          # init_gather (measured 2.7): 4 weights of 2 products each, a 4-term sum
C_CORR = 1.5          # corr_gather (measured 0.43): 128-term dot, / sqrt(C), 4-weight blend
E_EMB = 2.5e-7        # corr_gather embedding, absolute (measured 8.2e-8): accurate sincosf of the fp32 product vs fp64
C_HEAT = 3.0          # pips_heatmap (measured 0.7): 128-term dot, scale, 4 levels x 4 taps, fp32 source positions
C_TM_F32 = 6.0        # pips_tokenmix, CUDA-core fp32 kernel (measured 1.6): LayerNorms, two contractions, residual
C_TM_TC = 128.0       # wgmma token mixing, x (measured 38): each bf16x3 product carries ~2^-16 relative error
C_TM_Y = 128.0        # its LN2 output as hi + lo (measured 42): the 2^-17 split alone can be 128 units of |y|
C_POOL = 12.0         # pips_ln_pool fp32 output (measured 3.5)
C_UPD = 12.0          # pips_update ffeats (measured 3.2): GroupNorm(1,128), 128-term dot, exact GELU, residual
C_VIS = 2.5           # pips_vis_head (measured 0.61): 128-term dot
# pips_mixer_forward, max|delta - ref| / max|ref| against the fp64 oracle mixer (12 DeltaBlock layers, head_scale 1).
# bf16x3 operands carry 2^-17 relative error each, so ~1e-5 is its floor; bf16 does not meet 1e-3 px and is bounded loosely.
MIXER_REL = {"fp32": 4e-6, "bf16x3": 5e-5, "bf16": 2e-2}
# one pips_refine_iter: max error of out_px in px (stride 8), and of ffeats relative to max|ffeats|
REFINE_PX = {"fp32": 4e-5, "bf16x3": 2.5e-4, "bf16": 0.1}
REFINE_FF = {"fp32": 2e-6, "bf16x3": 2e-5, "bf16": 1e-2}


def _st():
    return torch.cuda.current_stream().cuda_stream


def _windows(cases, other, windows):
    """pytest params (*case, S): `cases` at S = 8 under their plain ids, `other` at each of the other window lengths"""
    tup = lambda c: c if isinstance(c, tuple) else (c,)
    name = lambda c: "-".join(map(str, tup(c)))
    return ([pytest.param(*tup(c), S, id=name(c)) for c in cases]
            + [pytest.param(*tup(c), s, id=f"{name(c)}-S{s}") for s in windows for c in other])


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32).cpu()


def _split_bf16(t):
    """The (hi, lo) pair the kernels write: hi = rn_bf16(v), lo = rn_bf16(v - hi)."""
    hi = t.to(torch.bfloat16)
    return hi, (t - hi.float()).to(torch.bfloat16)


def _ratio(got, ref, mag):
    """max |got - ref| / (U * mag) over all elements; got / ref / mag on the host."""
    err = (got.double().cpu() - ref.double().cpu()).abs()
    return (err / (U * mag.double().cpu() + 1e-300)).max().item()


def _report(name, value, bound):
    print(f"{name}: {value:.3g} (bound {bound:.3g})")
    assert value <= bound, f"{name}: {value:.3g} > {bound:.3g}"


def _pyramid(fmaps, nhwc=False):
    """fmaps (frames, 128, H, W) fp32 on the host -> the 4 device levels (fp32, bf16), NaN-poisoned before the call."""
    lib = L.load()
    frames, _, H, W = fmaps.shape
    f32, bf = [], []
    h, w = H, W
    for _ in range(L.LEVELS):
        f32.append(_nan(frames, h, w, 128))
        bf.append(_nan(frames, h, w, 128, dtype=torch.bfloat16))
        h, w = h // 2, w // 2
    if nhwc:
        src = fmaps.permute(0, 2, 3, 1).contiguous().to(DEV)
        L.check(lib.pips_pyramid_build_nhwc(L.ptr(src), frames, H, W, L.ptr_array(f32), L.ptr_array(bf), _st()))
    else:
        src = fmaps.contiguous().to(DEV)
        L.check(lib.pips_pyramid_build(L.ptr(src), frames, H, W, L.ptr_array(f32), L.ptr_array(bf), _st()))
    torch.cuda.synchronize()
    return f32, bf


def _host_levels(lv):
    """Device levels (frames, h, w, 128) as fp64 host tensors: exactly the values the kernels read."""
    return [t.cpu().double() for t in lv]


# ------------------------------------------------------------------------------------------------ 1. pyramid, initial gather

@pytest.mark.gpu
@pytest.mark.parametrize("nhwc", [False, True])
@pytest.mark.parametrize("H,W", [(8, 8), (9, 80), (15, 9), (45, 8), (8, 15)])
def test_pyramid_levels_bit_exact(H, W, nhwc):
    """Level 3 is a single pixel (or a single row / column) for every map here."""
    torch.manual_seed(101)
    fm = torch.randn(3, 128, H, W)
    f32, bf = _pyramid(fm, nhwc)
    ref = fm
    for l in range(L.LEVELS):
        if l:
            ref = F.avg_pool2d(ref, 2, stride=2)
        r = ref.permute(0, 2, 3, 1).contiguous()
        assert f32[l].shape == r.shape, (l, f32[l].shape, r.shape)
        assert torch.equal(_bits(f32[l]), _bits(r)), f"level {l} (fp32) differs from avg_pool2d"
        assert torch.equal(_bits(bf[l]), _bits(r.to(torch.bfloat16))), f"level {l} (bf16) differs"


def _frame_base(B, N, T, seed):
    g = torch.Generator().manual_seed(seed)
    fb = torch.randint(0, T + 4, (B, N), generator=g, dtype=torch.int32)
    fb.view(-1)[:4] = torch.tensor([0, T - 1, T, T + 7], dtype=torch.int32)      # clip end, past the clip end
    return fb


@pytest.mark.gpu
@pytest.mark.parametrize("T", [3, 13])
def test_init_gather_chained(T):
    """pips_init_gather with frame_base: track (b, n) samples frame b*T + min(frame_base, T-1) at its frame-0 query
    (utils/samp.py: indices clamped, weights not), and broadcasts the row over the S rows of ffeats."""
    _check_init_gather(T, chained=True)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [2, 5, 16])
def test_init_gather_window(S):
    """pips_init_gather without frame_base: track (b, n) samples frame b*S of a pyramid of B*S frames."""
    _check_init_gather(S, chained=False, S=S)


def _check_init_gather(T, chained, S=S):
    lib = L.load()
    torch.manual_seed(102)
    B, N, H, W = 2, 24, 11, 19
    fm = torch.randn(B * T, 128, H, W)
    f32, _ = _pyramid(fm)
    fb = _frame_base(B, N, T, 103) if chained else torch.zeros(B, N, dtype=torch.int32)
    coords = torch.rand(B, S, N, 2) * torch.tensor([W + 6.0, H + 6.0]) - 3.0
    c0 = coords[:, 0].reshape(-1, 2)
    c0[:6] = torch.tensor([[W - 1.0, H - 1.0], [0.0, 0.0], [W - 1.0, 2.0], [3.0, H - 1.0], [-0.5, H - 0.5], [W + 2.25, -2.75]])
    c0[6:8] = torch.tensor([[5.0, 7.0], [W - 1.5, H - 1.5]])
    coords[:, 0] = c0.reshape(B, N, 2)
    ffeat, ffeats = _nan(B * N + 1, 128), _nan(B * N + 1, S, 128)           # one row past the end stays NaN
    cd = coords.to(DEV).contiguous()
    fbd = fb.to(DEV).contiguous() if chained else None
    L.check(lib.pips_init_gather(L.ptr(f32[0]), B, S, N, H, W, L.ptr(cd), L.ptr(fbd), T if chained else 0, L.ptr(ffeat),
                                 L.ptr(ffeats), _st()))
    torch.cuda.synchronize()
    frame = (torch.arange(B).view(B, 1) * T + fb.clamp(max=T - 1)).reshape(-1).long()
    img = f32[0].cpu().double()[frame].permute(0, 3, 1, 2)                    # (B*N, 128, H, W): each track's frame
    x = coords[:, 0, :, 0].reshape(-1, 1).double()
    y = coords[:, 0, :, 1].reshape(-1, 1).double()
    ref = torch_path.sample_clamped(img, x, y)[:, 0]
    mag = torch_path.sample_clamped(img.abs(), x, y)[:, 0]                    # weights are >= 0
    got = ffeat[:B * N].cpu()
    tag = f"T={T}" if chained else f"S={S}"
    _report(f"init_gather {tag}: err / (U sum|terms|)", _ratio(got, ref, mag), C_INIT)
    assert torch.isnan(ffeat[B * N]).all() and torch.isnan(ffeats[B * N]).all()
    assert torch.equal(_bits(ffeats[:B * N]), _bits(got.unsqueeze(1).expand(-1, S, -1)))


# ------------------------------------------------------------------------------------------------ 2./3. corr_gather

def _allpairs(levels, fidx, q):
    """fp64 all-pairs volumes (nets/pips.py:384-398) of each unit's query q (B,S,N,C) against its own frame fidx
    (B,S,N): per level (B,S,N,h,w), and the same with |q| and |f| (the magnitudes of the summed terms)."""
    B, S_, N, C_ = q.shape
    vols, mags = [], []
    for f in levels:
        fr, h, w, _ = f.shape
        flat = f.reshape(fr, h * w, C_)
        v = torch.zeros(B, S_, N, h * w, dtype=torch.float64)
        a = torch.zeros_like(v)
        for i in fidx.unique().tolist():
            m = fidx == i
            v[m] = q[m] @ flat[i].t()
            a[m] = q[m].abs() @ flat[i].abs().t()
        vols.append(v.reshape(B, S_, N, h, w) / math.sqrt(C_))
        mags.append(a.reshape(B, S_, N, h, w) / math.sqrt(C_))
    return vols, mags


def _embed_ref(coords, times):
    """The motion embedding (utils/misc.py:44-69) of the fp32 flows: fp64 sin / cos of the fp32 product flow * div, as the
    reference computes it in fp32.  coords (B,S,N,2) fp32 -> (B*N, S, 195) fp64 and the (B*N, S, 3) fp32 flows."""
    B, S_, N, _ = coords.shape
    flow = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S_, 2)
    flow = torch.cat([flow, times.view(1, S_, 1).expand(B * N, -1, -1)], 2)            # fp32
    div = torch.arange(0, 64, 2, dtype=torch.float32) * (1000.0 / 64)
    parts = []
    for a in range(3):
        v = (flow[:, :, a:a + 1] * div).double()                                     # the fp32 product
        parts.append(torch.stack([v.sin(), v.cos()], -1).reshape(B * N, S_, 64))
    return torch.cat(parts + [flow.double()], 2), flow


def _pad_pow2(v):
    """Zero-pad a volume (..., h, w) to (2^a + 1, 2^b + 1) pixels.  Outside the map this is grid_sample's own zero
    padding, so the samples do not change; but with (size - 1) a power of two grid_sample's normalisation of the
    coordinates round-trips exactly (no spurious 1e-16 weight on a pixel a tap only touches), and a level that is a
    single pixel wide stays defined (size - 1 = 0 divides by zero)."""
    h, w = v.shape[-2:]
    return F.pad(v, (0, (1 << (w - 1).bit_length()) + 1 - w, 0, (1 << (h - 1).bit_length()) + 1 - h))


def _corr_ref(levels, fidx, coords, q):
    """fp64 CorrBlock.sample of the all-pairs volumes at coords: (B*N*S, 196) in mixer row order, and the bound's
    magnitude: sum|terms| plus the |terms| of all four corners of each tap, unweighted.  The second part covers the
    fp32 rounding of the tap's fractional position (x - floor(x) rounds for -1 < x < 0), which moves a weight by up
    to U."""
    B, S_, N, _ = coords.shape
    vols, mags = _allpairs(levels, fidx, q)
    vols, mags = [_pad_pow2(v) for v in vols], [_pad_pow2(a) for a in mags]
    c = coords.double().clamp(-1e4, 1e4)                 # grid_sample of +-inf is NaN; 1e4 px is as far outside
    ref = po.sample_allpairs(vols, c)
    mag = po.sample_allpairs(mags, c)                    # bilinear weights are >= 0
    # 4 x the bilinear sample at the centre of a tap's pixel square = the sum over its 4 corners
    box = torch.cat([4 * po.sample_allpairs([a], torch.floor(c / 2 ** l) + 0.5) for l, a in enumerate(mags)], -1)
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(B * N * S_, -1)
    return rows(ref), rows(mag + box)


def _special_coords(H, W):
    """Level-0 coordinates that sit on the edges of every level l (in level-l pixels, times 2^l): integers, the last
    pixel, half a pixel outside, the strip where only the outermost tap reaches the map, either side of the kernel's
    +-8 px clamp; then diverged tracks at +-1e9 and +-inf."""
    pts = []
    g = torch.Generator().manual_seed(7)
    for l in range(L.LEVELS):
        hl, wl, sc = H >> l, W >> l, float(1 << l)
        xs = [0.0, 1.0, wl - 1.0, -0.5, wl - 0.5, -3.5, -3.25, -7.75, -8.25, wl + 7.75, wl + 8.25]
        ys = [0.0, 1.0, hl - 1.0, -0.5, hl - 0.5, -3.5, -3.75, -7.75, -8.25, hl + 7.75, hl + 8.25]
        for x, y in zip(xs, ys):
            mx, my = (torch.rand(2, generator=g) * torch.tensor([W - 1.0, H - 1.0])).tolist()
            pts += [(x * sc, my), (mx, y * sc), (x * sc, y * sc)]
    far = [(1e9, 3.0), (-1e9, 2.0), (4.0, 1e9), (float("inf"), 1.0), (2.0, float("-inf")), (float("-inf"), float("inf"))]
    return torch.tensor(pts, dtype=torch.float32), torch.tensor(far, dtype=torch.float32)


def _corr_gather(lv, feat, B, N, H, W, coords, ff_rows, times, fb=None, T=0, outs=("f32",), ldx=576, S=S):
    """One pips_corr_gather call into NaN-filled buffers with one unit's rows of slack; returns {name: (M+8, ldx)}."""
    lib = L.load()
    M = B * N * S
    buf = {"f32": _nan(M + 8, ldx) if "f32" in outs else None,
           "hi": _nan(M + 8, ldx, dtype=torch.bfloat16) if "hi" in outs else None,
           "lo": _nan(M + 8, ldx, dtype=torch.bfloat16) if "lo" in outs else None}
    cd, fd, td = coords.to(DEV).contiguous(), ff_rows.to(DEV).contiguous(), times.to(DEV)
    fbd = None if fb is None else fb.to(DEV).contiguous()
    L.check(lib.pips_corr_gather(L.ptr_array(lv), L.FEAT_DTYPES[feat], B, S, N, H, W, L.ptr(cd), L.ptr(fd), L.ptr(td),
                                 L.ptr(fbd), T, L.ptr(buf["hi"]), L.ptr(buf["lo"]), L.ptr(buf["f32"]), ldx, _st()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in buf.items() if v is not None}


def _same(a, b):
    """Bitwise equal where finite, both NaN elsewhere (the bf16 NaN pattern of a conversion is not fixed)."""
    a, b = a.float(), b.float()
    fin = torch.isfinite(a) | torch.isfinite(b)
    return torch.equal(a[fin].view(torch.int32), b[fin].view(torch.int32)) and torch.equal(torch.isnan(a), torch.isnan(b))


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["fp32", "bf16"])
@pytest.mark.parametrize("H,W,ldx,S", _windows([(8, 8, 576), (9, 40, 584), (15, 8, 640), (45, 80, 576)],
                                               [(9, 40, 584), (45, 80, 576)], [2, 5, 9, 16]))
def test_corr_gather_against_allpairs(feat, H, W, ldx, S):
    """Other window lengths at N = 37: B*S*N is no multiple of a CTA's 8 warps, and at S = 16 it exceeds the warps of
    the persistent grid (8 per SM), so warps take a second unit."""
    B, N = 2, 12 if S == 8 else 37
    torch.manual_seed(104)
    f32, bf = _pyramid(torch.randn(B * S, 128, H, W))
    lv = bf if feat == "bf16" else f32
    coords = torch.rand(B, S, N, 2) * torch.tensor([W + 4.0, H + 4.0]) - 2.0
    pts, far = _special_coords(H, W)
    flat = coords.view(-1, 2)
    flat[:len(pts)] = pts
    flat[-len(far):] = far
    ff_rows = torch.randn(B * N, S, 128)
    times = po.times_axis(S)
    out = _corr_gather(lv, feat, B, N, H, W, coords, ff_rows, times, outs=("f32",), ldx=ldx, S=S)["f32"]
    pair = _corr_gather(lv, feat, B, N, H, W, coords, ff_rows, times, outs=("hi", "lo"), ldx=ldx, S=S)
    plain = _corr_gather(lv, feat, B, N, H, W, coords, ff_rows, times, outs=("hi",), ldx=ldx, S=S)["hi"]
    M = B * N * S
    assert torch.isnan(out[M:]).all() and torch.isnan(pair["hi"][M:]).all() and torch.isnan(pair["lo"][M:]).all()
    x = out[:M]
    assert torch.equal(_bits(x[:, 519:576]), torch.zeros(M, 57, dtype=torch.int32)), "K padding is not exact zero"
    assert torch.isnan(x[:, 576:]).all(), "columns past 576 of the row stride were written"
    assert torch.equal(_bits(x[:, :128]), _bits(ff_rows.reshape(M, 128))), "feature copy differs"

    fidx = (torch.arange(B).view(B, 1, 1) * S + torch.arange(S).view(1, S, 1)).expand(B, S, N)
    q = ff_rows.reshape(B, N, S, 128).permute(0, 2, 1, 3).double()
    ref, mag = _corr_ref(_host_levels(lv), fidx, coords, q)
    diverged = (coords.abs() >= 1e9).any(-1).permute(0, 2, 1).reshape(M)
    assert (x[diverged, 128:324] == 0).all(), "a diverged track's correlation is not exactly 0"
    r = _ratio(x[:, 128:324], ref, mag)
    tag = f"corr_gather {feat} {H}x{W}" + ("" if S == 8 else f" S={S}")
    _report(f"{tag}: corr err / (U sum|terms|)", r, C_CORR)

    emb, flow = _embed_ref(coords, times)
    flow = flow.reshape(M, 3)
    ok = torch.isfinite(flow).all(-1)
    e_emb = (x[ok, 324:516].double() - emb.reshape(M, 195)[ok, :192]).abs().max().item()
    _report(f"{tag}: embedding abs err", e_emb, E_EMB)
    assert _same(x[:, 516:519], flow), "flow / time columns differ"

    hi, lo = _split_bf16(x[:, :576])
    assert _same(pair["hi"][:M, :576], hi) and _same(pair["lo"][:M, :576], lo), "bf16 pair is not the split of the fp32 row"
    assert _same(plain[:M, :576], hi), "plain bf16 row is not rn_bf16 of the fp32 row"
    assert torch.isnan(pair["hi"][:M, 576:].float()).all() and torch.isnan(pair["lo"][:M, 576:].float()).all()
    assert torch.isnan(plain[:, 576:].float()).all()


def _chained_case(B, N, H, W, T, seed, S=S):
    torch.manual_seed(seed)
    fm = torch.randn(B * T, 128, H, W)
    fb = _frame_base(B, N, T, seed + 1)
    coords = torch.rand(B, S, N, 2) * torch.tensor([W + 6.0, H + 6.0]) - 3.0
    ff_rows = torch.randn(B * N, S, 128)
    # the window of track (b, n) is frames min(frame_base + s, T-1) of clip b
    fidx = torch.arange(B).view(B, 1, 1) * T + (fb.view(B, 1, N) + torch.arange(S).view(1, S, 1)).clamp(max=T - 1)
    return fm, fb, coords, ff_rows, fidx


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["fp32", "bf16"])
@pytest.mark.parametrize("T", [3, 13, 20])
def test_corr_gather_chained(feat, T):
    """frame_base / frames_per_batch with B = 2: a wrong batch stride reads another clip's frames."""
    B, N, H, W = 2, 10, 16, 24
    fm, fb, coords, ff_rows, fidx = _chained_case(B, N, H, W, T, 105 + T)
    f32, bf = _pyramid(fm)
    lv = bf if feat == "bf16" else f32
    times = po.times_axis(S)
    x = _corr_gather(lv, feat, B, N, H, W, coords, ff_rows, times, fb=fb, T=T)["f32"]
    M = B * N * S
    assert torch.isnan(x[M:]).all()
    assert torch.equal(_bits(x[:M, :128]), _bits(ff_rows.reshape(M, 128)))
    q = ff_rows.reshape(B, N, S, 128).permute(0, 2, 1, 3).double()
    ref, mag = _corr_ref(_host_levels(lv), fidx, coords, q)
    _report(f"corr_gather chained {feat} T={T}: corr err / (U sum|terms|)", _ratio(x[:M, 128:324], ref, mag), C_CORR)
    emb, _ = _embed_ref(coords, times)
    e_emb = (x[:M, 324:516].double() - emb.reshape(M, 195)[:, :192]).abs().max().item()
    _report(f"corr_gather chained {feat} T={T}: embedding abs err", e_emb, E_EMB)


def _module(sd):
    """What PackedWeights reads from a module: its state dict, here on the device."""
    dev = {k: v.to(DEV).contiguous() for k, v in sd.items()}
    return types.SimpleNamespace(state_dict=lambda: dev)


def _update_ref(sd64, delta, coords, coords0, ff_rows):
    """nets/pips.py:525-536 in fp64: delta (B*N, S, 130) -> new coords (B,S,N,2) and ffeats rows (B*N, S, 128)."""
    B, S, N, _ = coords.shape
    dfeat = delta[:, :, 2:].reshape(-1, 128)
    g = F.group_norm(dfeat, 1, sd64["norm.weight"], sd64["norm.bias"], 1e-5)
    ff = F.gelu(F.linear(g, sd64["ffeat_updater.0.weight"], sd64["ffeat_updater.0.bias"])) + ff_rows.double().reshape(-1, 128)
    c = coords.double() + delta[:, :, :2].reshape(B, N, S, 2).permute(0, 2, 1, 3)
    c[:, 0] = coords0[:, 0].double()
    return c, ff.reshape(B * N, S, 128)


@pytest.mark.gpu
@pytest.mark.parametrize("precision,S", _windows(["fp32", "bf16x3", "bf16"], ["fp32", "bf16x3", "bf16"], [5, 16]))
def test_refine_iter_chained(precision, S):
    """One pips_refine_iter on chained windows against the loop body (nets/pips.py:499-536) in fp64 on the same
    frames min(frame_base + s, T-1): all-pairs correlation, embedding, the oracle mixer, the state update."""
    lib = L.load()
    B, N, H, W, T, stride = 2, 10, 16, 24, 13, 8.0
    fm, fb, coords, ff_rows, fidx = _chained_case(B, N, H, W, T, 106, S=S)
    coords = torch.rand(B, S, N, 2) * torch.tensor([W - 1.0, H - 1.0])
    coords0 = coords.clone()
    coords0[:, 0] += 0.25                                      # the frame-0 lock must restore coords0, not keep coords
    f32, _ = _pyramid(fm)
    sd = po.init_state_dict(seed=5, head_scale=1.0, S=S)
    w = engine.PackedWeights(_module(sd), _st())
    prec = L.PRECISIONS[precision]
    ws = engine.Workspace(B * N, prec, DEV, S=S)
    times = po.times_axis(S).to(DEV)
    cd, c0d = coords.to(DEV).contiguous(), coords0.to(DEV).contiguous()
    fd, fbd = ff_rows.to(DEV).contiguous(), fb.to(DEV).contiguous()
    prob = L.Problem()
    prob.B, prob.S, prob.N, prob.H, prob.W = B, S, N, H, W
    prob.feat_dtype, prob.precision = L.FEAT_F32, prec
    for i in range(L.LEVELS):
        prob.lvl[i] = L.ptr(f32[i])
    prob.times, prob.coords, prob.coords0, prob.ffeats = L.ptr(times), L.ptr(cd), L.ptr(c0d), L.ptr(fd)
    prob.stride, prob.frame_base, prob.frames_per_batch = stride, L.ptr(fbd), T
    out = _nan(B, S, N, 2)
    L.check(lib.pips_refine_iter(C.byref(prob), C.byref(w.c), C.byref(ws.c), L.ptr(out), _st()), "pips_refine_iter")
    torch.cuda.synchronize()

    sd64 = {k: v.double() for k, v in sd.items()}
    q = ff_rows.reshape(B, N, S, 128).permute(0, 2, 1, 3).double()
    corr, _ = _corr_ref(_host_levels(f32), fidx, coords, q)
    emb, _ = _embed_ref(coords, po.times_axis(S))
    x0 = torch.cat([ff_rows.double(), corr.reshape(B * N, S, 196), emb], 2)
    delta = po.mixer(sd64, x0).reshape(B * N, S, 130)
    c_ref, ff_ref = _update_ref(sd64, delta, coords, coords0, ff_rows)
    e_px = (out.cpu().double() - c_ref * stride).abs().max().item()
    e_ff = (fd.cpu().double() - ff_ref).abs().max().item() / ff_ref.abs().max().item()
    assert torch.equal(_bits(cd), _bits(out / stride)), "coords state and out_px disagree"
    assert torch.equal(_bits(cd[:, 0]), _bits(coords0[:, 0].to(DEV))), "frame 0 is not re-locked to coords0"
    tag = f"refine_iter chained {precision}" + ("" if S == 8 else f" S={S}")
    print(f"{tag}: max|dpos| {e_px:.3g} px (|delta| max {delta[..., :2].abs().max().item():.3g} px), ffeats rel err {e_ff:.3g}")
    _report(f"{tag}: out_px err (px)", e_px, REFINE_PX[precision])
    _report(f"{tag}: ffeats rel err", e_ff, REFINE_FF[precision])


# ------------------------------------------------------------------------------------------------ 4. heat map

def _heat_ref(levels, q, H8, W8):
    """fp64 nets/pips.py:504-511: sum over levels of F.interpolate(all-pairs volume, align_corners=True).  q (B,S,J,C).
    The bound's magnitude weights each level by (1 + source x + source y): the kernel, like ATen in fp32, forms the
    source position dst * (in-1)/(out-1) in fp32, which moves a sample by up to ~2 U * position."""
    B, S_, J, _ = q.shape
    fidx = (torch.arange(B).view(B, 1, 1) * S_ + torch.arange(S_).view(1, S_, 1)).expand(B, S_, J)
    vols, mags = _allpairs(levels, fidx, q)
    ref = torch.zeros(B * S_, J, H8, W8, dtype=torch.float64)
    mag = torch.zeros_like(ref)
    up = lambda t: F.interpolate(t.reshape(B * S_, J, *t.shape[-2:]), (H8, W8), mode="bilinear", align_corners=True)
    for v, a in zip(vols, mags):
        h, w = v.shape[-2:]
        sy = torch.arange(H8, dtype=torch.float64).view(H8, 1) * ((h - 1) / max(H8 - 1, 1))
        sx = torch.arange(W8, dtype=torch.float64).view(1, W8) * ((w - 1) / max(W8 - 1, 1))
        ref += up(v)
        mag += up(a) * (1 + sx + sy)
    return ref, mag


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["fp32", "bf16"])
@pytest.mark.parametrize("n_sel", [1, 33, 70])
@pytest.mark.parametrize("H8,W8,S", _windows([(8, 8), (9, 15), (45, 80)], [(9, 15), (45, 80)], [2, 5, 12]))
def test_heatmap_against_allpairs(H8, W8, S, n_sel, feat):
    """n_sel 33 and 70 need two and three heat_corr launches.  Selections repeat and are unsorted.  n_sel 1: identity
    slots with a gap between frames; 33: a slot map with unused slots; 70: both."""
    lib = L.load()
    B, N = 2, 20
    torch.manual_seed(107 + n_sel)
    f32, bf = _pyramid(torch.randn(B * S, 128, H8, W8))
    lv = bf if feat == "bf16" else f32
    ffeats = torch.randn(B * N, S, 128)
    sel = torch.tensor([N - 1]) if n_sel == 1 else torch.randint(0, N, (n_sel,))
    P = H8 * W8
    if n_sel == 1:
        slot, n_slots, stride = None, 1, P + 37
    else:
        n_slots = n_sel + 11
        slot = torch.randperm(n_slots)[:n_sel]
        stride = n_slots * P + (5 if n_sel == 70 else 0)
    out = _nan(B * S * stride + 64)
    scratch = _nan(lib.pips_heatmap_scratch_floats(B * S, n_sel, H8, W8))
    seld = sel.to(torch.int32).to(DEV)
    slotd = None if slot is None else slot.to(torch.int32).to(DEV)
    fd = ffeats.to(DEV).contiguous()
    L.check(lib.pips_heatmap(L.ptr_array(lv), L.FEAT_DTYPES[feat], B, S, N, H8, W8, L.ptr(fd), L.ptr(seld), L.ptr(slotd),
                             n_sel, L.ptr(scratch), L.ptr(out), stride, _st()), "pips_heatmap")
    torch.cuda.synchronize()
    q = ffeats.reshape(B, N, S, 128)[:, sel].permute(0, 2, 1, 3).double()          # (B, S, n_sel, 128)
    ref, mag = _heat_ref(_host_levels(lv), q, H8, W8)
    got = out.cpu()
    frames = got[:B * S * stride].view(B * S, stride)
    slots = torch.arange(n_sel) if slot is None else slot
    live = torch.zeros(B * S, stride, dtype=torch.bool)
    for j in range(n_sel):
        live[:, slots[j] * P:(slots[j] + 1) * P] = True
    assert torch.isnan(frames[~live]).all(), "unused slots / the gap between frames were written"
    assert torch.isnan(got[B * S * stride:]).all()
    g = frames[:, :n_slots * P].reshape(B * S, n_slots, H8, W8)[:, slots]
    tag = f"heatmap {feat} {H8}x{W8} n_sel={n_sel}" + ("" if S == 8 else f" S={S}")
    _report(f"{tag}: err / (U sum|terms|)", _ratio(g, ref, mag), C_HEAT)


# ------------------------------------------------------------------------------------------------ 5. token mixing, pooling

def _layer(sd, l=4):
    p = f"{TD}.{l}"
    return {"ln1_w": sd[p + ".0.norm.weight"], "ln1_b": sd[p + ".0.norm.bias"], "w1": sd[p + ".0.fn.0.weight"][:, :, 0],
            "b1": sd[p + ".0.fn.0.bias"], "w2": sd[p + ".0.fn.3.weight"][:, :, 0], "b2": sd[p + ".0.fn.3.bias"],
            "ln2_w": sd[p + ".1.norm.weight"], "ln2_b": sd[p + ".1.norm.bias"],
            "out_w": sd[f"{TD}.13.weight"], "out_b": sd[f"{TD}.13.bias"]}


def _ln_mag(x, w, b):
    """Magnitude of the terms of LayerNorm(x) (fp64): (|x| + |mean|) * rstd * |w| + |b|."""
    m = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-5)
    return (x.abs() + m.abs()) * rstd * w.abs() + b.abs(), rstd


def _tokenmix_ref(x, lw):
    """fp64 nets/pips.py:117 + the LayerNorm of :118; x (seqs, 8, 512).  Returns x_new, y, and the term magnitudes."""
    w = {k: v.double() for k, v in lw.items()}
    y = po._ln(x, w["ln1_w"], w["ln1_b"])
    h = F.gelu(torch.einsum("js,rsc->rjc", w["w1"], y) + w["b1"].view(1, -1, 1))
    z = torch.einsum("sj,rjc->rsc", w["w2"], h) + w["b2"].view(1, -1, 1)
    ymag, _ = _ln_mag(x, w["ln1_w"], w["ln1_b"])
    hmag = torch.einsum("js,rsc->rjc", w["w1"].abs(), ymag) + w["b1"].abs().view(1, -1, 1)
    zmag = torch.einsum("sj,rjc->rsc", w["w2"].abs(), hmag) + w["b2"].abs().view(1, -1, 1)
    xn = x + z
    xmag = x.abs() + zmag
    y2 = po._ln(xn, w["ln2_w"], w["ln2_b"])
    _, rstd2 = _ln_mag(xn, w["ln2_w"], w["ln2_b"])
    y2mag = y2.abs() + rstd2 * w["ln2_w"].abs() * (xmag + xn.abs().mean(-1, keepdim=True))
    return xn, y2, xmag, y2mag


def _tokenmix_inputs(seqs, offset, seed, S=S):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(seqs, S, 512, generator=g)
    if offset:
        x = x + 100.0 + 20.0 * torch.randn(seqs, S, 1, generator=g)              # mean ~1e2, spread ~1
    return x


def _tokenmix_seqs(S=S):
    """1, 37, one track more than the wgmma kernel's persistent grid (its next-track prefetch and residual loop), 700.
    The grid is 4 CTAs per SM at S = 8, 3 at S < 8 (the frame guards need more registers) and 1 above 8 (two
    warpgroups)."""
    per_sm = 4 if S == 8 else 3 if S < 8 else 1
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    return [1, 37, per_sm * sms + 1, 700]


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("which,S", _windows(range(4), range(4), [2, 5, 9, 16]))
def test_tokenmix_outputs(which, S, offset):
    """pips_tokenmix as (hi, lo) [bf16x3: the wgmma kernel], (hi, NULL) [bf16: the wgmma kernel], f32 [the CUDA-core
    kernel], and pips_tokenmix_tc itself; x is updated in place.  A sequence past the end stays NaN.  Other window
    lengths go through pips_tokenmix_s and pips_tokenmix_tc_s: P = 8 padded below 8, P = 16 above."""
    lib = L.load()
    seqs = _tokenmix_seqs(S)[which]
    sd = po.init_state_dict(3, S=S)
    lw = _layer(sd)
    x = _tokenmix_inputs(seqs, offset, 108 + seqs, S=S)
    d = {k: v.to(DEV).contiguous() for k, v in lw.items()}
    w = (L.ptr(d["ln1_w"]), L.ptr(d["ln1_b"]), L.ptr(d["w1"]), L.ptr(d["b1"]), L.ptr(d["w2"]), L.ptr(d["b2"]),
         L.ptr(d["ln2_w"]), L.ptr(d["ln2_b"]))
    R = (seqs + 1) * S

    def run(fn, hi, lo, f32):
        xd = _nan(R, 512)
        xd[:seqs * S] = x.reshape(-1, 512).to(DEV)
        bufs = {"hi": _nan(R, 512, dtype=torch.bfloat16) if hi else None, "lo": _nan(R, 512, dtype=torch.bfloat16) if lo else None,
                "f32": _nan(R, 512) if f32 else None}
        args = (L.ptr(xd), seqs, *w, L.ptr(bufs["hi"]), L.ptr(bufs["lo"])) if S == 8 else \
            (L.ptr(xd), seqs, S, *w, L.ptr(bufs["hi"]), L.ptr(bufs["lo"]))
        L.check(fn(*args, _st()) if fn in (lib.pips_tokenmix_tc, lib.pips_tokenmix_tc_s) else fn(*args, L.ptr(bufs["f32"]), _st()))
        torch.cuda.synchronize()
        for t in [xd] + [v for v in bufs.values() if v is not None]:
            assert torch.isnan(t[seqs * S:].float()).all(), "a row past seqs was written"
        return xd[:seqs * S].cpu(), {k: v[:seqs * S].cpu() for k, v in bufs.items() if v is not None}

    tm, tm_tc = (lib.pips_tokenmix, lib.pips_tokenmix_tc) if S == 8 else (lib.pips_tokenmix_s, lib.pips_tokenmix_tc_s)
    x_pair, pair = run(tm, True, True, False)
    x_hi, plain = run(tm, True, False, False)
    x_f, f32 = run(tm, False, False, True)
    x_tc, tc = run(tm_tc, True, True, False)
    assert torch.equal(_bits(x_pair), _bits(x_tc)) and torch.equal(_bits(pair["hi"]), _bits(tc["hi"])) \
        and torch.equal(_bits(pair["lo"]), _bits(tc["lo"])), "pips_tokenmix (hi, lo) and pips_tokenmix_tc differ"
    assert torch.equal(_bits(x_hi), _bits(x_pair)) and torch.equal(_bits(plain["hi"]), _bits(pair["hi"])), \
        "(hi, NULL) is not the hi half of (hi, lo)"

    xn, y2, xmag, y2mag = _tokenmix_ref(x.double(), lw)
    xn, y2, xmag, y2mag = (t.reshape(-1, 512) for t in (xn, y2, xmag, y2mag))
    tag = f"tokenmix seqs={seqs} offset={offset}" + ("" if S == 8 else f" S={S}")
    _report(f"{tag} wgmma: x err / (U sum|terms|)", _ratio(x_pair, xn, xmag), C_TM_TC)
    _report(f"{tag} wgmma: hi+lo err / (U sum|terms|)", _ratio(pair["hi"].double() + pair["lo"].double(), y2, y2mag), C_TM_Y)
    _report(f"{tag} fp32: x err / (U sum|terms|)", _ratio(x_f, xn, xmag), C_TM_F32)
    _report(f"{tag} fp32: y err / (U sum|terms|)", _ratio(f32["f32"], y2, y2mag), C_TM_F32)
    rec = pair["hi"].double() + pair["lo"].double()
    assert ((plain["hi"].double() - rec).abs() <= 2.0 ** -8 * rec.abs()).all(), "hi is not rn_bf16 of hi + lo"


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("seqs,S", _windows([1, 37, 700], [1, 37, 700], [2, 5, 9, 16]))
def test_ln_pool_outputs(seqs, S, offset):
    """pips_ln_pool (nets/pips.py:120-121) as (hi, lo), (hi, NULL) and f32; pips_ln_pool_s at the other window lengths."""
    lib = L.load()
    lw = _layer(po.init_state_dict(3, S=S))
    x = _tokenmix_inputs(seqs, offset, 109 + seqs, S=S)
    xd = x.reshape(-1, 512).to(DEV).contiguous()
    gw, gb = lw["out_w"].to(DEV), lw["out_b"].to(DEV)
    outs = {}
    for name, parts in (("pair", ("hi", "lo")), ("plain", ("hi",)), ("f32", ("f32",))):
        b = {k: _nan(seqs + 1, 512, dtype=torch.float32 if k == "f32" else torch.bfloat16) if k in parts else None
             for k in ("hi", "lo", "f32")}
        outs_ = (L.ptr(gw), L.ptr(gb), L.ptr(b["hi"]), L.ptr(b["lo"]), L.ptr(b["f32"]), _st())
        L.check(lib.pips_ln_pool(L.ptr(xd), seqs, *outs_) if S == 8 else lib.pips_ln_pool_s(L.ptr(xd), seqs, S, *outs_))
        torch.cuda.synchronize()
        for v in b.values():
            if v is not None:
                assert torch.isnan(v[seqs].float()).all(), "a row past seqs was written"
        outs[name] = {k: v[:seqs].cpu() for k, v in b.items() if v is not None}
    w64, b64 = lw["out_w"].double(), lw["out_b"].double()
    xd64 = x.double()
    ref = po._ln(xd64, w64, b64).mean(1)
    mag, _ = _ln_mag(xd64, w64, b64)
    mag = mag.mean(1)
    pf = outs["f32"]["f32"]
    tag = f"ln_pool seqs={seqs} offset={offset}" + ("" if S == 8 else f" S={S}")
    _report(f"{tag}: f32 err / (U sum|terms|)", _ratio(pf, ref, mag), C_POOL)
    hi, lo = outs["pair"]["hi"].float(), outs["pair"]["lo"].float()
    rec = ((hi.double() + lo.double()) - pf.double()).abs() / pf.double().abs().clamp_min(1e-30)
    _report(f"{tag}: hi+lo vs f32, relative", rec.max().item(), 2.0 ** -16)
    assert torch.equal(_bits(outs["plain"]["hi"]), _bits(outs["pair"]["hi"])), "(hi, NULL) is not the hi half of (hi, lo)"


# ------------------------------------------------------------------------------------------------ 6. update, peers, vis head

def _update_case(B, N, seed, S=S):
    torch.manual_seed(seed)
    delta = torch.randn(B * N, S, 130)
    delta[: (B * N) // 3, :, 2:] += 50.0                     # GroupNorm rows with a large common offset
    delta[:, :, 2:] *= torch.rand(B * N, S, 1) * 3 + 0.1
    coords = torch.rand(B, S, N, 2) * 40
    coords0 = torch.rand(B, S, N, 2) * 40
    ffeats = torch.randn(B * N, S, 128)
    return delta, coords, coords0, ffeats


def _upd_call(sd, delta, coords, coords0, ffeats, stride, peer=None):
    """pips_update_peer with delta in rows of PIPS_DELTA_LD(S) floats, NaN in the pad columns of odd S."""
    lib = L.load()
    B, S, N, _ = coords.shape
    d = lambda t: t.to(DEV).contiguous()
    dd = _nan(B * N, L.delta_ld(S))
    dd[:, :S * 130] = d(delta.reshape(B * N, S * 130))
    cd, c0d, fd = d(coords), d(coords0), d(ffeats)
    gw, gb, wu, bu = d(sd["norm.weight"]), d(sd["norm.bias"]), d(sd["ffeat_updater.0.weight"]), d(sd["ffeat_updater.0.bias"])
    out = _nan(B, S, N, 2)
    L.check(lib.pips_update_peer(L.ptr(dd), L.ptr(cd), L.ptr(c0d), L.ptr(fd), L.ptr(gw), L.ptr(gb), L.ptr(wu), L.ptr(bu),
                                 L.ptr(out), stride, B, S, N, None if peer is None else C.byref(peer), _st()))
    torch.cuda.synchronize()
    return cd.cpu(), fd.cpu(), out.cpu()


@pytest.mark.gpu
def test_update_and_vis_head_fp64():
    _check_update_and_vis_head()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [2, 5, 9, 16])
def test_update_and_vis_head_fp64_window(S):
    """pips_update reads delta rows PIPS_DELTA_LD(S) floats apart (2 pad columns at odd S); pips_vis_head decodes the
    warp of (b, s, n) by S."""
    _check_update_and_vis_head(S)


def _check_update_and_vis_head(S=S):
    lib = L.load()
    sd = po.init_state_dict(4)
    sd64 = {k: v.double() for k, v in sd.items()}
    B, N, stride = 2, 45, 4.0
    delta, coords, coords0, ffeats = _update_case(B, N, 110, S=S)
    c, ff, out = _upd_call(sd, delta, coords, coords0, ffeats, stride)
    # coordinates: one fp32 add (frame 0: the copy of coords0), then one fp32 multiply -- exactly torch's fp32 results
    c_ref = coords + delta[:, :, :2].reshape(B, N, S, 2).permute(0, 2, 1, 3)
    c_ref[:, 0] = coords0[:, 0]
    assert torch.equal(_bits(c), _bits(c_ref)) and torch.equal(_bits(out), _bits(c_ref * stride))
    _, ff_ref = _update_ref(sd64, delta.double(), coords, coords0, ffeats)
    v = delta[:, :, 2:].double().reshape(-1, 128)
    gmag, _ = _ln_mag(v, sd64["norm.weight"], sd64["norm.bias"])                    # GroupNorm(1, 128) = LN over 128
    fmag = gmag @ sd64["ffeat_updater.0.weight"].abs().t() + sd64["ffeat_updater.0.bias"].abs() + ffeats.double().reshape(-1, 128).abs()
    tag = "" if S == 8 else f" S={S}"
    _report(f"update{tag}: ffeats err / (U sum|terms|)", _ratio(ff.reshape(-1, 128), ff_ref.reshape(-1, 128), fmag), C_UPD)

    vis = _nan(B, S, N + 1)
    fd = ff.to(DEV).contiguous()
    vw, vb = sd["vis_predictor.0.weight"].reshape(-1).to(DEV), sd["vis_predictor.0.bias"].to(DEV)
    L.check(lib.pips_vis_head(L.ptr(fd), L.ptr(vw), L.ptr(vb), L.ptr(vis), B, S, N, _st()))
    torch.cuda.synchronize()
    f64 = ff.double().reshape(B, N, S, 128).permute(0, 2, 1, 3)
    v_ref = f64 @ sd64["vis_predictor.0.weight"].reshape(-1) + sd64["vis_predictor.0.bias"]
    v_mag = f64.abs() @ sd64["vis_predictor.0.weight"].abs().reshape(-1) + sd64["vis_predictor.0.bias"].abs()
    got = vis.cpu().view(-1)[:B * S * N].view(B, S, N)
    _report(f"vis_head{tag}: err / (U sum|terms|)", _ratio(got, v_ref, v_mag), C_VIS)
    assert torch.isnan(vis.cpu().view(-1)[B * S * N:]).all()


@pytest.mark.gpu
def test_update_peer_stores_the_slice_into_every_peer():
    """The fused all-gather of pips_update_peer with three peers that are local buffers: particles [5, 5 + N) of
    n_total = N + 9, in all three, bit-equal to out_px; every other element stays NaN."""
    sd = po.init_state_dict(4)
    B, N, off, stride = 2, 21, 5, 8.0
    n_total = N + 9
    delta, coords, coords0, ffeats = _update_case(B, N, 111)
    peers = [_nan(B, S, n_total, 2) for _ in range(3)]
    peer = L.PeerOut()
    peer.n_peers, peer.n_offset, peer.n_total = 3, off, n_total
    for r, t in enumerate(peers):
        peer.out[r] = L.ptr(t)
    c, ff, out = _upd_call(sd, delta, coords, coords0, ffeats, stride, peer)
    c2, ff2, out2 = _upd_call(sd, delta, coords, coords0, ffeats, stride)
    assert torch.equal(_bits(out), _bits(out2)) and torch.equal(_bits(ff), _bits(ff2)), "peer stores changed the local result"
    for r, t in enumerate(peers):
        t = t.cpu()
        assert torch.equal(_bits(t[:, :, off:off + N]), _bits(out)), f"peer {r}: slice differs from out_px"
        mask = torch.ones(n_total, dtype=torch.bool)
        mask[off:off + N] = False
        assert torch.isnan(t[:, :, mask]).all(), f"peer {r}: written outside its slice"


@pytest.mark.gpu
@pytest.mark.parametrize("cols,cols_total,col_offset", [(8, 20, 4), (5, 13, 3)])
def test_peer_scatter_column_offset(cols, cols_total, col_offset):
    """pips_peer_scatter into two local buffers: the 16-byte path (multiples of 4) and the scalar path."""
    lib = L.load()
    rows = 37
    torch.manual_seed(112)
    src = torch.randn(rows, cols).to(DEV)
    dst = [_nan(rows, cols_total) for _ in range(2)]
    L.check(lib.pips_peer_scatter(L.ptr(src), rows, cols, L.ptr_array(dst), 2, cols_total, col_offset, _st()))
    torch.cuda.synchronize()
    for t in dst:
        t = t.cpu()
        assert torch.equal(_bits(t[:, col_offset:col_offset + cols]), _bits(src))
        assert torch.isnan(t[:, :col_offset]).all() and torch.isnan(t[:, col_offset + cols:]).all()


# ------------------------------------------------------------------------------------------------ 7. the whole mixer

_MIXER = {}


def _mixer_case(S=S):
    """Weights with head_scale 1 (the head does not shrink errors), 300 sequences of mixer input and the fp64 oracle
    mixer's delta for them.  Sequences are independent, so the first k rows serve every seqs = k."""
    if S not in _MIXER:
        sd = po.init_state_dict(seed=9, head_scale=1.0, S=S)
        g = torch.Generator().manual_seed(113)
        x0 = torch.randn(300, S, 519, generator=g)
        _MIXER[S] = dict(sd=sd, x0=x0, ref=po.mixer({k: v.double() for k, v in sd.items()}, x0.double()))
    return _MIXER[S]


_WS_ROWS = {"x0": "M", "x": "M", "y": "M", "h": "M", "p": "seqs", "delta": "seqs"}


def _mixer_run(w, ws, x0, seqs, prec, tail, S=S):
    """Fill the workspace's live rows with x0 and every row at or beyond M (beyond seqs for p / delta) with `tail`,
    run pips_mixer_forward (pips_mixer_forward_s at S != 8), return delta (all rows, PIPS_DELTA_LD(S) columns)."""
    lib = L.load()
    M = seqs * S
    for name, t in ws.keep.items():
        live = seqs if _WS_ROWS[name.split("_")[0]] == "seqs" else M
        if name.startswith("x0"):
            t.zero_()                                        # K padding of live rows: zero, as pips_corr_gather writes it
        else:
            t.fill_(float("nan"))                            # live rows a kernel fails to write stay NaN
        t[live:] = tail
    flat = x0[:seqs].reshape(M, 519).to(DEV)
    if prec == L.PREC_F32:
        ws.keep["x0_f32"][:M, :519] = flat
    else:
        hi, lo = _split_bf16(flat)
        ws.keep["x0_hi"][:M, :519] = hi
        if prec == L.PREC_BF16X3:
            ws.keep["x0_lo"][:M, :519] = lo
    if S == 8:
        L.check(lib.pips_mixer_forward(C.byref(w.c), C.byref(ws.c), seqs, prec, _st()), "pips_mixer_forward")
    else:
        L.check(lib.pips_mixer_forward_s(C.byref(w.c), C.byref(ws.c), seqs, S, prec, _st()), "pips_mixer_forward_s")
    torch.cuda.synchronize()
    return ws.keep["delta"].cpu()


_PRECISIONS = ["fp32", "bf16x3", "bf16"]


@pytest.mark.gpu
@pytest.mark.parametrize("precision,S", _windows(_PRECISIONS, _PRECISIONS, [2, 5, 9, 16]))
def test_mixer_forward_against_fp64(precision, S):
    """pips_mixer_forward (1 + 12 x 3 + 1 dense layers, token mixing, pooling) against the oracle mixer in fp64, at
    seqs 1, 37, 300; error relative to max|delta|.  At odd S the 2 pad columns of every delta row stay NaN."""
    case = _mixer_case(S)
    prec = L.PRECISIONS[precision]
    w = engine.PackedWeights(_module(case["sd"]), _st())
    ws = engine.Workspace(300, prec, DEV, S=S)
    n = L.head_n(S)
    for seqs in (1, 37, 300):
        d = _mixer_run(w, ws, case["x0"], seqs, prec, 0.0, S=S)
        ref = case["ref"][:seqs]
        assert torch.isnan(d[:seqs, n:]).all(), "pad columns of delta were written"
        rel = (d[:seqs, :n].double() - ref).abs().max().item() / ref.abs().max().item()
        tag = f"mixer {precision} seqs={seqs}" + ("" if S == 8 else f" S={S}")
        _report(f"{tag}: max|err| / max|delta| (max|delta| {ref.abs().max().item():.3g})", rel, MIXER_REL[precision])


@pytest.mark.gpu
@pytest.mark.parametrize("precision,S", _windows(_PRECISIONS, _PRECISIONS, [2, 5, 9, 16]))
def test_mixer_forward_tails_and_prefix(precision, S):
    """Rows past M (past seqs for p / delta) hold stale data when a workspace is reused for a smaller chunk: NaN there
    must not reach a live row, and delta rows >= seqs must not be written.  A sequence's delta must not depend on how
    many other sequences share the call (particle chunking relies on it)."""
    case = _mixer_case(S)
    prec = L.PRECISIONS[precision]
    w = engine.PackedWeights(_module(case["sd"]), _st())
    ws = engine.Workspace(300, prec, DEV, S=S)
    n = L.head_n(S)
    zero = _mixer_run(w, ws, case["x0"], 37, prec, 0.0, S=S)
    poisoned = _mixer_run(w, ws, case["x0"], 37, prec, float("nan"), S=S)
    assert torch.equal(_bits(poisoned[:37]), _bits(zero[:37])), "stale rows past M changed live rows"
    assert torch.isnan(poisoned[37:]).all(), "delta rows >= seqs were written"
    assert not torch.isnan(zero[:37, :n]).any()
    assert torch.isnan(zero[:37, n:]).all() and torch.isnan(poisoned[:37, n:]).all(), "pad columns of delta were written"
    full = _mixer_run(w, ws, case["x0"], 300, prec, 0.0, S=S)
    assert torch.equal(_bits(full[:37]), _bits(zero[:37])), "delta of the first 37 sequences depends on seqs"


# ------------------------------------------------------------------------------------------------ 8. host-side validation

def test_corr_gather_and_update_peer_validate_arguments_without_gpu():
    lib = L.load()
    p = C.c_void_p(256)
    lv = (C.c_void_p * 4)(256, 256, 256, 256)

    def cg(H=16, W=16, fb=None, T=0, hi=p, lo=p, f=p, ldx=576):
        return lib.pips_corr_gather(lv, 0, 1, 8, 4, H, W, p, p, p, fb, T, hi, lo, f, ldx, None)

    for ldx, what in ((568, "ldx < 576"), (580, "ldx % 8")):
        assert cg(ldx=ldx) != 0, what
        assert b"ldx must be >= 576 and a multiple of 8" in lib.pips_last_error()
    assert cg(hi=None, lo=p, f=p) != 0
    assert b"x_lo without x_hi" in lib.pips_last_error()
    assert cg(fb=p, T=0) != 0
    assert b"frame_base needs frames_per_batch > 0" in lib.pips_last_error()
    for H, W in ((7, 16), (16, 7)):
        assert cg(H=H, W=W) != 0
        assert b"level-0 map must be at least 8x8" in lib.pips_last_error()

    peer = L.PeerOut()
    peer.n_peers, peer.n_offset, peer.n_total = 2, 5, 12                                  # 5 + N(=8) > 12
    peer.out[0] = peer.out[1] = 256
    upd = lambda: lib.pips_update_peer(p, p, p, p, p, p, p, p, p, 8.0, 1, 8, 8, C.byref(peer), None)
    assert upd() != 0
    assert b"particle slice outside n_total" in lib.pips_last_error()
    peer.n_total = 13
    peer.n_peers = L.MAX_PEERS + 1
    assert upd() != 0
    assert b"more than PIPS_MAX_PEERS" in lib.pips_last_error()
    peer.n_peers = 2
    peer.out[1] = 260                                                                    # 4-byte aligned only
    assert upd() != 0
    assert b"null or misaligned peer result" in lib.pips_last_error()
