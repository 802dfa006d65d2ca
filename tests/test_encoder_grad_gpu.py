"""Training the feature encoder on the sm_90a kernels (Pips(encoder_path='cuda'), torch_path.encoder_cuda): the
convolution weight gradient, the flipped-weight input gradients, the InstanceNorm backward and the resize adjoint against
fp64, the whole encoder's forward and backward against fp64 autograd of the Encoder module, bit-equality with fnet_tc,
determinism, nn.DataParallel replicas, a training step against encoder_path='torch', memory and routing.  Output buffers
are filled with NaN before every call.  Kernel errors are per element in units of 2^-24 * sum|terms| (fp64); a bf16x3
product carries about 2^-17 relative error (128 units) and so does a (hi, lo) pair, hence bounds of 256 units."""
import zlib

import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path
from pips_b200 import encoder_fast as E
from pips_b200.encoder import Encoder

DEV = "cuda:0"
U = 2.0 ** -24


def _st():
    return torch.cuda.current_stream().cuda_stream


def _pair(v, cp):
    """(N, H, W, C) fp32 -> _Pair of channel pitch cp (padding zero); also the fp64 value hi + lo it carries"""
    N, H, W, C = v.shape
    p = E._Pair(N, H, W, cp, DEV)
    p.C = C
    full = torch.zeros(N, H, W, cp, device=DEV)
    full[..., :C] = v
    L.check(L.load().pips_split_bf16(L.ptr(full), L.ptr(p.hi), L.ptr(p.lo), full.numel(), _st()), "pips_split_bf16")
    return p, (p.hi.double() + p.lo.double())[..., :C]


def _units(got, ref, mag):
    """max |got - ref| / (2^-24 * mag) over the elements, with mag the fp64 sum of |terms|"""
    return ((got.double() - ref).abs() / (U * mag.clamp(min=1e-300))).max().item()


def _wgrad(dyp, step, xp, cout, R, S, stride, pad):
    lib = L.load()
    N, H, W = xp.shape
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - S) // stride + 1
    K = R * S * xp.Cp
    dw = torch.full((cout, K), float("nan"), device=DEV)
    n = lib.pips_conv_wgrad_scratch_floats(N, Ho, Wo, cout, K)
    scratch = torch.full((max(n, 1),), float("nan"), device=DEV)
    L.check(lib.pips_conv_wgrad(L.ptr(dyp.hi), L.ptr(dyp.lo), dyp.Cp, step, L.ptr(xp.hi), L.ptr(xp.lo), N, H, W, xp.Cp, cout, R, S,
                                stride, stride, pad, pad, L.ptr(scratch), L.ptr(dw), _st()), "pips_conv_wgrad")
    return dw


WGRAD_CASES = [  # (N, H, W, Cin, Cout, R, stride, pad): every encoder geometry, odd sizes where stride-2 boxes cross the border
    (2, 32, 40, 64, 64, 3, 1, 1),        # layer1
    (2, 33, 41, 64, 96, 3, 2, 1),        # layer2.0.conv1, odd input
    (2, 32, 40, 64, 96, 1, 2, 0),        # layer2.0.downsample
    (3, 17, 23, 96, 128, 1, 2, 0),       # layer3.0.downsample, odd input
    (2, 16, 20, 128, 128, 3, 1, 1),      # layer3/4 conv2
    (2, 16, 20, 416, 256, 3, 1, 1),      # head conv2 (448-channel pitch)
    (2, 16, 20, 256, 128, 1, 1, 0),      # head conv3
    (1, 7, 5, 128, 128, 3, 2, 1),        # tiny, tiles larger than the image
    (32, 96, 128, 64, 64, 3, 1, 1),      # many pixel tiles: the chunked reduction
]


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,pad", WGRAD_CASES)
@pytest.mark.parametrize("dilated", [False, True])
def test_conv_wgrad_matches_fp64(N, H, W, Cin, Cout, R, stride, pad, dilated):
    if dilated and stride == 1:
        pytest.skip("the zero-dilated gradient exists for stride-2 convolutions only")
    g = torch.Generator(device=DEV).manual_seed(N * 1000 + H + Cin)
    x = torch.randn(N, H, W, Cin, device=DEV, generator=g)
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    dy = torch.randn(N, Ho, Wo, Cout, device=DEV, generator=g)
    xp, x64 = _pair(x, E._pad64(Cin))
    if dilated:
        D = torch.zeros(N, H, W, Cout, device=DEV)
        D[:, ::2, ::2] = dy
        dyp, D64 = _pair(D, E._pad64(Cout))
        dy64 = D64[:, ::2, ::2]
    else:
        dyp, dy64 = _pair(dy, E._pad64(Cout))
    dw = _wgrad(dyp, 2 if dilated else 1, xp, Cout, R, R, stride, pad)
    dw = dw.view(Cout, R, R, xp.Cp)[..., :Cin].permute(0, 3, 1, 2)
    xn, dn = x64.permute(0, 3, 1, 2), dy64.permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(xn, (Cout, Cin, R, R), dn, stride=stride, padding=pad)
    mag = torch.nn.grad.conv2d_weight(xn.abs(), (Cout, Cin, R, R), dn.abs(), stride=stride, padding=pad)
    e = _units(dw, ref, mag)
    print(f"conv_wgrad N={N} {H}x{W} {Cin}->{Cout} {R}x{R}/{stride} dilated={dilated}: {e:.2f} units")
    assert torch.isfinite(dw).all() and e <= 256


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W", [(2, 64, 80), (1, 11, 9)])
def test_stem_wgrad_matches_fp64(N, H, W):
    """the stem's 4x1 convolution over pips_stem_pack's row-pair pixels, folded back to (64, 3, 7, 7)"""
    g = torch.Generator(device=DEV).manual_seed(H)
    rgb = torch.rand(N, 3, H, W, device=DEV, generator=g) * 255
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    unf = E._Pair(N, Ho + 3, Wo, 64, DEV)
    L.check(L.load().pips_stem_pack(L.ptr(rgb), 0, N, H, W, L.ptr(unf.hi), L.ptr(unf.lo), _st()), "pips_stem_pack")
    dy = torch.randn(N, Ho, Wo, 64, device=DEV, generator=g)
    dyp, dy64 = _pair(dy, 64)
    dw = _wgrad(dyp, 1, unf, 64, 4, 1, 1, 0)
    dw = dw.view(64, 8, 32)[:, :7, :21].reshape(64, 7, 7, 3).permute(0, 3, 1, 2)
    x64 = (unf.hi.double() + unf.lo.double())
    # the unfolded pixels hold the normalised image: the reference convolves the image the pack carries
    img = torch.zeros(N, 3, H, W, dtype=torch.float64, device=DEV)
    for j in range(Ho + 3):
        for half in (0, 1):
            y = 2 * j - 3 + half
            if 0 <= y < H:
                k = x64[:, j, :, 32 * half:32 * half + 21].reshape(N, Wo, 7, 3)      # [n, ox, s, colour] at x = 2ox + s - 3
                for s in range(7):
                    xs = torch.arange(Wo, device=DEV) * 2 + s - 3
                    ok = (xs >= 0) & (xs < W)
                    img[:, :, y, xs[ok]] = k[:, ok, s, :].permute(0, 2, 1)
    dn = dy64.permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(img, (64, 3, 7, 7), dn, stride=2, padding=3)
    mag = torch.nn.grad.conv2d_weight(img.abs(), (64, 3, 7, 7), dn.abs(), stride=2, padding=3)
    e = _units(dw, ref, mag)
    print(f"stem wgrad N={N} {H}x{W}: {e:.2f} units")
    assert torch.isfinite(dw).all() and e <= 256


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(32, 40), (33, 41)])
@pytest.mark.parametrize("Cin,Cout,R,stride", [(64, 64, 3, 1), (128, 128, 3, 1), (256, 128, 1, 1), (64, 96, 3, 2), (96, 128, 1, 2),
                                               (416, 256, 3, 1)])
def test_flipped_weight_input_gradient_matches_fp64(H, W, Cin, Cout, R, stride):
    g = torch.Generator(device=DEV).manual_seed(H * Cin + R)
    pad = R // 2
    N = 2
    w = torch.randn(Cout, Cin, R, R, device=DEV, generator=g) / (Cin * R * R) ** 0.5
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    dy = torch.randn(N, Ho, Wo, Cout, device=DEV, generator=g)
    if stride == 2:
        D = torch.zeros(N, H, W, Cout, device=DEV)
        D[:, ::2, ::2] = dy
        dyp, D64 = _pair(D, E._pad64(Cout))
        dy64 = D64[:, ::2, ::2]
    else:
        dyp, dy64 = _pair(dy, E._pad64(Cout))
    run = torch_path._EncRun(torch.device(DEV))
    parts = [(0, Cin)] if Cin <= 256 else [(0, 160), (160, Cin)]
    dx = torch.cat([run.dgrad(dyp, w, pad, rows=r) for r in parts], dim=-1)
    # the kernel's weight is the (hi, lo) pair of the flipped weight: the reference uses those values
    wt = w.flip(2, 3).transpose(0, 1)
    w64 = torch.cat([torch.stack(E.pack_conv_weight(wt[a:b])).double().sum(0)[:b - a].view(b - a, R, R, -1)[..., :Cout]
                     for a, b in parts]).permute(3, 0, 1, 2).flip(2, 3)                 # back to (Cout, Cin, R, R)
    dn = dy64.permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_input((N, Cin, H, W), w64, dn, stride=stride, padding=pad).permute(0, 2, 3, 1)
    mag = torch.nn.grad.conv2d_input((N, Cin, H, W), w64.abs(), dn.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    e = _units(dx, ref, mag)
    print(f"input gradient {H}x{W} {Cin}->{Cout} {R}x{R}/{stride}: {e:.2f} units")
    assert torch.isfinite(dx).all() and e <= 256


def _inorm_case(kind, N, H, W, C, g):
    y = torch.randn(N, H, W, C, device=DEV, generator=g) * 2 + 0.3
    if kind == "flat":                                   # every other channel constant: var 0, rstd = 1/sqrt(1e-5) ~ 316
        y[..., ::2] = torch.randn(N, 1, 1, C // 2, device=DEV, generator=g)
    elif kind == "offset":                               # mean / std ~ 1e3
        y = 1000.0 + torch.randn(N, H, W, C, device=DEV, generator=g)
    return y


def _stats(y):
    N, H, W, C = y.shape
    chunks = max(1, min(64, H * W // 256))
    partial = torch.empty(N, chunks, 3, C, device=DEV)
    st = torch.empty(N, 2, C, device=DEV)
    L.check(L.load().pips_inorm_stats(L.ptr(y), N, H * W, C, L.ptr(partial), chunks, L.ptr(st), _st()), "pips_inorm_stats")
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["plain", "flat", "offset"])
@pytest.mark.parametrize("relu_main,relu_out,residual,n_add,dil", [
    (1, 0, None, 1, False), (1, 0, None, 1, True), (1, 1, "plain", 3, False), (1, 1, "norm", 2, False),
    (0, 0, None, 1, True), (0, 0, None, 2, False), (1, 1, "norm", 1, True)])
def test_inorm_grad_matches_fp64(kind, relu_main, relu_out, residual, n_add, dil):
    N, H, W, C = 2, 13, 19, 96
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr((kind, relu_main, relu_out, residual, n_add, dil)).encode()))
    y = _inorm_case(kind, N, H, W, C, g)
    st = _stats(y)
    r = sr = None
    if residual is not None:
        r = torch.randn(N, H, W, C, device=DEV, generator=g)
        sr = _stats(r) if residual == "norm" else None
    adds = [torch.randn(N, H, W, C, device=DEV, generator=g) for _ in range(n_add)]
    lib = L.load()
    Hd, Wd = (2 * H - 1, 2 * W) if dil else (H, W)
    cp = 128
    hi = torch.full((N, Hd, Wd, cp), float("nan"), dtype=torch.bfloat16, device=DEV)
    lo = hi.clone()
    skip = torch.full_like(y, float("nan"))
    scratch = torch.full((lib.pips_inorm_grad_scratch_floats(N, H * W, C),), float("nan"), device=DEV)
    gp = adds + [None] * (3 - n_add)
    L.check(lib.pips_inorm_grad(L.ptr(y), L.ptr(st), L.ptr(r), L.ptr(sr), relu_main, relu_out, *(L.ptr(t) for t in gp), N, H, W, C,
                                L.ptr(scratch), L.ptr(hi), L.ptr(lo), cp, *((Hd, Wd) if dil else (0, 0)), L.ptr(skip), _st()),
            "pips_inorm_grad")
    torch.cuda.synchronize()
    out64 = hi.double() + lo.double()
    if dil:
        odd = torch.ones(Hd, Wd, dtype=torch.bool, device=DEV)
        odd[::2, ::2] = False
        assert (hi[:, odd] == 0).all() and (lo[:, odd] == 0).all() and not torch.signbit(hi[:, odd].float()).any()
        out64 = out64[:, ::2, ::2]
    assert (hi[..., C:] == 0).all() and (lo[..., C:] == 0).all()
    dy = out64[..., :C]
    # masks from the forward kernel's own fp32 output (pips_inorm_apply), the rest in fp64 from the same statistics
    v = torch.empty_like(y)
    L.check(lib.pips_inorm_apply(L.ptr(y), L.ptr(st), L.ptr(r), L.ptr(sr), relu_main, relu_out, L.ptr(v), None, 0, N, H * W, C,
                                 _st()), "pips_inorm_apply")
    main = torch.empty_like(y)
    L.check(lib.pips_inorm_apply(L.ptr(y), L.ptr(st), None, None, 0, 0, L.ptr(main), None, 0, N, H * W, C, _st()), "pips_inorm_apply")
    gsum = adds[0]
    for a in adds[1:]:
        gsum = gsum + a
    if relu_out:
        gsum = torch.where(v > 0, gsum, torch.zeros_like(gsum))
    assert torch.equal(skip, gsum)                                   # the residual branch's gradient, bit-exact
    gm = torch.where(main > 0, gsum, torch.zeros_like(gsum)) if relu_main else gsum
    m64, s64 = st[:, 0].double()[:, None, None], st[:, 1].double()[:, None, None]
    xh = (y.double() - m64) * s64
    g64 = gm.double()
    mg, mgx = g64.mean((1, 2), keepdim=True), (g64 * xh).mean((1, 2), keepdim=True)
    ref = s64 * (g64 - mg - xh * mgx)
    mag = s64 * (g64.abs() + g64.abs().mean((1, 2), keepdim=True) + xh.abs() * (g64 * xh).abs().mean((1, 2), keepdim=True))
    # the (hi, lo) pair of a fp32 value carries it to 2^-16 * 2^-8 relative: part of the bound
    e = _units(dy, ref, mag + ref.abs())
    print(f"inorm_grad {kind} relu {relu_main}{relu_out} residual {residual} addends {n_add} dilated {dil}: {e:.2f} units")
    assert e <= 256


@pytest.mark.gpu
@pytest.mark.parametrize("stride", [4, 8])
def test_resize_grad_matches_fp64(stride):
    H, W, N = 96, 160, 2
    H8, W8 = H // stride, W // stride
    widths = (64, 96, 128, 128)
    g = torch.Generator(device=DEV).manual_seed(stride)
    ld = 416
    gc = torch.randn(N, H8, W8, ld, device=DEV, generator=g)
    lib = L.load()
    c_off = 0
    for l, C in enumerate(widths):
        Hs, Ws = H // 2 ** (l + 1), W // 2 ** (l + 1)
        out = torch.full((N, Hs, Ws, C), float("nan"), device=DEV)
        L.check(lib.pips_resize_grad(L.ptr(gc), ld, c_off, N, H8, W8, L.ptr(out), Hs, Ws, C, _st()), "pips_resize_grad")
        gs = gc[..., c_off:c_off + C].double()
        # the transpose of the forward as pips_resize_pair computes it: its fp32 tap weights, summed in fp64
        Ay, Ax = _taps(Hs, H8), _taps(Ws, W8)
        ref = torch.einsum("ys,xt,nyxc->nstc", Ay, Ax, gs)
        mag = torch.einsum("ys,xt,nyxc->nstc", Ay, Ax, gs.abs())
        e = _units(out, ref, mag)
        # and fp64 autograd of F.interpolate, whose fp64 tap weights differ from fp32's by rounding
        src = torch.zeros(N, C, Hs, Ws, dtype=torch.float64, device=DEV, requires_grad=True)
        F.interpolate(src, (H8, W8), mode="bilinear", align_corners=True).backward(gs.permute(0, 3, 1, 2))
        e64 = ((out.double() - src.grad.permute(0, 2, 3, 1)).abs().max() / src.grad.abs().max()).item()
        print(f"resize_grad stride {stride} layer{l + 1} {Hs}x{Ws} -> {H8}x{W8}: {e:.2f} units; F.interpolate fp64 {e64:.1e}")
        assert torch.isfinite(out).all() and e <= 16 and e64 <= 1e-5
        c_off += C


def _taps(n_src, n_dst):
    """(n_dst, n_src) fp64 matrix of the fp32 bilinear tap weights of resize_split3_kernel (align_corners=True)"""
    A = torch.zeros(n_dst, n_src, dtype=torch.float64, device=DEV)
    sc = torch.tensor(float(n_src - 1), dtype=torch.float32) / torch.tensor(float(n_dst - 1), dtype=torch.float32) \
        if n_dst > 1 else torch.tensor(0.0)
    for o in range(n_dst):
        f = (sc * torch.tensor(float(o), dtype=torch.float32)).item()
        f = torch.tensor(f, dtype=torch.float32)
        i0 = int(f.item())
        lam = (f - torch.tensor(float(i0), dtype=torch.float32))
        A[o, i0] += (torch.tensor(1.0, dtype=torch.float32) - lam).item()
        A[o, i0 + (1 if i0 < n_src - 1 else 0)] += lam.item()
    return A


# ---------------------------------------------------------------------------------------------- the whole encoder

def _encoder(stride, seed=3):
    torch.manual_seed(seed)
    enc = Encoder(output_dim=128, stride=stride)
    with torch.no_grad():
        for m in enc.modules():
            if isinstance(m, torch.nn.Conv2d):
                m.bias.normal_(0, 0.1)
    return enc.to(DEV)


def _rgbs(B, S, H, W, seed, flat=False):
    if flat:
        c = torch.tensor([40.0, 200.0, 120.0]).view(1, 1, 3, 1, 1)
        return c.expand(B, S, 3, H, W).contiguous().to(DEV)
    return po.smooth_video(B, S, H, W, seed=seed).to(DEV).float()


def _cuda_masks(enc, rgbs):
    """Every ReLU decision of encoder_cuda's forward, in module order (stem; per ResBlock: after conv1's InstanceNorm,
    after conv2's, at the block output; head), as NCHW 0/1 tensors.  They are recomputed with fnet_tc's kernels from
    the block boundaries its forward keeps -- the recompute encoder_cuda's backward runs -- and the normalisation
    (y - mean) * rstd is evaluated in fp32 exactly as pips_inorm_apply evaluates it."""
    run = torch_path._EncRun(torch.device(DEV))
    raw = rgbs.flatten(0, 1).contiguous()
    _, convs = torch_path._encoder_params(enc)
    packs = {convs[n]: (E.pack_stem_weight if n == "conv1" else E.pack_conv_weight)(convs[n].weight.detach())
             for n in torch_path.ENCODER_CONVS}

    def pos(y, st):
        N, C = st.shape[0], st.shape[2]
        xh = (y - st[:, 0].view(N, 1, 1, C)) * st[:, 1].view(N, 1, 1, C)
        return (xh > 0).permute(0, 3, 1, 2)

    masks, keep = [], []
    with torch.no_grad():
        E._fnet_tc(enc, raw, packs=packs, keep=keep)
        _, y0, s0 = E.stem_tc(raw, packs[enc.conv1])
        masks.append(pos(y0, s0))
        b = 0
        for i in range(1, 5):
            for blk in getattr(enc, f"layer{i}"):
                xp = run.pair_of(keep[b])
                y1, s1 = E._conv_stats(run.ops, xp, blk.conv1, packs[blk.conv1])
                _, a1 = E._apply_pair(run.ops, y1, s1, relu_main=True)
                y2, s2 = E._conv_stats(run.ops, a1, blk.conv2, packs[blk.conv2])
                masks += [pos(y1, s1), pos(y2, s2), (keep[b + 1] > 0).permute(0, 3, 1, 2)]
                b += 1
        N, H, W = raw.shape[0], raw.shape[2] // enc.stride, raw.shape[3] // enc.stride
        cat = run.pair(N, H, W, 416)
        c_off = 0
        for l in range(4):
            X = keep[2 * l + 2]
            L.check(L.load().pips_resize_pair(L.ptr(X), N, X.shape[1], X.shape[2], X.shape[3], L.ptr(cat.hi), L.ptr(cat.lo), H, W,
                                              cat.Cp, c_off, _st()), "pips_resize_pair")
            c_off += X.shape[3]
        yh, sh = E._conv_stats(run.ops, cat, enc.conv2, packs[enc.conv2])
        masks.append(pos(yh, sh))
    return masks


def _masked_forward(e, x, masks):
    """Encoder.forward with every ReLU replaced by the product with a given 0/1 mask: the same function as long as the
    masks are the ReLU decisions, differentiable without them"""
    it = iter(masks)

    def relu(v):
        return v * next(it).to(v.dtype)

    def inorm(t):
        return F.instance_norm(t, eps=1e-5)

    size = (x.shape[-2] // e.stride, x.shape[-1] // e.stride)
    x = relu(inorm(e.conv1(x)))
    taps = []
    for i in range(1, 5):
        for blk in getattr(e, f"layer{i}"):
            y = relu(inorm(blk.conv1(x)))
            y = relu(inorm(blk.conv2(y)))
            if blk.downsample is not None:
                x = inorm(blk.downsample[0](x))
            x = relu(x + y)
        taps.append(F.interpolate(x, size, mode="bilinear", align_corners=True))
    x = relu(inorm(e.conv2(torch.cat(taps, dim=1))))
    return e.conv3(x)


def _module_grads(enc, rgbs, dfm, dtype, masks=None):
    e = _encoder(enc.stride).to(dtype)
    e.load_state_dict(enc.state_dict())
    B, S, C, H, W = rgbs.shape
    x = (2 * (rgbs.to(dtype) / 255.0) - 1.0).reshape(B * S, C, H, W)
    f = e(x) if masks is None else _masked_forward(e, x, masks)
    f.backward(dfm.to(dtype))
    return f.detach(), {n: p.grad.detach() for n, p in e.named_parameters()}


def _cuda_grads(enc, rgbs, dfm):
    enc.zero_grad(set_to_none=True)
    f = torch_path.encoder_cuda(enc, rgbs)
    B, S = rgbs.shape[:2]
    f.backward(dfm.view(B, S, *dfm.shape[1:]))
    return f.detach().flatten(0, 1), {n: p.grad.detach().clone() for n, p in enc.named_parameters() if p.grad is not None}


ENCODER_CASES = [  # (B, S, H, W, stride, flat)
    (1, 2, 128, 160, 8, False),
    (1, 2, 96, 128, 4, False),
    (1, 1, 64, 96, 8, True),
    (1, 1, 384, 512, 8, False),
    (1, 1, 100, 136, 8, False),          # odd layer sizes: 50x68, 25x34, 13x17, 7x9 -> 12x17
]
# A bf16x3 product or (hi, lo) pair carries about 2^-17 relative error; the longest chain the gradient of a weight goes
# through is about 20 convolutions and InstanceNorms forward and as many backward, so 64 such roundings bound it.
BF16X3_BOUND = 64 * 2.0 ** -17


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,H,W,stride,flat", ENCODER_CASES)
def test_encoder_cuda_matches_fp64_autograd(monkeypatch, B, S, H, W, stride, flat):
    """fmaps and every weight gradient against fp64 autograd of the Encoder evaluated with encoder_cuda's own ReLU
    decisions (_cuda_masks), error relative to each tensor's max |value|, bounded by max(2 x strict fp32's error under
    the same decisions, BF16X3_BOUND).  Against the plain fp64 module a ReLU whose input lies within the forward's
    rounding of zero can decide the other way, and with a gradient of random sign one such decision moves a weight
    gradient by about 1/sqrt(pixels) of its max: those errors are printed as well (and strict fp32's own), not bounded."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    enc = _encoder(stride)
    rgbs = _rgbs(B, S, H, W, seed=H + stride, flat=flat)
    g = torch.Generator(device=DEV).manual_seed(7)
    dfm = torch.randn(B * S, 128, H // stride, W // stride, device=DEV, generator=g)
    masks = _cuda_masks(enc, rgbs)
    f64, g64 = _module_grads(enc, rgbs, dfm, torch.float64, masks)
    f32, g32 = _module_grads(enc, rgbs, dfm, torch.float32, masks)
    _, u64 = _module_grads(enc, rgbs, dfm, torch.float64)
    _, u32 = _module_grads(enc, rgbs, dfm, torch.float32)
    fc, gc = _cuda_grads(enc, rgbs, dfm)
    flips = sum(((m.double() > 0) != (a > 0)).sum().item() for m, a in zip(masks, _fp64_pre_relu(enc, rgbs, masks)))

    def err(a, b):
        return ((a.double() - b).abs().max() / b.abs().max().clamp(min=1e-300)).item()

    total = torch.cat([t.flatten() for t in g64.values()]).norm().item()
    report = []
    for n in g64:
        if n.endswith("bias") and n != "conv3.bias":
            assert (gc[n] == 0).all(), n                  # the 21 biases before an InstanceNorm: exactly zero
            assert g64[n].norm().item() <= 1e-6 * total, n
            continue
        report.append((n, err(gc[n], g64[n]), err(g32[n], g64[n]), err(gc[n], u64[n]), err(u32[n], u64[n])))
    ef_c, ef_t = err(fc, f64), err(f32, f64)
    ratio = {n: ec / max(2 * et, BF16X3_BOUND) for n, ec, et, _, _ in report}
    w = max(ratio, key=ratio.get)
    issue = sum(ec <= max(2 * et, 1e-5) for _, ec, et, _, _ in report)
    print(f"encoder {B}x{S}x{H}x{W}/{stride} flat={flat}: {flips} ReLU decisions differ from fp64's; fmaps cuda {ef_c:.2e} "
          f"fp32 {ef_t:.2e}; same decisions, worst gradient {w} {ratio[w]:.2f} of its bound; {issue} of {len(report)} gradients "
          f"within max(2 x fp32, 1e-5)\n  same decisions cuda/fp32 | plain fp64 module cuda/fp32: "
          + ", ".join(f"{n} {a:.1e}/{b:.1e} | {c:.1e}/{d:.1e}" for n, a, b, c, d in report))
    assert ef_c <= max(2 * ef_t, BF16X3_BOUND / 2)
    assert ratio[w] <= 1.0


def _fp64_pre_relu(enc, rgbs, masks):
    """the inputs of every ReLU of the fp64 masked forward, in the order of _cuda_masks (for the count of differing
    decisions)"""
    e = _encoder(enc.stride).double()
    e.load_state_dict(enc.state_dict())
    B, S, C, H, W = rgbs.shape
    x = (2 * (rgbs.double() / 255.0) - 1.0).reshape(B * S, C, H, W)
    pre = []
    it = iter(masks)

    def relu(v):
        pre.append(v)
        return v * next(it).double()

    def inorm(t):
        return F.instance_norm(t, eps=1e-5)

    with torch.no_grad():
        size = (H // e.stride, W // e.stride)
        x = relu(inorm(e.conv1(x)))
        taps = []
        for i in range(1, 5):
            for blk in getattr(e, f"layer{i}"):
                y = relu(inorm(blk.conv1(x)))
                y = relu(inorm(blk.conv2(y)))
                if blk.downsample is not None:
                    x = inorm(blk.downsample[0](x))
                x = relu(x + y)
            taps.append(F.interpolate(x, size, mode="bilinear", align_corners=True))
        relu(inorm(e.conv2(torch.cat(taps, dim=1))))
    return pre


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_encoder_cuda_forward_is_fnet_tc(dtype):
    enc = _encoder(8)
    rgbs = _rgbs(2, 3, 96, 160, seed=4).to(dtype)
    with torch.no_grad():
        ref = E.fnet_tc(enc, rgbs.flatten(0, 1))
    f = torch_path.encoder_cuda(enc, rgbs)
    assert f.requires_grad
    assert torch.equal(f.permute(0, 1, 3, 4, 2).flatten(0, 1), ref)


@pytest.mark.gpu
def test_encoder_cuda_is_deterministic():
    enc = _encoder(8)
    rgbs = _rgbs(1, 4, 128, 160, seed=9)
    dfm = torch.randn(4, 128, 16, 20, device=DEV)
    f1, g1 = _cuda_grads(enc, rgbs, dfm)
    f2, g2 = _cuda_grads(enc, rgbs, dfm)
    assert torch.equal(f1, f2) and all(torch.equal(g1[n], g2[n]) for n in g1)


@pytest.mark.gpu
def test_frozen_parameters_get_no_gradient():
    """weights that do not require grad are skipped; the others keep the bits of a call with every parameter trained"""
    enc = _encoder(8)
    rgbs = _rgbs(1, 2, 96, 128, seed=6)
    dfm = torch.randn(2, 128, 12, 16, device=DEV)
    _, full = _cuda_grads(enc, rgbs, dfm)
    frozen = {n for n, _ in enc.named_parameters() if n.startswith(("conv1.", "layer1.", "layer3.0.downsample", "conv3.bias"))}
    for n, p in enc.named_parameters():
        p.requires_grad_(n not in frozen)
    _, part = _cuda_grads(enc, rgbs, dfm)
    assert set(part) == set(full) - frozen
    assert all(torch.equal(part[n], full[n]) for n in part)


@pytest.mark.gpu
def test_data_parallel_replica_on_one_gpu():
    """A replica made by torch.nn.parallel.replicate (what nn.DataParallel runs) lists no parameters: the gradients flow
    through its broadcast copies to the original parameters, with the bits of a direct call."""
    enc = _encoder(8)
    rgbs = _rgbs(1, 2, 96, 128, seed=2)
    dfm = torch.randn(2, 128, 12, 16, device=DEV)
    f1, g1 = _cuda_grads(enc, rgbs, dfm)
    enc.zero_grad(set_to_none=True)
    replica = torch.nn.parallel.replicate(enc, [0])[0]
    assert len(list(replica.parameters())) == 0
    f = torch_path.encoder_cuda(replica, rgbs)
    f.backward(dfm.view(1, 2, *dfm.shape[1:]))
    assert torch.equal(f.detach().flatten(0, 1), f1)
    assert all(torch.equal(p.grad, g1[n]) for n, p in enc.named_parameters())
    assert not hasattr(enc.conv2, "_wtc") and not hasattr(enc.conv1, "_wstem")      # no module caches written


def _train_model(encoder_path, seed=3):
    m = Pips(S=8, stride=8, loss_path="fused", mixer_path="cuda", encoder_path=encoder_path).to(DEV).train()
    m.load_state_dict(po.init_state_dict(seed=seed, head_scale=0.05), strict=True)
    return m


def _train_inputs(B=1, N=64, H=128, W=160, seed=5):
    rgbs = po.smooth_video(B, 8, H, W, seed=100 + seed).to(DEV)
    xys = po.random_queries(B, N, H, W, seed=200 + seed).to(DEV)
    g = torch.Generator().manual_seed(400 + seed)
    tg = (xys.cpu()[:, None] + torch.cumsum(torch.randn(B, 8, N, 2, generator=g) * 3.0, 1)).to(DEV)
    vg = (torch.rand(B, 8, N, generator=g) > 0.2).float().to(DEV)
    va = (torch.rand(B, 8, N, generator=g) > 0.1).float().to(DEV)
    return rgbs, xys, tg, vg, va


def _train_step(m, rgbs, xys, tg, vg, va, iters):
    m.zero_grad(set_to_none=True)
    _, _, _, losses = m(xys, rgbs, iters=iters, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    sum(losses).backward()
    return [l.detach() for l in losses], {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [1, 3])
def test_training_step_matches_torch_encoder(monkeypatch, iters):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    inputs = _train_inputs()
    lt, gt = _train_step(_train_model("torch"), *inputs, iters=iters)
    lc, gc = _train_step(_train_model("cuda"), *inputs, iters=iters)
    rel_l = [abs(a.item() - b.item()) / abs(b.item()) for a, b in zip(lc, lt)]
    assert set(gt) == set(gc)

    def rel(a, b):
        return ((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-300)).item()

    total = torch.cat([g.flatten() for g in gt.values()]).double().norm().item()
    # biases with an exact gradient of 0 (a following normalisation removes them) are compared to the whole norm
    zero = {n for n in gt if n.endswith("bias") and gt[n].double().norm().item() <= 1e-5 * total}
    fnet_zero = [n for n in gc if n.startswith("fnet.") and n.endswith("bias") and n != "fnet.conv3.bias"]
    assert set(fnet_zero) <= zero and len(fnet_zero) == 21
    rel_g = {n: rel(gc[n], gt[n]) for n in gt if n not in zero}
    noise = max((gc[n] - gt[n]).double().norm().item() / total for n in zero)
    worst = max(rel_g, key=rel_g.get)
    rel_all = rel(torch.cat([gc[n].flatten() for n in gt]), torch.cat([gt[n].flatten() for n in gt]))
    print(f"iters={iters}: losses relative {rel_l}; all gradients {rel_all:.2e}; worst gradient {worst} {rel_g[worst]:.2e}; "
          f"{len(zero)} zero-gradient biases, difference {noise:.2e} of the norm")
    # the encoder's gradients differ like test_encoder_cuda_matches_fp64_autograd's (ReLU decisions of a bf16x3 forward)
    assert max(rel_l) <= 1e-4 and rel_all <= 3e-2 and rel_g[worst] <= 3e-2 and noise <= 1e-5
    assert all((gc[n] == 0).all() for n in fnet_zero)


@pytest.mark.gpu
def test_memory_after_forward():
    """32 frames of 384x512: what the forward keeps until the backward, above its output"""
    enc = _encoder(8)
    rgbs = _rgbs(4, 8, 384, 512, seed=1)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    f = torch_path.encoder_cuda(enc, rgbs)
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - base - f.numel() * 4
    print(f"held after the forward at 32 x 384x512: {held / 2**20:.0f} MiB ({held / 32 / 2**20:.1f} MiB per frame)")
    assert held <= 32 * 64 * 2**20
    f.backward(torch.ones_like(f))
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_routing(monkeypatch):
    rgbs, xys, tg, vg, va = _train_inputs(N=16, seed=8)
    calls = []
    real = torch_path.encoder_cuda

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(torch_path, "encoder_cuda", spy)
    m = _train_model(None)
    assert m.encoder_path == "torch"
    m(xys, rgbs, iters=1, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert calls == []                                              # the default keeps the module
    monkeypatch.setenv("PIPS_B200_ENCODER", "cuda")
    m = _train_model(None)
    assert m.encoder_path == "cuda"
    _, _, _, losses = m(xys, rgbs, iters=1, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert calls == [1] and losses[0].requires_grad
    m(xys, rgbs.clone().requires_grad_(True), iters=1, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert calls == [1]                                             # an image that wants a gradient keeps the module
    mc = Pips(S=8, stride=8, encoder_path="cuda").train()
    mc.load_state_dict(po.init_state_dict(seed=3, head_scale=0.05))
    mc(xys.cpu(), rgbs.cpu()[..., :64, :64], iters=1, is_train=True)
    assert calls == [1]                                             # CPU tensors keep the module
    with torch.no_grad():                                           # plain inference: fnet_tc, untouched
        m(xys, rgbs, iters=1)
    assert calls == [1]
    # no_grad: the path keeps nothing but its output
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        out = real(m.fnet, rgbs)
    torch.cuda.synchronize()
    kept = torch.cuda.memory_allocated() - base
    print(f"kept under no_grad: {kept} B, output {out.numel() * 4} B")
    assert out.grad_fn is None and kept <= out.numel() * 4 + 2**20
    assert _train_model("torch").encoder_path == "torch"            # the argument wins over the environment


@pytest.mark.gpu
def test_encoder_cuda_rejects_bad_inputs():
    enc = _encoder(8)
    with pytest.raises(RuntimeError):
        torch_path.encoder_cuda(enc, torch.zeros(1, 1, 3, 64, 64))
    with pytest.raises(ValueError):
        torch_path.encoder_cuda(enc, torch.zeros(1, 3, 64, 64, device=DEV))
    with pytest.raises(ValueError):
        torch_path.encoder_cuda(enc, torch.zeros(1, 1, 3, 64, 64, device=DEV, requires_grad=True))
    with pytest.raises(ValueError):
        torch_path.encoder_cuda(torch.nn.Linear(3, 3).to(DEV), torch.zeros(1, 1, 3, 64, 64, device=DEV))
