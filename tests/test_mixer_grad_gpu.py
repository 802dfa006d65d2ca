"""Training the DeltaBlock mixer on the sm_90a kernels (Pips(mixer_path='cuda'), torch_path.delta_block_cuda): the
weight-gradient GEMM, the pre-activation GEMM epilogues and the fused LayerNorm / token-mixing backward against fp64,
the whole mixer's forward and backward against fp64 autograd of the DeltaBlock module, stale rows, determinism, a
training step against mixer_path='torch', memory, routing, and argument validation without a GPU.

The CUDA-core backward kernels (pips_tokenmix_grad, pips_ln_pool_grad) are checked per element against fp64 references
that follow their formulas, in units of U * magnitude: the magnitude is the same backward evaluated on absolute values
with every subtraction turned into an addition (test_loop_kernels_gpu.py's convention).  The bounds are the largest
ratio measured on an H100 80GB HBM3 with a margin of 2-4x.  The whole DeltaBlock is checked per tensor as
max|err| / max|ref|.  The GEMM pieces are checked norm-wise here (``_rel``) and bit for bit in test_tc_exact_gpu.py."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import pips_oracle as po
from pips_b200 import Pips, _lib as L, torch_path
from pips_b200.pips import DeltaBlock
from tests.test_loop_kernels_gpu import _bits, _ln_mag, _nan, _ratio, _report, _tokenmix_inputs

DEV = "cuda:0"

# Bounds, in units of U * magnitude (U = 2^-24), per element.  The kernels' sums run in a fixed order, so these inputs
# give the same ratios on every run.
C_TG_DX = 1.0          # pips_tokenmix_grad dx (measured 0.40, plain rows at 2049 sequences)
C_TG_LN2 = 6.0         # its ln2_w and ln2_b gradients (measured 2.3, plain, 1 sequence): dy is exact, so the magnitudes
                       # of their terms are tight
C_TG_PARAM = 0.5       # its other 1576 gradients (measured 0.19, tok_w1): their terms pass through dh and du, whose
                       # magnitudes carry the rounding of the recomputed hidden layer
C_LP_DX = 10.0         # pips_ln_pool_grad dx (measured 3.9, plain rows at 2049 sequences)
C_LP_PARAM = 12.0      # its ln_w and ln_b gradients (measured 4.9, ln_b at 37 sequences)
# The whole DeltaBlock, max|err| / max|ref| per tensor.  A bf16x3 product or (hi, lo) pair carries about 2^-17 relative
# error, and a gradient passes through the 38 GEMMs of the forward and about as many of the backward; the rounding
# errors mostly cancel, and the largest measured is 5.8 x 2^-17 (4.4e-5, block 11's FC1 bias at R = 3072, head x0.05).
# Strict fp32 torch stays below 4.2e-6, so this floor sets every bound.
MIX_FLOOR = 16 * 2.0 ** -17


def _rel(a, b):
    """norm-wise relative error ||a - b|| / ||b|| (in fp64)"""
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-300)).item()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _split(v, rows=None):
    """(hi, lo) bf16 of the fp32 matrix v, in buffers of `rows` rows (default: v's)"""
    v = v.float().contiguous()
    rows = rows or v.shape[0]
    hi = torch.full((rows, v.shape[1]), float("nan"), dtype=torch.bfloat16, device=DEV)
    lo = hi.clone()
    L.check(L.load().pips_split_bf16(L.ptr(v), L.ptr(hi), L.ptr(lo), v.numel(), _st()), "pips_split_bf16")
    return hi, lo


def _wgrad(g, x):
    lib = L.load()
    M, N = g.shape
    K = x.shape[1]
    gp, xp = _split(g), _split(x)
    dw = torch.full((N, K), float("nan"), device=DEV)
    n = lib.pips_wgrad_scratch_floats(M, N, K)
    scratch = torch.full((max(n, 1),), float("nan"), device=DEV)
    L.check(lib.pips_wgrad(L.ptr(gp[0]), L.ptr(gp[1]), N, L.ptr(xp[0]), L.ptr(xp[1]), K, M, N, K, L.ptr(scratch), L.ptr(dw),
                           _st()), "pips_wgrad")
    return dw


WGRAD_SHAPES = [  # (M, N, K): FC2 (dx^T h), FC1 (dh^T y), input layer, head over pooled rows; M not a multiple of a tile
    (8 * 3072, 512, 2048),
    (8 * 3071, 2048, 512),
    (8 * 37, 512, 576),
    (3072, 1040, 512),
    (37, 1040, 512),
    (8, 512, 576),
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", WGRAD_SHAPES)
def test_wgrad_matches_fp64(M, N, K):
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    G = torch.randn(M, N, device=DEV, generator=g)
    X = torch.randn(M, K, device=DEV, generator=g) + 0.5
    dw = _wgrad(G, X)
    ref = G.double().t() @ X.double()
    e, e32 = _rel(dw, ref), _rel(G.t() @ X, ref)
    print(f"wgrad M={M} N={N} K={K}: {e:.2e} (fp32 torch {e32:.2e})")
    assert torch.isfinite(dw).all()
    assert e <= 1e-4
    assert torch.equal(dw, _wgrad(G, X))                                  # the same bits on a second run


@pytest.mark.gpu
@pytest.mark.parametrize("M,N", [(8 * 3071, 2048), (37, 1040), (300, 512)])
def test_colsum_matches_fp64(M, N):
    lib = L.load()
    G = torch.randn(M, N, device=DEV) + 0.25
    out = torch.empty(N, device=DEV)
    n = lib.pips_colsum_scratch_floats(M, N)
    scratch = torch.empty(max(n, 1), device=DEV)
    L.check(lib.pips_colsum(L.ptr(G), None, None, N, M, N, L.ptr(scratch), L.ptr(out), _st()), "pips_colsum")
    hi, lo = _split(G)
    out2 = torch.empty(N, device=DEV)
    L.check(lib.pips_colsum(None, L.ptr(hi), L.ptr(lo), N, M, N, L.ptr(scratch), L.ptr(out2), _st()), "pips_colsum")
    ref = G.double().sum(0)
    print(f"colsum M={M} N={N}: fp32 {_rel(out, ref):.2e}, (hi, lo) {_rel(out2, ref):.2e}")
    assert _rel(out, ref) <= 1e-5 and _rel(out2, ref) <= 1e-4


def _gelu_grad64(x):
    return 0.5 * torch.erfc(-x / math.sqrt(2.0)) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [8 * 37, 2048 + 8])
def test_pre_activation_epilogues_match_fp64(M):
    lib = L.load()
    N, K = 2048, 512
    g = torch.Generator(device=DEV).manual_seed(M)
    A = torch.randn(M, K, device=DEV, generator=g)
    W = torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)
    b = torch.randn(N, device=DEV, generator=g)
    b[::7] += 9.0                                                         # pre-activations in both GELU tails, |x| > 6
    b[3::7] -= 9.0
    ap, wp = _split(A, 256 * ((M + 255) // 256)), _split(W)
    hi = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    lo = hi.clone()
    pre = torch.full((M, N), float("nan"), device=DEV)
    L.check(lib.pips_gemm_tc_aux(L.ptr(ap[0]), L.ptr(ap[1]), K, ap[0].shape[0], L.ptr(wp[0]), L.ptr(wp[1]), K, N, M, N, K,
                                 L.ptr(b), L.EPI_BIAS_GELU_PRE, None, 0, L.ptr(hi), L.ptr(lo), N, L.ptr(pre), N, _st()),
            "pips_gemm_tc_aux")
    h64 = A.double() @ W.double().t() + b.double()
    gelu64 = F.gelu(h64)
    e_pre, e_gelu = _rel(pre, h64), _rel(hi.double() + lo.double(), gelu64)
    tails = h64.abs() > 6
    e_tail = _rel((hi.double() + lo.double())[tails], gelu64[tails])
    # GELU_GRAD: (A W^T + b) * gelu'(pre), with the pre-activation just written
    dh_hi = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    dh_lo = dh_hi.clone()
    L.check(lib.pips_gemm_tc_aux(L.ptr(ap[0]), L.ptr(ap[1]), K, ap[0].shape[0], L.ptr(wp[0]), L.ptr(wp[1]), K, N, M, N, K,
                                 L.ptr(b), L.EPI_GELU_GRAD, None, 0, L.ptr(dh_hi), L.ptr(dh_lo), N, L.ptr(pre), N, _st()),
            "pips_gemm_tc_aux")
    dref = h64 * _gelu_grad64(pre.double())
    e_grad = _rel(dh_hi.double() + dh_lo.double(), dref)
    e_gtail = _rel((dh_hi.double() + dh_lo.double())[tails], dref[tails])
    print(f"M={M}: pre {e_pre:.2e}, gelu {e_gelu:.2e} (tails {e_tail:.2e}), gelu' product {e_grad:.2e} (tails {e_gtail:.2e}); "
          f"{int(tails.sum())} tail elements")
    assert tails.sum() > 1000
    assert max(e_pre, e_gelu, e_tail, e_grad, e_gtail) <= 1e-4


GELU_GRAD_ZERO = -0.7517915246935644                     # gelu'(h) = Phi(h) + h phi(h) = 0: its two terms cancel
TOK_PARAMS = ("ln1_w", "ln1_b", "tok_w1", "tok_b1", "tok_w2", "tok_b2", "ln2_w", "ln2_b")   # the order of the 2600 gradients


def _tok_params(seed):
    """Token-mixing block parameters.  Hidden units 0, 8, 16, 24 sit in GELU's positive tail (h > 6 nearly everywhere),
    units 1, 9, 17, 25 in its negative tail, and units 2, 10, 18, 26 within about 3e-3 of gelu''s zero crossing."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = {"ln1_w": 1 + 0.2 * torch.randn(512, generator=g, device=DEV), "ln1_b": 0.1 * torch.randn(512, generator=g, device=DEV),
         "tok_w1": torch.randn(32, 8, generator=g, device=DEV) / math.sqrt(8), "tok_b1": 0.3 * torch.randn(32, generator=g, device=DEV),
         "tok_w2": torch.randn(8, 32, generator=g, device=DEV) / math.sqrt(32), "tok_b2": 0.1 * torch.randn(8, generator=g, device=DEV),
         "ln2_w": 1 + 0.2 * torch.randn(512, generator=g, device=DEV), "ln2_b": 0.1 * torch.randn(512, generator=g, device=DEV)}
    P["tok_b1"][0::8] += 9.0
    P["tok_b1"][1::8] -= 9.0
    P["tok_w1"][2::8] *= 1e-3
    P["tok_b1"][2::8] = GELU_GRAD_ZERO
    return {k: v.contiguous() for k, v in P.items()}


def _tok_block64(x, P):
    """the token-mixing PreNormResidual and the LayerNorm of the channel-mixing one, in fp64: (x_mid, LN2(x_mid))"""
    u = F.layer_norm(x, (512,), P["ln1_w"], P["ln1_b"])
    h = F.gelu(torch.einsum("js,rsc->rjc", P["tok_w1"], u) + P["tok_b1"][None, :, None])
    x_mid = torch.einsum("sj,rjc->rsc", P["tok_w2"], h) + P["tok_b2"][None, :, None] + x
    return x_mid, F.layer_norm(x_mid, (512,), P["ln2_w"], P["ln2_b"])


def _ln_back64(x, dy, dymag, w):
    """fp64 LayerNorm backward over the last axis with ln_backward8's formulas (mixer_grad.cu): xh = (x - m) r and
    dx = r (w dy - mean(w dy) - xh mean(w dy xh)).  Returns dx and the per-element terms dy xh of the weight gradient,
    each with the magnitude of its terms: every subtraction becomes an addition, |x - m| becomes (|x| + |m|) r
    (_ln_mag), and dy comes with its own magnitude dymag."""
    m = x.mean(-1, keepdim=True)
    xhmag, r = _ln_mag(x, torch.ones_like(w), torch.zeros_like(w))
    xh = (x - m) * r
    gd, gdmag = dy * w, dymag * w.abs()
    a, amag = gd.mean(-1, keepdim=True), gdmag.mean(-1, keepdim=True)
    b, bmag = (gd * xh).mean(-1, keepdim=True), (gdmag * xhmag).mean(-1, keepdim=True)
    return r * (gd - a - xh * b), r * (gdmag + amag + xhmag * bmag), dy * xh, dymag * xhmag


def _gelu64(h, hmag):
    """gelu(h) and gelu'(h) in fp64 with the magnitudes of common.cuh's formulas: 0.5 h (1 + erf(h / sqrt 2)) and
    Phi(h) + h phi(h), each plus |its derivative| times the magnitude of h (the rounding of the recomputed h)."""
    phi = torch.exp(-0.5 * h * h) / math.sqrt(2.0 * math.pi)
    Phi = 0.5 * torch.erfc(-h / math.sqrt(2.0))
    d1, d2 = Phi + h * phi, phi * (2.0 - h * h)
    amag = 0.5 * h.abs() * (1.0 + torch.erf(h / math.sqrt(2.0)).abs()) + d1.abs() * hmag
    return h * Phi, amag, d1, Phi + h.abs() * phi + d2.abs() * hmag


def _tokenmix_grad64(x, xm, dy, dxo, P):
    """pips_tokenmix_grad in fp64, with the formulas of the comment above tokenmix_grad_kernel: dz = dxo + LN2^T(dy),
    da = W2^T dz, dh = da gelu'(h), du = W1^T dh, dx = dz + LN1^T(du), and the 8 parameter sums.  Every result comes as
    (value, magnitude): the same backward on absolute values (_ln_back64, _gelu64).  x, xm, dy, dxo: (seqs, 8, 512)."""
    d = {k: v.double() for k, v in P.items()}
    out = {}
    dl, dlmag, tw, twmag = _ln_back64(xm, dy, dy.abs(), d["ln2_w"])
    dz, dzmag = dxo + dl, dxo.abs() + dlmag
    out["ln2_w"], out["ln2_b"] = (tw.sum((0, 1)), twmag.sum((0, 1))), (dy.sum((0, 1)), dy.abs().sum((0, 1)))
    umag, r = _ln_mag(x, d["ln1_w"], d["ln1_b"])
    u = (x - x.mean(-1, keepdim=True)) * r * d["ln1_w"] + d["ln1_b"]
    w1, w2 = d["tok_w1"], d["tok_w2"]
    h = torch.einsum("js,rsc->rjc", w1, u) + d["tok_b1"][None, :, None]
    hmag = torch.einsum("js,rsc->rjc", w1.abs(), umag) + d["tok_b1"].abs()[None, :, None]
    a, amag, gp, gpmag = _gelu64(h, hmag)
    dh = torch.einsum("sj,rsc->rjc", w2, dz) * gp
    dhmag = torch.einsum("sj,rsc->rjc", w2.abs(), dzmag) * gpmag
    out["tok_w1"] = (torch.einsum("rjc,rsc->js", dh, u), torch.einsum("rjc,rsc->js", dhmag, umag))
    out["tok_b1"] = (dh.sum((0, 2)), dhmag.sum((0, 2)))
    out["tok_w2"] = (torch.einsum("rsc,rjc->sj", dz, a), torch.einsum("rsc,rjc->sj", dzmag, amag))
    out["tok_b2"] = (dz.sum((0, 2)), dzmag.sum((0, 2)))
    du, dumag = torch.einsum("js,rjc->rsc", w1, dh), torch.einsum("js,rjc->rsc", w1.abs(), dhmag)
    dl, dlmag, tw, twmag = _ln_back64(x, du, dumag, d["ln1_w"])
    out["ln1_w"], out["ln1_b"] = (tw.sum((0, 1)), twmag.sum((0, 1))), (du.sum((0, 1)), dumag.sum((0, 1)))
    out["dx"] = (dz + dl, dzmag + dlmag)
    return out


@pytest.mark.gpu
def test_tokenmix_grad_reference_matches_autograd():
    """_tokenmix_grad64 against fp64 autograd of _tok_block64, with x_mid = the forward's, on flat rows and GELU tails:
    the per-element reference of test_tokenmix_grad_per_element is the module's gradient."""
    P = _tok_params(5)
    x = _grad_rows("flat", 37, 501).double().to(DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    dy, dxo = (torch.randn(37, 8, 512, generator=g, device=DEV, dtype=torch.float64) for _ in range(2))
    P64 = {k: v.double().requires_grad_(True) for k, v in P.items()}
    x64 = x.clone().requires_grad_(True)
    x_mid, y = _tok_block64(x64, P64)
    ((y * dy).sum() + (x_mid * dxo).sum()).backward()
    ref = _tokenmix_grad64(x, x_mid.detach(), dy, dxo, P)
    errs = {k: _rel(ref[k][0], (x64 if k == "dx" else P64[k]).grad) for k in ("dx",) + TOK_PARAMS}
    print("explicit fp64 backward vs fp64 autograd: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) <= 1e-10


_ROWS = {}


def _grad_rows(kind, seqs, seed):
    """(seqs, 8, 512) fp32 rows on the host: "plain" randn, "offset" (_tokenmix_inputs: mean ~100, spread ~1), "flat"
    (randn with every third row and every fifth sequence made of one value repeated over the 512 channels) or
    "nearflat" (a common value per row and a spread of 1e-3: the variance, 1e-6, is below LayerNorm's epsilon).  Made
    at 2049 sequences and cut, so a smaller call sees the first rows of a larger one."""
    key = (kind, seed)
    if key not in _ROWS:
        x = _tokenmix_inputs(2049, kind == "offset", seed)
        if kind == "flat":
            flat = (torch.arange(2049 * 8) % 3 == 0).view(2049, 8)
            flat[::5] = True
            x[flat] = x[flat][:, :1].expand(-1, 512).contiguous()
        elif kind == "nearflat":
            x = 0.5 + torch.randn(2049, 8, 1, generator=torch.Generator().manual_seed(seed + 1)) + 1e-3 * x
        _ROWS[key] = x
    return _ROWS[key][:seqs]


def _padded(t, seqs):
    """t (seqs, 8, 512) on the device in a buffer of seqs + 1 sequences, the last one NaN"""
    out = torch.full((seqs + 1, 8, 512), float("nan"), device=DEV)
    out[:seqs] = t
    return out


def _tokenmix_grad_call(x, xm, dy, dxo, P, seqs):
    """pips_tokenmix_grad over the first `seqs` sequences of NaN-padded buffers, with NaN scratch and NaN grads 64 floats
    longer than the 2600 it writes.  Returns dx (all seqs + 1 sequences) and grads (2664 floats) on the host."""
    lib = L.load()
    dx = _padded(dxo[:seqs], seqs)
    scratch = _nan(lib.pips_tokenmix_grad_scratch_floats(seqs))
    grads = _nan(2600 + 64)
    ins = [_padded(t[:seqs], seqs) for t in (x, xm, dy)]
    L.check(lib.pips_tokenmix_grad(*(L.ptr(t) for t in ins), L.ptr(dx), seqs, *(L.ptr(P[k]) for k in TOK_PARAMS),
                                   L.ptr(scratch), L.ptr(grads), _st()), "pips_tokenmix_grad")
    torch.cuda.synchronize()
    return dx.cpu(), grads.cpu()


GRAD_KINDS = ["plain", "offset", "flat", "nearflat"]
GRAD_SEQS = [1, 37, 700, 2049]       # 700: a partial last CTA; 2049: 257 CTAs, so the partial rows take two colsum levels


@pytest.mark.gpu
@pytest.mark.parametrize("kind", GRAD_KINDS)
@pytest.mark.parametrize("seqs", GRAD_SEQS)
def test_tokenmix_grad_per_element(seqs, kind):
    """pips_tokenmix_grad per element against _tokenmix_grad64: dx and each of the 2600 gradients within C_TG_* units of
    U * magnitude.  x and x_mid are both inputs of the kernel and both take the row kind; the GELU-tail parameters
    of _tok_params throughout.  dx is updated in place and grads is written exactly; the bits repeat, and the first 37
    sequences' dx does not depend on how many sequences share the call."""
    P = _tok_params(seqs)
    x, xm = _grad_rows(kind, seqs, 111), _grad_rows(kind, seqs, 112)
    g = torch.Generator().manual_seed(113)
    dy, dxo = torch.randn(2049, 8, 512, generator=g)[:seqs], torch.randn(2049, 8, 512, generator=g)[:seqs]
    dev = [t.to(DEV) for t in (x, xm, dy, dxo)]
    dx, grads = _tokenmix_grad_call(*dev, P, seqs)
    assert torch.isnan(dx[seqs]).all(), "pips_tokenmix_grad wrote dx past the last sequence"
    assert not torch.isnan(grads[:2600]).any() and torch.isnan(grads[2600:]).all(), "grads: not exactly 2600 floats written"
    dx2, grads2 = _tokenmix_grad_call(*dev, P, seqs)
    assert torch.equal(_bits(dx), _bits(dx2)) and torch.equal(_bits(grads), _bits(grads2)), "a second run differs"
    if seqs > 37:
        dx37, _ = _tokenmix_grad_call(*dev, P, 37)
        assert torch.equal(_bits(dx[:37]), _bits(dx37[:37])), "dx of the first 37 sequences depends on seqs"
    ref = _tokenmix_grad64(*(t.double() for t in dev), P)
    tag = f"tokenmix_grad seqs={seqs} {kind}"
    u = F.layer_norm(dev[0].double(), (512,), P["ln1_w"].double(), P["ln1_b"].double())
    hidden = torch.einsum("js,rsc->rjc", P["tok_w1"].double(), u) + P["tok_b1"].double()[None, :, None]
    print(f"{tag}: {int((hidden > 6).sum())} h > 6, {int((hidden < -6).sum())} h < -6, "
          f"{int(((hidden - GELU_GRAD_ZERO).abs() < 0.01).sum())} |h - h0| < 0.01")
    _report(f"{tag} dx: err / (U mag)", _ratio(dx[:seqs], ref["dx"][0], ref["dx"][1]), C_TG_DX)
    off = 0
    for k in TOK_PARAMS:
        n = P[k].numel()
        _report(f"{tag} {k}: err / (U mag)", _ratio(grads[off:off + n], ref[k][0].reshape(-1), ref[k][1].reshape(-1)),
                C_TG_LN2 if k.startswith("ln2") else C_TG_PARAM)
        off += n


def _ln_pool_grad_call(x, dp, w, b, seqs):
    """pips_ln_pool_grad over `seqs` sequences: x and dx in buffers of seqs + 1 sequences (x's last NaN), NaN scratch and
    NaN grads 64 floats longer than the 1024 it writes.  Returns dx and grads on the host."""
    lib = L.load()
    xd = _padded(x, seqs)
    dx = _nan(seqs + 1, 8, 512)
    scratch = _nan(lib.pips_ln_pool_grad_scratch_floats(seqs))
    grads = _nan(1024 + 64)
    L.check(lib.pips_ln_pool_grad(L.ptr(xd), L.ptr(dp), seqs, L.ptr(w), L.ptr(b), L.ptr(dx), L.ptr(scratch), L.ptr(grads),
                                  _st()), "pips_ln_pool_grad")
    torch.cuda.synchronize()
    return dx.cpu(), grads.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", GRAD_KINDS[:3])
@pytest.mark.parametrize("seqs", GRAD_SEQS)
def test_ln_pool_grad_per_element(seqs, kind):
    """pips_ln_pool_grad (the backward of LayerNorm -> mean over the 8 rows) per element against fp64: dx within C_LP_DX
    and the 1024 gradients within C_LP_PARAM units of U * magnitude.  dx is overwritten (it starts NaN, rows past seqs
    stay NaN), ln_b is not read (NaN there gives the same bits), and exactly 1024 floats of grads are written."""
    g = torch.Generator(device=DEV).manual_seed(seqs)
    w = (1 + 0.2 * torch.randn(512, generator=g, device=DEV)).contiguous()
    b = 0.1 * torch.randn(512, generator=g, device=DEV)
    x = _grad_rows(kind, seqs, 121).to(DEV)
    dp = torch.randn(2049, 512, generator=torch.Generator().manual_seed(122))[:seqs].to(DEV)
    dx, grads = _ln_pool_grad_call(x, dp, w, b, seqs)
    assert not torch.isnan(dx[:seqs]).any() and torch.isnan(dx[seqs]).all(), "dx: not exactly the live rows written"
    assert not torch.isnan(grads[:1024]).any() and torch.isnan(grads[1024:]).all(), "grads: not exactly 1024 floats written"
    dx_nb, grads_nb = _ln_pool_grad_call(x, dp, w, torch.full_like(b, float("nan")), seqs)
    assert torch.equal(_bits(dx), _bits(dx_nb)) and torch.equal(_bits(grads), _bits(grads_nb)), "ln_b changed the result"
    x64, dp64 = x.double(), dp.double()
    gy = (dp64 / 8)[:, None, :].expand(-1, 8, -1)
    ref, mag, tw, twmag = _ln_back64(x64, gy, gy.abs(), w.double())
    tag = f"ln_pool_grad seqs={seqs} {kind}"
    _report(f"{tag} dx: err / (U mag)", _ratio(dx[:seqs], ref, mag), C_LP_DX)
    _report(f"{tag} ln_w: err / (U mag)", _ratio(grads[:512], tw.sum((0, 1)), twmag.sum((0, 1))), C_LP_PARAM)
    _report(f"{tag} ln_b: err / (U mag)", _ratio(grads[512:1024], gy.sum((0, 1)), gy.abs().sum((0, 1))), C_LP_PARAM)


def _delta_block(seed, head_scale, dtype=torch.float32):
    sd = po.init_state_dict(seed=seed, head_scale=head_scale)
    m = DeltaBlock().to(DEV, dtype)
    m.load_state_dict({k[len("delta_block."):]: v for k, v in sd.items() if k.startswith("delta_block.")})
    return m


def _mixer_input(R, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(R, 8, 519, generator=g, device=DEV)


def _fwd_bwd(m, x, cuda, dy):
    m.zero_grad(set_to_none=True)
    xr = x.clone().requires_grad_(True)
    out = torch_path.delta_block_cuda(m, xr) if cuda else m(xr)
    (out * dy).sum().backward()
    return out.detach(), xr.grad, {n: p.grad.detach().clone() for n, p in m.named_parameters()}


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 37, 3072])
@pytest.mark.parametrize("head_scale", [0.05, 1.0])
def test_delta_block_cuda_matches_fp64_autograd(monkeypatch, R, head_scale):
    """The output, dx and each of the 150 parameter gradients against fp64 autograd of the module, as max|err| / max|ref|
    per tensor, within max(2 x strict fp32 torch's own error, MIX_FLOOR).  The token-mixing FC2 biases have an exact
    gradient of 0 (every path from them meets a LayerNorm that removes a per-row constant): they are compared to the
    norm of all gradients instead."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    m = _delta_block(3, head_scale)
    m64 = _delta_block(3, head_scale, torch.float64)
    x = _mixer_input(R, R)
    dy = torch.randn(R, 8, 130, device=DEV, generator=torch.Generator(device=DEV).manual_seed(R + 1))
    o64, dx64, g64 = _fwd_bwd(m64, x.double(), False, dy.double())
    oc, dxc, gc = _fwd_bwd(m, x, True, dy)
    o32, dx32, g32 = _fwd_bwd(m, x, False, dy)
    assert len(gc) == 150
    total = torch.cat([g.flatten() for g in g64.values()]).norm().item()
    zero = {n for n in g64 if g64[n].norm().item() <= 1e-6 * total}
    assert all(n.endswith("0.fn.3.bias") for n in zero) and len(zero) == 12, zero
    noise = max((gc[n].double() - g64[n]).norm().item() / total for n in zero)

    def err(a, b):
        return ((a.double() - b).abs().max() / b.abs().max().clamp(min=1e-300)).item()

    cases = {"out": (oc, o32, o64), "dx": (dxc, dx32, dx64), **{n: (gc[n], g32[n], g64[n]) for n in g64 if n not in zero}}
    e = {n: (err(c, r), err(t, r)) for n, (c, t, r) in cases.items()}
    ratio = {n: ec / max(2 * et, MIX_FLOOR) for n, (ec, et) in e.items()}
    worst = max(ratio, key=ratio.get)
    top = sorted(e, key=lambda n: e[n][0], reverse=True)[:4]
    print(f"R={R} head x{head_scale}: max|err| / max|ref|, cuda / fp32 torch: out {e['out'][0]:.2e} / {e['out'][1]:.2e}, "
          f"dx {e['dx'][0]:.2e} / {e['dx'][1]:.2e}, largest " + ", ".join(f"{n} {e[n][0]:.2e} / {e[n][1]:.2e}" for n in top)
          + f"; worst against its bound {worst} {ratio[worst]:.2f}; {len(zero)} zero-gradient biases {noise:.2e} of the norm")
    assert ratio[worst] <= 1.0 and noise <= 1e-5


def _fwd_bwd_filled(m, x, dy, fill, monkeypatch):
    """_fwd_bwd on the CUDA path with every uninitialised allocation of the delta_block_cuda call (torch.empty and
    _MixerRun.rows, in its forward and its backward) filled with `fill`"""
    real = torch.empty

    def empty(*a, **k):
        return real(*a, **k).fill_(fill)

    m.zero_grad(set_to_none=True)
    xr = x.clone().requires_grad_(True)
    with monkeypatch.context() as mp:
        mp.setattr(torch, "empty", empty)
        mp.setattr(torch_path._MixerRun, "rows", lambda self, n, cols, dtype=torch.float32: empty(n, cols, dtype=dtype,
                                                                                                   device=self.dev))
        out = torch_path.delta_block_cuda(m, xr)
        (out * dy).sum().backward()
    return out.detach(), xr.grad, {n: p.grad.detach().clone() for n, p in m.named_parameters()}


@pytest.mark.gpu
def test_delta_block_cuda_stale_rows(monkeypatch):
    """Every buffer of a call holds whole 256-row tiles (M = 296 rows at R = 37 live in 512-row buffers) from the
    caching allocator, and rows past M are never written: whatever they hold must not reach a result.  With every
    uninitialised allocation filled with NaN, and then with zeros, the output, dx and all 150 gradients have the same
    bits, and no NaN."""
    m = _delta_block(3, 1.0)
    x = _mixer_input(37, 71)
    dy = torch.randn(37, 8, 130, device=DEV, generator=torch.Generator(device=DEV).manual_seed(72))
    nan = _fwd_bwd_filled(m, x, dy, float("nan"), monkeypatch)
    zero = _fwd_bwd_filled(m, x, dy, 0.0, monkeypatch)
    assert len(zero[2]) == 150
    for name, a, b in [("out", nan[0], zero[0]), ("dx", nan[1], zero[1])] + [(n, nan[2][n], zero[2][n]) for n in zero[2]]:
        assert not torch.isnan(b).any(), f"{name}: NaN with zero-filled buffers"
        assert torch.equal(_bits(a), _bits(b)), f"{name}: stale rows changed the result"


@pytest.mark.gpu
def test_delta_block_cuda_prefix():
    """The output and dx of a sequence do not depend on how many other sequences share the call: the first 37 rows are
    the same bits at R = 37 and R = 300."""
    m = _delta_block(3, 1.0)
    x = _mixer_input(300, 73)
    dy = torch.randn(300, 8, 130, device=DEV, generator=torch.Generator(device=DEV).manual_seed(74))
    o300, dx300, _ = _fwd_bwd(m, x, True, dy)
    o37, dx37, _ = _fwd_bwd(m, x[:37], True, dy[:37])
    assert torch.equal(_bits(o300[:37]), _bits(o37)), "the output of the first 37 sequences depends on R"
    assert torch.equal(_bits(dx300[:37]), _bits(dx37)), "dx of the first 37 sequences depends on R"


@pytest.mark.gpu
def test_delta_block_cuda_is_deterministic():
    m = _delta_block(4, 0.05)
    x = _mixer_input(3000, 9)
    dy = torch.randn(3000, 8, 130, device=DEV)
    a, b = _fwd_bwd(m, x, True, dy), _fwd_bwd(m, x, True, dy)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(a[2][n], b[2][n]) for n in a[2])


def _train_model(mixer_path, seed=3):
    m = Pips(S=8, stride=8, loss_path="fused", mixer_path=mixer_path).to(DEV).train()
    m.load_state_dict(po.init_state_dict(seed=seed, head_scale=0.05), strict=True)
    return m


def _train_inputs(B=2, N=64, H=128, W=128, seed=5):
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
def test_training_step_matches_torch_mixer(monkeypatch, iters):
    # strict fp32 and deterministic cuDNN, as in test_losses_grad_gpu.py: the comparison then measures the mixer
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    inputs = _train_inputs()
    lt, gt = _train_step(_train_model("torch"), *inputs, iters=iters)
    lc, gc = _train_step(_train_model("cuda"), *inputs, iters=iters)
    rel_l = [abs(a.item() - b.item()) / abs(b.item()) for a, b in zip(lc, lt)]
    assert gt.keys() == gc.keys() and len(gt) > 0
    total = torch.cat([g.flatten() for g in gt.values()]).double().norm().item()
    rel_all = _rel(torch.cat([gc[n].flatten() for n in gt]), torch.cat([gt[n].flatten() for n in gt]))
    # Biases with an exact gradient of 0 (a following normalisation removes them: the token-mixing FC2 biases, fnet's conv
    # biases) are compared to the whole norm.  Every other gradient is compared to its own norm: at iters=1 the mixer's
    # are small against fnet's, but the kernels' errors are relative to each gradient.
    zero = {n for n in gt if n.endswith("bias") and gt[n].double().norm().item() <= 1e-5 * total}
    rel_g = {n: _rel(gc[n], gt[n]) for n in gt if n not in zero}
    noise = max([(gc[n] - gt[n]).double().norm().item() / total for n in zero], default=0.0)
    worst = max(rel_g, key=rel_g.get)
    print(f"iters={iters}: losses cuda {[l.item() for l in lc]} vs torch {[l.item() for l in lt]}: relative {rel_l}; all "
          f"gradients {rel_all:.2e}; {len(rel_g)} parameter gradients, worst {worst} {rel_g[worst]:.2e}; {len(zero)} "
          f"zero-gradient biases, difference {noise:.2e} of the gradient's norm")
    assert max(rel_l) <= 1e-3
    assert rel_all <= 1e-3 and rel_g[worst] <= 1e-3 and noise <= 1e-5


@pytest.mark.gpu
def test_memory_at_train_shape():
    """train.py's per-GPU shape: B=4, N=768 -> R = 3072 sequences, M = 24576 mixer rows."""
    R = 3072
    x = _mixer_input(R, 1)
    dy = torch.randn(R, 8, 130, device=DEV)
    peaks, held = {}, {}
    for name in ("cuda", "torch"):
        m = _delta_block(3, 0.05)
        xr = x.clone().requires_grad_(True)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = torch_path.delta_block_cuda(m, xr) if name == "cuda" else m(xr)
        torch.cuda.synchronize()
        held[name] = torch.cuda.memory_allocated() - base             # kept from the forward until the backward
        (out * dy).sum().backward()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del m, xr, out
    # What a call keeps between forward and backward -- a training step holds one such set per iteration: the residual
    # stream at 13 block boundaries, the (hi, lo) input rows, the output, and the packs the backward reads (fc1_w, fc1_w^T
    # and fc2_w^T as (hi, lo) bf16 per block, 12 MiB each, plus the small ones), and 32 MiB of slack.  The fp32 weight
    # copies (~100 MiB) and the forward-only packs (~52 MiB) do not fit in it.
    M = 8 * R
    budget = 13 * M * 512 * 4 + M * 576 * 4 + R * 1040 * 4 + 12 * 12 * 2**20 + 8 * 2**20 + 32 * 2**20
    print(f"DeltaBlock forward + backward at M = {M}: peak above inputs: cuda {peaks['cuda'] / 2**30:.2f} GiB, "
          f"torch {peaks['torch'] / 2**30:.2f} GiB; held from forward to backward: cuda {held['cuda'] / 2**20:.0f} MiB "
          f"(budget {budget / 2**20:.0f} MiB), torch {held['torch'] / 2**20:.0f} MiB")
    assert peaks["cuda"] <= 2.5 * 2**30
    assert held["cuda"] <= budget


@pytest.mark.gpu
def test_routing(monkeypatch):
    rgbs, xys, tg, vg, va = _train_inputs(B=1, N=16, seed=8)
    calls = []
    real = torch_path.delta_block_cuda

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(torch_path, "delta_block_cuda", spy)
    m = _train_model(None)
    assert m.mixer_path == "torch"
    mod_calls = []
    h = m.delta_block.register_forward_hook(lambda *a: mod_calls.append(1))
    m(xys, rgbs, iters=2, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert calls == [] and mod_calls == [1, 1]                       # the default keeps the torch module
    h.remove()
    monkeypatch.setenv("PIPS_B200_MIXER", "cuda")
    m = _train_model(None)
    assert m.mixer_path == "cuda"
    _, _, _, losses = m(xys, rgbs, iters=2, trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    assert calls == [1, 1] and losses[0].requires_grad
    # no gradients: the path runs and keeps nothing but its output; with gradients a call keeps the block boundaries
    mod, x = m.delta_block, _mixer_input(64, 2)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        out = torch_path.delta_block_cuda(mod, x)
    torch.cuda.synchronize()
    kept_no_grad = torch.cuda.memory_allocated() - base
    assert out.grad_fn is None and out.shape == (64, 8, 130)
    del out
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    out = torch_path.delta_block_cuda(mod, x)
    torch.cuda.synchronize()
    kept_grad = torch.cuda.memory_allocated() - base
    print(f"kept after a call: no_grad {kept_no_grad} B (output {64 * 1040 * 4} B), with gradients {kept_grad / 2**20:.1f} MiB")
    assert kept_no_grad <= 64 * 1040 * 4 + 4096
    assert kept_grad >= 13 * 512 * 512 * 4 and out.grad_fn is not None
    del out
    assert _train_model("torch").mixer_path == "torch"               # the argument wins over the environment


def test_routing_without_gpu(monkeypatch):
    with pytest.raises(ValueError):
        Pips(S=8, stride=8, mixer_path="fast")
    monkeypatch.setenv("PIPS_B200_MIXER", "bogus")
    with pytest.raises(ValueError):
        Pips(S=8, stride=8)
    # CPU tensors keep the torch module
    from tests.golden.make_golden import LOSS_CASE, case_inputs, loss_targets
    c = LOSS_CASE
    m = Pips(S=8, stride=8, mixer_path="cuda").train()
    m.load_state_dict(po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"]))
    calls = []
    m.delta_block.register_forward_hook(lambda *a: calls.append(1))
    rgbs, xys, _ = case_inputs(c)
    tg, vg, va = loss_targets(c, xys)
    _, _, _, losses = m(xys[:1, :3], rgbs[:1], iters=1, trajs_g=tg[:1, :, :3], vis_g=vg[:1, :, :3], valids=va[:1, :, :3],
                        is_train=True)
    assert calls == [1]
    sum(losses).backward()
    assert m.delta_block.to_delta[0].weight.grad is not None
    with pytest.raises(RuntimeError):
        torch_path.delta_block_cuda(m.delta_block, torch.zeros(2, 8, 519))


def test_mixer_grad_entry_points_validate_arguments_without_gpu():
    lib = L.load()
    p = C.c_void_p(256)
    q = C.c_void_p(264)                                                   # 8-byte aligned only
    wg = lib.pips_wgrad
    assert wg(None, p, 512, p, p, 512, 100, 512, 512, p, p, None) != 0
    assert b"pips_wgrad: null pointer" in lib.pips_last_error()
    assert wg(p, p, 512, p, p, 512, 0, 512, 512, p, p, None) != 0
    assert b"empty problem" in lib.pips_last_error()
    assert wg(p, p, 1036, p, p, 512, 100, 1036, 512, p, p, None) != 0     # N not a multiple of 8
    assert b"multiples of 8" in lib.pips_last_error()
    assert wg(p, p, 256, p, p, 512, 100, 512, 512, p, p, None) != 0      # ldg < N
    assert wg(q, p, 512, p, p, 512, 100, 512, 512, p, p, None) != 0      # misaligned G
    assert b"16-byte aligned" in lib.pips_last_error()
    assert wg(p, p, 512, p, p, 512, 5000, 512, 512, None, p, None) != 0  # several splits, no scratch
    assert b"scratch" in lib.pips_last_error()
    assert lib.pips_wgrad_scratch_floats(2048, 512, 512) == 0
    assert lib.pips_wgrad_scratch_floats(2049, 512, 512) == 2 * 512 * 512

    cs = lib.pips_colsum
    assert cs(None, None, None, 512, 10, 512, None, p, None) != 0
    assert b"pips_colsum: null pointer" in lib.pips_last_error()
    assert cs(p, None, None, 100, 10, 512, None, p, None) != 0          # ld < N
    assert cs(p, None, None, 512, 1000, 512, None, p, None) != 0        # several splits, no scratch
    assert b"scratch" in lib.pips_last_error()
    assert lib.pips_colsum_scratch_floats(256, 10) == 0 and lib.pips_colsum_scratch_floats(257, 10) == 20

    tg = lib.pips_tokenmix_grad
    args = [p] * 4 + [4] + [p] * 10
    bad = list(args)
    bad[1] = None
    assert tg(*bad, None) != 0 and b"pips_tokenmix_grad: null pointer" in lib.pips_last_error()
    bad = list(args)
    bad[4] = 0
    assert tg(*bad, None) != 0 and b"no sequences" in lib.pips_last_error()
    bad = list(args)
    bad[3] = q
    assert tg(*bad, None) != 0 and b"16-byte aligned" in lib.pips_last_error()

    lp = lib.pips_ln_pool_grad
    assert lp(p, None, 4, p, p, p, p, p, None) != 0 and b"pips_ln_pool_grad: null pointer" in lib.pips_last_error()
    assert lp(p, p, 0, p, p, p, p, p, None) != 0 and b"no sequences" in lib.pips_last_error()
    assert lp(p, q, 4, p, p, p, p, p, None) != 0 and b"16-byte aligned" in lib.pips_last_error()
    # one partial row of P floats per CTA of 8 sequences; above 256 CTAs pips_colsum adds them in two levels, with one
    # more row per split of 256
    for fn, P in ((lib.pips_ln_pool_grad_scratch_floats, 1024), (lib.pips_tokenmix_grad_scratch_floats, 2600)):
        for seqs in (1, 2048, 2049):
            ctas = (seqs + 7) // 8
            assert fn(seqs) == ctas * P + ((ctas + 255) // 256 * P if ctas > 256 else 0), (P, seqs)
    assert lib.pips_ln_pool_grad_scratch_floats(0) == 0

    ga = lib.pips_gemm_tc_aux
    assert ga(p, p, 512, 256, p, p, 512, 2048, 256, 2048, 512, p, L.EPI_GELU_GRAD, None, 0, p, p, 2048, None, 0, None) != 0
    assert b"aux" in lib.pips_last_error()
    assert ga(p, None, 512, 256, p, None, 512, 2048, 256, 2048, 512, p, L.EPI_BIAS_GELU_PRE, None, 0, p, p, 2048, p, 2048,
              None) != 0
    assert b"bf16x3 only" in lib.pips_last_error()
    assert lib.pips_gemm_tc(p, p, 512, 256, p, p, 512, 2048, 256, 2048, 512, p, L.EPI_GELU_GRAD, None, 0, p, p, 2048, None) != 0


@pytest.mark.gpu
def test_delta_block_cuda_rejects_bad_inputs():
    m = _delta_block(3, 0.05)
    with pytest.raises(ValueError):
        torch_path.delta_block_cuda(m, torch.zeros(2, 7, 519, device=DEV))          # S != 8
    with pytest.raises(ValueError):
        torch_path.delta_block_cuda(m, torch.zeros(2, 8, 520, device=DEV))
    with pytest.raises(ValueError):
        torch_path.delta_block_cuda(m, torch.zeros(2, 8, 519, device=DEV, dtype=torch.float64))


@pytest.mark.gpu
def test_data_parallel_replica_on_one_gpu():
    """A replica made by torch.nn.parallel.replicate (what nn.DataParallel runs, train.py:254) lists no parameters: its
    broadcast copies are plain attributes.  delta_block_cuda finds them by name, and the gradients flow back through the
    broadcast to the original parameters, with the bits of a direct call."""
    m = _delta_block(3, 0.05)
    replica = torch.nn.parallel.replicate(m, [0])[0]
    print(f"replica lists {len(list(replica.parameters()))} parameters")
    x = _mixer_input(37, 5)
    dy = torch.randn(37, 8, 130, device=DEV)
    m.zero_grad(set_to_none=True)
    out_r = torch_path.delta_block_cuda(replica, x)
    (out_r * dy).sum().backward()
    via_replica = {n: p.grad for n, p in m.named_parameters()}
    _, _, direct = _fwd_bwd(m, x, True, dy)
    assert all(via_replica[n] is not None for n in direct), [n for n in direct if via_replica[n] is None]
    assert all(torch.equal(via_replica[n], direct[n]) for n in direct)
    assert torch.equal(out_r.detach(), torch_path.delta_block_cuda(m, x).detach())


@pytest.mark.gpu
def test_data_parallel_matches_one_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    m = _delta_block(3, 0.05)

    class Wrap(torch.nn.Module):
        def __init__(self, mod):
            super().__init__()
            self.mod = mod

        def forward(self, x):
            return torch_path.delta_block_cuda(self.mod, x)

    x = _mixer_input(64, 3)
    dy = torch.randn(64, 8, 130, device=DEV)
    w = Wrap(m)
    w.zero_grad()
    (w(x) * dy).sum().backward()
    one = {n: p.grad.clone() for n, p in m.named_parameters()}
    w.zero_grad()
    (torch.nn.DataParallel(w, device_ids=[0, 1])(x) * dy).sum().backward()
    e = max(_rel(p.grad, one[n]) for n, p in m.named_parameters() if one[n].norm() > 0)
    print(f"DataParallel over 2 GPUs vs one: worst gradient {e:.2e}")
    assert e <= 1e-5
