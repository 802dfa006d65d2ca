"""The tensor-core GEMMs and convolutions (csrc/gemm_tc.cu, conv_tc.cu, conv_rows.cu, conv_grad.cu) checked bit for bit
with exactly representable operands.

The wgmma kernels evaluate a bf16x3 product as hi.hi + lo.hi + hi.lo (lo.lo is skipped) with fp32 accumulation.  A
product of two bf16 values is exact in fp32, and a sum of values on a grid q is exact as long as every partial sum stays
below 2^24 q.  So operands whose hi parts are small integers and whose lo parts are small multiples of q make the
kernel's correct output a known fp32 number, whatever the accumulation order, tile shape or split: the tests compare it
with the fp64 three-term product and count differing elements, which must be zero.  A dropped term, a wrong stride, a
ring stage read twice or a tail tile computed wrongly changes at least one element.  For every case `exact_budget` works
out the worst-case sum of |terms| from the value ranges (bias and residual included) and asserts that it stays below
2^24 times the finest grid.

Outputs are poisoned with NaN before every call, as are operand rows past the problem, pitch columns and the rows of
output allocations past the problem: they must not reach a stored element, and what is not stored must stay NaN.

Only where a transcendental epilogue sits on the accumulator (GELU, GELU') is a bound needed, and section 5 bounds the
rounding on randn data: per element c * 2^-24 * sum|three terms| of the pairs the kernel was given.  Every test prints its
measured error; the constants c are the largest ratio measured on an H100 80GB HBM3 with a margin of about 2-4x."""
import math
from typing import NamedTuple

import pytest
import torch
import torch.nn.functional as F

from pips_b200 import _lib as L

DEV = "cuda:0"
U = 2.0 ** -24                                # fp32 unit roundoff
Q = 2.0 ** -8                                 # grid of the lo parts
TILES = ["pair", "256", "128", "64", ""]      # PIPS_B200_GEMM_TILE; "" = the automatic choice

# Bounds, in units of U (times |value| unless stated otherwise).
C_GELU_HL = 256.0     # BIAS_GELU as hi + lo vs fp64 gelu(v), |gelu(v)| units (measured 129): the (hi, lo) split alone
                      # can be 2^-16 (half an ulp of lo)
C_GELU_H = 2.0 ** 16 + 256   # hi alone (out_lo = NULL), |gelu(v)| units (measured 65300): half a bf16 ulp is <= 2^16 units
C_GELU_ABS = 1.0      # v < 0, beyond the relative term: |error| in units of U |v| (measured 0.27): 1/2 - Phi(-|v|)
                      # rounded near 1/2, the fit's 7.8e-9, ex2.approx
C_GELU_GRAD = 256.0   # GELU_GRAD, (acc + b) gelu'(aux) as hi + lo, units of |acc + b| (Phi + |z phi|) (measured 130)
C_STATS = 4.0         # InstanceNorm statistics of an exact output: mean in U mean|y| (measured 1.23), rstd in U rstd (1.68)
C_GEMM = 64.0         # section 5, randn data: pips_gemm_tc (measured 23.2, FC2)
C_WGRAD = 48.0        # pips_wgrad (measured 14.9)
C_CONV = 64.0         # pips_conv_tc / conv_rows (measured 26.1, the head's 3x3 over 416 channels)
C_CONV_WGRAD = 6.0    # pips_conv_wgrad (measured 1.85)


# ------------------------------------------------------------------------------------------------ exact operands

class Ranges(NamedTuple):
    """largest |hi| and the grid hi lies on; largest |lo| and its grid"""
    hi: float
    hi_grid: float
    lo: float
    lo_grid: float


class Spec(NamedTuple):
    """(hi, lo) operand values scale * (h + l q): h integer in [-hi, hi], l in +-[1, lo] (never zero, so each of the three
    terms contributes); scale and q powers of two."""
    hi: int
    lo: int
    q: float = Q
    scale: float = 1.0

    @property
    def ranges(self):
        return Ranges(self.hi * self.scale, self.scale, self.lo * self.q * self.scale, self.q * self.scale)

    def draw(self, shape, g):
        dev = g.device
        h = torch.randint(-self.hi, self.hi + 1, shape, generator=g, device=dev).float()
        l = torch.randint(1, self.lo + 1, shape, generator=g, device=dev).float()
        l = l * (torch.randint(0, 2, shape, generator=g, device=dev).float() * 2 - 1)
        return (h * self.scale).to(torch.bfloat16), (l * (self.q * self.scale)).to(torch.bfloat16)


def exact_budget(K, a, w, terms=3, extra=0.0):
    """Worst-case sum of |terms| of one output element -- K products of `a` and `w` values (Ranges) plus `extra` (bias,
    residual, all on the product grid) -- and the finest grid they lie on.  Asserts that every partial sum is exact in
    fp32: below 2^24 times that grid."""
    per, grid = a.hi * w.hi, a.hi_grid * w.hi_grid
    if terms == 3:
        per += a.lo * w.hi + a.hi * w.lo
        grid = min(grid, a.lo_grid * w.hi_grid, a.hi_grid * w.lo_grid)
    total = K * per + extra
    assert total < 2.0 ** 24 * grid, f"sum|terms| {total} is not exact on the grid {grid}"
    return total, grid


def on_grid(shape, vmax, grid, g):
    """fp32 values on `grid` with |v| <= vmax"""
    n = int(vmax / grid)
    return torch.randint(-n, n + 1, shape, generator=g, device=g.device).double().mul(grid).float()


def ref3(a_hi, a_lo, w_hi, w_lo, terms=3):
    """fp64 A W^T of the pairs: hi.hi (+ lo.hi + hi.lo), without lo.lo -- what the kernels compute"""
    ah, wh = a_hi.double(), w_hi.double()
    r = ah @ wh.t()
    if terms == 3:
        r = r + a_lo.double() @ wh.t() + ah @ w_lo.double().t()
    return r


def mag3(a_hi, a_lo, w_hi, w_lo, terms=3):
    """fp64 sum of |terms| of ref3"""
    return ref3(a_hi.abs(), a_lo.abs(), w_hi.abs(), w_lo.abs(), terms)


def test_exact_operands_without_gpu():
    """the exactness bound and the fp64 reference, on the host: the reference must equal an int64 computation on the
    scaled integers, and a budget past 2^24 grid units must be refused"""
    g = torch.Generator().manual_seed(0)
    for (M, N, K), sa, sw in [((7, 5, 64), Spec(3, 8), Spec(3, 8)), ((33, 17, 576), Spec(3, 8), Spec(3, 8, scale=2.0 ** -5)),
                              ((9, 40, 2048), Spec(1, 2, 2.0 ** -6), Spec(1, 2, 2.0 ** -6))]:
        total, grid = exact_budget(K, sa.ranges, sw.ranges)
        a_hi, a_lo = sa.draw((M, K), g)
        w_hi, w_lo = sw.draw((N, K), g)
        r = ref3(a_hi, a_lo, w_hi, w_lo)
        # integer units of the operands: a = ua * ga, w = uw * gw with ga * gw = grid
        ga, gw = sa.ranges.lo_grid, sw.ranges.lo_grid
        assert ga * gw <= grid
        ua = [(t.double() / ga).long() for t in (a_hi, a_lo)]
        uw = [(t.double() / gw).long() for t in (w_hi, w_lo)]
        assert all(torch.equal(u.double() * ga, t.double()) for u, t in zip(ua, (a_hi, a_lo)))
        exact = ua[0] @ uw[0].t() + ua[1] @ uw[0].t() + ua[0] @ uw[1].t()                # int64, in units of ga * gw
        assert torch.equal(r, exact.double() * (ga * gw))
        assert r.abs().max().item() <= total and torch.equal(r.float().double(), r)     # and it survives fp32
        print(f"exact operands {M}x{N}x{K}: budget {total:.0f} of {2.0 ** 24 * grid:.0f}")
    with pytest.raises(AssertionError):
        exact_budget(8 * 3072, Spec(3, 8).ranges, Spec(3, 8).ranges)
    with pytest.raises(AssertionError):
        exact_budget(64, Spec(3, 8).ranges, Spec(3, 8).ranges, extra=2.0 ** 16)


# ------------------------------------------------------------------------------------------------ helpers (GPU)

def _st():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _differ(got, ref):
    """number of elements of got that are not exactly ref (NaN differs from everything)"""
    return int((~(got.double() == ref.double())).sum().item())


def _operand(spec, rows, valid, K, ld, g):
    """(hi, lo) of `rows` x `ld`: spec values in [:valid, :K], NaN elsewhere (rows past the problem, pitch columns)"""
    hi, lo = _nan(rows, ld, dtype=torch.bfloat16), _nan(rows, ld, dtype=torch.bfloat16)
    h, l = spec.draw((valid, K), g)
    hi[:valid, :K], lo[:valid, :K] = h, l
    return hi, lo


def _gemm(a, w, M, N, K, bias, epi, of=None, oh=None, ol=None, x3=True, aux=None, ld_aux=0):
    (a_hi, a_lo), (w_hi, w_lo) = a, w
    lib = L.load()
    L.check(lib.pips_gemm_tc_aux(L.ptr(a_hi), L.ptr(a_lo) if x3 else None, a_hi.shape[1], a_hi.shape[0],
                                 L.ptr(w_hi), L.ptr(w_lo) if x3 else None, w_hi.shape[1], w_hi.shape[0], M, N, K, L.ptr(bias), epi,
                                 L.ptr(of), of.shape[1] if of is not None else 0, L.ptr(oh), L.ptr(ol),
                                 oh.shape[1] if oh is not None else 0, L.ptr(aux), ld_aux, _st()), "pips_gemm_tc")


def _tail_spec(K, sa, sw):
    """sw scaled by a power of two so that |acc| <= 2: with biases of +8 / -16 every pre-activation then lies in GELU's
    flat tails, where the kernel's GELU returns exactly v (v >= 6) or 0 (v <= -14)"""
    total, _ = exact_budget(K, sa.ranges, sw.ranges)
    return sw._replace(scale=sw.scale * 2.0 ** -math.ceil(math.log2(total / 2.0)))


def _tail_bias(N, g):
    return torch.where(torch.rand(N, generator=g, device=DEV) < 0.5, 8.0, -16.0).float()


def _gelu_tail_expected(v):
    """(hi, lo) the kernel must write for pre-activations v in GELU's flat tails"""
    assert ((v >= 6) | (v <= -14)).all()
    gv = torch.where(v >= 6, v, torch.zeros_like(v)).float()
    hi = gv.to(torch.bfloat16)
    return hi, (gv - hi.float()).to(torch.bfloat16)


def check_exact_gemm(M, N, K, epi, terms, g, sa=Spec(3, 8), sw=Spec(3, 8), w_rows=None, with_lo=True, ldo=None,
                     zero_w_pad=False):
    """One exact pips_gemm_tc call at lda = K + 8, ldw = K + 8, ldo = N + 4 (or `ldo`), ldh = N + 8, NaN around everything.
    BIAS / BIAS_RESID: out == fp64; BIAS_GELU: pre-activations in the flat tails, hi and lo == expected.  -> (differing
    elements, a description of any poison that was overwritten).  zero_w_pad: W rows [N, w_rows) are 0, as PackedWeights
    pads the head, so a column past N that the kernel stores holds 0 instead of the NaN the poison already is."""
    x3 = terms == 3
    gelu = epi == L.EPI_BIAS_GELU
    if gelu:
        sa = sw = Spec(3, 2, q=2.0 ** -4)
        sw = _tail_spec(K, sa, sw)
    a_rows = (M // 256 + 1) * 256                      # rows [M, a_rows) NaN, a multiple of 256 (pair kernel)
    w_rows = w_rows or (N // 256 + 1) * 256
    a = _operand(sa, a_rows, M, K, K + 8, g)
    w = _operand(sw, w_rows, N, K, K + 8, g)
    if zero_w_pad:
        w[0][N:], w[1][N:] = 0, 0
    ra, rw = sa.ranges, sw.ranges
    _, grid = exact_budget(K, ra, rw, terms)
    bias = _tail_bias(N, g) if gelu else on_grid((N,), 4.0, grid, g)
    resid = on_grid((M, N), 4.0, grid, g) if epi == L.EPI_BIAS_RESID else None
    exact_budget(K, ra, rw, terms, extra=bias.abs().max().item() + (4.0 if resid is not None else 0.0))
    acc = ref3(a[0][:M, :K], a[1][:M, :K], w[0][:N, :K], w[1][:N, :K], terms) + bias.double()
    extra_rows = 70
    bad = []
    if gelu:
        oh = _nan(M + extra_rows, N + 8, dtype=torch.bfloat16)
        ol = _nan(M + extra_rows, N + 8, dtype=torch.bfloat16) if with_lo else None
        _gemm(a, w, M, N, K, bias, epi, oh=oh, ol=ol, x3=x3)
        torch.cuda.synchronize()
        e_hi, e_lo = _gelu_tail_expected(acc)
        n = _differ(oh[:M, :N], e_hi) + (_differ(ol[:M, :N], e_lo) if with_lo else 0)
        for name, o in (("hi", oh), ("lo", ol)):
            if o is not None and not (torch.isnan(o[M:].float()).all() and torch.isnan(o[:M, N:].float()).all()):
                bad.append(name)
        return n, bad
    of = _nan(M + extra_rows, ldo or N + 4)
    if resid is not None:
        of[:M, :N] = resid
        acc = acc + resid.double()
    _gemm(a, w, M, N, K, bias, epi, of=of, x3=x3)
    torch.cuda.synchronize()
    n = _differ(of[:M, :N], acc)
    if not (torch.isnan(of[M:]).all() and torch.isnan(of[:M, N:]).all()):
        bad.append("out")
    return n, bad


# ------------------------------------------------------------------------------------------------ 1. calibration

@pytest.mark.gpu
@pytest.mark.parametrize("signs", ["positive", "mixed"])
def test_calibration_one_tile_at_the_largest_values(signs, monkeypatch):
    """One 128 x 256 tile at the largest sum this file uses (the head convolution's K = 9 x 448 at hi = 3, lo = 8 q):
    the H100 tensor cores must add such values exactly.  'positive': every term has the same sign, so the running sum
    grows to its bound and the q-sized lo terms are added to a sum of ~2^15."""
    monkeypatch.setenv("PIPS_B200_GEMM_TILE", "256")
    g = _gen(1)
    M, N, K = 128, 256, 4032
    spec = Spec(3, 8)
    total, grid = exact_budget(K, spec.ranges, spec.ranges, extra=4.0)
    a = _operand(spec, 256, M, K, K, g)
    w = _operand(spec, 256, N, K, K, g)
    if signs == "positive":                             # hi = 3, lo > 0 everywhere: the sum grows to its bound
        a[0][:M], w[0][:N] = 3.0, 3.0
        a[1].abs_()
        w[1].abs_()
    bias = torch.full((N,), 4.0, device=DEV) if signs == "positive" else on_grid((N,), 4.0, grid, g)
    of = _nan(M, N)
    _gemm(a, w, M, N, K, bias, L.EPI_BIAS, of=of)
    torch.cuda.synchronize()
    ref = ref3(a[0][:M], a[1][:M], w[0][:N], w[1][:N]) + bias.double()
    n = _differ(of, ref)
    d = (of.double() - ref)
    print(f"calibration ({signs}): max |sum| {ref.abs().max().item():.1f} (budget {total:.0f} < {2.0 ** 24 * grid:.0f}); "
          f"{n} differing elements, max |diff| {d.abs().max().item() / grid:.0f} grid units")
    assert n == 0


# ------------------------------------------------------------------------------------------------ 2. pips_gemm_tc

# The production shapes, the tile variants and bf16x3 / bf16 are tested bit for bit by test_kernels_gpu.py::test_gemm_tc
# through check_exact_gemm (above); this file adds the edges, the persistent loop, GELU's centre, FC1 -> FC2 under PDL.
PROD_SHAPES = {   # name: (M, N, K, epilogue, weight rows)
    "gemm_in": (8 * 300, 512, 576, L.EPI_BIAS, None),
    "fc1": (8 * 300, 2048, 512, L.EPI_BIAS_GELU, None),
    "fc2": (8 * 300, 512, 2048, L.EPI_BIAS_RESID, None),
    "head": (300, 1040, 512, L.EPI_BIAS, L.HEAD_PAD),
}


EDGE_M = [1, 63, 64, 65, 127, 129, 255, 257]
EDGE_N = [8, 40, 264, 1040]


@pytest.mark.gpu
@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("terms", [3, 1])
def test_gemm_exact_edges(terms, tile, monkeypatch):
    """M past a 64-row half, a pair CTA past M, partial halves; N in partial 32-column chunks and one chunk past a 256
    tile.  The epilogue cycles through BIAS, BIAS_RESID and BIAS_GELU (with and without lo)."""
    monkeypatch.setenv("PIPS_B200_GEMM_TILE", tile)
    g = _gen(11 + terms)
    fails = []
    i = 0
    for M in EDGE_M:
        for N in EDGE_N:
            epi = [L.EPI_BIAS, L.EPI_BIAS_RESID, L.EPI_BIAS_GELU][i % 3]
            n, bad = check_exact_gemm(M, N, 128, epi, terms, g, with_lo=(i % 2 == 0))
            if n or bad:
                fails.append((M, N, epi, n, bad))
            i += 1
    print(f"gemm edges tile={tile or 'auto'} terms={terms}: {len(EDGE_M) * len(EDGE_N)} shapes, failing: {fails or 'none'}")
    assert not fails


def check_exact_gemm_f32(M, N, K, g, ldo, w_rows):
    """One exact pips_gemm_f32 (BIAS) call at lda = ldw = K + 8: A on the grid Q (hi + lo of Spec(3, 8), exact in fp32),
    W small integers, so every product and partial sum is exact.  NaN in A's and W's rows past the problem and pitch
    columns, and around the output.  -> (differing elements, whether any poison was overwritten)"""
    sa, sw = Spec(3, 8), Spec(3, 8)
    a_hi, a_lo = _operand(sa, (M // 256 + 1) * 256, M, K, K + 8, g)
    w_hi, _ = _operand(sw, w_rows, N, K, K + 8, g)
    a, w = a_hi.float() + a_lo.float(), w_hi.float()
    ra = sa.ranges
    _, grid = exact_budget(K, Ranges(ra.hi + ra.lo, ra.lo_grid, 0.0, ra.lo_grid), sw.ranges, terms=1)
    bias = on_grid((N,), 4.0, grid, g)
    exact_budget(K, Ranges(ra.hi + ra.lo, ra.lo_grid, 0.0, ra.lo_grid), sw.ranges, terms=1, extra=4.0)
    of = _nan(M + 70, ldo)
    L.check(L.load().pips_gemm_f32(L.ptr(a), a.shape[1], L.ptr(w), w.shape[1], M, N, K, L.ptr(bias), L.EPI_BIAS, L.ptr(of),
                                   ldo, _st()), "pips_gemm_f32")
    torch.cuda.synchronize()
    ref = a[:M, :K].double() @ w[:N, :K].double().t() + bias.double()
    return _differ(of[:M, :N], ref), not (torch.isnan(of[M:]).all() and torch.isnan(of[:M, N:]).all())


@pytest.mark.gpu
@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("terms", [3, 1])
def test_gemm_exact_head_every_window(terms, tile, monkeypatch):
    """The head Linear(512 -> 130 S) of every window length 2..16 as pips_mixer_forward_s runs it: N = 130 S over
    PIPS_HEAD_PAD(S) weight rows, into delta rows of PIPS_DELTA_LD(S) floats.  At odd S, N % 8 is 2 or 6, so the bias
    guards of the last column group and the TMA store's clipping of a partial 32-column box are live, and the 2 pad
    columns of every row must stay NaN (W's pad rows are zero, as in the packed weights).  M = 300 (512 rows allocated) reaches the pair kernel.  pips_gemm_f32, the fp32
    precision's head, is checked at the same N and ldo."""
    monkeypatch.setenv("PIPS_B200_GEMM_TILE", tile)
    g = _gen(31 + terms)
    fails = []
    for S in range(2, L.S_MAX + 1):
        N, w_rows, ldo = L.head_n(S), L.head_pad(S), L.delta_ld(S)
        for M in (1, 65, 300):
            n, bad = check_exact_gemm(M, N, 512, L.EPI_BIAS, terms, g, w_rows=w_rows, ldo=ldo, zero_w_pad=True)
            if n or bad:
                fails.append(("tc", S, M, n, bad))
            if terms == 3 and tile == "":
                n, bad = check_exact_gemm_f32(M, N, 512, g, ldo, w_rows)
                if n or bad:
                    fails.append(("f32", S, M, n, bad))
    print(f"gemm head S=2..16 tile={tile or 'auto'} terms={terms}: 45 shapes, failing: {fails or 'none'}")
    assert not fails


def _persistent_m(tile, N):
    """M such that every CTA (cluster) of the variant takes at least 3 tiles and the last wave is partial"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if tile in ("pair", ""):
        workers, tm, tn = sms // 2, 256, (N + 255) // 256
    else:
        workers, tm, tn = sms, 128, (N + int(tile) - 1) // int(tile)
    tiles = 3 * workers + workers // 2
    return ((tiles + tn - 1) // tn) * tm - 37


@pytest.mark.gpu
@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("terms", [3, 1])
@pytest.mark.parametrize("epi", [L.EPI_BIAS_RESID, L.EPI_BIAS_GELU])
def test_gemm_exact_persistent_loop(epi, terms, tile, monkeypatch):
    """several tiles per CTA and a partial last wave: the handoff buffer's ho_full / ho_empty phases cycle many times"""
    monkeypatch.setenv("PIPS_B200_GEMM_TILE", tile)
    N, K = 512, 256
    M = _persistent_m(tile, N)
    n, bad = check_exact_gemm(M, N, K, epi, terms, _gen(M + terms))
    print(f"gemm persistent M={M} tile={tile or 'auto'} terms={terms} epi={epi}: {n} differing elements, "
          f"poison overwritten: {bad or 'none'}")
    assert n == 0 and not bad


def _bf16_ulp(hi):
    """spacing of the bf16 values around hi (0 for hi = 0); frexp, as a device log2 can miss an exact power of two"""
    m, e = torch.frexp(hi.double())
    return torch.where(hi.double() == 0, torch.zeros_like(m), torch.ldexp(torch.ones_like(m), e - 8))


def _gelu_errors(v, hi, lo, bound):
    """The bound per element is U (bound |gelu(v)| + C_GELU_ABS |v|).  -> (max error / (U |gelu(v)|) over v >= 0; over
    v < 0, the largest error beyond U bound |gelu(v)| in units of U |v|; whether |lo| <= ulp(hi) / 2)"""
    got = hi.double() + (lo.double() if lo is not None else 0.0)
    ref = F.gelu(v)
    err = (got - ref).abs()
    pos = v >= 0
    c_rel = (err[pos] / (U * ref[pos].abs()).clamp(min=1e-300)).max().item()
    neg = ~pos
    c_abs = ((err[neg] - bound * U * ref[neg].abs()).clamp(min=0) / (U * v[neg].abs())).max().item() if neg.any() else 0.0
    lo_ok = True if lo is None else bool((lo.double().abs() <= _bf16_ulp(hi) / 2).all())
    return c_rel, c_abs, lo_ok


def check_gelu_bounded(M, N, K, terms, with_lo, label):
    """BIAS_GELU with exact pre-activations over GELU's centre and both tails: hi (+ lo) per element against fp64 gelu(v)
    within U (C |gelu(v)| + C_GELU_ABS |v|), |lo| <= ulp(hi) / 2, and NaN poison past M and in the pitch kept"""
    g = _gen(5)
    sa, sw = Spec(3, 8, scale=2.0 ** -3), Spec(3, 8, scale=2.0 ** -3)
    a, w = _operand(sa, (M // 256 + 1) * 256, M, K, K + 8, g), _operand(sw, (N + 255) // 256 * 256, N, K, K + 8, g)
    _, grid = exact_budget(K, sa.ranges, sw.ranges, terms)
    bias = on_grid((N,), 2.0, grid, g)
    bias[::5] += 12.0
    bias[2::5] -= 20.0
    exact_budget(K, sa.ranges, sw.ranges, terms, extra=bias.abs().max().item())
    x3 = terms == 3
    v = ref3(a[0][:M, :K], a[1][:M, :K], w[0][:N, :K], w[1][:N, :K], terms) + bias.double()
    oh = _nan(M + 70, N + 8, dtype=torch.bfloat16)
    ol = _nan(M + 70, N + 8, dtype=torch.bfloat16) if with_lo else None
    _gemm(a, w, M, N, K, bias, L.EPI_BIAS_GELU, oh=oh, ol=ol, x3=x3)
    torch.cuda.synchronize()
    bound = C_GELU_HL if with_lo else C_GELU_H
    c_rel, c_abs, lo_ok = _gelu_errors(v, oh[:M, :N], ol[:M, :N] if with_lo else None, bound)
    n_pos, n_neg, n_mid = int((v > 6).sum()), int((v < -6).sum()), int((v.abs() < 3).sum())
    print(f"gemm gelu {label} terms={terms} lo={with_lo}: {c_rel:.3g} units of |gelu| (bound {bound}), "
          f"{c_abs:.3g} units of |v| for v < 0 (bound {C_GELU_ABS}); {n_neg} / {n_mid} / {n_pos} left tail / centre / right tail")
    assert min(n_pos, n_neg, n_mid) > M * N // 16
    assert lo_ok, "|lo| > ulp(hi) / 2"
    poison = [o for o in (oh, ol) if o is not None]
    assert all(torch.isnan(o[M:].float()).all() and torch.isnan(o[:M, N:].float()).all() for o in poison)
    assert c_rel <= bound and c_abs <= C_GELU_ABS


@pytest.mark.gpu
@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("terms,with_lo", [(3, False), (1, True)])
def test_gemm_gelu_bounded(terms, with_lo, tile, monkeypatch):
    """FC1's GELU with the lo output the forward does not use: out_lo = NULL in bf16x3, lo written in plain bf16 (the
    other two combinations run in test_kernels_gpu.py::test_gemm_tc)"""
    monkeypatch.setenv("PIPS_B200_GEMM_TILE", tile)
    check_gelu_bounded(8 * 300, 2048, 512, terms, with_lo, f"tile={tile or 'auto'}")


@pytest.mark.gpu
@pytest.mark.parametrize("tile", TILES)
def test_fc1_then_fc2_without_host_sync(tile, monkeypatch):
    """FC1 (BIAS_GELU into hi, lo) and FC2 (BIAS_RESID reading FC1's output) back to back on one stream, launched with
    programmatic dependent launch (the default): FC1's pre-activations lie in GELU's flat tails, so both are exact."""
    monkeypatch.setenv("PIPS_B200_GEMM_TILE", tile)
    M, D, H = 8 * 300, 512, 2048
    g = _gen(21)
    # FC1: A nonzero in its first 64 columns only (a budget of 64 products), W scaled so that |acc| <= 8; biases +14 / -30
    # put v in [6, 22] or [-38, -22] on the grid 1/32, where hi + lo holds v exactly (10 significant bits)
    sa, s1 = Spec(1, 1, q=0.5), Spec(1, 1, q=0.5, scale=2.0 ** -4)
    K1 = 64
    total1, grid1 = exact_budget(K1, sa.ranges, s1.ranges)
    a = _operand(sa, 2560, M, D, D + 8, g)
    a[0][:M, K1:D] = 0
    a[1][:M, K1:D] = 0
    w1 = _operand(s1, H, H, D, D + 8, g)
    b1 = torch.where(torch.rand(H, generator=g, device=DEV) < 0.5, 14.0, -30.0).float()
    assert total1 <= 8 and grid1 == 1 / 32
    # FC2 reads (hi, lo) with |value| <= 22 on the grid 1/32: hi <= 22 on 1/32, lo <= 1/16 on 1/32
    s2 = Spec(1, 1, q=0.5)
    h_ranges = Ranges(22.0, 1 / 32, 1 / 16, 1 / 32)
    _, grid2 = exact_budget(H, h_ranges, s2.ranges, extra=8.0)
    w2 = _operand(s2, D, D, H, H + 8, g)
    b2 = on_grid((D,), 4.0, grid2, g)
    x = on_grid((M, D), 4.0, grid2, g)
    hh = _nan(2560, H + 8, dtype=torch.bfloat16)
    hl = _nan(2560, H + 8, dtype=torch.bfloat16)
    of = _nan(M + 70, D + 4)
    of[:M, :D] = x
    torch.cuda.synchronize()
    _gemm(a, w1, M, H, D, b1, L.EPI_BIAS_GELU, oh=hh, ol=hl)
    _gemm((hh, hl), w2, M, D, H, b2, L.EPI_BIAS_RESID, of=of)
    torch.cuda.synchronize()
    v = ref3(a[0][:M, :D], a[1][:M, :D], w1[0][:, :D], w1[1][:, :D]) + b1.double()
    e_hi, e_lo = _gelu_tail_expected(v)
    assert torch.equal(e_hi.double() + e_lo.double(), torch.where(v >= 6, v, torch.zeros_like(v)))
    n1 = _differ(hh[:M, :H], e_hi) + _differ(hl[:M, :H], e_lo)
    ref = ref3(e_hi, e_lo, w2[0][:, :H], w2[1][:, :H]) + b2.double() + x.double()
    n2 = _differ(of[:M, :D], ref)
    print(f"fc1 -> fc2 tile={tile or 'auto'}: {n1} differing FC1 elements, {n2} differing FC2 elements")
    assert n1 == 0 and n2 == 0
    assert torch.isnan(of[M:]).all() and torch.isnan(of[:M, D:]).all()


# ------------------------------------------------------------------------------------------------ 3. training GEMMs

def _gelu_grad64(x):
    return 0.5 * torch.erfc(-x / math.sqrt(2.0)) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(8 * 300, 2048, 512), (8 * 300 + 5, 512, 2048), (129, 264, 128)])
def test_gemm_aux_epilogues(M, N, K):
    """BIAS_GELU_PRE: pre bit-exact, GELU hi / lo bounded.  GELU_GRAD: aux holds exact pre-activations in the centre and
    both tails; (acc + b) gelu'(aux) per element against fp64.  ld_aux = N + 8 with a NaN pitch."""
    g = _gen(M + N)
    sa, sw = Spec(3, 8, scale=2.0 ** -3), Spec(3, 8, scale=2.0 ** -3)
    a, w = _operand(sa, (M // 256 + 1) * 256, M, K, K + 8, g), _operand(sw, N, N, K, K + 8, g)
    _, grid = exact_budget(K, sa.ranges, sw.ranges)
    bias = on_grid((N,), 2.0, grid, g)
    bias[::5] += 12.0
    bias[2::5] -= 20.0
    exact_budget(K, sa.ranges, sw.ranges, extra=bias.abs().max().item())
    v = ref3(a[0][:M, :K], a[1][:M, :K], w[0][:N, :K], w[1][:N, :K]) + bias.double()
    hi, lo = _nan(M + 70, N + 8, dtype=torch.bfloat16), _nan(M + 70, N + 8, dtype=torch.bfloat16)
    pre = _nan(M + 70, N + 8)
    _gemm(a, w, M, N, K, bias, L.EPI_BIAS_GELU_PRE, oh=hi, ol=lo, aux=pre, ld_aux=N + 8)
    torch.cuda.synchronize()
    n_pre = _differ(pre[:M, :N], v)
    c_rel, c_abs, lo_ok = _gelu_errors(v, hi[:M, :N], lo[:M, :N], C_GELU_HL)
    poison = all(torch.isnan(t[M:].float()).all() and torch.isnan(t[:M, N:].float()).all() for t in (hi, lo, pre))
    # GELU_GRAD: a fresh aux of exact pre-activations (grid 1/64) over the centre and both tails
    aux = _nan(M + 70, N + 8)
    z = on_grid((M, N), 4.0, 1 / 64, g)
    z[:, ::5] += 12.0
    z[:, 2::5] -= 20.0
    aux[:M, :N] = z
    dh, dl = _nan(M + 70, N + 8, dtype=torch.bfloat16), _nan(M + 70, N + 8, dtype=torch.bfloat16)
    _gemm(a, w, M, N, K, bias, L.EPI_GELU_GRAD, oh=dh, ol=dl, aux=aux, ld_aux=N + 8)
    torch.cuda.synchronize()
    z64 = z.double()
    dref = v * _gelu_grad64(z64)
    got = dh[:M, :N].double() + dl[:M, :N].double()
    # units of U |acc + b| (Phi(z) + |z phi(z)|), the size of gelu's two terms (they cancel near z = -0.75); below
    # ~2^-126 the fp32 gelu' and the product are subnormal: an absolute floor of 2^-120 |acc + b|
    gmag = v.abs() * (0.5 * torch.erfc(-z64 / math.sqrt(2.0)) + (z64 * torch.exp(-0.5 * z64 * z64)).abs() / math.sqrt(2.0 * math.pi))
    c_grad = ((got - dref).abs() / (U * gmag + 2.0 ** -120 * v.abs()).clamp(min=1e-300)).max().item()
    aux_kept = torch.equal(aux[:M, :N], z) and torch.isnan(aux[:M, N:]).all() and torch.isnan(aux[M:]).all()
    poison = poison and all(torch.isnan(t[M:].float()).all() and torch.isnan(t[:M, N:].float()).all() for t in (dh, dl))
    print(f"aux {M}x{N}x{K}: pre {n_pre} differing; gelu {c_rel:.3g} units of |gelu| (bound {C_GELU_HL}), {c_abs:.3g} "
          f"units of |v| (bound {C_GELU_ABS}); gelu' product {c_grad:.3g} units (bound {C_GELU_GRAD})")
    assert n_pre == 0 and lo_ok and poison and aux_kept
    assert c_rel <= C_GELU_HL and c_abs <= C_GELU_ABS and c_grad <= C_GELU_GRAD


WGRAD_SHAPES = [(8 * 3072, 512, 2048), (8 * 3071, 2048, 512), (8 * 37, 512, 576), (3072, 1040, 512), (37, 1040, 512),
                (8, 512, 576)]
WGRAD_EDGES = [(M, N, K) for M in (2047, 2048, 2049, 4096 + 31) for N in (8, 136) for K in (8, 136)]


def _wgrad_spec(M):
    return Spec(3, 8) if M <= 4200 else Spec(1, 2, q=2.0 ** -6)


def _wgrad_call(gp, xp, M, N, K):
    lib = L.load()
    dw = _nan(N, K)
    n = lib.pips_wgrad_scratch_floats(M, N, K)
    scratch = _nan(max(n, 1))
    L.check(lib.pips_wgrad(L.ptr(gp[0]), L.ptr(gp[1]), gp[0].shape[1], L.ptr(xp[0]), L.ptr(xp[1]), xp[0].shape[1], M, N, K,
                           L.ptr(scratch), L.ptr(dw), _st()), "pips_wgrad")
    return dw


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", WGRAD_SHAPES + WGRAD_EDGES)
def test_wgrad_exact(M, N, K):
    """dW = G^T X bit-exact: the 2048-row splits and their reduction, a partial 32-row K-block, N and K past a tile;
    ldg = N + 8, ldx = K + 8 with NaN pitch columns (TMA zero-fills past N and K, never reads them), NaN scratch"""
    g = _gen(M * 7 + N + K)
    spec = _wgrad_spec(M)
    exact_budget(M, spec.ranges, spec.ranges)
    gp = _operand(spec, M, M, N, N + 8, g)
    xp = _operand(spec, M, M, K, K + 8, g)
    dw = _wgrad_call(gp, xp, M, N, K)
    torch.cuda.synchronize()
    ref = ref3(gp[0][:, :N].t(), gp[1][:, :N].t(), xp[0][:, :K].t(), xp[1][:, :K].t())
    n = _differ(dw, ref)
    print(f"wgrad {M}x{N}x{K}: {n} differing elements")
    assert n == 0


@pytest.mark.gpu
@pytest.mark.parametrize("M,N", [(8 * 3071, 2048), (37, 1040), (300, 512)])
def test_colsum_exact(M, N):
    lib = L.load()
    g = _gen(M + N)
    spec = Spec(1, 2, q=2.0 ** -6)                   # M values hi + lo, |.| <= 1 + 2q on the grid q
    exact_budget(M, Ranges(1.0 + 2 * spec.q, spec.q, 0.0, spec.q), Ranges(1.0, 1.0, 0.0, 1.0), terms=1)
    hi, lo = _operand(spec, M, M, N, N + 8, g)
    G = hi.float() + lo.float()                      # exact in fp32
    scratch = _nan(max(lib.pips_colsum_scratch_floats(M, N), 1))
    out, out2 = _nan(N), _nan(N)
    L.check(lib.pips_colsum(L.ptr(G), None, None, N + 8, M, N, L.ptr(scratch), L.ptr(out), _st()), "pips_colsum")
    L.check(lib.pips_colsum(None, L.ptr(hi), L.ptr(lo), N + 8, M, N, L.ptr(scratch), L.ptr(out2), _st()), "pips_colsum")
    torch.cuda.synchronize()
    ref = G[:, :N].double().sum(0)
    n1, n2 = _differ(out, ref), _differ(out2, ref)
    print(f"colsum {M}x{N}: fp32 {n1}, (hi, lo) {n2} differing elements")
    assert n1 == 0 and n2 == 0


# ------------------------------------------------------------------------------------------------ 4. convolutions

def _pad64(c):
    return (c + 63) // 64 * 64


class XPair(NamedTuple):
    hi: torch.Tensor       # (N, H, W, Cp) bf16, channels [C, Cp) zero
    lo: torch.Tensor
    C: int


def _xpair(spec, N, H, W, C, g, pitch=None, pad_value=0.0):
    cp = pitch or _pad64(C)
    hi = torch.full((N, H, W, cp), pad_value, dtype=torch.bfloat16, device=DEV)
    lo = hi.clone()
    h, l = spec.draw((N, H, W, C), g)
    hi[..., :C], lo[..., :C] = h, l
    return XPair(hi, lo, C)


def _nchw(p, part):
    return getattr(p, part)[..., :p.C].permute(0, 3, 1, 2).double()


def _wpack(spec, cout, cin, R, S, g):
    """(BN, R*S*Cp) (hi, lo) filter pack [k = (r*S + s)*Cp + ci]: rows [Cout, BN) NaN, channels [Cin, Cp) zero; and the
    (Cout, Cin, R, S) fp64 hi and lo"""
    cp = _pad64(cin)
    bn = 64 if cout <= 64 else (128 if cout <= 128 else 256)
    h, l = spec.draw((cout, R, S, cin), g)
    packs = []
    for t in (h, l):
        p = torch.zeros(bn, R, S, cp, dtype=torch.bfloat16, device=DEV)
        p[:cout, ..., :cin] = t
        p[cout:] = float("nan")
        packs.append(p.reshape(bn, R * S * cp).contiguous())
    return packs, (h.permute(0, 3, 1, 2).double(), l.permute(0, 3, 1, 2).double())


def _conv3(x, w, stride, pad, conv=F.conv2d):
    """fp64 three-term convolution of (hi, lo) pairs: x_hi w_hi + x_lo w_hi + x_hi w_lo"""
    return conv(x[0], w[0], stride=stride, padding=pad) + conv(x[1], w[0], stride=stride, padding=pad) + \
        conv(x[0], w[1], stride=stride, padding=pad)


def _conv_call(x, packs, cout, R, S, sy, sx, py, px, bias, Ho, Wo, stats):
    """pips_conv_tc (_aniso for unequal strides or paddings; _stats) into an output allocation with a NaN tail
    -> (out, tail, statistics or None)"""
    lib = L.load()
    N, H, W, cp = x.hi.shape
    size = N * Ho * Wo * cout
    buf = _nan(size + 4096)
    if stats:
        chunks = lib.pips_conv_tc_chunks(H, W, R, S, sy, sx, py, px)
        partial = _nan(N, chunks, 3, cout)
        st = _nan(N, 2, cout)
        L.check(lib.pips_conv_tc_stats(L.ptr(x.hi), L.ptr(x.lo), N, H, W, cp, L.ptr(packs[0]), L.ptr(packs[1]), cout, R, S, sy, sx,
                                       py, px, L.ptr(bias), L.ptr(buf), L.ptr(partial), _st()), "pips_conv_tc_stats")
        L.check(lib.pips_inorm_finalize(L.ptr(partial), N, chunks, Ho * Wo, cout, L.ptr(st), _st()), "pips_inorm_finalize")
    elif sy == sx and py == px:
        st = None
        L.check(lib.pips_conv_tc(L.ptr(x.hi), L.ptr(x.lo), N, H, W, cp, L.ptr(packs[0]), L.ptr(packs[1]), cout, R, S, sy, py,
                                 L.ptr(bias), L.ptr(buf), _st()), "pips_conv_tc")
    else:
        st = None
        L.check(lib.pips_conv_tc_aniso(L.ptr(x.hi), L.ptr(x.lo), N, H, W, cp, L.ptr(packs[0]), L.ptr(packs[1]), cout, R, S, sy, sx,
                                       py, px, L.ptr(bias), L.ptr(buf), _st()), "pips_conv_tc_aniso")
    torch.cuda.synchronize()
    return buf[:size].view(N, Ho, Wo, cout), buf[size:], st


def _stats_units(st, y):
    """InstanceNorm statistics of y (N, Ho, Wo, C) against fp64: mean error in U mean|y|, rstd error in U rstd"""
    y = y.double()
    mean = y.mean(dim=(1, 2))
    rstd = 1.0 / torch.sqrt(y.var(dim=(1, 2), unbiased=False) + 1e-5)
    e_mean = ((st[:, 0].double() - mean).abs() / (U * y.abs().mean(dim=(1, 2)))).max().item()
    e_rstd = ((st[:, 1].double() - rstd).abs() / (U * rstd)).max().item()
    return e_mean, e_rstd


CONV_CASES = [  # (N, H, W, Cin, Cout, R, stride, pad, bias): the geometries of test_conv_tc, then those of the weight gradient
    (2, 24, 40, 64, 64, 3, 1, 1, False), (1, 45, 80, 64, 64, 3, 1, 1, False), (2, 48, 64, 64, 96, 3, 2, 1, False),
    (2, 48, 64, 64, 96, 1, 2, 0, False), (1, 23, 40, 96, 96, 3, 1, 1, False), (1, 12, 16, 416, 256, 3, 1, 1, False),
    (3, 12, 16, 256, 128, 1, 1, 0, True), (1, 192, 256, 64, 64, 3, 1, 1, False), (2, 45, 80, 64, 64, 3, 1, 1, False),
    (5, 24, 32, 128, 128, 3, 1, 1, False), (3, 15, 24, 64, 96, 3, 2, 1, False),
    (2, 32, 40, 64, 64, 3, 1, 1, True), (2, 33, 41, 64, 96, 3, 2, 1, False), (2, 32, 40, 64, 96, 1, 2, 0, True),
    (3, 17, 23, 96, 128, 1, 2, 0, False), (2, 16, 20, 128, 128, 3, 1, 1, False), (2, 16, 20, 416, 256, 3, 1, 1, True),
    (2, 16, 20, 256, 128, 1, 1, 0, False), (1, 7, 5, 128, 128, 3, 2, 1, False), (32, 96, 128, 64, 64, 3, 1, 1, False),
]


def _conv_exact(x, packs, w64, cout, R, S, sy, sx, py, px, bias, g, stats=True):
    """conv_tc (aniso) and conv_tc_stats on the same operands: both bit-exact, the same bits, the NaN tail untouched,
    the statistics bounded -> (differing elements, stats units or None)"""
    N, H, W, _ = x.hi.shape
    Ho, Wo = (H + 2 * py - R) // sy + 1, (W + 2 * px - S) // sx + 1
    ref = _conv3((_nchw(x, "hi"), _nchw(x, "lo")), w64, (sy, sx), (py, px))
    if bias is not None:
        ref = ref + bias.double().view(1, -1, 1, 1)
    ref = ref.permute(0, 2, 3, 1)
    out, tail, _ = _conv_call(x, packs, cout, R, S, sy, sx, py, px, bias, Ho, Wo, False)
    n = _differ(out, ref) + int((~torch.isnan(tail)).sum())
    if not stats:
        return n, None
    out2, tail2, st = _conv_call(x, packs, cout, R, S, sy, sx, py, px, bias, Ho, Wo, True)
    n += int((~(out2.view(torch.int32) == out.view(torch.int32))).sum()) + int((~torch.isnan(tail2)).sum())
    return n, _stats_units(st, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,pad,bias", CONV_CASES)
def test_conv_tc_exact(N, H, W, Cin, Cout, R, stride, pad, bias):
    g = _gen(N * 100 + H + Cin + Cout)
    spec = Spec(3, 8)
    x = _xpair(spec, N, H, W, Cin, g)
    packs, w64 = _wpack(spec, Cout, Cin, R, R, g)
    total, grid = exact_budget(R * R * Cin, spec.ranges, spec.ranges, extra=4.0)
    b = on_grid((Cout,), 4.0, grid, g) if bias else None
    n, (e_mean, e_rstd) = _conv_exact(x, packs, w64, Cout, R, R, stride, stride, pad, pad, b, g)
    print(f"conv_tc {N}x{H}x{W} {Cin}->{Cout} {R}x{R}/{stride}: {n} differing elements; statistics: mean {e_mean:.3g}, "
          f"rstd {e_rstd:.3g} units (bound {C_STATS})")
    assert n == 0 and e_mean <= C_STATS and e_rstd <= C_STATS


@pytest.mark.gpu
@pytest.mark.parametrize("geometry", ["stem4x1", "3x1/2"])
def test_conv_tc_aniso_exact(geometry):
    """the stem's 4x1 convolution over an input shaped like pips_stem_pack's (N, Ho + 3, Wo, 64), and a 3x1 filter with
    stride (2, 1), padding (1, 0)"""
    g = _gen(3)
    spec = Spec(3, 8)
    if geometry == "stem4x1":
        N, H, W, R, S, sy, sx, py, px, cout = 2, 67, 80, 4, 1, 1, 1, 0, 0, 64
    else:
        N, H, W, R, S, sy, sx, py, px, cout = 2, 33, 41, 3, 1, 2, 1, 1, 0, 96
    x = _xpair(spec, N, H, W, 64, g)
    packs, w64 = _wpack(spec, cout, 64, R, S, g)
    exact_budget(R * S * 64, spec.ranges, spec.ranges)
    n, (e_mean, e_rstd) = _conv_exact(x, packs, w64, cout, R, S, sy, sx, py, px, None, g)
    print(f"conv_tc_aniso {geometry}: {n} differing elements; statistics: mean {e_mean:.3g}, rstd {e_rstd:.3g} units")
    assert n == 0 and e_mean <= C_STATS and e_rstd <= C_STATS


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W", [(2, 24, 40), (1, 45, 300), (3, 7, 130), (2, 192, 256), (1, 90, 160), (1, 33, 640)])
def test_conv_rows_exact(N, H, W):
    """the row-ring 3x3 kernel: bit-exact, the same bits as conv_tc on the same operands, statistics bounded"""
    lib = L.load()
    g = _gen(N + H + W)
    spec = Spec(3, 8)
    x = _xpair(spec, N, H, W, 64, g)
    packs, w64 = _wpack(spec, 64, 64, 3, 3, g)
    exact_budget(9 * 64, spec.ranges, spec.ranges)
    ref = _conv3((_nchw(x, "hi"), _nchw(x, "lo")), w64, 1, 1).permute(0, 2, 3, 1)
    size = N * H * W * 64
    buf = _nan(size + 4096)
    chunks = lib.pips_conv_rows_chunks(H, W)
    partial = _nan(N, chunks, 3, 64)
    st = _nan(N, 2, 64)
    L.check(lib.pips_conv_rows(L.ptr(x.hi), L.ptr(x.lo), N, H, W, L.ptr(packs[0]), L.ptr(packs[1]), L.ptr(buf), L.ptr(partial),
                               _st()), "pips_conv_rows")
    L.check(lib.pips_inorm_finalize(L.ptr(partial), N, chunks, H * W, 64, L.ptr(st), _st()), "pips_inorm_finalize")
    torch.cuda.synchronize()
    out = buf[:size].view(N, H, W, 64)
    gen, _, _ = _conv_call(x, packs, 64, 3, 3, 1, 1, 1, 1, None, H, W, False)
    n = _differ(out, ref) + int((~torch.isnan(buf[size:])).sum())
    same = torch.equal(out.view(torch.int32), gen.view(torch.int32))
    e_mean, e_rstd = _stats_units(st, ref)
    print(f"conv_rows {N}x{H}x{W}: {n} differing elements, same bits as conv_tc: {same}; statistics: mean {e_mean:.3g}, "
          f"rstd {e_rstd:.3g} units (bound {C_STATS})")
    assert n == 0 and same and e_mean <= C_STATS and e_rstd <= C_STATS


WGRAD_CASES = [  # (N, H, W, Cin, Cout, R, stride, pad): every encoder geometry
    (2, 32, 40, 64, 64, 3, 1, 1), (2, 33, 41, 64, 96, 3, 2, 1), (2, 32, 40, 64, 96, 1, 2, 0), (3, 17, 23, 96, 128, 1, 2, 0),
    (2, 16, 20, 128, 128, 3, 1, 1), (2, 16, 20, 416, 256, 3, 1, 1), (2, 16, 20, 256, 128, 1, 1, 0), (1, 7, 5, 128, 128, 3, 2, 1),
    (32, 96, 128, 64, 64, 3, 1, 1),
]


def _conv_wgrad_exact(N, H, W, Cin, Cout, R, S, sy, sx, py, px, step, g):
    lib = L.load()
    Ho, Wo = (H + 2 * py - R) // sy + 1, (W + 2 * px - S) // sx + 1
    pixels = N * Ho * Wo
    spec = Spec(3, 8) if pixels * 9.2 < 2 ** 16 else Spec(1, 1, q=2.0 ** -4)
    exact_budget(pixels, spec.ranges, spec.ranges)
    x = _xpair(spec, N, H, W, Cin, g)
    ldy = _pad64(Cout)
    if step == 2:                                        # zero-dilated on the input's grid, output pixel (oy, ox) at (2oy, 2ox)
        d = _xpair(spec, N, Ho, Wo, Cout, g)
        dyp = XPair(torch.zeros(N, H, W, ldy, dtype=torch.bfloat16, device=DEV), torch.zeros(N, H, W, ldy, dtype=torch.bfloat16,
                                                                                           device=DEV), Cout)
        dyp.hi[:, ::2, ::2], dyp.lo[:, ::2, ::2] = d.hi, d.lo
        dyp.hi[..., Cout:], dyp.lo[..., Cout:] = float("nan"), float("nan")
    else:
        d = dyp = _xpair(spec, N, Ho, Wo, Cout, g, pad_value=float("nan"))     # channels [Cout, ldy) NaN
    K = R * S * x.hi.shape[-1]
    dw = _nan(Cout, K)
    scratch = _nan(max(lib.pips_conv_wgrad_scratch_floats(N, Ho, Wo, Cout, K), 1))
    L.check(lib.pips_conv_wgrad(L.ptr(dyp.hi), L.ptr(dyp.lo), ldy, step, L.ptr(x.hi), L.ptr(x.lo), N, H, W, x.hi.shape[-1], Cout, R, S,
                                sy, sx, py, px, L.ptr(scratch), L.ptr(dw), _st()), "pips_conv_wgrad")
    torch.cuda.synchronize()
    xs = (_nchw(x, "hi"), _nchw(x, "lo"))
    ds = (_nchw(d, "hi"), _nchw(d, "lo"))
    cw = torch.nn.grad.conv2d_weight
    shape = (Cout, Cin, R, S)
    ref = cw(xs[0], shape, ds[0], stride=(sy, sx), padding=(py, px)) + cw(xs[0], shape, ds[1], stride=(sy, sx), padding=(py, px)) + \
        cw(xs[1], shape, ds[0], stride=(sy, sx), padding=(py, px))
    got = dw.view(Cout, R, S, -1)
    n = _differ(got[..., :Cin], ref.permute(0, 2, 3, 1)) + _differ(got[..., Cin:], torch.zeros_like(got[..., Cin:]))
    return n, pixels


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,pad", WGRAD_CASES)
@pytest.mark.parametrize("step", [1, 2])
def test_conv_wgrad_exact(N, H, W, Cin, Cout, R, stride, pad, step):
    """bit-exact dW, the chunked reduction over pixels included; dY channels [Cout, ldy) NaN, NaN scratch"""
    if step == 2 and stride == 1:
        pytest.skip("the zero-dilated gradient exists for stride-2 convolutions only")
    n, pixels = _conv_wgrad_exact(N, H, W, Cin, Cout, R, R, stride, stride, pad, pad, step, _gen(N * 31 + H + Cin))
    print(f"conv_wgrad N={N} {H}x{W} {Cin}->{Cout} {R}x{R}/{stride} step={step} ({pixels} pixels): {n} differing elements")
    assert n == 0


@pytest.mark.gpu
def test_conv_wgrad_stem_exact():
    """the stem's 4x1 convolution over pips_stem_pack-shaped row-pair pixels"""
    n, pixels = _conv_wgrad_exact(2, 67, 80, 64, 64, 4, 1, 1, 1, 0, 0, 1, _gen(4))
    print(f"conv_wgrad stem 4x1 ({pixels} pixels): {n} differing elements")
    assert n == 0


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,R,stride", [(64, 64, 3, 1), (64, 96, 3, 2), (96, 128, 1, 2), (416, 256, 3, 1)])
def test_input_gradient_exact(Cin, Cout, R, stride):
    """torch_path._EncRun.dgrad: pips_conv_tc with the flipped, transposed weight (the head in 160 + 256 channel parts),
    over dY zero-dilated for stride 2; bit-exact against fp64 conv2d_input.  The weights k 2^-10, |k| < 1024, split
    exactly into their (hi, lo) pack."""
    from pips_b200 import encoder_fast as E
    from pips_b200 import torch_path
    g = _gen(Cin + R)
    N, H, W, pad = 2, 33, 41, R // 2
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    w = torch.randint(-1023, 1024, (Cout, Cin, R, R), generator=g, device=DEV).float() * 2.0 ** -10
    spec = Spec(1, 1, q=0.25)
    exact_budget(R * R * Cout, spec.ranges, Ranges(1.0, 2.0 ** -10, 2.0 ** -9, 2.0 ** -10))
    d = _xpair(spec, N, Ho, Wo, Cout, g)
    dyp = E._Pair(N, H, W, Cout, DEV)
    dyp.hi.zero_()
    dyp.lo.zero_()
    dyp.hi[:, ::stride, ::stride], dyp.lo[:, ::stride, ::stride] = d.hi, d.lo
    run = torch_path._EncRun(torch.device(DEV))
    parts = [(0, Cin)] if Cin <= 256 else [(0, 160), (160, Cin)]
    dx = torch.cat([run.dgrad(dyp, w, pad, rows=r) for r in parts], dim=-1)
    torch.cuda.synchronize()
    wh = w.to(torch.bfloat16)
    wl = (w - wh.float()).to(torch.bfloat16)
    assert torch.equal(wh.double() + wl.double(), w.double()) and (wl != 0).any()
    # the pack holds exactly these (hi, lo): check one part against them
    ph, pl = E.pack_conv_weight(w.flip(2, 3).transpose(0, 1)[:16])
    assert torch.equal(ph.view(-1, R, R, _pad64(Cout))[:16, ..., :Cout], wh.flip(2, 3).transpose(0, 1)[:16].permute(0, 2, 3, 1))
    ci = torch.nn.grad.conv2d_input
    ds = (_nchw(d, "hi"), _nchw(d, "lo"))
    ref = ci((N, Cin, H, W), wh.double(), ds[0], stride=stride, padding=pad) + \
        ci((N, Cin, H, W), wh.double(), ds[1], stride=stride, padding=pad) + \
        ci((N, Cin, H, W), wl.double(), ds[0], stride=stride, padding=pad)
    n = _differ(dx, ref.permute(0, 2, 3, 1))
    print(f"input gradient {Cin}->{Cout} {R}x{R}/{stride}: {n} differing elements")
    assert n == 0


# ------------------------------------------------------------------------------------------------ 5. randn data

def _randn_pair(shape, g, rows=None, ld=None):
    v = torch.randn(shape, generator=g, device=DEV)
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    if rows is None:
        return hi, lo
    out = []
    for t in (hi, lo):
        p = _nan(rows, ld, dtype=torch.bfloat16)
        p[:shape[0], :shape[1]] = t
        out.append(p)
    return tuple(out)


def _units(got, ref, mag):
    return ((got.double() - ref).abs() / (U * mag).clamp(min=1e-300)).max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("tile", ["", "128"])
@pytest.mark.parametrize("shape", ["gemm_in", "fc2", "head"])
def test_gemm_rounding_on_randn(shape, tile, monkeypatch):
    monkeypatch.setenv("PIPS_B200_GEMM_TILE", tile)
    M, N, K, epi, w_rows = PROD_SHAPES[shape]
    g = _gen(M + K)
    a = _randn_pair((M, K), g, (M // 256 + 1) * 256, K)
    w = _randn_pair((N, K), g, w_rows or N, K)
    bias = torch.randn(N, generator=g, device=DEV)
    of = _nan(M, N)
    ref = ref3(a[0][:M], a[1][:M], w[0][:N], w[1][:N]) + bias.double()
    mag = mag3(a[0][:M], a[1][:M], w[0][:N], w[1][:N]) + bias.double().abs()
    if epi == L.EPI_BIAS_RESID:
        x = torch.randn(M, N, generator=g, device=DEV)
        of.copy_(x)
        ref, mag = ref + x.double(), mag + x.double().abs()
    _gemm(a, w, M, N, K, bias, epi, of=of)
    torch.cuda.synchronize()
    e = _units(of, ref, mag)
    print(f"gemm {shape} tile={tile or 'auto'} on randn: {e:.3g} units of U sum|terms| (bound {C_GEMM})")
    assert e <= C_GEMM


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(8 * 3072, 512, 2048), (8 * 3071, 2048, 512), (3072, 1040, 512)])
def test_wgrad_rounding_on_randn(M, N, K):
    g = _gen(M)
    gp, xp = _randn_pair((M, N), g), _randn_pair((M, K), g)
    dw = _wgrad_call(gp, xp, M, N, K)
    torch.cuda.synchronize()
    args = (gp[0].t(), gp[1].t(), xp[0].t(), xp[1].t())
    e = _units(dw, ref3(*args), mag3(*args))
    print(f"wgrad {M}x{N}x{K} on randn: {e:.3g} units (bound {C_WGRAD})")
    assert e <= C_WGRAD


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,pad", [(2, 96, 128, 64, 64, 3, 1, 1), (2, 16, 20, 416, 256, 3, 1, 1),
                                                         (2, 48, 64, 64, 96, 3, 2, 1)])
def test_conv_rounding_on_randn(N, H, W, Cin, Cout, R, stride, pad):
    lib = L.load()
    g = _gen(H + Cin)
    v = torch.randn(N, H, W, Cin, generator=g, device=DEV)
    hi = torch.zeros(N, H, W, _pad64(Cin), dtype=torch.bfloat16, device=DEV)
    lo = hi.clone()
    hi[..., :Cin] = v.to(torch.bfloat16)
    lo[..., :Cin] = (v - hi[..., :Cin].float()).to(torch.bfloat16)
    x = XPair(hi, lo, Cin)
    wv = torch.randn(Cout, Cin, R, R, generator=g, device=DEV) / math.sqrt(Cin * R * R)
    wh, wl = wv.to(torch.bfloat16), (wv - wv.to(torch.bfloat16).float()).to(torch.bfloat16)
    from pips_b200.encoder_fast import pack_conv_weight
    packs = pack_conv_weight(wv)
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    out, _, _ = _conv_call(x, packs, Cout, R, R, stride, stride, pad, pad, None, Ho, Wo, False)
    xs = (_nchw(x, "hi"), _nchw(x, "lo"))
    ref = _conv3(xs, (wh.double(), wl.double()), stride, pad).permute(0, 2, 3, 1)
    mag = _conv3((xs[0].abs(), xs[1].abs()), (wh.double().abs(), wl.double().abs()), stride, pad).permute(0, 2, 3, 1)
    e = _units(out, ref, mag)
    msg = f"conv_tc {N}x{H}x{W} {Cin}->{Cout} {R}x{R}/{stride} on randn: {e:.3g} units"
    if (Cin, Cout, R, stride) == (64, 64, 3, 1):
        buf = _nan(N * H * W * 64)
        chunks = lib.pips_conv_rows_chunks(H, W)
        partial = _nan(N, chunks, 3, 64)
        L.check(lib.pips_conv_rows(L.ptr(x.hi), L.ptr(x.lo), N, H, W, L.ptr(packs[0]), L.ptr(packs[1]), L.ptr(buf), L.ptr(partial),
                                   _st()), "pips_conv_rows")
        torch.cuda.synchronize()
        e_rows = _units(buf.view(N, H, W, 64), ref, mag)
        msg += f", conv_rows {e_rows:.3g} units"
        e = max(e, e_rows)
    print(f"{msg} (bound {C_CONV})")
    assert e <= C_CONV


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,Cin,Cout,R,stride,pad", [(32, 96, 128, 64, 64, 3, 1, 1), (2, 16, 20, 416, 256, 3, 1, 1),
                                                         (2, 33, 41, 64, 96, 3, 2, 1)])
def test_conv_wgrad_rounding_on_randn(N, H, W, Cin, Cout, R, stride, pad):
    lib = L.load()
    g = _gen(N + H + Cin)
    Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1

    def pair(n, h, w, c):
        v = torch.randn(n, h, w, c, generator=g, device=DEV)
        hi = torch.zeros(n, h, w, _pad64(c), dtype=torch.bfloat16, device=DEV)
        lo = hi.clone()
        hi[..., :c] = v.to(torch.bfloat16)
        lo[..., :c] = (v - hi[..., :c].float()).to(torch.bfloat16)
        return XPair(hi, lo, c)

    x, d = pair(N, H, W, Cin), pair(N, Ho, Wo, Cout)
    K = R * R * x.hi.shape[-1]
    dw = _nan(Cout, K)
    scratch = _nan(max(lib.pips_conv_wgrad_scratch_floats(N, Ho, Wo, Cout, K), 1))
    L.check(lib.pips_conv_wgrad(L.ptr(d.hi), L.ptr(d.lo), d.hi.shape[-1], 1, L.ptr(x.hi), L.ptr(x.lo), N, H, W, x.hi.shape[-1], Cout,
                                R, R, stride, stride, pad, pad, L.ptr(scratch), L.ptr(dw), _st()), "pips_conv_wgrad")
    torch.cuda.synchronize()
    xs, ds = (_nchw(x, "hi"), _nchw(x, "lo")), (_nchw(d, "hi"), _nchw(d, "lo"))
    cw = torch.nn.grad.conv2d_weight
    shape = (Cout, Cin, R, R)

    def three(xa, da):
        return cw(xa[0], shape, da[0], stride=stride, padding=pad) + cw(xa[0], shape, da[1], stride=stride, padding=pad) + \
            cw(xa[1], shape, da[0], stride=stride, padding=pad)

    ref = three(xs, ds)
    mag = three(tuple(t.abs() for t in xs), tuple(t.abs() for t in ds))
    got = dw.view(Cout, R, R, -1)[..., :Cin].permute(0, 3, 1, 2)
    e = _units(got, ref, mag)
    print(f"conv_wgrad N={N} {H}x{W} {Cin}->{Cout} {R}x{R}/{stride} on randn: {e:.3g} units (bound {C_CONV_WGRAD})")
    assert e <= C_CONV_WGRAD
