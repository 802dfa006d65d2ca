"""The score-map loss and its gradient kernels (csrc/scoremap_loss.cu, scoremap_grad.cu) checked bit for bit in the flat
tails of softplus and the sigmoid, and the basis kernels per element against fp64.

The loss and gradient kernels put a transcendental epilogue on the score s = <F_row, G_pixel> of a bf16x3 wgmma.  With
the kernels' own fp32 formulas, softplus(v) = max(v, 0) + log1pf(__expf(-|v|)) is exactly v for v >= 24 (e^-24 is below
half an ulp of 24) and exactly 0 for v <= -128 (__expf underflows).  The score gradient is -cpos / (1 + __expf(s)) at the
target pixel: exactly -cpos for s <= -24 and -0 for s >= 128 (__expf overflows); elsewhere cneg / (1 + __expf(-s)),
exactly cneg for s >= 24 and 0 for s <= -128.  So the operands below put every score in those tails:

  G[p] = sigma_p m_p u + g'  on the first 96 channels, 1 on the last 32   (u a fixed sign vector, sigma_p a sign,
  F[r] = tau_r a_r u + f'    on the first 96 channels, -b_r on the last 32   m_p = 2 on "strong" pixels, else 1,
                                                                            a_r, b_r in {2, 3} per channel)

with hi parts integers and lo parts small multiples of Q (test_tc_exact_gpu.py's scheme).  A score is then about
+-240 m_p - 80: positive ones are >= 92, negative ones <= -252, and targets sit on strong pixels, whose positive scores are
>= 284.  Every score is exact (its three-term product on the grid Q), the loss's per-split sum of positive non-target
scores is exact, and the score gradient takes only the values cneg, 0, -cpos and -0 with cpos and cneg powers of two, so
dF = sum_p c G and dG = sum_i sum_n c F are sums of exact products too.  Per output the tests work out the actual sum of
|terms| and assert through `exact_budget` that it stays below 2^24 times its grid; the pixel signs are balanced in each
64-pixel tile, which keeps the largest split's sum of positive scores near 53 000 of the 65 536 allowed.  The expected fp32
outputs are then known, whatever the tile order or split, and the tests require zero differing elements.  A target
column off by one, a masked column let through, a split running past its end, a wrong (hi, lo) operand or a mis-mapped
row or K-block changes at least one element.

Every output buffer is NaN-poisoned with trailing slack that must stay NaN.  The basis G and its adjoint have no
transcendental to flatten and are checked per element against fp64 (section 5), and section 6 bounds the rounding of the
loss and both gradients on randn data, with scores in the sigmoid's live range: per element c * 2^-24 * sum|terms|,
where a score's term counts its sum of |terms| times the derivative of what consumes it.  Every test prints its
measured error; the constants c are the largest ratio measured on an H100 80GB HBM3 (700 W) with a margin of about 2-4x.
"""
import math
from typing import NamedTuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pips_b200 import _lib as L
from tests.test_tc_exact_gpu import (DEV, Q, Ranges, Spec, _bf16_ulp, _differ, _nan, _st, _units, exact_budget, mag3, ref3)

C = 128
S = 8
SPLIT = 512                                   # pixels per split of pips_scoremap_loss
MAIN = 96                                     # channels that carry the sign vector; the other 32 carry the offset
CPOS, CNEG = 2.0 ** -1, 2.0 ** -4             # the gradient coefficients of the exact tests: powers of two
SLACK = 1024                                  # NaN elements after every output

# Bounds, in units of U times the sum of |terms| of the element.
C_BASIS = 512.0       # pips_scoremap_basis, hi + lo vs fp64 (measured 156, 45x80): the (hi, lo) split alone can be 2^-16
                      # (256 units), and the fp32 tap coordinate s * v is off by about U v, which a small weight does not scale
C_BASIS_GRAD = 512.0  # pips_scoremap_basis_grad vs the fp64 adjoint (measured 135, 45x80 level 1; 4.9 at 8x8): the same
                      # coordinate error, without the split
C_LOSS = 32.0         # pips_scoremap_loss on randn: neg_part and pos_part (measured 14.2)
C_DF = 768.0          # pips_scoremap_grad_feats on randn (measured 280): the (hi, lo) split of c alone can be 2^-16 a term
C_DG = 512.0          # pips_scoremap_grad_basis on randn (measured 177)

# (H8, W8, N, B): one tile; a partial tile; level 3 a single pixel (9, 15) and (15, 8); P = 512 exactly; a 17-pixel last
# split; 8 splits with a 16-pixel tail; the evaluation shape
CASES = [(8, 8, 1, 1), (8, 9, 63, 2), (9, 15, 64, 1), (15, 8, 65, 2), (16, 32, 129, 1), (23, 23, 300, 2),
         (45, 80, 65, 1), (48, 64, 129, 2)]
RANDN_CASES = [(9, 15, 129, 1), (23, 23, 65, 2), (45, 80, 300, 1), (48, 64, 129, 2)]
# other window lengths (pips_scoremap_loss_window), all with B = 2 so that a wrong b*S frame stride shows
WINDOWS = [2, 5, 12, 16]
WINDOW_CASES = [CASES[1], CASES[5], CASES[7]]


def _ids(cases):
    return [f"{h}x{w}-N{n}-B{b}" for h, w, n, b in cases]


def _windows(cases, other, windows):
    """pytest params (H8, W8, N, B, S): `cases` at S = 8 under their plain ids, `other` at each of `windows`"""
    return ([pytest.param(*c, S, id=i) for c, i in zip(cases, _ids(cases))]
            + [pytest.param(*c, s, id=f"{i}-S{s}") for s in windows for c, i in zip(other, _ids(other))])


# ------------------------------------------------------------------------------------------------ problems

class Problem(NamedTuple):
    H8: int
    W8: int
    N: int
    B: int
    g_hi: torch.Tensor        # (frames, P, C) bf16
    g_lo: torch.Tensor
    f_hi: torch.Tensor        # (I, frames, N, C) bf16; the fp32 ffeats are hi + lo
    f_lo: torch.Tensor
    target: torch.Tensor      # (frames, N) int32: pixel, or -1
    S: int = S                # window length: frame b*S + s of the basis serves row ((b N + n), s)

    @property
    def frames(self):
        return self.B * self.S

    @property
    def P(self):
        return self.H8 * self.W8

    @property
    def I(self):
        return self.f_hi.shape[0]

    @property
    def n_split(self):
        return (self.P + SPLIT - 1) // SPLIT

    @property
    def f(self):
        return self.f_hi.float() + self.f_lo.float()

    def to(self, dev):
        return self._replace(**{k: getattr(self, k).to(dev) for k in ("g_hi", "g_lo", "f_hi", "f_lo", "target")})


def _signs(shape, g):
    return torch.randint(0, 2, shape, generator=g).float() * 2 - 1


def edge_pixels(P):
    """pixel 0 and P - 1, both sides of the first tile edge and of the first split edge, the last tile's first pixel"""
    return sorted({p for p in (0, 1, 63, 64, 511, 512, (P - 1) // 64 * 64, P - 2, P - 1) if 0 <= p < P})


def _targets(P, N, frames, strong, g):
    """every fifth row -1; the first rows of each frame on the edge pixels in turn, the others on random strong pixels"""
    edges = edge_pixels(P)
    target = torch.empty(frames, N, dtype=torch.int32)
    for fr in range(frames):
        pool = strong[fr].nonzero().flatten()
        t = pool[torch.randint(0, len(pool), (N,), generator=g)]
        k = min(N, 2 * len(edges))
        t[:k] = torch.tensor([edges[(fr + n) % len(edges)] for n in range(k)])
        target[fr] = t.int()
    rows = torch.arange(frames * N).view(frames, N)
    target[rows % 5 == 3] = -1
    return target


def exact_problem(H8, W8, N, B, I, seed, S=S):
    """the tail operands of the module docstring, on the host"""
    g = torch.Generator().manual_seed(seed)
    frames, P = B * S, H8 * W8
    u = _signs((C,), g)
    half = torch.tensor([1.0] * 32 + [-1.0] * 32)
    tiles = (P + 63) // 64
    sigma = torch.stack([torch.cat([half[torch.randperm(64, generator=g)] for _ in range(tiles)])[:P] for _ in range(frames)])
    strong = torch.rand(frames, P, generator=g) < 1 / 16
    strong[:, edge_pixels(P)] = True
    g_hi = torch.ones(frames, P, C)
    g_hi[..., :MAIN] = (sigma * (1.0 + strong.float()))[..., None] * u[:MAIN]
    _, g_lo = Spec(0, 2).draw((frames, P, C), g)
    tau = _signs((I, frames, N, 1), g)
    f_hi = -torch.randint(2, 4, (I, frames, N, C), generator=g).float()
    f_hi[..., :MAIN] *= -tau * u[:MAIN]
    _, f_lo = Spec(0, 1).draw((I, frames, N, C), g)
    return Problem(H8, W8, N, B, g_hi.to(torch.bfloat16), g_lo, f_hi.to(torch.bfloat16), f_lo,
                   _targets(P, N, frames, strong, g), S)


def randn_problem(H8, W8, N, B, I, seed, S=S):
    """randn G and F scaled so that the scores are about N(0, 4^2): in the sigmoid's live range"""
    g = torch.Generator().manual_seed(seed)
    frames, P = B * S, H8 * W8
    G = torch.randn(frames, P, C, generator=g) * 0.35
    Fv = torch.randn(I, frames, N, C, generator=g)
    g_hi, f_hi = G.to(torch.bfloat16), Fv.to(torch.bfloat16)
    target = torch.randint(0, P, (frames, N), generator=g, dtype=torch.int32)
    target[torch.rand(frames, N, generator=g) < 0.2] = -1
    return Problem(H8, W8, N, B, g_hi, (G - g_hi.float()).to(torch.bfloat16), f_hi, (Fv - f_hi.float()).to(torch.bfloat16),
                   target, S)


# ------------------------------------------------------------------------------------------------ fp64 references

def scores(p, mag=False):
    """(I, frames, N, P) fp64 three-term scores (or their sums of |terms|) of every iteration, row and pixel"""
    fn = mag3 if mag else ref3
    out = torch.empty(p.I, p.frames, p.N, p.P, dtype=torch.float64, device=p.g_hi.device)
    for fr in range(p.frames):
        a_hi, a_lo = p.f_hi[:, fr].reshape(-1, C), p.f_lo[:, fr].reshape(-1, C)
        out[:, fr] = fn(a_hi, a_lo, p.g_hi[fr], p.g_lo[fr]).view(p.I, p.N, p.P)
    return out


def _target_mask(p):
    """(frames, N, P) True at each row's target pixel; (frames, N) True for rows with a target"""
    t = p.target.long()
    return torch.arange(p.P, device=t.device) == t[..., None], t >= 0


def _split_sums(x, p):
    """(..., P) -> (rows, n_split): sums over each split's pixels"""
    x = F.pad(x, (0, p.n_split * SPLIT - p.P))
    return x.reshape(-1, p.n_split, SPLIT).sum(-1)


def assert_in_tails(p, s):
    """every score where the kernels' epilogues are flat: targets <= -24 or >= 128, the others >= 24 or <= -128"""
    is_t, _ = _target_mask(p)
    ok = torch.where(is_t, (s <= -24) | (s >= 128), (s >= 24) | (s <= -128))
    assert bool(ok.all()), f"{int((~ok).sum())} scores outside the flat tails"


def expected_loss(p, s):
    """(neg_part (rows, n_split), pos_part (rows,)) of one iteration's exact tail scores s (frames, N, P)"""
    is_t, kept = _target_mask(p)
    neg = _split_sums(torch.where(~is_t & (s > 0) & kept[..., None], s, 0.0), p)
    st = s.gather(-1, p.target.long().clamp(min=0)[..., None])[..., 0]
    pos = torch.where(kept & (st < 0), -st, 0.0).reshape(-1)
    return neg, pos


def expected_c(p, s):
    """(I, frames, N, P): the score gradient of the tail scores, in {cneg, 0, -cpos}"""
    is_t, kept = _target_mask(p)
    c = torch.where(is_t, torch.where(s < 0, -CPOS, 0.0), torch.where(s > 0, CNEG, 0.0))
    return c.double() * kept[..., None]


def grad_refs(p, c):
    """dF (I, frames, N, C) = c (G_hi + G_lo) and dG (frames, P, C) = sum_i c^T (F_hi + F_lo) in fp64: with c_lo = 0
    (or for a true fp64 reference) the three-term products the kernels compute"""
    g = p.g_hi.double() + p.g_lo.double()
    f = p.f_hi.double() + p.f_lo.double()
    dF = torch.einsum("ifnp,fpc->ifnc", c, g)
    dG = torch.einsum("ifnp,ifnc->fpc", c, f)
    return dF, dG


def grad_mags(p, w):
    """the same sums with |weights| w and |hi| + |lo|"""
    g = p.g_hi.double().abs() + p.g_lo.double().abs()
    f = p.f_hi.double().abs() + p.f_lo.double().abs()
    return torch.einsum("ifnp,fpc->ifnc", w, g), torch.einsum("ifnp,ifnc->fpc", w, f)


def _sum_budget(total, grid):
    """exact_budget for a sum of values on `grid` whose sum of |terms| is `total`"""
    return exact_budget(1, Ranges(total, grid, 0.0, grid), Ranges(1.0, 1.0, 0.0, 1.0))


R_F = Ranges(3.0, 1.0, Q, Q)                  # F: hi in +-{2, 3}, lo = +-Q
R_G = Ranges(2.0, 1.0, 2 * Q, Q)              # G: hi in {+-1, +-2}, lo in +-{1, 2} Q


def exact_budgets(p, s):
    """asserts that the scores, the loss's split sums, dF and dG of the exact problem are exact in fp32"""
    exact_budget(C, R_F, R_G)
    neg, _ = expected_loss(p, s[0])
    _sum_budget(neg.max().item(), Q)
    grid = min(CPOS, CNEG) * Q
    dF_mag, dG_mag = grad_mags(p, expected_c(p, s).abs())
    _sum_budget(dF_mag.max().item(), grid)
    _sum_budget(dG_mag.max().item(), grid)
    return neg.max().item(), dF_mag.max().item(), dG_mag.max().item()


# ------------------------------------------------------------------------------------------------ 1. on the host

def _softplus32(v):
    v = np.asarray(v, dtype=np.float32)
    return np.maximum(v, np.float32(0)) + np.log1p(np.exp(-np.abs(v)))


def _score_grad32(s, at_target):
    s = np.asarray(s, dtype=np.float32)
    with np.errstate(over="ignore"):
        one = np.float32(1)
        return np.where(at_target, np.float32(-CPOS) / (one + np.exp(s)), np.float32(CNEG) / (one + np.exp(-s)))


def test_flat_tails_and_exact_operands_without_gpu():
    """In float32, the kernels' softplus and score gradient are flat past the tails the tests use.  The operands put every
    score in those tails, every output passes exact_budget, and the fp64 references equal int64 computations in grid
    units: Q^2 for scores and split sums, CNEG Q for dF and dG."""
    up = np.arange(24, 4096, 0.125, dtype=np.float32)
    down = -np.arange(128, 4096, 0.125, dtype=np.float32)
    assert (_softplus32(up) == up).all() and (_softplus32(down) == 0).all()
    assert (_score_grad32(-up, True) == np.float32(-CPOS)).all()
    g = _score_grad32(-down, True)
    assert (g == 0).all() and np.signbit(g).all()                             # -0
    assert (_score_grad32(up, False) == np.float32(CNEG)).all() and (_score_grad32(down, False) == 0).all()

    for case, I in ((CASES[3], 3), (CASES[5], 2), (CASES[7], 1)):
        p = exact_problem(*case, I=I, seed=sum(case))
        s = scores(p)
        assert_in_tails(p, s)
        budgets = exact_budgets(p, s)
        # the operands are what the kernels see: hi = rn_bf16(hi + lo) for the fp32 ffeats the kernels split
        assert torch.equal(p.f.to(torch.bfloat16), p.f_hi) and torch.equal((p.f - p.f_hi.float()).to(torch.bfloat16), p.f_lo)
        # the float32 epilogues on the fp64 scores give the expected values
        is_t, kept = _target_mask(p)
        s32 = s.float()
        assert torch.equal(s32.double(), s)
        c32 = torch.from_numpy(_score_grad32(s32.numpy(), is_t.expand_as(s).numpy()).astype(np.float64)) * kept[..., None]
        assert torch.equal(c32, expected_c(p, s))
        sp = torch.from_numpy(_softplus32(s32[0].numpy()).astype(np.float64))
        neg, pos = expected_loss(p, s[0])
        assert torch.equal(_split_sums(torch.where(~is_t & kept[..., None], sp, 0.0), p), neg)
        spt = torch.from_numpy(_softplus32(-s32[0].numpy()).astype(np.float64)).gather(-1, p.target.long().clamp(min=0)[..., None])
        assert torch.equal(torch.where(kept, spt[..., 0], 0.0).reshape(-1), pos)
        # int64 in grid units
        u = {k: (getattr(p, k).double() / Q).long() for k in ("f_hi", "f_lo", "g_hi", "g_lo")}
        assert all(torch.equal(u[k].double() * Q, getattr(p, k).double()) for k in u)
        su = torch.einsum("ifnc,fpc->ifnp", u["f_hi"] + u["f_lo"], u["g_hi"]) + torch.einsum("ifnc,fpc->ifnp", u["f_hi"], u["g_lo"])
        assert torch.equal(su.double() * Q * Q, s)
        negu = _split_sums(torch.where(~is_t & (su[0] > 0) & kept[..., None], su[0], 0), p)
        assert torch.equal(negu.double() * Q * Q, neg)
        c = expected_c(p, s)
        cu = (c / CNEG).long()
        assert torch.equal(cu.double() * CNEG, c)
        dF, dG = grad_refs(p, c)
        dFu = torch.einsum("ifnp,fpc->ifnc", cu, u["g_hi"] + u["g_lo"])
        dGu = torch.einsum("ifnp,ifnc->fpc", cu, u["f_hi"] + u["f_lo"])
        assert torch.equal(dFu.double() * (CNEG * Q), dF) and torch.equal(dGu.double() * (CNEG * Q), dG)
        print(f"exact score-map problem {case} I={I}: largest split sum {budgets[0]:.0f} of {2.0 ** 24 * Q:.0f}, "
              f"dF {budgets[1]:.1f} and dG {budgets[2]:.1f} of {2.0 ** 24 * CNEG * Q:.0f}")


# ------------------------------------------------------------------------------------------------ GPU helpers

def _buf(*shape):
    """a NaN tensor of `shape` followed by SLACK NaN elements: (the view, the whole buffer)"""
    n = math.prod(shape)
    whole = _nan(n + SLACK)
    return whole[:n].view(shape), whole


def _slack_ok(whole, n):
    return bool(torch.isnan(whole[n:]).all())


def _rows_layout(f, S=S):
    """(frames, N, C) ffeats of one iteration -> pips_scoremap_loss's ((b N + n), s, c)"""
    frames, N, _ = f.shape
    return f.view(frames // S, S, N, C).permute(0, 2, 1, 3).contiguous()


def run_loss(p, i):
    neg, neg_w = _buf(p.frames * p.N, p.n_split)
    pos, pos_w = _buf(p.frames * p.N)
    ff = _rows_layout(p.f[i], p.S)
    lib = L.load()
    fn, name = (lib.pips_scoremap_loss, "pips_scoremap_loss") if p.S == 8 else \
        (lib.pips_scoremap_loss_window, "pips_scoremap_loss_window")
    L.check(fn(L.ptr(p.g_hi), L.ptr(p.g_lo), L.ptr(ff), p.B, p.S, p.N, p.H8, p.W8, L.ptr(p.target), L.ptr(neg), L.ptr(pos),
               _st()), name)
    torch.cuda.synchronize()
    return neg, pos, _slack_ok(neg_w, neg.numel()) and _slack_ok(pos_w, pos.numel())


def run_grads(p, coef):
    lib = L.load()
    dF, dF_w = _buf(p.I, p.frames, p.N, C)
    dG, dG_w = _buf(p.frames, p.P, C)
    f = p.f.contiguous()
    L.check(lib.pips_scoremap_grad_feats(L.ptr(p.g_hi), L.ptr(p.g_lo), L.ptr(f), p.I, p.B, S, p.N, p.H8, p.W8,
                                         L.ptr(p.target), L.ptr(coef), L.ptr(dF), _st()), "pips_scoremap_grad_feats")
    L.check(lib.pips_scoremap_grad_basis(L.ptr(p.g_hi), L.ptr(p.g_lo), L.ptr(p.f_hi), L.ptr(p.f_lo), p.I, p.B, S, p.N, p.H8,
                                         p.W8, L.ptr(p.target), L.ptr(coef), L.ptr(dG), _st()), "pips_scoremap_grad_basis")
    torch.cuda.synchronize()
    return dF, dG, _slack_ok(dF_w, dF.numel()) and _slack_ok(dG_w, dG.numel())


# ------------------------------------------------------------------------------------------------ 3. the loss, exact

@pytest.mark.gpu
@pytest.mark.parametrize("H8,W8,N,B,S", _windows(CASES, WINDOW_CASES, WINDOWS))
def test_scoremap_loss_exact(H8, W8, N, B, S):
    """neg_part per (row, split) and pos_part bit-equal to the sums of the tail scores; rows without a target hold 0.
    Other window lengths through pips_scoremap_loss_window."""
    p = exact_problem(H8, W8, N, B, I=2, seed=H8 * W8 + N + B, S=S).to(DEV)
    s = scores(p)
    assert_in_tails(p, s)
    exact_budgets(p, s)
    _, kept = _target_mask(p)
    msgs, fails = [], 0
    for i in range(p.I):
        e_neg, e_pos = expected_loss(p, s[i])
        neg, pos, slack = run_loss(p, i)
        n_neg, n_pos = _differ(neg, e_neg), _differ(pos, e_pos)
        dropped = ~kept.reshape(-1)
        zeros = bool((neg[dropped] == 0).all() and (pos[dropped] == 0).all())
        msgs.append(f"iteration {i}: neg {n_neg}, pos {n_pos} differing; dropped rows 0: {zeros}; slack NaN: {slack}")
        fails += n_neg + n_pos + (not zeros) + (not slack)
    print(f"scoremap_loss {H8}x{W8} N={N} B={B} S={S} ({p.n_split} splits): " + "; ".join(msgs))
    assert fails == 0


# ------------------------------------------------------------------------------------------------ 4. the gradients, exact

@pytest.mark.gpu
@pytest.mark.parametrize("I", [1, 3, 6])
@pytest.mark.parametrize("H8,W8,N,B", CASES, ids=_ids(CASES))
def test_scoremap_grads_exact(H8, W8, N, B, I):
    """dF (pips_scoremap_grad_feats) and dG (pips_scoremap_grad_basis) bit-equal to the sums of c * operand with c in
    {cneg, 0, -cpos, -0}; dF of rows without a target is 0"""
    p = exact_problem(H8, W8, N, B, I=I, seed=7 * I + H8 * W8 + N + B).to(DEV)
    s = scores(p)
    assert_in_tails(p, s)
    exact_budgets(p, s)
    e_dF, e_dG = grad_refs(p, expected_c(p, s))
    coef = torch.tensor([CPOS, CNEG], device=DEV)
    dF, dG, slack = run_grads(p, coef)
    n_dF, n_dG = _differ(dF, e_dF), _differ(dG, e_dG)
    _, kept = _target_mask(p)
    zeros = bool((dF[:, ~kept] == 0).all())
    print(f"scoremap grads {H8}x{W8} N={N} B={B} I={I}: dF {n_dF}, dG {n_dG} differing elements; dropped rows 0: {zeros}; "
          f"slack NaN: {slack}")
    assert n_dF == 0 and n_dG == 0 and zeros and slack


# ------------------------------------------------------------------------------------------------ 5. the basis and its adjoint

def _level_shapes(H8, W8):
    return [(H8 >> l, W8 >> l) for l in range(4)]


def basis_ref(levels, H8, W8):
    """sum_l interpolate(level_l, align_corners=True) / sqrt(128) of channels-last levels (frames, h, w, C) ->
    (frames, P, C), in the levels' dtype"""
    frames = levels[0].shape[0]
    out = sum(F.interpolate(lv.permute(0, 3, 1, 2), (H8, W8), mode="bilinear", align_corners=True) for lv in levels)
    return (out / math.sqrt(C)).permute(0, 2, 3, 1).reshape(frames, H8 * W8, C)


@pytest.mark.gpu
@pytest.mark.parametrize("H8,W8,N,B", CASES, ids=_ids(CASES))
def test_scoremap_basis_per_element(H8, W8, N, B):
    """pips_scoremap_basis: hi + lo within C_BASIS U of the fp64 basis of the fp32 levels (units of the basis of
    |levels|), and (hi, lo) a canonical split: |lo| <= ulp(hi) / 2"""
    g = torch.Generator(device=DEV).manual_seed(H8 * W8 + B)
    frames, P = B * S, H8 * W8
    lv = [torch.randn(frames, h, w, C, generator=g, device=DEV) for h, w in _level_shapes(H8, W8)]
    hi = _nan(frames * P * C + SLACK, dtype=torch.bfloat16)
    lo = _nan(frames * P * C + SLACK, dtype=torch.bfloat16)
    L.check(L.load().pips_scoremap_basis(L.ptr_array(lv), frames, H8, W8, L.ptr(hi), L.ptr(lo), _st()), "pips_scoremap_basis")
    torch.cuda.synchronize()
    n = frames * P * C
    slack = bool(torch.isnan(hi[n:].float()).all() and torch.isnan(lo[n:].float()).all())
    hi_, lo_ = hi[:n].view(frames, P, C), lo[:n].view(frames, P, C)
    ref = basis_ref([v.double() for v in lv], H8, W8)
    mag = basis_ref([v.double().abs() for v in lv], H8, W8)
    e = _units(hi_.double() + lo_.double(), ref, mag)
    canonical = bool((lo_.double().abs() <= _bf16_ulp(hi_) / 2).all())
    print(f"scoremap_basis {H8}x{W8} B={B}: {e:.3g} units of U sum|terms| (bound {C_BASIS}); |lo| <= ulp(hi)/2: "
          f"{canonical}; slack NaN: {slack}")
    assert e <= C_BASIS and canonical and slack


@pytest.mark.gpu
@pytest.mark.parametrize("H8,W8,N,B", CASES, ids=_ids(CASES))
def test_scoremap_basis_grad_per_element(H8, W8, N, B):
    """pips_scoremap_basis_grad against the fp64 autograd of basis_ref for a randn dG, per element within C_BASIS_GRAD U
    times the adjoint applied to |dG|, on every level (level 3 is a single row or column below H8 or W8 = 16, where the
    gather's range is the whole fine axis)"""
    g = torch.Generator(device=DEV).manual_seed(3 * H8 * W8 + B)
    frames, P = B * S, H8 * W8
    dG = torch.randn(frames, P, C, generator=g, device=DEV)
    shapes = _level_shapes(H8, W8)
    bufs = [_buf(frames, h, w, C) for h, w in shapes]
    L.check(L.load().pips_scoremap_basis_grad(L.ptr(dG), frames, H8, W8, L.ptr_array([b[0] for b in bufs]), _st()),
            "pips_scoremap_basis_grad")
    torch.cuda.synchronize()
    lv = [torch.zeros(frames, h, w, C, dtype=torch.float64, device=DEV, requires_grad=True) for h, w in shapes]
    out = basis_ref(lv, H8, W8)
    ref = torch.autograd.grad(out, lv, dG.double(), retain_graph=True)
    mag = torch.autograd.grad(out, lv, dG.double().abs())
    es = [_units(b[0], r, m) for b, r, m in zip(bufs, ref, mag)]
    slack = all(_slack_ok(w, b.numel()) for b, w in bufs)
    print(f"scoremap_basis_grad {H8}x{W8} B={B} (levels {shapes}): " + ", ".join(f"{e:.3g}" for e in es)
          + f" units of U sum|terms| (bound {C_BASIS_GRAD}); slack NaN: {slack}")
    assert max(es) <= C_BASIS_GRAD and slack


# ------------------------------------------------------------------------------------------------ 6. randn data

@pytest.mark.gpu
@pytest.mark.parametrize("H8,W8,N,B,S", _windows(RANDN_CASES, [RANDN_CASES[1]], [5, 16]))
def test_scoremap_rounding_on_randn(H8, W8, N, B, S):
    """the loss and both gradients with scores in the sigmoid's live range, per element: a score's term counts
    softplus(s) + sigma(s) sum|terms of s| in the loss, |c| + |dc/ds| sum|terms of s| in the gradients, times |Y|.
    At other window lengths the loss alone (pips_scoremap_loss_window): the gradient kernels take S = 8 only."""
    I = 3
    p = randn_problem(H8, W8, N, B, I, seed=H8 + W8 + N + B, S=S).to(DEV)
    s, m = scores(p), scores(p, mag=True)
    is_t, kept = _target_mask(p)
    k = int(kept.sum()) * I
    coef = torch.tensor([1.0 / k, 1.0 / (k * (p.P - 1))], device=DEV)
    cpos, cneg = coef.double().tolist()
    st = torch.where(is_t, -s, s)                  # the argument of each softplus: -s at the target
    sp, sig = F.softplus(st), torch.sigmoid(st)
    mask = kept[..., None]
    # loss, every iteration
    e_loss = 0.0
    fails = 0
    for i in range(I):
        neg, pos, slack = run_loss(p, i)
        nt = ~is_t & mask
        e_neg = _split_sums(torch.where(nt, sp[i], 0.0), p)
        m_neg = _split_sums(torch.where(nt, sp[i] + sig[i] * m[i], 0.0), p)
        tt = is_t & mask
        e_pos = torch.where(tt, sp[i], 0.0).sum(-1).reshape(-1)
        m_pos = torch.where(tt, sp[i] + sig[i] * m[i], 0.0).sum(-1).reshape(-1)
        e_loss = max(e_loss, _units(neg, e_neg, m_neg), _units(pos, e_pos, m_pos))
        fails += not slack
    if S != 8:
        print(f"scoremap {H8}x{W8} N={N} B={B} S={S} I={I} on randn: loss {e_loss:.3g} (bound {C_LOSS}) units of U "
              f"sum|terms|; slack NaN: {not fails}")
        assert e_loss <= C_LOSS and not fails
        return
    # gradients: c = -cpos sigma(-s) at the target, cneg sigma(s) elsewhere
    c = torch.where(is_t, -cpos * sig, cneg * sig) * mask
    dc = torch.where(is_t, cpos, cneg).double() * sig * (1 - sig) * mask
    e_dF, e_dG = grad_refs(p, c)
    m_dF, m_dG = grad_mags(p, c.abs() + dc * m)
    dF, dG, slack = run_grads(p, coef)
    fails += not slack
    u_dF, u_dG = _units(dF, e_dF, m_dF), _units(dG, e_dG, m_dG)
    print(f"scoremap {H8}x{W8} N={N} B={B} I={I} on randn: loss {e_loss:.3g} (bound {C_LOSS}), dF {u_dF:.3g} (bound {C_DF}), "
          f"dG {u_dG:.3g} (bound {C_DG}) units of U sum|terms|; slack NaN: {not fails}")
    assert e_loss <= C_LOSS and u_dF <= C_DF and u_dG <= C_DG and not fails
