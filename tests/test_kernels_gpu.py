"""Per-kernel parity: every C-ABI entry point against the CPU oracle on seeded inputs."""
import math

import pytest
import torch

from oracle import pips_oracle as po
from pips_b200 import _lib as L

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _st():
    return torch.cuda.current_stream().cuda_stream


def _sync_check():
    torch.cuda.synchronize()


def _pyramid_gpu(fmaps, feat_dtype):
    lib = L.load()
    B, S, C, H, W = fmaps.shape
    f32, bf = [], []
    h, w = H, W
    for _ in range(4):
        f32.append(torch.empty(B * S, h, w, 128, device=DEV))
        bf.append(torch.empty(B * S, h, w, 128, device=DEV, dtype=torch.bfloat16))
        h, w = h // 2, w // 2
    fm = fmaps.reshape(B * S, C, H, W).contiguous().to(DEV)
    L.check(lib.pips_pyramid_build(L.ptr(fm), B * S, H, W, L.ptr_array(f32),
                                   L.ptr_array(bf) if feat_dtype == L.FEAT_BF16 else None, _st()))
    _sync_check()
    return f32, bf


@pytest.mark.parametrize("H,W", [(16, 16), (45, 80), (23, 37)])
def test_pyramid_build(H, W):
    torch.manual_seed(0)
    fmaps = torch.randn(1, 8, 128, H, W)
    ref = po.build_pyramid(fmaps)
    f32, bf = _pyramid_gpu(fmaps, L.FEAT_BF16)
    for l in range(4):
        r = ref[l][0].permute(0, 2, 3, 1).contiguous()
        assert f32[l].shape == r.shape
        assert torch.equal(f32[l].cpu(), r), f"level {l} not bit-exact"
        assert torch.equal(bf[l].cpu(), r.to(torch.bfloat16))


def test_pyramid_build_nhwc_input():
    lib = L.load()
    torch.manual_seed(2)
    fmaps = torch.randn(1, 8, 128, 23, 37)
    ref = po.build_pyramid(fmaps)
    src = fmaps[0].permute(0, 2, 3, 1).contiguous().to(DEV)          # (8, H, W, 128)
    f32, bf = [], []
    h, w = 23, 37
    for _ in range(4):
        f32.append(torch.empty(8, h, w, 128, device=DEV))
        bf.append(torch.empty(8, h, w, 128, device=DEV, dtype=torch.bfloat16))
        h, w = h // 2, w // 2
    L.check(lib.pips_pyramid_build_nhwc(L.ptr(src), 8, 23, 37, L.ptr_array(f32), L.ptr_array(bf), _st()))
    _sync_check()
    for l in range(4):
        r = ref[l][0].permute(0, 2, 3, 1).contiguous()
        assert torch.equal(f32[l].cpu(), r) and torch.equal(bf[l].cpu(), r.to(torch.bfloat16))


def test_init_gather_clamps_indices():
    lib = L.load()
    torch.manual_seed(1)
    B, S, N, H, W = 2, 8, 40, 20, 28
    fmaps = torch.randn(B, S, 128, H, W)
    coords = torch.rand(B, S, N, 2) * torch.tensor([W + 6.0, H + 6.0]) - 3.0
    coords[0, 0, 0] = torch.tensor([0.0, 0.0])
    coords[0, 0, 1] = torch.tensor([W - 1.0, H - 1.0])
    coords[0, 0, 2] = torch.tensor([5.0, 7.0])
    ref = po.bilinear_sample2d(fmaps[:, 0], coords[:, 0, :, 0], coords[:, 0, :, 1])
    f32, _ = _pyramid_gpu(fmaps, L.FEAT_F32)
    ffeat = torch.empty(B * N, 128, device=DEV)
    ffeats = torch.empty(B * N, S, 128, device=DEV)
    cd = coords.to(DEV).contiguous()
    L.check(lib.pips_init_gather(L.ptr(f32[0]), B, S, N, H, W, L.ptr(cd), None, 0, L.ptr(ffeat), L.ptr(ffeats), _st()))
    _sync_check()
    assert (ffeat.cpu().reshape(B, N, 128) - ref).abs().max() < 1e-5
    assert torch.equal(ffeats.cpu(), ffeat.cpu().unsqueeze(1).expand(-1, S, -1))


def _corr_case(B, N, H, W, seed, wild):
    torch.manual_seed(seed)
    S = 8
    fmaps = torch.randn(B, S, 128, H, W)
    coords = torch.rand(B, S, N, 2) * torch.tensor([W - 1.0, H - 1.0])
    if wild:
        coords = torch.rand(B, S, N, 2) * torch.tensor([W + 20.0, H + 20.0]) - 10.0
        coords[0, 0, 0] = torch.tensor([3.0, 4.0])            # exact integers
        coords[0, 1, 0] = torch.tensor([-0.0, H - 1.0])
        coords[0, 2, 0] = torch.tensor([1e9, -1e9])           # diverged track
        coords[0, 3, 0] = torch.tensor([W + 2.5, -3.25])
    ffeats = torch.randn(B, S, N, 128)
    return fmaps, coords, ffeats


@pytest.mark.parametrize("feat", ["fp32", "bf16"])
@pytest.mark.parametrize("B,N,H,W,wild", [(1, 5, 16, 16, False), (2, 37, 24, 40, True), (1, 700, 45, 80, True)])
def test_corr_gather(feat, B, N, H, W, wild):
    lib = L.load()
    S = 8
    fmaps, coords, ffeats = _corr_case(B, N, H, W, 3, wild)
    feat_dtype = L.FEAT_DTYPES[feat]
    pyr_src = fmaps
    f32, bf = _pyramid_gpu(pyr_src, feat_dtype)
    lv = bf if feat_dtype == L.FEAT_BF16 else f32
    # oracle on the same (possibly bf16-rounded) pyramid values
    pyr = [t.float().cpu().reshape(B, S, *t.shape[1:]).permute(0, 1, 4, 2, 3).contiguous() for t in lv]
    finite = coords.clamp(-1e4, 1e4)
    ref_corr = po.corr_local(pyr, ffeats, finite)                                  # (B,S,N,196)
    flows = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
    times = po.times_axis(S).reshape(1, S, 1).repeat(B * N, 1, 1)
    emb = po.embedding3d(torch.cat([flows, times], 2), 64)                          # (B*N,S,195)
    ff_rows = ffeats.permute(0, 2, 1, 3).reshape(B * N, S, 128)
    ref = torch.cat([ff_rows, ref_corr.permute(0, 2, 1, 3).reshape(B * N, S, 196), emb], 2)

    M = B * N * S
    x_hi = torch.full((M, 576), 7.0, device=DEV, dtype=torch.bfloat16)
    x_lo = torch.full((M, 576), 7.0, device=DEV, dtype=torch.bfloat16)
    x_f = torch.full((M, 576), 7.0, device=DEV)
    cd, fd = coords.to(DEV).contiguous(), ff_rows.to(DEV).contiguous()
    td = po.times_axis(S).to(DEV)
    L.check(lib.pips_corr_gather(L.ptr_array(lv), feat_dtype, B, S, N, H, W, L.ptr(cd), L.ptr(fd), L.ptr(td), None, 0,
                                 L.ptr(x_hi), L.ptr(x_lo), L.ptr(x_f), 576, _st()))
    _sync_check()
    got = x_f.cpu().reshape(B * N, S, 576)
    assert torch.equal(got[..., 519:], torch.zeros_like(got[..., 519:]))
    assert torch.equal(got[..., :128], ff_rows)
    ok = flows.abs().amax(-1) < 1e5                                             # skip the diverged track's embedding
    d_corr = (got[..., 128:324] - ref[..., 128:324]).abs().max()
    assert d_corr < 2e-4, d_corr
    d_emb = (got[..., 324:519][ok] - ref[..., 324:519][ok]).abs()
    # sin/cos of arguments up to ~1e4 rad: 2 ulp of the argument reduction
    print('corr err', float(d_corr), 'emb err', float(d_emb.max()))
    assert d_emb.max() < (2e-3 if wild else 1e-5), d_emb.max()
    # hi/lo split reproduces the fp32 row to ~2^-17 relative
    rec = x_hi.float().cpu() + x_lo.float().cpu()
    xf = x_f.cpu()
    fin = torch.isfinite(xf)
    assert ((rec - xf)[fin].abs() <= xf[fin].abs() * 2 ** -15 + 1e-30).all()


def _gemm_ref(a, w, bias, epi, resid=None):
    out = a.double() @ w.double().t() + bias.double()
    if epi == L.EPI_BIAS_GELU:
        out = torch.nn.functional.gelu(out)
    if epi == L.EPI_BIAS_RESID:
        out = out + resid.double()
    return out.float()


@pytest.mark.parametrize("M,N,K", [(64, 64, 64), (100, 130, 576), (257, 512, 512)])
@pytest.mark.parametrize("epi", [L.EPI_BIAS, L.EPI_BIAS_GELU, L.EPI_BIAS_RESID])
def test_gemm_f32(M, N, K, epi):
    lib = L.load()
    torch.manual_seed(5)
    a, w, bias = torch.randn(M, K), torch.randn(N, K) / math.sqrt(K), torch.randn(N)
    out0 = torch.randn(M, N)
    ref = _gemm_ref(a, w, bias, epi, out0)
    ad, wd, bd, od = a.to(DEV), w.to(DEV), bias.to(DEV), out0.clone().to(DEV)
    L.check(lib.pips_gemm_f32(L.ptr(ad), K, L.ptr(wd), K, M, N, K, L.ptr(bd), epi, L.ptr(od), N, _st()))
    _sync_check()
    assert (od.cpu() - ref).abs().max() < 1e-4


def _split(t):
    hi = t.to(torch.bfloat16)
    lo = (t - hi.float()).to(torch.bfloat16)
    return hi, lo


@pytest.mark.parametrize("pair", [False, True, 128, 64, "auto"])
@pytest.mark.parametrize("terms", [3, 1])
@pytest.mark.parametrize("M,N,K,epi", [
    (128, 256, 64, L.EPI_BIAS),            # one tile, one K block
    (128, 256, 512, L.EPI_BIAS),           # K pipeline wraps
    (96, 512, 576, L.EPI_BIAS),            # partial M tile, 2 N tiles   (first Linear)
    (1000, 2048, 512, L.EPI_BIAS_GELU),    # FC1
    (1000, 512, 2048, L.EPI_BIAS_RESID),   # FC2
    (300, 1040, 512, L.EPI_BIAS),          # head: partial N tile, 1280 weight rows
    (40000, 512, 512, L.EPI_BIAS_RESID),   # more tiles than SMs: persistent loop
    (8 * 300, 512, 576, L.EPI_BIAS),       # the first Linear at 300 sequences
    (8 * 300, 512, 2048, L.EPI_BIAS_RESID),  # FC2 at 300 sequences
])
def test_gemm_tc(terms, M, N, K, epi, pair, monkeypatch):
    """pair=True: the cluster kernel (256x256 per cluster of two CTAs, W multicast); False / 128 / 64: the single-CTA kernel with
    128 x 256 / 128 / 64 tiles; "auto": the shape pips_gemm_tc picks from the problem size.  Exact operands
    (tests/test_tc_exact_gpu.py): the output must equal the fp64 three-term product bit for bit, at lda = ldw = K + 8,
    ldo = N + 4, ldh = N + 8, with NaN operand rows past M and N, NaN pitch columns and NaN output rows past M that must
    stay NaN.  BIAS_GELU: bit for bit with pre-activations in GELU's flat tails, then bounded per element against fp64
    with pre-activations over the centre and both tails."""
    from tests.test_tc_exact_gpu import check_exact_gemm, check_gelu_bounded
    tile = "pair" if pair is True else "" if pair == "auto" else str(pair or 256)
    monkeypatch.setenv("PIPS_B200_GEMM_TILE", tile)
    g = torch.Generator(device=DEV).manual_seed(M + N + K + terms)
    n, bad = check_exact_gemm(M, N, K, epi, terms, g, with_lo=terms == 3)
    print(f"gemm_tc {M}x{N}x{K} epi={epi} terms={terms} tile={tile or 'auto'}: {n} differing elements, poison overwritten: {bad or 'none'}")
    assert n == 0 and not bad
    if epi == L.EPI_BIAS_GELU:
        check_gelu_bounded(M, N, K, terms, terms == 3, f"tile={tile or 'auto'}")


@pytest.mark.parametrize("terms", [3, 1])
@pytest.mark.parametrize("M,N,K,epi", [(1000, 2048, 512, L.EPI_BIAS_GELU), (2048, 512, 2048, L.EPI_BIAS_RESID),
                                       (300, 1040, 512, L.EPI_BIAS),
                                       # partial last wave of the pair kernel (66 clusters on 132 SMs):
                                       (33000, 512, 512, L.EPI_BIAS_RESID),       # 258 tiles = 3 waves + 60
                                       (2400, 2048, 512, L.EPI_BIAS_GELU)])       # 80 tiles = 1 wave + 14
def test_gemm_tile_shapes_are_bit_identical(terms, M, N, K, epi, monkeypatch):
    """Every tile shape accumulates an output element over K in the same order: the schedule that pips_gemm_tc picks
    from the problem size (pair / 256 / 128 / 64) must not change a single bit -- particle sharding and chunking,
    which change M, rely on it."""
    lib = L.load()
    torch.manual_seed(5)
    Ma, Na = (M + 255) // 256 * 256, (N + 255) // 256 * 256
    a = torch.zeros(Ma, K)
    a[:M] = torch.randn(M, K)
    w = torch.zeros(Na, K)
    w[:N] = torch.randn(N, K) / math.sqrt(K)
    a_hi, a_lo = (t.to(DEV).contiguous() for t in _split(a))
    w_hi, w_lo = (t.to(DEV).contiguous() for t in _split(w))
    bias = torch.randn(N).to(DEV)
    out0 = torch.randn(M, N)
    x3 = terms == 3
    outs = {}
    for tile in ("pair", "256", "128", "64", ""):                  # "" = automatic choice
        monkeypatch.setenv("PIPS_B200_GEMM_TILE", tile)
        of = out0.clone().to(DEV)
        oh = torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)
        ol = torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)
        L.check(lib.pips_gemm_tc(L.ptr(a_hi), L.ptr(a_lo) if x3 else 0, K, Ma, L.ptr(w_hi), L.ptr(w_lo) if x3 else 0, K, Na,
                                 M, N, K, L.ptr(bias), epi, L.ptr(of), N, L.ptr(oh), L.ptr(ol) if x3 else 0, N, _st()))
        _sync_check()
        outs[tile] = (of.cpu(), oh.cpu().view(torch.int16), ol.cpu().view(torch.int16))
    for tile, o in outs.items():
        for x, y in zip(o, outs["pair"]):
            assert torch.equal(x, y), f"tile {tile!r} differs from the pair kernel"


@pytest.mark.parametrize("seqs,tc", [(37, False), (37, True), (700, True)])
def test_tokenmix_and_ln_pool(seqs, tc):
    """tc=True: the tensor-core token-mixing kernel (pips_tokenmix_tc); tc=False: the CUDA-core kernel."""
    lib = L.load()
    sd = po.init_state_dict(3)
    torch.manual_seed(11)
    x = torch.randn(seqs, 8, 512) * 2 + 0.3
    p = "delta_block.to_delta.4"
    y = po._ln(x, sd[p + ".0.norm.weight"], sd[p + ".0.norm.bias"])
    h = torch.nn.functional.gelu(torch.einsum("js,rsc->rjc", sd[p + ".0.fn.0.weight"][:, :, 0], y) + sd[p + ".0.fn.0.bias"].view(1, -1, 1))
    x_ref = x + torch.einsum("sj,rjc->rsc", sd[p + ".0.fn.3.weight"][:, :, 0], h) + sd[p + ".0.fn.3.bias"].view(1, -1, 1)
    y_ref = po._ln(x_ref, sd[p + ".1.norm.weight"], sd[p + ".1.norm.bias"])
    g = {k: v.to(DEV).contiguous() for k, v in sd.items() if k.startswith(p) or ".13." in k}
    xd = x.to(DEV).contiguous()
    y_hi = torch.empty(seqs * 8, 512, dtype=torch.bfloat16, device=DEV)
    y_lo = torch.empty_like(y_hi)
    y_f = torch.empty(seqs * 8, 512, device=DEV)
    w1 = g[p + ".0.fn.0.weight"].reshape(32, 8).contiguous()
    w2 = g[p + ".0.fn.3.weight"].reshape(8, 32).contiguous()
    args = (L.ptr(xd), seqs, L.ptr(g[p + ".0.norm.weight"]), L.ptr(g[p + ".0.norm.bias"]), L.ptr(w1),
            L.ptr(g[p + ".0.fn.0.bias"]), L.ptr(w2), L.ptr(g[p + ".0.fn.3.bias"]),
            L.ptr(g[p + ".1.norm.weight"]), L.ptr(g[p + ".1.norm.bias"]), L.ptr(y_hi), L.ptr(y_lo))
    if tc:
        L.check(lib.pips_tokenmix_tc(*args, _st()))
    else:
        L.check(lib.pips_tokenmix(*args, L.ptr(y_f), _st()))
    _sync_check()
    ex = (xd.cpu() - x_ref).abs().max().item()
    rec = (y_hi.float() + y_lo.float()).cpu().reshape(seqs, 8, 512)
    ey = (rec - y_ref).abs().max().item()
    print(f"tokenmix tc={tc} seqs={seqs}: max|dx| {ex:.2e}  max|dy| {ey:.2e}")
    assert ex < (1e-4 if tc else 2e-5)
    assert ey < 3e-4
    if not tc:
        assert (y_f.cpu().reshape(seqs, 8, 512) - y_ref).abs().max() < 2e-5

    td = "delta_block.to_delta"
    pooled_ref = po._ln(x_ref, sd[f"{td}.13.weight"], sd[f"{td}.13.bias"]).mean(1)
    pf = torch.empty(seqs, 512, device=DEV)
    ph = torch.empty(seqs, 512, dtype=torch.bfloat16, device=DEV)
    L.check(lib.pips_ln_pool(L.ptr(xd), seqs, L.ptr(g[f"{td}.13.weight"]), L.ptr(g[f"{td}.13.bias"]), L.ptr(ph), 0, L.ptr(pf), _st()))
    _sync_check()
    assert (pf.cpu() - pooled_ref).abs().max() < 1e-5
    assert (ph.float().cpu() - pooled_ref).abs().max() < 2e-2


def test_update_and_vis_head():
    lib = L.load()
    sd = po.init_state_dict(4)
    torch.manual_seed(13)
    B, S, N = 2, 8, 45
    delta = torch.randn(B * N, S, 130)
    coords = torch.rand(B, S, N, 2) * 40
    coords0 = torch.rand(B, S, N, 2) * 40
    ffeats = torch.randn(B * N, S, 128)
    # oracle: nets/pips.py:525-539
    g = torch.nn.functional.group_norm(delta[:, :, 2:].reshape(-1, 128), 1, sd["norm.weight"], sd["norm.bias"], 1e-5)
    ff_ref = torch.nn.functional.gelu(torch.nn.functional.linear(g, sd["ffeat_updater.0.weight"], sd["ffeat_updater.0.bias"])) + ffeats.reshape(-1, 128)
    c_ref = coords + delta[:, :, :2].reshape(B, N, S, 2).permute(0, 2, 1, 3)
    c_ref[:, 0] = coords0[:, 0]
    d = lambda t: t.to(DEV).contiguous()
    dd, cd, c0d, fd = d(delta.reshape(B * N, S * 130)), d(coords), d(coords0), d(ffeats)
    out = torch.empty(B, S, N, 2, device=DEV)
    # keep the device copies alive: a temporary's block would be recycled by the caching allocator
    gw, gb, wu, bu = d(sd["norm.weight"]), d(sd["norm.bias"]), d(sd["ffeat_updater.0.weight"]), d(sd["ffeat_updater.0.bias"])
    L.check(lib.pips_update(L.ptr(dd), L.ptr(cd), L.ptr(c0d), L.ptr(fd), L.ptr(gw), L.ptr(gb), L.ptr(wu), L.ptr(bu), L.ptr(out), 4.0,
                            B, S, N, _st()))
    _sync_check()
    assert (cd.cpu() - c_ref).abs().max() < 1e-6
    assert (out.cpu() - c_ref * 4.0).abs().max() < 1e-5
    assert (fd.cpu().reshape(-1, 128) - ff_ref).abs().max() < 2e-5
    vis = torch.empty(B, S, N, device=DEV)
    vw, vb = d(sd["vis_predictor.0.weight"].reshape(-1)), d(sd["vis_predictor.0.bias"])
    L.check(lib.pips_vis_head(L.ptr(fd), L.ptr(vw), L.ptr(vb), L.ptr(vis), B, S, N, _st()))
    _sync_check()
    v_ref = torch.nn.functional.linear(ff_ref, sd["vis_predictor.0.weight"], sd["vis_predictor.0.bias"]).reshape(B, N, S).permute(0, 2, 1)
    assert (vis.cpu() - v_ref).abs().max() < 1e-4


@pytest.mark.parametrize("N,H,W,cin,cout,k,stride,pad,bias", [
    (2, 24, 40, 64, 64, 3, 1, 1, False),      # layer1-like, two tile rows
    (1, 45, 80, 64, 64, 3, 1, 1, False),      # odd height, partial tiles
    (2, 48, 64, 64, 96, 3, 2, 1, False),      # stride 2, Cout padded 96 -> 128
    (2, 48, 64, 64, 96, 1, 2, 0, False),      # 1x1 stride-2 projection
    (1, 23, 40, 96, 96, 3, 1, 1, False),      # Cin padded 96 -> 128
    (1, 12, 16, 416, 256, 3, 1, 1, False),    # head conv, K = 9 x 448
    (3, 12, 16, 256, 128, 1, 1, 0, True),     # final 1x1 with bias; odd number of tiles
    (1, 192, 256, 64, 64, 3, 1, 1, False),    # full-size layer1 map: many tiles per pair
    (2, 45, 80, 64, 64, 3, 1, 1, False),      # 45 x 80: odd tile count per image (a tile past the last one), several groups
    (5, 24, 32, 128, 128, 3, 1, 1, False),    # layer4-like: 3 pair tiles per image, odd image count
    (3, 15, 24, 64, 96, 3, 2, 1, False),      # stride 2 onto an 8 x 12 map: a single, partly empty tile per image
])
def test_conv_tc(N, H, W, cin, cout, k, stride, pad, bias):
    from pips_b200.encoder_fast import _Pair, conv_tc
    torch.manual_seed(17)
    conv = torch.nn.Conv2d(cin, cout, k, stride=stride, padding=pad).to(DEV)
    x = torch.randn(N, H, W, cin, device=DEV)
    pair = _Pair(N, H, W, cin, DEV)
    pair.hi.zero_(); pair.lo.zero_()            # K padding [cin, Cp): in the encoder the producing kernels write it as zero
    hi = x.to(torch.bfloat16)
    pair.hi[..., :cin] = hi
    pair.lo[..., :cin] = (x - hi.float()).to(torch.bfloat16)
    out = conv_tc(pair, conv, bias=bias)
    out2, st = conv_tc(pair, conv, bias=bias, stats=True)       # same kernel + InstanceNorm partial statistics in the epilogue
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    mean = out.double().mean(dim=(1, 2))
    rstd = 1.0 / torch.sqrt(out.double().var(dim=(1, 2), unbiased=False) + 1e-5)
    e_mean = (st[:, 0].double() - mean).abs().max().item()
    e_rstd = ((st[:, 1].double() - rstd) / rstd).abs().max().item()
    print(f"conv_tc statistics: mean err {e_mean:.2e}, rstd rel err {e_rstd:.2e}")
    assert e_mean < 1e-5 and e_rstd < 1e-5
    ref = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), conv.weight.double(),
                                     conv.bias.double() if bias else None, stride=stride, padding=pad).permute(0, 2, 3, 1).float()
    assert out.shape == ref.shape
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"conv_tc {cin}->{cout} k{k} s{stride}: max err {err:.2e} (|out| max {scale:.2f})")
    assert err < 3e-4 * max(1.0, scale)


@pytest.mark.parametrize("N,H,W", [(2, 24, 40), (1, 45, 300), (3, 7, 130), (2, 192, 256), (1, 90, 160), (1, 33, 640)])
def test_conv_rows(N, H, W):
    """The row-ring 3x3 convolution of layer1 (csrc/conv_rows.cu; nets/pips.py:135-136, :154-157): output against an
    fp64 convolution, the InstanceNorm statistics from its epilogue against the statistics of its own output, and the
    generic tap-by-tap kernel (conv_tc.cu) on the same operands.  Widths below / across the 256-pixel pair block,
    heights that are no multiple of the 8-row work item."""
    from pips_b200.encoder_fast import _Pair, conv_rows, conv_rows_ok, conv_tc
    torch.manual_seed(23)
    conv = torch.nn.Conv2d(64, 64, 3, stride=1, padding=1).to(DEV)
    x = torch.randn(N, H, W, 64, device=DEV)
    pair = _Pair(N, H, W, 64, DEV)
    hi = x.to(torch.bfloat16)
    pair.hi.copy_(hi)
    pair.lo.copy_((x - hi.float()).to(torch.bfloat16))
    assert conv_rows_ok(pair, conv) == (W / (((W + 255) // 256) * 256) >= 0.75)      # narrow last pair blocks use conv_tc in the encoder
    out, st = conv_rows(pair, conv)
    gen = conv_tc(pair, conv)
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), conv.weight.double(), None, stride=1, padding=1).permute(0, 2, 3, 1)
    err = (out.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    mean = out.double().mean(dim=(1, 2))
    rstd = 1.0 / torch.sqrt(out.double().var(dim=(1, 2), unbiased=False) + 1e-5)
    e_mean = (st[:, 0].double() - mean).abs().max().item()
    e_rstd = ((st[:, 1].double() - rstd) / rstd).abs().max().item()
    print(f"conv_rows {N}x{H}x{W}: max err {err:.2e} (|out| max {scale:.2f}); vs conv_tc {float((out - gen).abs().max()):.2e}; "
          f"stats: mean err {e_mean:.2e}, rstd rel err {e_rstd:.2e}")
    assert err < 3e-4 * max(1.0, scale)
    assert (out - gen).abs().max().item() < 1e-4 * max(1.0, scale)     # same products, same K order: fp32 accumulation noise only
    assert e_mean < 1e-5 and e_rstd < 1e-5
