"""pips_encode on the GPU: the same bits as the Python sequence of entry points it replaced, kept below as a
restatement; the block boundaries encoder_cuda saves; a short workspace; CUDA graph capture; Pips.forward on the demo
clip; and examples/track.c, the whole forward from plain C."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import pips_oracle as po          # weight generator only
from pips_b200 import Pips, _lib as L, encoder_fast as E, saverloader, torch_path
from pips_b200.encoder import Encoder

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _st():
    return torch.cuda.current_stream().cuda_stream


def restated(enc, rgb, packs=None, keep=None):
    """The encoder as encoder_fast._fnet_tc sequenced it in Python before pips_encode, one entry point call at a time.
    -> (fmaps (N, H/stride, W/stride, 128), kernels launched)."""
    E.LAUNCHES[0] = 0
    rgb = rgb.contiguous()
    ops = E._Ops(rgb.device)
    N, _, H, W = rgb.shape
    H8, W8 = H // enc.stride, W // enc.stride
    _, y, s_stem = E.stem_tc(rgb, E._packed_stem_weight(enc.conv1) if packs is None else packs[enc.conv1])
    X, XP = E._apply_pair(ops, y, s_stem, relu_main=True, plain=True)
    pk = (lambda conv: None) if packs is None else packs.__getitem__
    if keep is not None:
        keep.append(X)
    cat = E._Pair(N, H8, W8, 64 + 96 + 128 + 128, rgb.device)
    c_off = 0
    for i in range(1, 5):
        for blk in getattr(enc, f"layer{i}"):
            y1, s1 = E._conv_stats(ops, XP, blk.conv1, pk(blk.conv1))
            _, AP = E._apply_pair(ops, y1, s1, relu_main=True)
            y2, s2 = E._conv_stats(ops, AP, blk.conv2, pk(blk.conv2))
            if blk.downsample is not None:
                d, sd = E._conv_stats(ops, XP, blk.downsample[0], pk(blk.downsample[0]))
                X, XP = E._apply_pair(ops, y2, s2, r=d, stats_r=sd, relu_main=True, relu_out=True, plain=True)
            else:
                X, XP = E._apply_pair(ops, y2, s2, r=X, relu_main=True, relu_out=True, plain=True)
            if keep is not None:
                keep.append(X)
        Ns, Hs, Ws, Cs = X.shape
        L.check(ops.lib.pips_resize_pair(L.ptr(X), Ns, Hs, Ws, Cs, L.ptr(cat.hi), L.ptr(cat.lo), H8, W8, cat.Cp, c_off, _st()),
                "pips_resize_pair")
        E.LAUNCHES[0] += 1
        c_off += Cs
    y, sy = E._conv_stats(ops, cat, enc.conv2, pk(enc.conv2))
    _, AP = E._apply_pair(ops, y, sy, relu_main=True)
    out = E.conv_tc(AP, enc.conv3, bias=True, w=pk(enc.conv3))
    return out, E.LAUNCHES[0]


_ENC = {}


def _enc(stride):
    if stride not in _ENC:
        torch.manual_seed(stride)
        e = Encoder(stride=stride)
        with torch.no_grad():
            for m in e.modules():
                if isinstance(m, torch.nn.Conv2d):
                    m.bias.normal_(0, 0.1)
        _ENC[stride] = e.to(DEV)
    return _ENC[stride]


def _rgb(N, H, W, dtype, seed):
    g = torch.Generator(DEV).manual_seed(seed)
    return (torch.rand(N, 3, H, W, device=DEV, generator=g) * 255.0).to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 32])
@pytest.mark.parametrize("H,W", [(100, 136), (128, 160), (384, 512), (720, 1280)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("stride", [4, 8])
def test_encode_is_the_python_sequence(stride, dtype, H, W, N):
    enc = _enc(stride)
    rgb = _rgb(N, H, W, dtype, seed=H + N)
    with torch.no_grad():
        ref, launches = restated(enc, rgb)
        out = E.fnet_tc(enc, rgb)
    assert out.shape == (N, H // stride, W // stride, 128)
    assert torch.equal(out, ref)
    assert E.LAUNCHES[0] == launches == L.load().pips_encode_launches(N, H, W, stride)


@pytest.mark.gpu
@pytest.mark.parametrize("stride,H,W", [(8, 100, 136), (4, 96, 128)])
def test_keep_is_what_encoder_cuda_saved(monkeypatch, stride, H, W):
    """encoder_cuda's forward saves the block boundaries pips_encode keeps: the restatement's, bit for bit, and its
    output is the restatement's too"""
    enc = _enc(stride)
    rgbs = po.smooth_video(2, 3, H, W, seed=7).to(DEV).float()
    seen = {}
    inner = E._fnet_tc

    def spy(e, rgb, packs=None, keep=None):
        out = inner(e, rgb, packs=packs, keep=keep)
        seen.update(rgb=rgb, packs=packs, keep=None if keep is None else list(keep))
        return out

    monkeypatch.setattr(E, "_fnet_tc", spy)
    f = torch_path.encoder_cuda(enc, rgbs)
    assert f.requires_grad and seen["keep"] is not None and len(seen["keep"]) == 9
    old = []
    with torch.no_grad():
        ref, _ = restated(enc, seen["rgb"], packs=seen["packs"], keep=old)
    assert torch.equal(f.permute(0, 1, 3, 4, 2).flatten(0, 1), ref)
    assert [tuple(k.shape) for k in seen["keep"]] == [tuple(k.shape) for k in old] == E.keep_shapes(6, H, W)
    for i, (a, b) in enumerate(zip(seen["keep"], old)):
        assert torch.equal(a, b), i
    f.backward(torch.ones_like(f))                       # the backward recomputes from these boundaries
    assert enc.conv1.weight.grad is not None and torch.isfinite(enc.conv1.weight.grad).all()
    enc.zero_grad(set_to_none=True)


@pytest.mark.gpu
def test_workspace_one_byte_short_is_refused():
    enc = _enc(8)
    N, H, W = 2, 100, 136
    rgb = _rgb(N, H, W, torch.float32, seed=3)
    lib = L.load()
    with torch.no_grad():
        w, hold = E.encoder_weights(enc)
        need = lib.pips_encode_workspace_bytes(N, H, W, 8)
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
        out = torch.full((N, H // 8, W // 8, 128), float("nan"), device=DEV)
        torch.cuda.synchronize()
        rc = lib.pips_encode(C.byref(w), L.ptr(rgb), 0, N, H, W, 8, L.ptr(ws), need - 1, L.ptr(out), None, _st())
        assert rc != 0 and b"workspace too small" in lib.pips_last_error()
        torch.cuda.synchronize()
        assert out.isnan().all()                         # refused before any launch
        L.check(lib.pips_encode(C.byref(w), L.ptr(rgb), 0, N, H, W, 8, L.ptr(ws), need, L.ptr(out), None, _st()), "pips_encode")
        assert torch.equal(out, restated(enc, rgb)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_encode_in_a_cuda_graph(dtype):
    enc = _enc(8)
    a, b = _rgb(4, 128, 160, dtype, seed=1), _rgb(4, 128, 160, dtype, seed=2)
    with torch.no_grad():
        ref_a, ref_b = E.fnet_tc(enc, a), E.fnet_tc(enc, b)
        x = a.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            E.fnet_tc(enc, x)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = E.fnet_tc(enc, x)
        for src, ref in ((b, ref_b), (a, ref_a), (b, ref_b)):
            x.copy_(src)
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, ref)
        assert torch.equal(E.fnet_tc_graphed(enc, b), ref_b)


def _demo():
    """the demo clip's 8 frames resized to 360x640 on the device and its 16x16 query grid (tests/golden/make_golden.py)"""
    pytest.importorskip("PIL")
    from tests.golden.make_golden import DEMO_CASE, demo_decode, demo_inputs
    gold = np.load(os.path.join(ROOT, "tests", "golden", "reference_demo.npz"))
    raw = demo_decode([gold[f"jpeg{i}"].tobytes() for i in range(8)])
    rgbs, xy = demo_inputs(raw.to(DEV))
    sd = po.init_state_dict(seed=DEMO_CASE["seed"], head_scale=DEMO_CASE["head_scale"])
    return DEMO_CASE, rgbs.contiguous(), xy.to(DEV).contiguous(), sd


@pytest.mark.gpu
def test_forward_on_the_demo_clip_is_unchanged(monkeypatch):
    c, rgbs, xy, sd = _demo()
    model = Pips(S=8, stride=c["stride"]).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    with torch.no_grad():
        after = model(xy, rgbs, iters=c["iters"])
    monkeypatch.setattr(E, "_fnet_tc", lambda enc, rgb, packs=None, keep=None: restated(enc, rgb, packs, keep)[0])
    model.fnet.__dict__.pop("_fnet_plans", None)         # the captured encoder graphs hold the pips_encode call
    with torch.no_grad():
        before = model(xy, rgbs, iters=c["iters"])
    assert all(torch.equal(p, q) for p, q in zip(after[0], before[0])) and len(after[0]) == c["iters"]
    assert torch.equal(after[2], before[2])


@pytest.mark.gpu
def test_track_c_is_pips_forward(tmp_path):
    """examples/track.c, built with the host compiler against the header and the library, on the demo clip with the
    weight pack saverloader writes: the trajectories of every iteration and the visibility logits of Pips.forward at
    precision='bf16x3', bit for bit."""
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no host C compiler")
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc")))
    libdir = os.path.dirname(L.lib_path())
    exe = str(tmp_path / "track")
    r = subprocess.run([cc, "-std=c99", "-O2", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "examples", "track.c"),
                        "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"), "-L" + libdir, "-lpips_b200",
                        "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-lm", "-Wl,-rpath," + libdir, "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    c, rgbs, xy, sd = _demo()
    B, S, _, H, W = rgbs.shape
    N, iters, stride = xy.shape[1], c["iters"], c["stride"]
    model = Pips(S=S, stride=stride, precision="bf16x3", feat_dtype="fp32").to(DEV).eval()
    ck = tmp_path / "ckpt"
    ck.mkdir()
    torch.save({"optimizer_state_dict": {}, "model_state_dict": sd}, str(ck / "model-000000001.pth"))
    saverloader.load(str(ck), model)                    # loads the parameters and writes model-000000001.pack
    pack_path = ck / "model-000000001.pack"
    assert pack_path.exists()
    with torch.no_grad():
        preds, _, vis_e, _ = model(xy, rgbs, iters=iters)
    rgbs.cpu().numpy().astype(np.float32).tofile(tmp_path / "frames.f32")
    xy.cpu().numpy().astype(np.float32).tofile(tmp_path / "queries.f32")
    args = [exe, str(pack_path), str(tmp_path / "frames.f32"), str(tmp_path / "queries.f32"), *map(str, (B, S, H, W, N, stride, iters)),
            str(tmp_path / "trajs.f32"), str(tmp_path / "vis.f32")]
    env = dict(os.environ, LD_LIBRARY_PATH=libdir + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
    r = subprocess.run(args, capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    trajs = np.fromfile(tmp_path / "trajs.f32", dtype=np.float32).reshape(iters, B, S, N, 2)
    vis = np.fromfile(tmp_path / "vis.f32", dtype=np.float32).reshape(B, S, N)
    ref = torch.stack(preds).cpu().numpy()
    assert np.array_equal(trajs.view(np.int32), ref.view(np.int32)), np.abs(trajs - ref).max()
    assert np.array_equal(vis.view(np.int32), vis_e.cpu().numpy().view(np.int32)), np.abs(vis - vis_e.cpu().numpy()).max()
