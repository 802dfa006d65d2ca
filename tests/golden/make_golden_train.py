"""Golden training gradients from the UNMODIFIED reference: each loss's gradient in every parameter, per tensor digest.

    python tests/golden/make_golden_train.py          # needs the reference checkout (see make_golden.py)

For each case the reference's ``Pips(S, stride).train()`` runs one step with ground truth (``is_train=True``) on
weights from ``oracle.pips_oracle.init_state_dict`` and inputs from ``case_inputs``, both made under the default fp32
dtype with make_golden_window.py's seeding.  Each of the three losses (sequence, visibility, score map) is
differentiated on its own (``torch.autograd.grad`` with ``retain_graph``), twice:

* ``ref64``: the model ``.double()`` and the inputs in fp64, so every intermediate is fp64.  The model's constants keep
  the values the fp32 model uses -- ``linspace(0, S, S)``, ``div_term``, ``sqrt(C)`` and the +-3 window are made in
  fp32 as the code says and promote to fp64 where they meet an fp64 operand -- and the scoped shims below turn the
  reference's fp32 buffers and casts into fp64 ones, for the duration of the forward only:

  ===========================  ==============================================  =========================================
  reference site               what it does in fp32                            under ref64
  ===========================  ==============================================  =========================================
  nets/pips.py:429             ``torch.tensor(0.0).cuda()``                    ``Tensor.cuda`` is the identity (both
                                                                               runs, as in make_golden_window.py)
  nets/pips.py:382             ``CorrBlock.sample`` returns ``.float()``       ``Tensor.float`` returns an fp64 tensor
                                                                               unchanged
  utils/samp.py:11-12          ``x.float()``, ``y.float()`` of the query       the same ``Tensor.float`` shim
  utils/misc.py:53-55          ``pe_x/y/z = torch.zeros(.., float32)``: the    ``utils.misc`` sees a ``torch`` whose
                               sin/cos embedding is stored rounded to fp32     ``zeros`` makes fp64 buffers
  nets/pips.py:397             ``sqrt(torch.tensor(C).float())``               no shim: an fp32 constant (int -> float
                                                                               is untouched by the ``Tensor.float`` shim)
  nets/pips.py:504             ``fcp = torch.zeros(.., float32)``              no shim: 0 + fp64 level is exact, fp64
  nets/pips.py:519             ``torch.linspace(0, S, S)``                     no shim: an fp32 constant
  utils/misc.py:51             ``div_term`` in fp32                            no shim: an fp32 constant
  utils/samp.py:13-14, 54-57   ``H_f``, ``W_f``, ``x0.float()`` ...            no shim: integers, exact in fp32
  ===========================  ==============================================  =========================================

* ``ref32``: as shipped (only the ``Tensor.cuda`` shim), so the reference's own fp32 error is known per tensor.

The full gradients are 29 M floats per loss at S = 8, so ``digest`` keeps per tensor: max|g|, 16 elements at seeded
positions (always the first and the last) and 4 projections onto seeded +-1 vectors (each a signed sum of every
element), all in fp64.  Positions and vectors are regenerated from ``digest_seed`` by the tests.  ``has`` records which
parameters a loss reaches at all (``allow_unused``), ``gnorm`` the 2-norm of a loss's whole gradient.  Of ref32 only
its losses and ``err``, its ``digest_error`` against ref64 per loss and tensor (0 where a loss does not reach one),
are kept: that is all the tests use of it, and the file stays under 1 MB.  Each case also records its ``xys`` and a digest of its ``rgbs``, so the tests can check that they regenerate
the same inputs with the same helpers.
"""
import os
import sys
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import pips_oracle as po  # noqa: E402

FILE = os.path.join(HERE, "reference_train.npz")
LOSSES = ("seq", "vis", "ce")
DIGEST = ("max", "samples", "proj")
K_SAMPLES, K_PROJ = 16, 4

# name: dict(S, B, N, H, W, stride, iters, head_scale, seed).  H / stride and W / stride >= 16 (the reference's own
# grid_sample divides by zero on a level one pixel high: DESIGN.md section 7)
CASES = {
    "s8_st8": dict(S=8, B=2, N=13, H=128, W=160, stride=8, iters=3, head_scale=0.05, seed=31),
    "s8_st4": dict(S=8, B=1, N=16, H=64, W=96, stride=4, iters=2, head_scale=0.05, seed=32),
    "s8_undamped": dict(S=8, B=1, N=16, H=128, W=160, stride=8, iters=1, head_scale=1.0, seed=33),
    "s2_st8": dict(S=2, B=2, N=13, H=128, W=160, stride=8, iters=3, head_scale=0.05, seed=34),
    "s12_st8": dict(S=12, B=1, N=16, H=128, W=128, stride=8, iters=3, head_scale=0.05, seed=35),
    "s16_st8": dict(S=16, B=1, N=11, H=128, W=128, stride=8, iters=2, head_scale=0.05, seed=36),
}


def case_inputs(c):
    """Shared with tests/: rgbs, xys, trajs_g, vis_g, valids (fp32, CPU) of a case.  Queries on the four frame edges and
    corners as well as inside, two tracks whose ground truth leaves the map (the score-map loss drops those rows), one
    track never visible, about 10% of the valids zero -- tests/test_train_window_gpu.py's _inputs."""
    B, S, N, H, W, seed = c["B"], c["S"], c["N"], c["H"], c["W"], c["seed"]
    rgbs = po.smooth_video(B, S, H, W, seed=100 + seed)
    xys = po.random_queries(B, N, H, W, seed=200 + seed)
    edge = torch.tensor([[0.0, 0.0], [W - 1.0, 0.0], [0.0, H - 1.0], [W - 1.0, H - 1.0],
                         [W / 2 + 0.3, 0.0], [W / 2 - 0.7, H - 1.0], [0.0, H / 2 + 0.4], [W - 1.0, H / 2 - 0.2]])
    k = min(len(edge), N // 2)
    xys[:, :k] = edge[:k]
    g = torch.Generator().manual_seed(400 + seed)
    tg = xys[:, None] + torch.cumsum(torch.randn(B, S, N, 2, generator=g) * 3.0, 1)
    tg[:, S // 2:, k, 0] = -20.0                    # left of the map
    tg[:, S - 1:, k + 1, 1] = H + 20.0              # below it
    vg = (torch.rand(B, S, N, generator=g) > 0.2).float()
    vg[0, :, k + 2] = 0
    va = (torch.rand(B, S, N, generator=g) > 0.1).float()
    return rgbs, xys, tg, vg, va


def digest_seed(case_seed, name):
    return case_seed * 1_000_003 + zlib.crc32(name.encode())


def digest(tensors, seed):
    """fp64 digest of same-shaped tensors (None: no gradient) -> (max (T,), samples (T, 16), projections (T, 4)) with
    T = len(tensors); the positions and the +-1 vectors depend on the seed and the element count only"""
    n = next(t for t in tensors if t is not None).numel()
    g = torch.Generator().manual_seed(seed)
    pos = torch.cat([torch.tensor([0, n - 1]), torch.randint(0, n, (K_SAMPLES - 2,), generator=g)])
    signs = torch.randint(0, 2, (K_PROJ, n), generator=g, dtype=torch.int8).double() * 2 - 1
    mx, smp, prj = np.zeros(len(tensors)), np.zeros((len(tensors), K_SAMPLES)), np.zeros((len(tensors), K_PROJ))
    for i, t in enumerate(tensors):
        if t is None:
            continue
        v = t.detach().double().flatten().cpu()
        mx[i], smp[i], prj[i] = v.abs().max().item(), v[pos].numpy(), (signs @ v).numpy()
    return mx, smp, prj


def loss_grads(losses, params):
    """each loss's gradient in every parameter (None where a loss does not reach it)"""
    out = []
    for i, l in enumerate(losses):
        out.append(torch.autograd.grad(l, params, retain_graph=i < len(losses) - 1, allow_unused=True))
    return out


def digest_step(losses, names, grads, case_seed):
    """the record of one step: losses (3,), has (3,T), gnorm (3,), max (3,T), samples (3,T,16), proj (3,T,4)"""
    T = len(names)
    rec = dict(losses=np.array([l.item() for l in losses], dtype=np.float64),
               has=np.array([[g is not None for g in gl] for gl in grads]),
               gnorm=np.array([torch.cat([g.detach().double().flatten() for g in gl if g is not None]).norm().item()
                               for gl in grads]),
               max=np.zeros((3, T)), samples=np.zeros((3, T, K_SAMPLES)), proj=np.zeros((3, T, K_PROJ)))
    for j, n in enumerate(names):
        mx, smp, prj = digest([gl[j] for gl in grads], digest_seed(case_seed, n))
        rec["max"][:, j], rec["samples"][:, j], rec["proj"][:, j] = mx, smp, prj
    return rec


class _Fp64Buffers:
    """utils.misc's view of torch for ref64: torch, except that zeros(.., dtype=float32) makes fp64 buffers"""

    def __init__(self, real):
        self._real = real

    def __getattr__(self, name):
        return getattr(self._real, name)

    def zeros(self, *a, dtype=None, **k):
        return self._real.zeros(*a, dtype=torch.float64 if dtype == torch.float32 else dtype, **k)


def _run_reference(Pips, misc, c, sd, inputs, fp64):
    model = Pips(S=c["S"], stride=c["stride"]).train()
    model.load_state_dict(sd, strict=True)
    names = [n for n, _ in model.named_parameters()]
    if fp64:
        model.double()
        inputs = [t.double() for t in inputs]
    rgbs, xys, tg, vg, va = inputs
    real_float, real_torch = torch.Tensor.float, misc.torch
    if fp64:
        torch.Tensor.float = lambda self, *a, **k: self if self.dtype == torch.float64 else real_float(self, *a, **k)
        misc.torch = _Fp64Buffers(real_torch)
    try:
        _, _, _, losses = model(xys, rgbs, iters=c["iters"], trajs_g=tg, vis_g=vg, valids=va, is_train=True)
    finally:
        torch.Tensor.float, misc.torch = real_float, real_torch
    assert all(l.dtype == (torch.float64 if fp64 else torch.float32) for l in losses), [l.dtype for l in losses]
    return names, losses, loss_grads(losses, list(model.parameters()))


def structurally_zero(name):
    """parameters whose gradient is 0 in exact arithmetic: the fnet conv and downsample biases in front of an
    InstanceNorm, and the token-mixing FC2 biases (a per-frame constant that every consumer's LayerNorm removes)"""
    return (name.startswith("fnet.") and name.endswith("bias") and name != "fnet.conv3.bias") or name.endswith("0.fn.3.bias")


def entry(rec, i, j):
    """(max, samples, proj) of loss i's gradient in tensor j"""
    return tuple(rec[k][i, j] for k in DIGEST)


def error_scale(rec, i, j, name):
    """what an error in loss i's gradient in tensor j is measured against: its max|g|, or for a structurally zero
    tensor the 2-norm of the loss's whole gradient"""
    return rec["gnorm"][i] if structurally_zero(name) else max(rec["max"][i, j], 1e-300)


def digest_error(a, b, n, scale):
    """max over a digest's entries of |a - b| / scale; the projections (sums of n signed terms) count in units of
    sqrt(n) * scale.  a, b: (max, samples, proj) of one tensor of n elements"""
    return max(abs(a[0] - b[0]), np.abs(a[1] - b[1]).max(), np.abs(a[2] - b[2]).max() / np.sqrt(n)) / scale


def main():
    sys.path.insert(0, "/root/reference")
    torch.Tensor.cuda = lambda self, *a, **k: self
    import utils.misc as misc
    from nets.pips import Pips  # the reference, unmodified

    assert torch.get_default_dtype() == torch.float32
    torch.set_num_threads(8)
    out, names = {}, None
    for name, c in CASES.items():
        sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"], S=c["S"])
        inputs = case_inputs(c)
        shapes = {k: v.numel() for k, v in sd.items()}
        recs = {}
        for tag, fp64 in (("ref64", True), ("ref32", False)):
            nm, losses, grads = _run_reference(Pips, misc, c, sd, inputs, fp64)
            assert names is None or nm == names
            names = nm
            recs[tag] = digest_step(losses, names, grads, c["seed"])
        r64, r32 = recs["ref64"], recs["ref32"]
        assert (r64["has"] == r32["has"]).all()
        l_err = np.abs(r32["losses"] - r64["losses"]) / np.abs(r64["losses"])
        err32 = np.zeros(r64["has"].shape)
        for i in range(3):
            for j, n in enumerate(names):
                if r64["has"][i, j]:
                    err32[i, j] = digest_error(entry(r32, i, j), entry(r64, i, j), shapes[n], error_scale(r64, i, j, n))
        errs = err32[r64["has"]]
        print(f"{name}: losses {r64['losses']}; |ref32 - ref64| / |ref64|: losses {l_err.max():.2e}, gradient "
              f"digests max {max(errs):.2e} (median {np.median(errs):.2e})")
        # fp32 level: the worst tensors are fnet weights, where fp32 and fp64 take a few encoder ReLUs differently
        assert l_err.max() < 1e-6 and np.median(errs) < 1e-4 and max(errs) < 5e-2, (name, l_err, max(errs))
        for k, v in r64.items():
            out[f"{name}/ref64/{k}"] = v
        out[f"{name}/ref32/losses"], out[f"{name}/ref32/err"] = r32["losses"], err32
        out[f"{name}/xys"] = inputs[1].numpy()
        for k, v in zip(DIGEST, digest([inputs[0]], digest_seed(c["seed"], "rgbs"))):
            out[f"{name}/rgbs/{k}"] = v[0]
    out["names"] = np.array(names)
    np.savez_compressed(FILE, **out)
    print("wrote", FILE, f"{os.path.getsize(FILE) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
