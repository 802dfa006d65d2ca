"""Differentiable PyTorch path of ``Pips.forward`` for the cases the CUDA inference loop does not
cover: ground truth given (losses requested, nets/pips.py:600-606), ``is_train=True`` (no frame-0
lock, gradients needed) or a summary writer that wants to log this step.  It runs wherever the
tensors live (it is what ``train.py`` / ``test_on_flt.py`` exercise) and keeps the reference's
semantics, including the dense score map ``fcps`` that only the score-map loss consumes -- except with
``model.loss_path == 'fused'`` on CUDA tensors, where ``fused_score_map_loss`` computes that loss and its gradients
without ``fcps``, and with ``model.mixer_path == 'cuda'`` on CUDA tensors, where ``delta_block_cuda`` runs the
DeltaBlock mixer forward and backward on the sm_90a kernels, with ``model.encoder_path == 'cuda'`` on CUDA tensors
that need no gradient, where ``encoder_cuda`` does the same for the feature encoder, and with ``model.corr_path ==
'cuda'`` on CUDA tensors (feature maps of at least 8x8), where ``local_corr_cuda`` computes the local correlation
and its gradients without the all-pairs volumes.

Not used -- and not a fallback -- for plain inference: that path is CUDA-only (pips.py).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def masked_mean(x, mask, eps=1e-6):
    """utils/basic.py:59 (reduce_masked_mean over all dims)."""
    return (x * mask).sum() / (eps + mask.sum())


def balanced_ce_loss(pred, gt, valid=None):
    """nets/pips.py:14-37."""
    assert pred.shape == gt.shape
    valid = torch.ones_like(gt) if valid is None else valid
    assert valid.shape == gt.shape
    pos, neg = (gt > 0.95).float(), (gt < 0.05).float()
    a = -(pos * 2.0 - 1.0) * pred
    b = F.relu(a)
    loss = b + torch.log(torch.exp(-b) + torch.exp(a - b))
    return masked_mean(loss, pos * valid) + masked_mean(loss, neg * valid), loss


def sequence_loss(flow_preds, flow_gt, vis, valids, gamma=0.8):
    """nets/pips.py:39-56."""
    B, S, N, D = flow_gt.shape
    assert D == 2 and vis.shape[1] == S and valids.shape[1] == S
    n = len(flow_preds)
    total = 0.0
    for i, pred in enumerate(flow_preds):
        l1 = (pred - flow_gt).abs().mean(dim=3)
        total = total + gamma ** (n - i - 1) * masked_mean(l1, valids)
    return total / n


def score_map_loss(fcps, trajs_g, vis_g, valids):
    """nets/pips.py:58-90: balanced CE between every iteration's score map and a one-hot at the
    rounded ground-truth position, over visible + valid + in-bounds targets."""
    B, S, I, N, H8, W8 = fcps.shape
    fcp = fcps.permute(0, 1, 3, 2, 4, 5).reshape(B * S * N, I, H8, W8)
    xy = trajs_g.reshape(B * S * N, 2).round().long()
    x, y = xy[:, 0], xy[:, 1]
    keep = (x >= 0) & (x <= W8 - 1) & (y >= 0) & (y <= H8 - 1) & (valids.reshape(-1) > 0) & (vis_g.reshape(-1) > 0)
    fcp, x, y = fcp[keep], x[keep], y[keep]
    gt = torch.zeros_like(fcp)
    gt[torch.arange(fcp.shape[0], device=fcp.device), :, y, x] = 1
    loss, _ = balanced_ce_loss(fcp.reshape(-1), gt.reshape(-1))
    return loss


def score_map_targets(trajs_g, vis_g, valids, H8, W8):
    """The rows score_map_loss keeps (nets/pips.py:63-67: rounded half to even, inside the map, valid and visible) and
    their target pixel y*W8 + x, -1 for every other row: the (B,S,N) int32 targets of pips_scoremap_loss.  trajs_g is
    in feature-map pixels."""
    B, S, N, _ = trajs_g.shape
    xy = trajs_g.reshape(B * S * N, 2).round().long()
    x, y = xy[:, 0], xy[:, 1]
    keep = (x >= 0) & (x <= W8 - 1) & (y >= 0) & (y <= H8 - 1) & (valids.reshape(-1) > 0) & (vis_g.reshape(-1) > 0)
    return torch.where(keep, y * W8 + x, torch.full_like(x, -1)).to(torch.int32).reshape(B, S, N).contiguous()


def _window_entry(name, S):
    """The C entry point for a window of S frames: ``name`` itself at S = 8, its ``_window`` sibling (2 <= S <= 16; the
    same kernel, so the same bits at S = 8) otherwise."""
    return name if S == 8 else name + "_window"


class _FusedScoreMapLoss(torch.autograd.Function):
    """score_map_loss from the per-iteration ffeats and the pyramid, without the dense score maps, forward and backward
    on the CUDA kernels of csrc/scoremap_loss.cu and csrc/scoremap_grad.cu.  Saves G (hi, lo), the targets and the
    ffeats; the backward recomputes the scores tile by tile."""

    @staticmethod
    def forward(ctx, target, n_iters, *tensors):
        from . import _lib as L
        from .engine import _score_map_loss
        lib = L.load()
        ffeats, levels = tensors[:n_iters], tensors[n_iters:]
        B, S, N, C = ffeats[0].shape
        H8, W8 = levels[0].shape[-2:]
        P, dev = H8 * W8, ffeats[0].device
        st = torch.cuda.current_stream(dev).cuda_stream
        lvls = [lv.detach().float().permute(0, 1, 3, 4, 2).contiguous() for lv in levels]       # channels-last
        g_hi = torch.empty(B * S, P, C, dtype=torch.bfloat16, device=dev)
        g_lo = torch.empty_like(g_hi)
        L.check(lib.pips_scoremap_basis(L.ptr_array(lvls), B * S, H8, W8, L.ptr(g_hi), L.ptr(g_lo), st), "pips_scoremap_basis")
        del lvls
        n_split = lib.pips_scoremap_splits(H8, W8)
        neg = torch.empty(n_iters, B * S * N, n_split, device=dev)
        pos = torch.empty(n_iters, B * S * N, device=dev)
        name = _window_entry("pips_scoremap_loss", S)
        for i, f in enumerate(ffeats):
            fi = f.detach().float().permute(0, 2, 1, 3).contiguous()        # ((b*N + n), s, c): free for the loop's state
            L.check(getattr(lib, name)(L.ptr(g_hi), L.ptr(g_lo), L.ptr(fi), B, S, N, H8, W8, L.ptr(target),
                                       L.ptr(neg[i]), L.ptr(pos[i]), st), name)
        ctx.save_for_backward(g_hi, g_lo, target, *ffeats)
        ctx.n_iters, ctx.level_shapes = n_iters, [lv.shape for lv in levels]
        return _score_map_loss(neg, pos, target, n_iters, P)

    @staticmethod
    def backward(ctx, grad):
        from . import _lib as L
        lib = L.load()
        g_hi, g_lo, target, *ffeats = ctx.saved_tensors
        I = ctx.n_iters
        B, S, N, C = ffeats[0].shape
        H8, W8 = ctx.level_shapes[0][-2:]
        P, dev = H8 * W8, g_hi.device
        st = torch.cuda.current_stream(dev).cuda_stream
        # dloss/dpos and dloss/dneg of engine._score_map_loss, on the device
        k = (target >= 0).sum().double() * I
        g = grad.detach().double()
        coef = torch.stack([g / (1e-6 + k), g / (1e-6 + k * (P - 1))]).float()
        F_ = torch.stack([f.detach().float() for f in ffeats])            # (I, B, S, N, C): frame-major
        need_f = any(ctx.needs_input_grad[2:2 + I])
        need_l = any(ctx.needs_input_grad[2 + I:])
        dF = None
        if need_f:
            dF = torch.empty_like(F_)
            name = _window_entry("pips_scoremap_grad_feats", S)
            L.check(getattr(lib, name)(L.ptr(g_hi), L.ptr(g_lo), L.ptr(F_), I, B, S, N, H8, W8, L.ptr(target),
                                       L.ptr(coef), L.ptr(dF), st), name)
        dls = [None] * len(ctx.level_shapes)
        if need_l:
            f_hi = torch.empty(F_.shape, dtype=torch.bfloat16, device=dev)
            f_lo = torch.empty_like(f_hi)
            L.check(lib.pips_split_bf16(L.ptr(F_), L.ptr(f_hi), L.ptr(f_lo), F_.numel(), st), "pips_split_bf16")
            del F_
            dG = torch.empty(B * S, P, C, device=dev)
            name = _window_entry("pips_scoremap_grad_basis", S)
            L.check(getattr(lib, name)(L.ptr(g_hi), L.ptr(g_lo), L.ptr(f_hi), L.ptr(f_lo), I, B, S, N, H8, W8,
                                       L.ptr(target), L.ptr(coef), L.ptr(dG), st), name)
            del f_hi, f_lo
            dl = [torch.empty(B * S, sh[-2], sh[-1], C, device=dev) for sh in ctx.level_shapes]
            L.check(lib.pips_scoremap_basis_grad(L.ptr(dG), B * S, H8, W8, L.ptr_array(dl), st), "pips_scoremap_basis_grad")
            dls = [d.view(B, S, d.shape[1], d.shape[2], C).permute(0, 1, 4, 2, 3) for d in dl]   # logical (B,S,C,h,w)
        dFs = [None] * I if dF is None else list(dF.unbind(0))
        return (None, None, *dFs, *dls)


def fused_score_map_loss(ffeats_per_iter, pyramid, trajs_g, vis_g, valids):
    """score_map_loss (nets/pips.py:58-90) of the score maps <ffeats_i, G> without building them, differentiable in the
    ffeats and the pyramid.  ffeats_per_iter: the I (B,S,N,128) ffeats at the start of each iteration; pyramid: the 4
    (B,S,128,H8>>l,W8>>l) levels; trajs_g (B,S,N,2) in feature-map pixels, vis_g and valids (B,S,N).  CUDA tensors only.
    Returns the same 0-dim fp32 loss as score_map_loss, summed in fp64 in a fixed order."""
    ffeats_per_iter, pyramid = list(ffeats_per_iter), list(pyramid)
    if not ffeats_per_iter:
        raise ValueError("fused_score_map_loss: no iterations")
    if not all(t.is_cuda for t in ffeats_per_iter + pyramid + [trajs_g, vis_g, valids]):
        raise RuntimeError("fused_score_map_loss runs on the CUDA kernels only; use score_map_loss for CPU tensors")
    B, S, N, C = ffeats_per_iter[0].shape
    H8, W8 = pyramid[0].shape[-2:]
    assert all(tuple(f.shape) == (B, S, N, C) for f in ffeats_per_iter), "every iteration's ffeats must be (B,S,N,128)"
    assert len(pyramid) == 4 and all(tuple(lv.shape) == (B, S, C, H8 >> l, W8 >> l) for l, lv in enumerate(pyramid)), \
        "pyramid must be the 4 avg-pooled levels (B,S,128,H8>>l,W8>>l)"
    target = score_map_targets(trajs_g, vis_g, valids, H8, W8)
    return _FusedScoreMapLoss.apply(target, len(ffeats_per_iter), *ffeats_per_iter, *pyramid)


def _round_up(v, m):
    return (v + m - 1) // m * m


class _MixerRun:
    """Launch helpers of one delta_block_cuda call: its packs, device, stream and row counts.  Row buffers are allocated
    with whole 256-row tiles (the pair GEMM kernel's condition) from torch's caching allocator on the call's device."""

    def __init__(self, packs, R, dev):
        from . import _lib as L
        self.L, self.lib, self.w, self.dev = L, L.load(), packs, dev
        self.st = torch.cuda.current_stream(dev).cuda_stream
        self.R, self.M = R, R * 8
        self.Ra, self.Ma = _round_up(R, 256), _round_up(R * 8, 256)
        self.zero = torch.zeros(L.HIDDEN, device=dev)                 # the bias of the input-gradient GEMMs

    def rows(self, n, cols, dtype=torch.float32):
        return torch.empty(n, cols, dtype=dtype, device=self.dev)

    def pair(self, n, cols):
        return self.rows(n, cols, torch.bfloat16), self.rows(n, cols, torch.bfloat16)

    def split(self, src, n_rows=None):
        """(hi, lo) of the fp32 rows src (n, cols), in buffers of whole tiles"""
        hi, lo = self.pair(_round_up(src.shape[0], 256), src.shape[1])
        self.L.check(self.lib.pips_split_bf16(self.L.ptr(src), self.L.ptr(hi), self.L.ptr(lo), src.numel(), self.st),
                     "pips_split_bf16")
        return hi, lo

    def gemm(self, a, M, K, wname, N, bias, epi, out=None, ldo=0, oh=(None, None), ldh=0, aux=None):
        L, w = self.L, self.w
        self.L.check(self.lib.pips_gemm_tc_aux(
            L.ptr(a[0]), L.ptr(a[1]), a[0].shape[1], a[0].shape[0], L.ptr(w[wname + "_hi"]), L.ptr(w[wname + "_lo"]),
            w[wname + "_hi"].shape[1], w[wname + "_hi"].shape[0], M, N, K, L.ptr(bias), epi, L.ptr(out), ldo,
            L.ptr(oh[0]), L.ptr(oh[1]), ldh, L.ptr(aux), 0 if aux is None else aux.shape[1], self.st), "pips_gemm_tc")

    def wgrad(self, g, N, x, K, M):
        L = self.L
        dw = torch.empty(N, K, device=self.dev)
        n = self.lib.pips_wgrad_scratch_floats(M, N, K)
        scratch = torch.empty(n, device=self.dev) if n else None
        L.check(self.lib.pips_wgrad(L.ptr(g[0]), L.ptr(g[1]), g[0].shape[1], L.ptr(x[0]), L.ptr(x[1]), x[0].shape[1], M, N, K,
                                    L.ptr(scratch), L.ptr(dw), self.st), "pips_wgrad")
        return dw

    def colsum(self, g32=None, pair=(None, None), N=0, M=0):
        L = self.L
        out = torch.empty(N, device=self.dev)
        n = self.lib.pips_colsum_scratch_floats(M, N)
        scratch = torch.empty(n, device=self.dev) if n else None
        ld = (g32 if g32 is not None else pair[0]).shape[1]
        L.check(self.lib.pips_colsum(L.ptr(g32), L.ptr(pair[0]), L.ptr(pair[1]), ld, M, N, L.ptr(scratch), L.ptr(out), self.st),
                "pips_colsum")
        return out

    def block_forward(self, l, x, y, h):
        """block l in place on the residual stream x (Ma, 512); y, h: (hi, lo) buffers of LN2's output and FC1's"""
        L, w, q = self.L, self.w, f"layer{l}."
        L.check(self.lib.pips_tokenmix(L.ptr(x), self.R, *(L.ptr(w[q + n]) for n in
                                                          ("ln1_w", "ln1_b", "tok_w1", "tok_b1", "tok_w2", "tok_b2", "ln2_w", "ln2_b")),
                                       L.ptr(y[0]), L.ptr(y[1]), None, self.st), "pips_tokenmix")
        self.gemm(y, self.M, L.DIM, q + "fc1_w", L.HIDDEN, w[q + "fc1_b"], L.EPI_BIAS_GELU, oh=h, ldh=L.HIDDEN)
        self.gemm(h, self.M, L.HIDDEN, q + "fc2_w", L.DIM, w[q + "fc2_b"], L.EPI_BIAS_RESID, out=x, ldo=L.DIM)


# DeltaBlock parameter names in named_parameters order: the order of delta_block_cuda's inputs and gradients
def _delta_param_names(depth=12):
    names = ["to_delta.0.weight", "to_delta.0.bias"]
    for l in range(depth):
        p = f"to_delta.{l + 1}"
        for half in (0, 1):                 # PreNormResidual registers fn before norm
            names += [f"{p}.{half}.fn.0.weight", f"{p}.{half}.fn.0.bias", f"{p}.{half}.fn.3.weight", f"{p}.{half}.fn.3.bias",
                      f"{p}.{half}.norm.weight", f"{p}.{half}.norm.bias"]
    return names + ["to_delta.13.weight", "to_delta.13.bias", "to_delta.15.weight", "to_delta.15.bias"]


DELTA_PARAMS = tuple(_delta_param_names())


def _delta_shapes():
    """the parameter shapes of a DeltaBlock(), by name (built on the meta device: no memory, no initialisation)"""
    global _DELTA_SHAPES
    if _DELTA_SHAPES is None:
        from .pips import DeltaBlock
        with torch.device("meta"):
            _DELTA_SHAPES = {n: tuple(p.shape) for n, p in DeltaBlock().named_parameters()}
    return _DELTA_SHAPES


_DELTA_SHAPES = None


def _delta_block_params(delta_block):
    """The 150 parameter tensors of ``delta_block`` in DELTA_PARAMS order, found by attribute lookup along each dotted
    name.  named_parameters() would not do: an nn.DataParallel replica (torch.nn.parallel.replicate) keeps its broadcast
    parameters as plain attributes and lists none."""
    params = []
    for n in DELTA_PARAMS:
        mod_name, attr = n.rsplit(".", 1)
        try:
            t = getattr(delta_block.get_submodule(mod_name), attr)
        except AttributeError:
            t = None
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != _delta_shapes()[n]:
            raise ValueError(f"delta_block_cuda: the module is not a 12-block DeltaBlock(dim=512, S=8) (at {n})")
        params.append(t)
    return params


# pack entries only the forward reads: dropped before the pack is kept for the backward
_FORWARD_ONLY = ("in_w_hi", "in_w_lo", "head_w_hi", "head_w_lo") + tuple(
    f"layer{l}.fc2_w_{part}" for l in range(12) for part in ("hi", "lo"))


class _DeltaBlockFn(torch.autograd.Function):
    """DeltaBlock.forward on the sm_90a kernels, bf16x3 throughout, with the parameters as explicit inputs (so gradients
    reach nn.DataParallel replicas' broadcast parameters).  The forward saves the block boundaries only: the (hi, lo)
    input rows, the residual stream at the entry of each of the 12 blocks and before the final LayerNorm.  The backward
    recomputes each block from its entry with the forward's kernels, so the recomputed activations are the forward's
    bits, and runs the block's backward: FC1 recompute (keeping the pre-activation), FC2 weight / input gradients (the
    GELU derivative in the GEMM epilogue), FC1 weight / input gradients, then one CUDA-core kernel for the LayerNorms and
    the token mixing."""

    @staticmethod
    def forward(ctx, save, x, *params):
        from .engine import PackedWeights
        R = x.shape[0]
        dev = x.device
        with torch.cuda.device(dev):
            sd = {"delta_block." + n: p.detach() for n, p in zip(DELTA_PARAMS, params)}
            run = _MixerRun(None, R, dev)
            L = run.L
            run.w = PackedWeights.pack_mapping(sd, run.st, transposed=save, f32_copies=False)
            M, Ma = run.M, run.Ma
            xin = torch.zeros(M, L.KPAD, device=dev)
            xin[:, :519] = x.detach().reshape(M, 519)
            x0 = run.split(xin)
            del xin
            xs = torch.empty(L.DEPTH + 1 if save else 1, Ma, L.DIM, device=dev)
            run.gemm(x0, M, L.KPAD, "in_w", L.DIM, run.w["in_b"], L.EPI_BIAS, out=xs[0], ldo=L.DIM)
            y, h = run.pair(Ma, L.DIM), run.pair(Ma, L.HIDDEN)
            for l in range(L.DEPTH):
                cur = xs[l + 1] if save else xs[0]
                if save:
                    cur.copy_(xs[l])
                run.block_forward(l, cur, y, h)
            del y, h
            xf = xs[-1]
            p = run.pair(run.Ra, L.DIM)
            L.check(run.lib.pips_ln_pool(L.ptr(xf), R, L.ptr(run.w["out_ln_w"]), L.ptr(run.w["out_ln_b"]), L.ptr(p[0]),
                                         L.ptr(p[1]), None, run.st), "pips_ln_pool")
            delta = torch.empty(R, L.HEAD, device=dev)
            run.gemm(p, R, L.DIM, "head_w", L.HEAD, run.w["head_b"], L.EPI_BIAS, out=delta, ldo=L.HEAD)
        if save:
            ctx.save_for_backward(x0[0], x0[1], xs)
            ctx.packs = {k: v for k, v in run.w.items() if k not in _FORWARD_ONLY}
            ctx.shapes = [p.shape for p in params]
        return delta.view(R, 8, L.HEAD // 8)

    @staticmethod
    def backward(ctx, grad):
        from . import _lib as L
        x0_hi, x0_lo, xs = ctx.saved_tensors
        dev = xs.device
        R = grad.shape[0]
        with torch.cuda.device(dev):
            run = _MixerRun(ctx.packs, R, dev)
            w, lib, M, Ma, Ra = run.w, run.lib, run.M, run.Ma, run.Ra
            g = {}
            # head: delta = p . head_w^T + head_b over the R pooled rows; K padded to 1280 with zeros
            dd = torch.zeros(R, L.HEAD_PAD, device=dev)
            dd[:, :L.HEAD] = grad.reshape(R, L.HEAD)
            ddp = run.split(dd)
            p = run.pair(Ra, L.DIM)
            L.check(lib.pips_ln_pool(L.ptr(xs[-1]), R, L.ptr(w["out_ln_w"]), L.ptr(w["out_ln_b"]), L.ptr(p[0]), L.ptr(p[1]), None,
                                     run.st), "pips_ln_pool")
            g["to_delta.15.weight"] = run.wgrad(ddp, L.HEAD, p, L.DIM, R)
            g["to_delta.15.bias"] = run.colsum(g32=dd, N=L.HEAD, M=R)
            del p
            dp = run.rows(Ra, L.DIM)
            run.gemm(ddp, R, L.HEAD_PAD, "head_wT", L.DIM, run.zero, L.EPI_BIAS, out=dp, ldo=L.DIM)
            del dd, ddp
            dX = run.rows(Ma, L.DIM)
            lp = torch.empty(lib.pips_ln_pool_grad_scratch_floats(R), device=dev)
            lpg = torch.empty(2 * L.DIM, device=dev)
            L.check(lib.pips_ln_pool_grad(L.ptr(xs[-1]), L.ptr(dp), R, L.ptr(w["out_ln_w"]), L.ptr(w["out_ln_b"]), L.ptr(dX),
                                          L.ptr(lp), L.ptr(lpg), run.st), "pips_ln_pool_grad")
            g["to_delta.13.weight"], g["to_delta.13.bias"] = lpg[:L.DIM], lpg[L.DIM:]
            del dp, lp
            # the 12 blocks, last first
            work = run.rows(Ma, L.DIM)
            y, gh = run.pair(Ma, L.DIM), run.pair(Ma, L.HIDDEN)
            dh = run.pair(Ma, L.HIDDEN)
            hpre = run.rows(Ma, L.HIDDEN)
            dy = run.rows(Ma, L.DIM)
            tg = torch.empty(lib.pips_tokenmix_grad_scratch_floats(R), device=dev)
            for l in reversed(range(L.DEPTH)):
                q, pn = f"layer{l}.", f"to_delta.{l + 1}"
                work.copy_(xs[l])
                L.check(lib.pips_tokenmix(L.ptr(work), R, *(L.ptr(w[q + n]) for n in
                                                           ("ln1_w", "ln1_b", "tok_w1", "tok_b1", "tok_w2", "tok_b2", "ln2_w", "ln2_b")),
                                          L.ptr(y[0]), L.ptr(y[1]), None, run.st), "pips_tokenmix")
                run.gemm(y, M, L.DIM, q + "fc1_w", L.HIDDEN, w[q + "fc1_b"], L.EPI_BIAS_GELU_PRE, oh=gh, ldh=L.HIDDEN, aux=hpre)
                dXp = run.split(dX[:M])
                g[pn + ".1.fn.3.weight"] = run.wgrad(dXp, L.DIM, gh, L.HIDDEN, M)
                g[pn + ".1.fn.3.bias"] = run.colsum(g32=dX, N=L.DIM, M=M)
                run.gemm(dXp, M, L.DIM, q + "fc2_wT", L.HIDDEN, run.zero, L.EPI_GELU_GRAD, oh=dh, ldh=L.HIDDEN, aux=hpre)
                del dXp
                g[pn + ".1.fn.0.weight"] = run.wgrad(dh, L.HIDDEN, y, L.DIM, M)
                g[pn + ".1.fn.0.bias"] = run.colsum(pair=dh, N=L.HIDDEN, M=M)
                run.gemm(dh, M, L.HIDDEN, q + "fc1_wT", L.DIM, run.zero, L.EPI_BIAS, out=dy, ldo=L.DIM)
                tk = torch.empty(2600, device=dev)
                L.check(lib.pips_tokenmix_grad(L.ptr(xs[l]), L.ptr(work), L.ptr(dy), L.ptr(dX), R,
                                               *(L.ptr(w[q + n]) for n in ("ln1_w", "ln1_b", "tok_w1", "tok_b1", "tok_w2",
                                                                           "tok_b2", "ln2_w", "ln2_b")),
                                               L.ptr(tg), L.ptr(tk), run.st), "pips_tokenmix_grad")
                for name, a, b in ((".0.norm.weight", 0, 512), (".0.norm.bias", 512, 1024), (".0.fn.0.weight", 1024, 1280),
                                   (".0.fn.0.bias", 1280, 1312), (".0.fn.3.weight", 1312, 1568), (".0.fn.3.bias", 1568, 1576),
                                   (".1.norm.weight", 1576, 2088), (".1.norm.bias", 2088, 2600)):
                    g[pn + name] = tk[a:b]
            del work, y, gh, dh, hpre, dy, tg
            # input layer: x = x0 . in_w^T + in_b
            dXp = run.split(dX[:M])
            dx0 = run.rows(Ma, L.KPAD)
            run.gemm(dXp, M, L.DIM, "in_wT", L.KPAD, run.zero, L.EPI_BIAS, out=dx0, ldo=L.KPAD)
            g["to_delta.0.weight"] = run.wgrad(dXp, L.DIM, (x0_hi, x0_lo), L.KPAD, M)[:, :519].contiguous()
            g["to_delta.0.bias"] = run.colsum(g32=dX, N=L.DIM, M=M)
            dx = dx0[:M, :519].reshape(R, 8, 519)
        grads = [g[n].reshape(sh) for n, sh in zip(DELTA_PARAMS, ctx.shapes)]
        return (None, dx if ctx.needs_input_grad[1] else None, *grads)


def delta_block_cuda(delta_block, x):
    """``DeltaBlock.forward`` (nets/pips.py:304-311) on the sm_90a kernels, differentiable in ``x`` and in every one of
    the block's 150 parameters: x (R, 8, 519) fp32 CUDA -> (R, 8, 130).  The arithmetic is bf16x3 (fp32-class) whatever
    PIPS_B200_PRECISION says.  Allocates through torch's caching allocator on x's device and runs on its current stream;
    the weights are packed from the parameters on every call (nn.DataParallel replicas hold new tensors each step).
    ``delta_block`` may be a DeltaBlock or an nn.DataParallel replica of one; the gradients flow to whatever tensors its
    parameter attributes hold (a replica's broadcast copies, and through them the original parameters)."""
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise RuntimeError("delta_block_cuda runs on the CUDA kernels only; use the DeltaBlock module for CPU tensors")
    if x.dim() != 3 or x.shape[1] != 8 or x.shape[2] != 519:
        raise ValueError(f"delta_block_cuda: x must be (R, 8, 519) (S = 8 frames); got {tuple(x.shape)}")
    if x.dtype != torch.float32:
        raise ValueError(f"delta_block_cuda: x must be float32; got {x.dtype}")
    if x.shape[0] == 0:
        raise ValueError("delta_block_cuda: no rows")
    params = _delta_block_params(delta_block)
    if any(p.device != x.device or p.dtype != torch.float32 for p in params):
        raise ValueError("delta_block_cuda: the parameters must be float32 on x's device")
    save = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
    return _DeltaBlockFn.apply(save, x.contiguous(), *params)


# Encoder convolutions in named_parameters order; each contributes (weight, bias) to encoder_cuda's inputs
ENCODER_CONVS = ("conv1",) + tuple(
    f"layer{i}.{j}.{c}" for i in range(1, 5) for j in (0, 1)
    for c in ("conv1", "conv2") + (("downsample.0",) if i > 1 and j == 0 else ())) + ("conv2", "conv3")
ENCODER_PARAMS = tuple(f"{c}.{p}" for c in ENCODER_CONVS for p in ("weight", "bias"))
_ENCODER_SHAPES = None


def _encoder_params(fnet):
    """The 44 parameter tensors of the Encoder ``fnet`` in ENCODER_PARAMS order, by attribute lookup (nn.DataParallel
    replicas list no parameters), and its convolution modules by name."""
    global _ENCODER_SHAPES
    if _ENCODER_SHAPES is None:
        from .encoder import Encoder
        with torch.device("meta"):
            _ENCODER_SHAPES = {n: tuple(p.shape) for n, p in Encoder().named_parameters()}
    params, convs = [], {}
    for n in ENCODER_PARAMS:
        mod_name, attr = n.rsplit(".", 1)
        try:
            mod = fnet.get_submodule(mod_name)
            t = getattr(mod, attr)
        except AttributeError:
            mod = t = None
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != _ENCODER_SHAPES[n]:
            raise ValueError(f"encoder_cuda: the module is not a BasicEncoder(output_dim=128) (at {n})")
        params.append(t)
        convs[mod_name] = mod
    return params, convs


class _EncRun:
    """Launch helpers of one encoder_cuda backward: device, stream and the raw entry points."""

    def __init__(self, dev):
        from . import _lib as L
        from . import encoder_fast as E
        self.L, self.E, self.lib, self.dev = L, E, L.load(), dev
        self.st = torch.cuda.current_stream(dev).cuda_stream
        self.ops = E._Ops(dev)

    def pair(self, N, H, W, C):
        return self.E._Pair(N, H, W, C, self.dev)

    def pair_of(self, x):
        """the (hi, lo) pair of an fp32 activation: the bits pips_inorm_apply_pair wrote for it in the forward"""
        return self.E._apply_pair(self.ops, x, None, relu_main=False)[1]

    def wgrad(self, dy, step, x, conv_w, R, S, stride, pad):
        """dL/dW (Cout, Cin, R, S) of a convolution over the pair x, from the pair dy"""
        L = self.L
        N, H, W = x.shape
        cout, cin = conv_w.shape[:2]
        Ho, Wo = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - S) // stride + 1
        K = R * S * x.Cp
        dw = torch.empty(cout, K, device=self.dev)
        n = self.lib.pips_conv_wgrad_scratch_floats(N, Ho, Wo, cout, K)
        scratch = torch.empty(n, device=self.dev) if n else None
        L.check(self.lib.pips_conv_wgrad(L.ptr(dy.hi), L.ptr(dy.lo), dy.Cp, step, L.ptr(x.hi), L.ptr(x.lo), N, H, W, x.Cp, cout, R, S,
                                         stride, stride, pad, pad, L.ptr(scratch), L.ptr(dw), self.st), "pips_conv_wgrad")
        return dw.view(cout, R, S, x.Cp)[..., :cin].permute(0, 3, 1, 2)

    def dgrad(self, dy, conv_w, pad, rows=None):
        """input gradient of a convolution: pips_conv_tc over the pair dy (zero-dilated for stride 2) with the weight
        flipped in (r, s) and transposed in channels; ``rows`` = (first, end) input channel"""
        L = self.L
        wt = conv_w.detach().flip(2, 3).transpose(0, 1)
        if rows is not None:
            wt = wt[rows[0]:rows[1]]
        hi, lo = self.E.pack_conv_weight(wt)
        N, H, W = dy.shape
        cout, _, R, S = wt.shape
        out = torch.empty(N, H, W, cout, device=self.dev)
        L.check(self.lib.pips_conv_tc(L.ptr(dy.hi), L.ptr(dy.lo), N, H, W, dy.Cp, L.ptr(hi), L.ptr(lo), cout, R, S, 1, pad, None,
                                      L.ptr(out), self.st), "pips_conv_tc")
        return out

    def inorm_grad(self, y, stats, addends, r=None, stats_r=None, relu_main=True, relu_out=False, dil=None, skip=False):
        """-> (dy pair, g after the output ReLU's mask or None); dil = (H, W) of a zero-dilated output grid"""
        L = self.L
        N, H, W, C = y.shape
        dy = self.pair(N, *(dil or (H, W)), C)
        g_out = torch.empty_like(y) if skip else None
        scratch = torch.empty(self.lib.pips_inorm_grad_scratch_floats(N, H * W, C), device=self.dev)
        g = list(addends) + [None] * (3 - len(addends))
        L.check(self.lib.pips_inorm_grad(L.ptr(y), L.ptr(stats), L.ptr(r), L.ptr(stats_r), int(relu_main), int(relu_out),
                                         *(L.ptr(t) for t in g), N, H, W, C, L.ptr(scratch), L.ptr(dy.hi), L.ptr(dy.lo), dy.Cp,
                                         *(dil or (0, 0)), L.ptr(g_out), self.st), "pips_inorm_grad")
        return dy, g_out


class _EncoderFn(torch.autograd.Function):
    """Encoder.forward on the sm_90a kernels of fnet_tc, bf16x3, with the 44 parameters as explicit inputs.  The forward
    saves the block boundaries only (the stem output and the output of every ResBlock, fp32) and the image; the backward
    recomputes each block from its saved input with the forward's kernels -- so the recomputed activations are the
    forward's bits -- and runs its backward last block first: ReLU masks and InstanceNorm backward (pips_inorm_grad),
    weight gradients (pips_conv_wgrad), input gradients (pips_conv_tc over flipped weights), the resize adjoint of the
    head's input (pips_resize_grad).

    The biases of the 21 convolutions that feed an InstanceNorm get an exact zero gradient: InstanceNorm removes a
    per-channel constant again, so the forward never adds them (conv_tc(..., bias=False)) and the function computed
    does not depend on them.  conv3's bias gets the column sum of the output gradient."""

    @staticmethod
    def forward(ctx, save, convs, rgb, *params):
        from . import encoder_fast as E
        dev = rgb.device
        with torch.cuda.device(dev):
            ws = dict(zip(ENCODER_PARAMS, params))
            packs = {}
            for name in ENCODER_CONVS:
                w = ws[name + ".weight"].detach()
                packs[convs[name]] = E.pack_stem_weight(w) if name == "conv1" else E.pack_conv_weight(w)
            keep = [] if save else None
            out = E._fnet_tc(convs[""], rgb, packs=packs, keep=keep)
        if save:
            ctx.save_for_backward(rgb, *keep, *(ws[c + ".weight"] for c in ENCODER_CONVS))
            ctx.convs, ctx.packs = convs, {n: packs[convs[n]] for n in ENCODER_CONVS}
            ctx.shapes = [p.shape for p in params]
        return out

    @staticmethod
    def backward(ctx, gout):
        rgb, *rest = ctx.saved_tensors
        X, wl = rest[:9], dict(zip(ENCODER_CONVS, rest[9:]))
        convs, packs = ctx.convs, ctx.packs
        dev = rgb.device
        g = {}
        need = dict(zip(ENCODER_PARAMS, ctx.needs_input_grad[3:]))       # weight gradients of frozen convolutions are skipped
        with torch.cuda.device(dev):
            run = _EncRun(dev)
            L, lib, st, ops = run.L, run.lib, run.st, run.ops
            E = run.E
            N, H8, W8, _ = gout.shape
            gout = gout.contiguous()
            # ---- head: fmaps = conv3(relu(IN(conv2(cat)))) + b3
            widths = (64, 96, 128, 128)
            cat = run.pair(N, H8, W8, sum(widths))
            c_off = 0
            for l, C in enumerate(widths):
                Xl = X[2 * l + 2]
                L.check(lib.pips_resize_pair(L.ptr(Xl), N, Xl.shape[1], Xl.shape[2], C, L.ptr(cat.hi), L.ptr(cat.lo), H8, W8, cat.Cp,
                                             c_off, st), "pips_resize_pair")
                c_off += C
            yh, sh = E._conv_stats(ops, cat, convs["conv2"], packs["conv2"])
            _, ah = E._apply_pair(ops, yh, sh, relu_main=True)
            gp = run.pair(N, H8, W8, 128)
            L.check(lib.pips_split_bf16(L.ptr(gout), L.ptr(gp.hi), L.ptr(gp.lo), gout.numel(), st), "pips_split_bf16")
            if need["conv3.weight"]:
                g["conv3.weight"] = run.wgrad(gp, 1, ah, wl["conv3"], 1, 1, 1, 0)
            if need["conv3.bias"]:
                M = N * H8 * W8
                n = lib.pips_colsum_scratch_floats(M, 128)
                scratch = torch.empty(n, device=dev) if n else None
                b3 = torch.empty(128, device=dev)
                L.check(lib.pips_colsum(L.ptr(gout), None, None, 128, M, 128, L.ptr(scratch), L.ptr(b3), st), "pips_colsum")
                g["conv3.bias"] = b3
            dah = run.dgrad(gp, wl["conv3"], 0)
            del gp, ah
            dyh, _ = run.inorm_grad(yh, sh, [dah])
            del dah, yh
            if need["conv2.weight"]:
                g["conv2.weight"] = run.wgrad(dyh, 1, cat, wl["conv2"], 3, 3, 1, 1)
            del cat
            # conv_tc covers 256 output channels: the 416 of the head's input gradient in two launches, split between
            # layer2 and layer3 so that every layer's slice lies in one of them
            dcat = (run.dgrad(dyh, wl["conv2"], 1, rows=(0, 160)), run.dgrad(dyh, wl["conv2"], 1, rows=(160, 416)))
            del dyh
            gl = []
            for l, (part, off) in enumerate(((0, 0), (0, 64), (1, 0), (1, 128))):
                Xl = X[2 * l + 2]
                d = torch.empty_like(Xl)
                src = dcat[part]
                L.check(lib.pips_resize_grad(L.ptr(src), src.shape[-1], off, N, H8, W8, L.ptr(d), Xl.shape[1], Xl.shape[2], Xl.shape[3],
                                             st), "pips_resize_grad")
                gl.append(d)
            del dcat
            # ---- the 8 ResBlocks, last first; `addends` holds the gradient of the current block's output
            addends = [gl[3]]
            for b in reversed(range(8)):
                i, j = b // 2 + 1, b % 2
                q = f"layer{i}.{j}."
                ds = i > 1 and j == 0
                stride = 2 if ds else 1
                x_in = X[b]
                xp = run.pair_of(x_in)
                y1, s1 = E._conv_stats(ops, xp, convs[q + "conv1"], packs[q + "conv1"])
                _, a1 = E._apply_pair(ops, y1, s1, relu_main=True)
                y2, s2 = E._conv_stats(ops, a1, convs[q + "conv2"], packs[q + "conv2"])
                if ds:
                    d, sd = E._conv_stats(ops, xp, convs[q + "downsample.0"], packs[q + "downsample.0"])
                    r, sr = d, sd
                else:
                    r, sr = x_in, None
                dy2, go = run.inorm_grad(y2, s2, addends, r=r, stats_r=sr, relu_out=True, skip=True)
                del addends, y2
                if need[q + "conv2.weight"]:
                    g[q + "conv2.weight"] = run.wgrad(dy2, 1, a1, wl[q + "conv2"], 3, 3, 1, 1)
                da1 = run.dgrad(dy2, wl[q + "conv2"], 1)
                del dy2, a1
                dil = tuple(x_in.shape[1:3]) if ds else None
                dy1, _ = run.inorm_grad(y1, s1, [da1], dil=dil)
                del da1, y1
                if need[q + "conv1.weight"]:
                    g[q + "conv1.weight"] = run.wgrad(dy1, stride, xp, wl[q + "conv1"], 3, 3, stride, 1)
                dx1 = run.dgrad(dy1, wl[q + "conv1"], 1)
                del dy1
                if ds:
                    dd, _ = run.inorm_grad(d, sd, [go], relu_main=False, dil=dil)
                    del d, go
                    if need[q + "downsample.0.weight"]:
                        g[q + "downsample.0.weight"] = run.wgrad(dd, 2, xp, wl[q + "downsample.0"], 1, 1, 2, 0)
                    addends = [dx1, run.dgrad(dd, wl[q + "downsample.0"], 0)]
                    del dd
                else:
                    addends = [go, dx1]
                if ds:
                    addends.append(gl[i - 2])                 # the block's input is layer i-1's output
                del xp
            # ---- stem: X0 = relu(IN(conv1(image))); no gradient for the image
            # the stem has no input gradient: with its weight frozen there is nothing left to do
            if need["conv1.weight"]:
                Ho, Wo = X[0].shape[1:3]
                unf, y0, s0 = E.stem_tc(rgb, packs["conv1"])
                dy0, _ = run.inorm_grad(y0, s0, addends)
                del addends, y0
                K = 4 * 64
                dw = torch.empty(64, K, device=dev)
                n = lib.pips_conv_wgrad_scratch_floats(N, Ho, Wo, 64, K)
                scratch = torch.empty(n, device=dev) if n else None
                L.check(lib.pips_conv_wgrad(L.ptr(dy0.hi), L.ptr(dy0.lo), dy0.Cp, 1, L.ptr(unf.hi), L.ptr(unf.lo), N, Ho + 3, Wo, 64,
                                            64, 4, 1, 1, 1, 0, 0, L.ptr(scratch), L.ptr(dw), st), "pips_conv_wgrad")
                # (64, 4*64) over the row pairs -> (64, 3, 7, 7): k = filter row * 32 + s*3 + colour (pack_stem_weight)
                g["conv1.weight"] = dw.view(64, 8, 32)[:, :7, :21].reshape(64, 7, 7, 3).permute(0, 3, 1, 2)
        grads = []
        for n_, sh_ in zip(ENCODER_PARAMS, ctx.shapes):
            t = g.get(n_)
            grads.append(None if not need[n_] else torch.zeros(sh_, device=dev) if t is None else t.contiguous())
        return (None, None, None, *grads)


def encoder_cuda(fnet, rgbs):
    """``Pips.encode`` (nets/pips.py:436-445, the BasicEncoder) on the sm_90a kernels of fnet_tc, differentiable in the
    encoder's 44 parameters (not in the image): rgbs (B,S,3,H,W) CUDA with values 0..255 -> fmaps (B,S,128,H/stride,
    W/stride) fp32, a view of the channels-last result like Pips.encode's.  The forward has the bits of fnet_tc; the
    arithmetic is bf16x3 whatever PIPS_B200_PRECISION or fnet_mode say.  The filters are packed from the parameters on
    every call, without the modules' caches, and no CUDA graph is used: ``fnet`` may be an nn.DataParallel replica run
    from a worker thread.  With gradients on, the forward keeps the block boundaries only (about 49 MiB per 384x512
    frame); under no_grad, nothing but its output."""
    if not isinstance(rgbs, torch.Tensor) or not rgbs.is_cuda:
        raise RuntimeError("encoder_cuda runs on the CUDA kernels only; use the Encoder module for CPU tensors")
    if rgbs.dim() != 5 or rgbs.shape[2] != 3:
        raise ValueError(f"encoder_cuda: rgbs must be (B, S, 3, H, W); got {tuple(rgbs.shape)}")
    if rgbs.requires_grad:
        raise ValueError("encoder_cuda computes no gradient for the image; use the Encoder module when rgbs requires grad")
    B, S, C, H, W = rgbs.shape
    params, convs = _encoder_params(fnet)
    stride = fnet.stride
    if H // stride == 0 or W // stride == 0:
        raise ValueError(f"encoder_cuda: a {H}x{W} frame has no feature pixel at stride {stride}")
    if any(p.device != rgbs.device or p.dtype != torch.float32 for p in params):
        raise ValueError("encoder_cuda: the parameters must be float32 on rgbs's device")
    convs[""] = fnet
    raw = rgbs if rgbs.dtype in (torch.float32, torch.bfloat16) else rgbs.float()
    raw = raw.reshape(B * S, C, H, W).contiguous()
    save = torch.is_grad_enabled() and any(p.requires_grad for p in params)
    f = _EncoderFn.apply(save, convs, raw, *params)
    H8, W8 = f.shape[1:3]
    return f.reshape(B, S, H8, W8, f.shape[-1]).permute(0, 1, 4, 2, 3)


class _LocalCorrFn(torch.autograd.Function):
    """The 196 correlation columns of pips_corr_gather, differentiable in the ffeats and the 4 levels.  The forward is
    pips_corr_gather into an fp32 row buffer, so it has the bits the inference path feeds its mixer; the backward is
    pips_corr_grad_feats and pips_corr_grad_levels (their _window siblings at S != 8).  Saves the inputs only: no
    all-pairs volume exists in either direction."""

    @staticmethod
    def forward(ctx, coords, ffeat_rows, *levels):
        from . import _lib as L
        lib = L.load()
        B, S, N, _ = coords.shape
        H, W = levels[0].shape[1:3]
        dev = coords.device
        st = torch.cuda.current_stream(dev).cuda_stream
        x = torch.empty(B * N * S, L.KPAD, device=dev)
        times = torch.zeros(S, device=dev)                      # the embedding columns are not returned
        L.check(lib.pips_corr_gather(L.ptr_array(levels), L.FEAT_F32, B, S, N, H, W, L.ptr(coords), L.ptr(ffeat_rows),
                                     L.ptr(times), None, 0, None, None, L.ptr(x), L.KPAD, st), "pips_corr_gather")
        ctx.save_for_backward(coords, ffeat_rows, *levels)
        return x[:, 128:324].reshape(B * N, S, 196).contiguous()      # frees the other 380 columns of the row buffer

    @staticmethod
    def backward(ctx, grad):
        from . import _lib as L
        lib = L.load()
        coords, ffeat_rows, *levels = ctx.saved_tensors
        B, S, N, _ = coords.shape
        H, W = levels[0].shape[1:3]
        dev = coords.device
        st = torch.cuda.current_stream(dev).cuda_stream
        # the gradient of a column slice of the mixer input arrives with the mixer input's row stride
        if grad.stride(2) != 1 or grad.stride(0) != S * grad.stride(1) or grad.stride(1) < 196:
            grad = grad.contiguous()
        ld = grad.stride(1)
        dff = None
        if ctx.needs_input_grad[1]:
            dff = torch.empty(B * N, S, 128, device=dev)
            name = _window_entry("pips_corr_grad_feats", S)
            L.check(getattr(lib, name)(L.ptr_array(levels), B, S, N, H, W, L.ptr(coords), L.ptr(grad), ld, L.ptr(dff), st),
                    name)
        dls = [None] * len(levels)
        if any(ctx.needs_input_grad[2:]):
            dls = [torch.empty_like(lv) for lv in levels]
            name = _window_entry("pips_corr_grad_levels", S)
            L.check(getattr(lib, name)(B, S, N, H, W, L.ptr(coords), L.ptr(ffeat_rows), L.ptr(grad), ld, L.ptr_array(dls),
                                       st), name)
        return (None, dff, *dls)


def local_corr_cuda(ffeat_rows, levels, coords):
    """The local correlation of forward_torch (nets/pips.py:355-398: the all-pairs volumes of the 4 levels sampled at
    the 49 taps around each track) on the sm_90a kernels, differentiable in ``ffeat_rows`` and in each level, never in
    ``coords`` (detached at the top of every iteration, nets/pips.py:500).  ffeat_rows (B*N, S, 128) fp32; levels the 4
    channels-last (B*S, H>>l, W>>l, 128) fp32 pyramid levels; coords (B, S, N, 2) fp32 in feature-map pixels.  Returns
    fcorr (B*N, S, 196): channel l*49 + a*7 + b samples x = cx/2^l + a - 3, y = cy/2^l + b - 3, as forward_torch's.
    Neither direction builds an all-pairs volume.  Windows of 2 <= S <= 16 frames (S = 8 runs the S = 8 entry points,
    any other S their _window siblings: the same kernels) and a level 0 of at least 8x8 only; the window length is
    checked before any tensor is touched.  Allocates through torch's caching allocator on the inputs' device and runs on
    its current stream, with no CUDA graph and no cache."""
    levels = list(levels)
    if not isinstance(coords, torch.Tensor) or coords.dim() != 4 or not 2 <= coords.shape[1] <= 16 or coords.shape[3] != 2:
        shape = tuple(coords.shape) if isinstance(coords, torch.Tensor) else type(coords).__name__
        raise ValueError(f"local_corr_cuda: coords must be (B, S, N, 2) with 2 <= S <= 16 frames; got {shape}")
    if not all(isinstance(t, torch.Tensor) and t.is_cuda for t in [ffeat_rows, coords] + levels):
        raise RuntimeError("local_corr_cuda runs on the CUDA kernels only; use forward_torch's matmul + grid_sample "
                           "for CPU tensors")
    B, S, N, _ = coords.shape
    if B == 0 or N == 0:
        raise ValueError("local_corr_cuda: no tracks")
    if tuple(ffeat_rows.shape) != (B * N, S, 128):
        raise ValueError(f"local_corr_cuda: ffeat_rows must be (B*N, S, 128) = {(B * N, S, 128)}; got {tuple(ffeat_rows.shape)}")
    if len(levels) != 4 or levels[0].dim() != 4:
        raise ValueError("local_corr_cuda: levels must be the 4 channels-last pyramid levels (B*S, H>>l, W>>l, 128)")
    H, W = levels[0].shape[1:3]
    if H < 8 or W < 8:
        raise ValueError(f"local_corr_cuda: level 0 must be at least 8x8; got {H}x{W}")
    for l, lv in enumerate(levels):
        if tuple(lv.shape) != (B * S, H >> l, W >> l, 128):
            raise ValueError(f"local_corr_cuda: level {l} must be {(B * S, H >> l, W >> l, 128)}; got {tuple(lv.shape)}")
    if any(t.dtype != torch.float32 or t.device != coords.device for t in [ffeat_rows] + levels) \
            or coords.dtype != torch.float32:
        raise ValueError("local_corr_cuda: every input must be float32 on one device")
    with torch.cuda.device(coords.device):
        return _LocalCorrFn.apply(coords.detach().contiguous(), ffeat_rows.contiguous(), *(lv.contiguous() for lv in levels))


def sample_clamped(im, x, y):
    """utils/samp.py:5-78: bilinear sample with clamped indices and unclamped weights -> (B,N,C)."""
    B, C, H, W = im.shape
    x0, y0 = torch.floor(x), torch.floor(y)
    x1, y1 = x0 + 1, y0 + 1
    flat = im.permute(0, 2, 3, 1).reshape(B, H * W, C)

    def tap(yy, xx):
        idx = yy.long().clamp(0, H - 1) * W + xx.long().clamp(0, W - 1)
        return torch.gather(flat, 1, idx.unsqueeze(-1).expand(-1, -1, C))

    return (((x1 - x) * (y1 - y)).unsqueeze(-1) * tap(y0, x0) + ((x - x0) * (y1 - y)).unsqueeze(-1) * tap(y0, x1)
            + ((x1 - x) * (y - y0)).unsqueeze(-1) * tap(y1, x0) + ((x - x0) * (y - y0)).unsqueeze(-1) * tap(y1, x1))


def motion_embedding(flow, C=64):
    """utils/misc.py:44-69 with cat_coords=True."""
    div = (torch.arange(0, C, 2, device=flow.device, dtype=torch.float32) * (1000.0 / C)).view(1, 1, -1)
    out = []
    for a in range(3):
        v = flow[:, :, a:a + 1] * div
        out.append(torch.stack([v.sin(), v.cos()], dim=-1).flatten(2))
    return torch.cat(out + [flow], dim=2)


def forward_torch(model, xys, rgbs, coords_init=None, feat_init=None, iters=3, trajs_g=None, vis_g=None, valids=None,
                  sw=None, return_feat=False, is_train=False):
    B, N, _ = xys.shape
    _, S, C, H, W = rgbs.shape
    stride = model.stride
    H8, W8 = H // stride, W // stride
    L, r = model.corr_levels, model.corr_radius

    if getattr(model, "encoder_path", "torch") == "cuda" and rgbs.is_cuda and not rgbs.requires_grad:
        fmaps = encoder_cuda(model.fnet, rgbs)                # sm_90a forward and backward, no CUDA graphs (DataParallel-safe)
    else:
        fmaps = model.encode(rgbs, torch_only=True)      # no CUDA graphs / custom kernels on this path (DataParallel-safe)
    if sw is not None and getattr(sw, "save_this", False) and hasattr(sw, "summ_feats"):
        sw.summ_feats("1_model/0_fmaps", fmaps.unbind(1))                       # nets/pips.py:447-448

    coords = (xys.clone() / float(stride)).reshape(B, 1, N, 2).repeat(1, S, 1, 1) if coords_init is None \
        else coords_init.clone() / stride
    pyramid = [fmaps]
    for _ in range(L - 1):
        f = F.avg_pool2d(pyramid[-1].flatten(0, 1), 2, stride=2)
        pyramid.append(f.reshape(B, S, *f.shape[1:]))
    ffeat = sample_clamped(fmaps[:, 0], coords[:, 0, :, 0], coords[:, 0, :, 1]) if feat_init is None else feat_init
    ffeats = ffeat.unsqueeze(1).repeat(1, S, 1, 1)
    coords0 = coords.clone()

    offs = torch.linspace(-r, r, 2 * r + 1, device=coords.device)
    window = torch.stack(torch.meshgrid(offs, offs, indexing="ij"), dim=-1).view(1, 2 * r + 1, 2 * r + 1, 2)
    times = torch.linspace(0, S, S, device=coords.device).reshape(1, S, 1)

    # loss_path='fused': the score-map loss comes from fused_score_map_loss over each iteration's starting ffeats, so the
    # dense score maps fcps (B,S,iters,N,H8,W8) are never built
    fused = (trajs_g is not None and getattr(model, "loss_path", "torch") == "fused"
             and all(t.is_cuda for t in (rgbs, trajs_g, vis_g, valids)))
    # corr_path='cuda': the correlation comes from local_corr_cuda over channels-last levels (built once; a no-op after
    # encoder_cuda, whose channels-last strides avg_pool2d keeps), so no all-pairs volume is kept for a backward; the
    # volumes are only built where the dense score maps need them
    corr_cuda = (getattr(model, "corr_path", "torch") == "cuda" and rgbs.is_cuda and H8 >= 8 and W8 >= 8)
    if corr_cuda:
        levels_cl = [lv.permute(0, 1, 3, 4, 2).contiguous().flatten(0, 1) for lv in pyramid]
    preds, anim, fcps, ffeats_per_iter = [], [coords.detach() * stride] * 2, [], []
    for _ in range(iters):
        coords = coords.detach()
        feats_ = ffeats.permute(0, 2, 1, 3).reshape(B * N, S, -1)
        vols = None
        if not (corr_cuda and fused):
            vols = [torch.matmul(ffeats, f.flatten(3)).reshape(B, S, N, *f.shape[-2:]) / torch.sqrt(torch.tensor(float(f.shape[2])))
                    for f in pyramid]                                           # :384-398
        if fused:
            ffeats_per_iter.append(ffeats)
        else:
            fcp = sum(F.interpolate(v.flatten(0, 1), (H8, W8), mode="bilinear", align_corners=True).reshape(B, S, N, H8, W8)
                      for v in vols)                                            # :504-511
            fcps.append(fcp)
        if corr_cuda:
            fcorr = local_corr_cuda(feats_, levels_cl, coords)                  # :355-382 on sm_90a
        else:
            taps = []
            for i, v in enumerate(vols):                                        # :355-382
                h, w = v.shape[-2:]
                loc = coords.reshape(B * S * N, 1, 1, 2) / 2 ** i + window
                if h > 1 and w > 1:
                    grid = torch.cat([2 * loc[..., :1] / (w - 1) - 1, 2 * loc[..., 1:] / (h - 1) - 1], dim=-1)
                    taps.append(F.grid_sample(v.reshape(B * S * N, 1, h, w), grid, align_corners=True).view(B, S, N, -1))
                else:
                    # a level one pixel high or wide (level 3 of an 8 to 15 px map): align_corners=True divides by
                    # size - 1 = 0 and every tap is NaN.  align_corners=False puts pixel j at j as well, so this is the
                    # same bilinear sample with zero padding, the one local_corr_cuda and pips_corr_gather take.
                    grid = torch.cat([(2 * loc[..., :1] + 1) / w - 1, (2 * loc[..., 1:] + 1) / h - 1], dim=-1)
                    taps.append(F.grid_sample(v.reshape(B * S * N, 1, h, w), grid, align_corners=False).view(B, S, N, -1))
            fcorr = torch.cat(taps, dim=-1).permute(0, 2, 1, 3).reshape(B * N, S, -1)
        flow = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        flow = torch.cat([flow, times.expand(B * N, -1, -1)], dim=2)
        x_mix = torch.cat([feats_, fcorr, motion_embedding(flow)], dim=2)
        if getattr(model, "mixer_path", "torch") == "cuda" and x_mix.is_cuda:
            delta = delta_block_cuda(model.delta_block, x_mix)                                      # :524 on sm_90a
        else:
            delta = model.delta_block(x_mix)                                                        # :524
        dfeat = delta[:, :, 2:].reshape(B * N * S, -1)
        feats_ = model.ffeat_updater(model.norm(dfeat)) + feats_.reshape(B * N * S, -1)             # :530
        ffeats = feats_.reshape(B, N, S, -1).permute(0, 2, 1, 3)
        coords = coords + delta[:, :, :2].reshape(B, N, S, 2).permute(0, 2, 1, 3)                   # :533
        if not is_train:
            coords[:, 0] = coords0[:, 0]                                                            # :535-536
        preds.append(coords * stride)
        anim.append(coords * stride)
    vis_e = model.vis_predictor(ffeats.reshape(B * S * N, -1)).reshape(B, S, N)                     # :559
    anim += [coords * stride] * 2

    losses = None
    if fused:
        losses = (sequence_loss(preds, trajs_g, vis_g, valids, 0.8), balanced_ce_loss(vis_e, vis_g, valids)[0],
                  fused_score_map_loss(ffeats_per_iter, pyramid, trajs_g / float(stride), vis_g, valids))
    elif trajs_g is not None:
        fcps_t = torch.stack(fcps, dim=2)
        losses = (sequence_loss(preds, trajs_g, vis_g, valids, 0.8), balanced_ce_loss(vis_e, vis_g, valids)[0],
                  score_map_loss(fcps_t, trajs_g / float(stride), vis_g, valids))
    if return_feat:
        return preds, anim, vis_e, ffeat, losses
    return preds, anim, vis_e, losses
