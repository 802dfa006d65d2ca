"""Differentiable PyTorch path of ``Pips.forward`` for the cases the CUDA inference loop does not
cover: ground truth given (losses requested, nets/pips.py:600-606), ``is_train=True`` (no frame-0
lock, gradients needed) or a summary writer that wants to log this step.  It runs wherever the
tensors live (it is what ``train.py`` / ``test_on_flt.py`` exercise) and keeps the reference's
semantics, including the dense score map ``fcps`` that only the score-map loss consumes -- except with
``model.loss_path == 'fused'`` on CUDA tensors, where ``fused_score_map_loss`` computes that loss and its gradients
without ``fcps``.

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
        for i, f in enumerate(ffeats):
            fi = f.detach().float().permute(0, 2, 1, 3).contiguous()        # ((b*N + n), s, c): free for the loop's state
            L.check(lib.pips_scoremap_loss(L.ptr(g_hi), L.ptr(g_lo), L.ptr(fi), B, S, N, H8, W8, L.ptr(target),
                                           L.ptr(neg[i]), L.ptr(pos[i]), st), "pips_scoremap_loss")
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
            L.check(lib.pips_scoremap_grad_feats(L.ptr(g_hi), L.ptr(g_lo), L.ptr(F_), I, B, S, N, H8, W8, L.ptr(target),
                                                 L.ptr(coef), L.ptr(dF), st), "pips_scoremap_grad_feats")
        dls = [None] * len(ctx.level_shapes)
        if need_l:
            f_hi = torch.empty(F_.shape, dtype=torch.bfloat16, device=dev)
            f_lo = torch.empty_like(f_hi)
            L.check(lib.pips_split_bf16(L.ptr(F_), L.ptr(f_hi), L.ptr(f_lo), F_.numel(), st), "pips_split_bf16")
            del F_
            dG = torch.empty(B * S, P, C, device=dev)
            L.check(lib.pips_scoremap_grad_basis(L.ptr(g_hi), L.ptr(g_lo), L.ptr(f_hi), L.ptr(f_lo), I, B, S, N, H8, W8,
                                                 L.ptr(target), L.ptr(coef), L.ptr(dG), st), "pips_scoremap_grad_basis")
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

    fmaps = model.encode(rgbs, torch_only=True)          # no CUDA graphs / custom kernels on this path (DataParallel-safe)
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
    preds, anim, fcps, ffeats_per_iter = [], [coords.detach() * stride] * 2, [], []
    for _ in range(iters):
        coords = coords.detach()
        vols = [torch.matmul(ffeats, f.flatten(3)).reshape(B, S, N, *f.shape[-2:]) / torch.sqrt(torch.tensor(float(f.shape[2])))
                for f in pyramid]                                               # :384-398
        if fused:
            ffeats_per_iter.append(ffeats)
        else:
            fcp = sum(F.interpolate(v.flatten(0, 1), (H8, W8), mode="bilinear", align_corners=True).reshape(B, S, N, H8, W8)
                      for v in vols)                                            # :504-511
            fcps.append(fcp)
        taps = []
        for i, v in enumerate(vols):                                            # :355-382
            h, w = v.shape[-2:]
            loc = coords.reshape(B * S * N, 1, 1, 2) / 2 ** i + window
            grid = torch.cat([2 * loc[..., :1] / (w - 1) - 1, 2 * loc[..., 1:] / (h - 1) - 1], dim=-1)
            taps.append(F.grid_sample(v.reshape(B * S * N, 1, h, w), grid, align_corners=True).view(B, S, N, -1))
        fcorr = torch.cat(taps, dim=-1).permute(0, 2, 1, 3).reshape(B * N, S, -1)
        flow = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        flow = torch.cat([flow, times.expand(B * N, -1, -1)], dim=2)
        feats_ = ffeats.permute(0, 2, 1, 3).reshape(B * N, S, -1)
        delta = model.delta_block(torch.cat([feats_, fcorr, motion_embedding(flow)], dim=2))      # :524
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
