"""Differentiable PyTorch path of ``Pips.forward`` for the cases the CUDA inference loop does not
cover: ground truth given (losses requested, nets/pips.py:600-606), ``is_train=True`` (no frame-0
lock, gradients needed) or a summary writer that wants to log this step.  It runs wherever the
tensors live (it is what ``train.py`` / ``test_on_flt.py`` exercise) and keeps the reference's
semantics, including the dense score map ``fcps`` that only the score-map loss consumes.

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

    preds, anim, fcps = [], [coords.detach() * stride] * 2, []
    for _ in range(iters):
        coords = coords.detach()
        vols = [torch.matmul(ffeats, f.flatten(3)).reshape(B, S, N, *f.shape[-2:]) / torch.sqrt(torch.tensor(float(f.shape[2])))
                for f in pyramid]                                               # :384-398
        fcp = sum(F.interpolate(v.flatten(0, 1), (H8, W8), mode="bilinear", align_corners=True).reshape(B, S, N, H8, W8)
                  for v in vols)                                                # :504-511
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
    if trajs_g is not None:
        fcps_t = torch.stack(fcps, dim=2)
        losses = (sequence_loss(preds, trajs_g, vis_g, valids, 0.8), balanced_ce_loss(vis_e, vis_g, valids)[0],
                  score_map_loss(fcps_t, trajs_g / float(stride), vis_g, valids))
    if return_feat:
        return preds, anim, vis_e, ffeat, losses
    return preds, anim, vis_e, losses
