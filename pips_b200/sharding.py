"""Particle-axis sharding over the GPUs of one node (SURVEY.md section 8e).

Tracks are independent -- the mixer mixes over the S frames and the channels of one track, never
across particles (nets/pips.py:517-524) -- so rank g refines particles [g*N/G, (g+1)*N/G) against its
own full copy of the feature pyramid.  The only exchange is the results (every rank returns the full
``coord_predictions`` / ``vis_e`` / ``ffeat``; <= 1 MB per iteration at the BASELINE configs):

  * ``refine_sharded_p2p`` (default when all ranks share a host): every rank's update kernel stores its slice
    straight into all ranks' result slabs over NVLink (pips_b200/peer.py, csrc/peer.cu), two flag barriers fence
    the slab; no collective library call on the data path, everything inside the per-shape CUDA graph;
  * ``refine_sharded_nccl``: one asynchronous ``all_gather_into_tensor`` per iteration plus two at the end
    (ranks on different hosts, ``PIPS_B200_GATHER=nccl``, or slab set-up failed -- decided collectively).

``encode_sharded`` splits the encoder's frames over the ranks and exchanges the feature maps the same way
(peer stores between two flag barriers; NCCL all-gather as the fallback).
Both paths are bit-identical to the unsharded run (tools/check_sharded.py on 2 / 8 GPUs; the host logic is
covered by the world-size-2 gloo tests in tests/test_sharding_cpu.py).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.distributed as dist


TRACE = None        # tools/diag_scale.py: a list that receives (label, cuda event) at the phase boundaries of a sharded forward


def _mark(label: str) -> None:
    if TRACE is not None:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        TRACE.append((label, ev))


def shard_bounds(N: int, rank: int, world: int) -> Tuple[int, int, int]:
    """Equal-size shards of ceil(N/world) particles (the tail is padded by repeating the last track)."""
    per = (N + world - 1) // world
    n0 = min(rank * per, N)
    n1 = min(n0 + per, N)
    return n0, n1, per


def _pad_particles(t: torch.Tensor, dim: int, per: int) -> torch.Tensor:
    n = t.shape[dim]
    if n == per:
        return t.contiguous()
    if n == 0:
        shape = list(t.shape)
        shape[dim] = per
        return torch.zeros(shape, dtype=t.dtype, device=t.device)
    last = t.narrow(dim, n - 1, 1)
    reps = [1] * t.dim()
    reps[dim] = per - n
    return torch.cat([t, last.repeat(*reps)], dim=dim).contiguous()


def gather_mode(model) -> str:
    """'p2p' (peer-mapped slabs, stores fused into the update kernel) or 'nccl' (all-gathers).  Decided once per
    model: PIPS_B200_GATHER overrides; p2p needs every rank on this host and at most 16 of them."""
    mode = getattr(model, "_gather_mode", None)
    if mode is None:
        import os
        from . import _lib as L
        from .peer import same_host
        _, world, group = model._shard
        mode = os.environ.get("PIPS_B200_GATHER", "")
        if mode not in ("p2p", "nccl"):
            mode = "p2p" if (world <= L.MAX_PEERS and same_host(group)) else "nccl"
        model._gather_mode = mode
    return mode


def refine_sharded(model, fmaps: torch.Tensor, coords: torch.Tensor, feat_init: Optional[torch.Tensor], iters: int,
                   stride: float):
    if coords.is_cuda and iters > 0 and gather_mode(model) == "p2p":
        return refine_sharded_p2p(model, fmaps, coords, feat_init, iters, stride)
    return refine_sharded_nccl(model, fmaps, coords, feat_init, iters, stride)


def shard_sizes(N: int, weights, quantum: int = 32):
    """Speed-weighted shard sizes: ``weights[r]`` ~ particles per second of rank r.  Sizes are multiples of ``quantum``
    tracks (32 tracks = one 256-row GEMM tile) where N allows, at least 1, and sum to N.  Deterministic in its inputs,
    so every rank computes the same list."""
    world = len(weights)
    if N < world:
        return None
    q = quantum if N >= 4 * quantum * world else 1
    tot = float(sum(weights))
    ideal = [N * w / tot for w in weights]
    sizes = [max(1 if q == 1 else q, int(x // q) * q) for x in ideal]
    # hand the remainder out in quantum steps to the ranks furthest below their ideal share (ties: lowest rank)
    while sum(sizes) > N:
        r = max(range(world), key=lambda i: (sizes[i] - ideal[i], -i))
        sizes[r] -= min(q, sum(sizes) - N)
    while sum(sizes) < N:
        r = min(range(world), key=lambda i: (sizes[i] - ideal[i], i))
        sizes[r] += min(q, N - sum(sizes))
    return sizes if min(sizes) >= 1 else None


class _Balance:
    """Speed-weighted particle shards.  The GPUs of one box do not run at one clock under the power cap (1.47-1.78 GHz
    seen on a multi-GPU node), and every forward ends in an exchange of results, so with equal shards the step time is the
    SLOWEST GPU's.  After ``warm`` sharded forwards each rank times ``measure`` refinement calls with CUDA events, the
    rates (particles per second) are exchanged once, and from then on rank r gets a share proportional to its rate."""

    def __init__(self, warm: int = 2, measure: int = 3):
        self.warm, self.measure = warm, measure
        self.calls, self.events, self.weights = 0, [], None

    def before(self):
        self.calls += 1
        if self.weights is None and self.calls > self.warm:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            return ev
        return None

    def after(self, ev, n_particles: int, group) -> None:
        if ev is None:
            return
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        self.events.append((ev, e1, n_particles))
        if len(self.events) >= self.measure:               # same call count on every rank: collective below is matched
            torch.cuda.synchronize()
            rate = sum(n for _, _, n in self.events) / max(1e-6, sum(a.elapsed_time(b) for a, b, _ in self.events))
            rates = [None] * dist.get_world_size(group)
            dist.all_gather_object(rates, float(rate), group=group)
            self.weights = rates
            self.events = []


def refine_sharded_p2p(model, fmaps: torch.Tensor, coords: torch.Tensor, feat_init: Optional[torch.Tensor], iters: int,
                       stride: float):
    """No collective on the data path: every rank's update kernel writes its predictions into all ranks' result
    slabs over NVLink (pips_peer_out), two flag barriers fence the slab's reuse and its completion."""
    from . import _lib as L
    from .peer import PeerPlan, PeerSlab
    rank, world, group = model._shard
    B, S, N, _ = coords.shape
    n0, n1, per = shard_bounds(N, rank, world)
    bal = getattr(model, "_balance", None)
    sizes = shard_sizes(N, bal.weights) if (bal is not None and bal.weights is not None) else None
    if sizes is not None:                                                   # speed-weighted shards, no padding
        n0 = sum(sizes[:rank]); n1 = n0 + sizes[rank]; per = sizes[rank]
    dev = coords.device
    need = 4 * PeerPlan.words_needed(world, iters, B, S, per, None if sizes is None else N)
    slab = getattr(model, "_peer_slab", None)
    if slab is None or slab.nbytes < need or slab.device != dev:           # collective: all ranks see the same shapes
        grown = 0
        if slab is not None:
            grown = 2 * slab.nbytes                                         # amortise slowly growing particle counts
            slab.close()
        model._peer_slab = None
        model.engine.invalidate(graphs_only=True)   # captured update kernels store through the old slab's peer mappings
        try:
            model._peer_slab = slab = PeerSlab(max(need, grown, 1 << 16), rank, world, group, dev)
        except L.PipsCudaError as e:        # raised on every rank together (peer.py): all fall back to NCCL
            import warnings
            warnings.warn(f"{e}; exchanging results with NCCL all-gathers instead")
            model._gather_mode = "nccl"
            return refine_sharded_nccl(model, fmaps, coords, feat_init, iters, stride)
    plan = PeerPlan(slab, iters, B, S, per, sizes)
    my_coords = _pad_particles(coords[:, :, n0:n1], 2, per)
    my_feat = None if feat_init is None else _pad_particles(feat_init[:, n0:n1], 1, per)

    _mark("inputs")
    slab.barrier()                      # every rank has copied the previous call's results out of its slab
    _mark("barrier0")
    ev = bal.before() if bal is not None else None
    _, vis, ffeat = model.engine.refine(model, fmaps, my_coords, my_feat, iters, stride, peer=plan)
    if bal is not None:
        bal.after(ev, B * per, group)
    _mark("refine")
    lib, st = L.load(), torch.cuda.current_stream(dev).cuda_stream
    vis, ffeat = vis.contiguous(), ffeat.contiguous()
    L.check(lib.pips_peer_scatter(L.ptr(vis), B * S, per, slab.region_ptrs(plan.off_vis), world, plan.n_total,
                                  plan.n_offset, st), "pips_peer_scatter")
    L.check(lib.pips_peer_scatter(L.ptr(ffeat), B, per * ffeat.shape[-1], slab.region_ptrs(plan.off_ffeat), world,
                                  plan.n_total * ffeat.shape[-1], plan.n_offset * ffeat.shape[-1], st), "pips_peer_scatter")
    slab.barrier()                      # every rank's stores into this slab have landed
    _mark("barrier1")
    c_all, v_all, f_all = plan.views()
    out = c_all[:, :, :, :N].clone(), v_all[:, :, :N].clone(), f_all[:, :N].clone()
    _mark("copy_out")
    return out


def refine_sharded_nccl(model, fmaps: torch.Tensor, coords: torch.Tensor, feat_init: Optional[torch.Tensor], iters: int,
                        stride: float):
    rank, world, group = model._shard
    B, S, N, _ = coords.shape
    n0, n1, per = shard_bounds(N, rank, world)
    my_coords = _pad_particles(coords[:, :, n0:n1], 2, per)
    my_feat = None if feat_init is None else _pad_particles(feat_init[:, n0:n1], 1, per)

    dev = coords.device
    # (world, iters, B, S, per, 2): one gather per iteration, issued as soon as that iteration is enqueued
    gathered = torch.empty(world, iters, B, S, per, 2, dtype=torch.float32, device=dev)
    works = []

    def gather_iter(it, coords_px):
        out = torch.empty(world * B, S, per, 2, dtype=torch.float32, device=dev)     # concatenated along dim 0
        works.append((dist.all_gather_into_tensor(out, coords_px, group=group, async_op=True), out.view(world, B, S, per, 2), it))

    _mark("inputs")
    preds, vis, ffeat = model.engine.refine(model, fmaps, my_coords, my_feat, iters, stride, on_iter=gather_iter)
    _mark("refine")
    if len(works) != iters:                      # particles were chunked inside the engine: gather at the end
        works.clear()
        for it in range(iters):
            gather_iter(it, preds[it].contiguous())
    vis_cat = torch.empty(world * B, S, per, dtype=torch.float32, device=dev)
    wv = dist.all_gather_into_tensor(vis_cat, vis.contiguous(), group=group, async_op=True)
    ff_cat = torch.empty(world * B, per, ffeat.shape[-1], dtype=torch.float32, device=dev)
    wf = dist.all_gather_into_tensor(ff_cat, ffeat.contiguous(), group=group, async_op=True)
    vis_all, ff_all = vis_cat.view(world, B, S, per), ff_cat.view(world, B, per, -1)
    for wk, out, it in works:
        wk.wait()
        gathered[:, it] = out
    wv.wait()
    wf.wait()
    preds_full = gathered.permute(1, 2, 3, 0, 4, 5).reshape(iters, B, S, world * per, 2)[:, :, :, :N].contiguous()
    vis_full = vis_all.permute(1, 2, 0, 3).reshape(B, S, world * per)[:, :, :N].contiguous()
    ff_full = ff_all.permute(1, 0, 2, 3).reshape(B, world * per, -1)[:, :N].contiguous()
    _mark("gathers")
    return preds_full, vis_full, ff_full


def _fmap_slab(model, need_bytes: int, dev):
    """The peer slab the frame-sharded encoder's feature maps are exchanged through (collective create / regrow).
    Returns None -- on every rank together -- when the slabs cannot be set up; the caller then uses NCCL."""
    from . import _lib as L
    from .peer import PeerSlab
    rank, world, group = model._shard
    slab = getattr(model, "_fmap_peer_slab", None)
    if slab is not None and slab.nbytes >= need_bytes and slab.device == dev:
        return slab
    if slab is not None:
        slab.close()
    model._fmap_peer_slab = None
    try:
        model._fmap_peer_slab = PeerSlab(need_bytes, rank, world, group, dev)
    except L.PipsCudaError as e:            # raised on every rank together (peer.py)
        import warnings
        warnings.warn(f"{e}; exchanging the feature maps with an NCCL all-gather instead")
        model._fmap_exchange = "nccl"
    return model._fmap_peer_slab


def encode_sharded(model, rgbs: torch.Tensor) -> torch.Tensor:
    """Frame-sharded fnet (SURVEY.md section 8e-3): the B*S frames are independent (InstanceNorm is per frame,
    nets/pips.py:412), so rank g encodes frames [g*F/G, (g+1)*F/G) and every rank ends up with all feature maps.
    Bit-identical to the unsharded encoder: every kernel of the 'tc' encoder works per image.

    Exchange: like the results, through peer-mapped slabs when all ranks share a host -- each rank stores its
    frames' channels-last maps into every rank's slab over NVLink (``pips_peer_scatter``, 512-byte runs per warp)
    between two flag barriers (slab reuse / stores landed); no collective library call.  Otherwise (ranks on
    several hosts, ``PIPS_B200_GATHER=nccl``, set-up failed) one NCCL all-gather."""
    from . import _lib as L
    from .peer import FLAG_WORDS
    rank, world, group = model._shard
    B, S, C, H, W = rgbs.shape
    F_ = B * S
    per = (F_ + world - 1) // world
    flat = rgbs.reshape(F_, C, H, W)
    idx = torch.arange(rank * per, (rank + 1) * per, device=rgbs.device).clamp_(max=F_ - 1)     # tail ranks repeat the last frame
    _mark("begin")
    mine = model.encode(flat[idx].unsqueeze(0))                                                  # (1, per, 128, H8, W8), NHWC memory
    _mark("fnet_local")
    H8, W8 = mine.shape[-2:]
    local = mine[0].permute(0, 2, 3, 1).contiguous()                                             # (per, H8, W8, 128)
    dev = local.device
    words = local.numel()                                                                        # per rank
    mode = (getattr(model, "_fmap_exchange", None) or gather_mode(model)) if local.is_cuda else "nccl"
    slab = _fmap_slab(model, 4 * (FLAG_WORDS + world * words), dev) if mode == "p2p" else None
    if slab is None:
        full = torch.empty(world * per, H8, W8, local.shape[-1], dtype=local.dtype, device=dev)
        dist.all_gather_into_tensor(full, local, group=group)
        _mark("fmaps_exchange")
        return full[:F_].reshape(B, S, H8, W8, -1).permute(0, 1, 4, 2, 3)                        # logical (B,S,128,H8,W8)
    slab.barrier()                      # every rank has copied the previous call's maps out of its slab
    L.check(L.load().pips_peer_scatter(L.ptr(local), 1, words, slab.region_ptrs(FLAG_WORDS), world, world * words, rank * words,
                                       torch.cuda.current_stream(dev).cuda_stream), "pips_peer_scatter")
    slab.barrier()                      # every rank's stores into this slab have landed
    full = slab.words[FLAG_WORDS:FLAG_WORDS + world * words].view(world * per, H8, W8, local.shape[-1])[:F_].clone()
    _mark("fmaps_exchange")
    return full.reshape(B, S, H8, W8, -1).permute(0, 1, 4, 2, 3)                                 # logical (B,S,128,H8,W8)
