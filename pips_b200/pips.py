"""Drop-in for the reference's ``nets.pips.Pips`` (nets/pips.py:400-611).

Same constructor, same ``forward(xys, rgbs, coords_init, feat_init, iters, trajs_g, vis_g, valids,
sw, return_feat, is_train)`` signature and return tuples, same ``state_dict`` keys -- so ``demo.py``,
``chain_demo.py``, ``test_on_*.py`` and ``saverloader.load`` work unchanged -- but at inference the
per-iteration refinement loop (nets/pips.py:459-559) runs in hand-written sm_90a CUDA
(libpips_b200.so) instead of ~150 eager torch ops per iteration, and the all-pairs correlation
volume is never materialised.

Window length: plain inference (forward, refine, score_maps) and evaluation with ground truth under no_grad with
loss_path 'cuda' / 'fused' run models of any S from 2 to 16 on the CUDA path (the token-mixing kernels pad the frame
axis to 8 or 16).  Training with mixer_path='cuda', chained tracking and streaming (pips_b200.chain /
pips_b200.stream) and particle-sharded models need S = 8 and raise ValueError otherwise; a clip whose frame count
differs from the model's S, S = 1 and S > 16 raise PipsCudaError on the CUDA path.

Extra, optional knobs (keyword-only; the reference signature is unchanged):
  precision   'bf16x3' (default; wgmma with hi/lo-split bf16 operands, fp32-class accuracy, meets
              the 1e-3 px parity target), 'bf16' (fast, ~1e-2 px), 'fp32' (CUDA-core GEMMs, exact)
  feat_dtype  'fp32' (default) or 'bf16' storage of the correlation pyramid
  fnet_mode   'tc' (default; residual stages and head as wgmma implicit-GEMM convolutions with bf16x3
              operands, element-wise stages fused, channels-last), 'fast' (cuDNN TF32 tensor-core
              convolutions over hi/lo-split operands instead), 'x3' (the same cuDNN convolutions through
              eager torch ops) or 'plain' (strict fp32 cuDNN)
  loss_path   'torch' (default), 'cuda' or 'fused': where a call WITH ground truth (trajs_g, vis_g, valids) runs when no
              gradient is wanted.  'torch' is the dense differentiable path (torch_path.forward_torch); 'cuda' runs
              the encoder and refinement loop of plain inference and computes the score-map loss with
              pips_scoremap_loss, which never stores the (B,S,iters,N,H8,W8) score maps.  'fused' does what 'cuda' does,
              and every other call with ground truth (gradients on, is_train=True: train.py) runs the differentiable
              path with torch_path.fused_score_map_loss, whose forward and backward are CUDA kernels that never build
              the score maps either (CPU tensors keep the dense loss)
  mixer_path  'torch' (default) or 'cuda': where the differentiable path (torch_path.forward_torch: ground truth,
              is_train=True, train.py) runs the DeltaBlock mixer.  'torch' is the nn.Module under autograd, which keeps
              every intermediate of every block; 'cuda' is torch_path.delta_block_cuda, one autograd node whose forward
              and backward run on sm_90a kernels (wgmma GEMMs, recompute per block from the saved block inputs) in
              bf16x3 arithmetic -- always, since PIPS_B200_PRECISION is an inference knob.  CPU tensors keep the module.
              Independent of loss_path; loss_path='fused', mixer_path='cuda' puts both on the CUDA kernels
  encoder_path 'torch' (default) or 'cuda': where the differentiable path runs the feature encoder.  'torch' is the
              Encoder module under autograd in strict fp32 (Pips.encode(torch_only=True)), which keeps every convolution
              output, InstanceNorm input and ReLU output until the backward; 'cuda' is torch_path.encoder_cuda, one
              autograd node whose forward (the kernels of fnet_tc, same bits) and backward (wgmma weight and input
              gradients, recompute per ResBlock from the saved block boundaries) run on sm_90a in bf16x3.  CPU tensors and
              an rgbs that requires grad keep the module; plain inference is unaffected.  Independent of loss_path and
              mixer_path
  corr_path   'torch' (default) or 'cuda': where the differentiable path computes the local correlation.  'torch' is
              the reference's formulation under autograd: all-pairs volumes (B,S,N,h,w) of the 4 levels by matmul, 196
              taps by grid_sample, every volume kept until the backward (whose grid_sample adjoint accumulates with
              atomics).  'cuda' is torch_path.local_corr_cuda: pips_corr_gather's 8x8 footprints forward and
              deterministic gather kernels backward, with no volume; volumes are then built only for the dense score
              maps (loss_path other than 'fused').  Any window of 2 to 16 frames: S != 8 runs the _window entry points
              of the same gradient kernels.  CPU tensors and maps under 8x8 keep the torch formulation; plain inference
              is unaffected.  Independent of the other paths
Environment overrides: PIPS_B200_PRECISION, PIPS_B200_FEAT, PIPS_B200_FNET, PIPS_B200_LOSSES, PIPS_B200_MIXER,
PIPS_B200_ENCODER, PIPS_B200_CORR.
"""
from __future__ import annotations

import contextlib
import os
from typing import Optional

import torch
import torch.nn as nn

from .encoder import Encoder
from .engine import RefineEngine

LATENT = 128
CORR_LEVELS = 4
CORR_RADIUS = 3


class PreNormResidual(nn.Module):
    def __init__(self, dim: int, fn: nn.Module):
        super().__init__()
        self.fn = fn
        self.norm = nn.LayerNorm(dim)

    def forward(self, x):
        return self.fn(self.norm(x)) + x


class _MeanOverFrames(nn.Module):
    def forward(self, x):                      # (R, S, C) -> (R, C)
        return x.mean(dim=1)


def _feed_forward(dim: int, dense) -> nn.Sequential:
    # indices 0 and 3 carry the parameters, like the reference's FeedForward (nets/pips.py:102-109);
    # the Dropout(0.) slots are identities
    return nn.Sequential(dense(dim, dim * 4), nn.GELU(), nn.Identity(), dense(dim * 4, dim), nn.Identity())


def _conv1(cin, cout):
    return nn.Conv1d(cin, cout, kernel_size=1)


class DeltaBlock(nn.Module):
    """MLP-Mixer over the S x 519 token stack of one track (nets/pips.py:283-311, :111-123)."""

    def __init__(self, input_dim=LATENT, corr_levels=CORR_LEVELS, corr_radius=CORR_RADIUS, S=8, dim=512, depth=12):
        super().__init__()
        self.input_dim, self.S = input_dim, S
        kitchen = corr_levels * (2 * corr_radius + 1) ** 2 + input_dim + 64 * 3 + 3
        blocks = [nn.Sequential(PreNormResidual(dim, _feed_forward(S, _conv1)),
                                PreNormResidual(dim, _feed_forward(dim, nn.Linear))) for _ in range(depth)]
        self.to_delta = nn.Sequential(nn.Linear(kitchen, dim), *blocks, nn.LayerNorm(dim), _MeanOverFrames(),
                                      nn.Linear(dim, S * (input_dim + 2)))

    def forward(self, x):                      # x: (R, S, 519) already concatenated
        return self.to_delta(x).reshape(x.shape[0], self.S, self.input_dim + 2)


@contextlib.contextmanager
def _conv_math(allow_tf32: bool):
    """Pin cuDNN's conv math for fnet.  torch enables plain TF32 convolutions by default on Ampere+, which
    alone moves trajectories by ~1e-2 px (measured: fmaps error 2.5e-2); fnet therefore runs either in
    strict fp32 ('plain') or in the 3xTF32 split mode ('x3', fp32-class accuracy on the tensor cores)."""
    c, m = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = c, m


class Pips(nn.Module):
    def __init__(self, S=8, stride=8, *, precision: Optional[str] = None, feat_dtype: Optional[str] = None,
                 fnet_mode: Optional[str] = None, max_seqs: int = 32768, loss_path: Optional[str] = None,
                 mixer_path: Optional[str] = None, encoder_path: Optional[str] = None, corr_path: Optional[str] = None):
        super().__init__()
        self.S = S
        self.stride = stride
        self.hidden_dim = 256
        self.latent_dim = LATENT
        self.corr_levels = CORR_LEVELS
        self.corr_radius = CORR_RADIUS

        self.fnet = Encoder(output_dim=LATENT, stride=stride)
        self.delta_block = DeltaBlock(input_dim=LATENT, corr_levels=CORR_LEVELS, corr_radius=CORR_RADIUS, S=S)
        self.norm = nn.GroupNorm(1, LATENT)
        self.ffeat_updater = nn.Sequential(nn.Linear(LATENT, LATENT), nn.GELU())
        self.vis_predictor = nn.Sequential(nn.Linear(LATENT, 1))

        precision = precision or os.environ.get("PIPS_B200_PRECISION", "bf16x3")
        feat_dtype = feat_dtype or os.environ.get("PIPS_B200_FEAT", "fp32")
        self._engine = RefineEngine(precision=precision, feat_dtype=feat_dtype, max_seqs=max_seqs)
        self._shard = None                      # (rank, world, group) when particle-sharded
        self.shard_fnet = True                  # sharded runs also split the encoder's frames over the ranks
        self.fnet_mode = fnet_mode or os.environ.get("PIPS_B200_FNET", "tc")
        if self.fnet_mode not in ("tc", "fast", "x3", "plain"):
            raise ValueError("fnet_mode must be 'tc' (wgmma implicit-GEMM convolutions, bf16x3), 'fast' (cuDNN 3xTF32 "
                             "convolutions, channels-last, fused element-wise kernels), 'x3' (3xTF32 convolutions through "
                             "eager torch ops) or 'plain' (strict fp32 cuDNN)")
        self.loss_path = loss_path or os.environ.get("PIPS_B200_LOSSES", "torch")
        if self.loss_path not in ("torch", "cuda", "fused"):
            raise ValueError("loss_path must be 'torch' (dense differentiable score maps), 'cuda' (fused score-map "
                             "loss kernel, inference only) or 'fused' ('cuda', and the fused loss with its CUDA backward "
                             "on the differentiable path)")
        self.mixer_path = mixer_path or os.environ.get("PIPS_B200_MIXER", "torch")
        if self.mixer_path not in ("torch", "cuda"):
            raise ValueError("mixer_path must be 'torch' (the DeltaBlock module under autograd) or 'cuda' (its forward and "
                             "backward on the sm_90a kernels, bf16x3)")
        self.encoder_path = encoder_path or os.environ.get("PIPS_B200_ENCODER", "torch")
        if self.encoder_path not in ("torch", "cuda"):
            raise ValueError("encoder_path must be 'torch' (the Encoder module under autograd) or 'cuda' (its forward and "
                             "backward on the sm_90a kernels, bf16x3)")
        self.corr_path = corr_path or os.environ.get("PIPS_B200_CORR", "torch")
        if self.corr_path not in ("torch", "cuda"):
            raise ValueError("corr_path must be 'torch' (all-pairs volumes and grid_sample under autograd) or 'cuda' (the "
                             "local correlation and its gradients on the sm_90a kernels, without the volumes)")

    # ------------------------------------------------------------------ configuration
    @property
    def engine(self) -> RefineEngine:
        return self._engine

    def shard_particles(self, group=None, balance: Optional[bool] = None) -> "Pips":
        """Particle-axis data parallelism (SURVEY.md section 8e): every rank owns a share of the tracks and a
        full copy of the feature pyramid; results are exchanged so each rank returns the full
        result.  Call after ``torch.distributed.init_process_group``.
        ``balance`` (default off; PIPS_B200_BALANCE=1 turns it on): after a few forwards the shares become proportional to
        each GPU's measured speed (sharding._Balance).  Under a power cap a GPU's speed drifts from step to step and WHICH
        GPU is slowest can change between runs, so a share fixed from a few samples need not beat equal shares -- an
        option for nodes with a persistently slow GPU (not measured on H100).
        Results do not depend on the shares (tracks are independent): bit-exact either way (tools/check_sharded.py)."""
        import torch.distributed as dist
        self._shard = (dist.get_rank(group), dist.get_world_size(group), group)
        if balance is None:
            balance = os.environ.get("PIPS_B200_BALANCE", "0") == "1"
        if balance and self._shard[1] > 1:
            from .sharding import _Balance
            self._balance = _Balance()
        else:
            self._balance = None
        return self

    def close_peer_slabs(self) -> None:
        """Collective: release the peer-mapped slabs of a particle-sharded model (results and feature maps).  They are
        re-created on demand by the next sharded forward."""
        for name in ("_peer_slab", "_fmap_peer_slab"):
            slab = getattr(self, name, None)
            if slab is not None:
                slab.close()
                setattr(self, name, None)
        self._engine.invalidate(graphs_only=True)

    # ------------------------------------------------------------------ forward
    def encode(self, rgbs: torch.Tensor, torch_only: bool = False) -> torch.Tensor:
        """nets/pips.py:436-445: normalise to [-1,1], fnet per frame -> (B,S,128,H8,W8) fp32.
        ``torch_only``: the plain torch module with strict-fp32 cuDNN math -- what the supervised / training path
        (torch_path.forward_torch) uses: it may run on nn.DataParallel replicas from worker threads (train.py:254),
        where per-parameter-pointer graph caches would be re-captured on every call and stream capture is unsafe."""
        B, S, C, H, W = rgbs.shape
        # the split paths detach the weights: inference only (the training path keeps plain cuDNN + autograd)
        infer = rgbs.is_cuda and not torch.is_grad_enabled() and not torch_only
        H8, W8 = H // self.stride, W // self.stride
        if self.fnet_mode == "tc" and infer:
            from .encoder_fast import fnet_tc, fnet_tc_graphed
            raw = rgbs if rgbs.dtype in (torch.float32, torch.bfloat16) else rgbs.float()
            run = fnet_tc_graphed if self._engine.use_graph else fnet_tc
            f = run(self.fnet, raw.reshape(B * S, C, H, W).contiguous())  # normalisation fused into the stem
            return f.reshape(B, S, H8, W8, self.latent_dim).permute(0, 1, 4, 2, 3)   # logical (B,S,128,H8,W8)
        x = 2 * (rgbs.float() / 255.0) - 1.0
        if self.fnet_mode == "fast" and infer:
            from .encoder_fast import fnet_fast
            with _conv_math(allow_tf32=True):
                f = fnet_fast(self.fnet, x.reshape(B * S, C, H, W))       # (B*S, H8, W8, 128) NHWC
            return f.reshape(B, S, H8, W8, self.latent_dim).permute(0, 1, 4, 2, 3)  # logical (B,S,128,H8,W8)
        x3 = self.fnet_mode in ("x3", "fast", "tc") and infer
        self.fnet.mode = "x3" if x3 else "plain"
        with _conv_math(allow_tf32=x3):
            fmaps = self.fnet(x.reshape(B * S, C, H, W))
        return fmaps.reshape(B, S, self.latent_dim, H8, W8)

    def forward(self, xys, rgbs, coords_init=None, feat_init=None, iters=3, trajs_g=None, vis_g=None, valids=None,
                sw=None, return_feat=False, is_train=False):
        B, N, D = xys.shape
        assert (D == 2)
        B, S, C, H, W = rgbs.shape

        save_this = sw is not None and getattr(sw, "save_this", False)
        # evaluation with ground truth (test_on_flt.py:87, test_on_crohd.py:133): no gradient wanted, so the score-map
        # loss can come from the fused kernel instead of the dense score maps -- when loss_path asks for it
        cuda_losses = (trajs_g is not None and self.loss_path in ("cuda", "fused") and not is_train and not save_this
                       and all(t is not None and t.is_cuda for t in (rgbs, trajs_g, vis_g, valids))
                       and not torch.is_grad_enabled() and (self._shard is None or self._shard[1] == 1))
        slow = not cuda_losses and (trajs_g is not None or is_train or save_this)
        if S != 8 and rgbs.is_cuda:                 # what stays S = 8, refused before the encoder runs
            if self._shard is not None and self._shard[1] > 1:
                raise ValueError(f"pips_b200.Pips: particle-sharded models need S=8; this model has S={self.S}")
            if slow and self.mixer_path == "cuda" and (is_train or torch.is_grad_enabled()):
                raise ValueError(f"pips_b200.Pips: mixer_path='cuda' trains models of S=8 only; this model has S={self.S}")
        if slow:
            from .torch_path import forward_torch
            return forward_torch(self, xys, rgbs, coords_init=coords_init, feat_init=feat_init, iters=iters,
                                 trajs_g=trajs_g, vis_g=vis_g, valids=valids, sw=sw, return_feat=return_feat,
                                 is_train=is_train)
        if N == 0:
            # the reference fails on an empty particle axis (F.interpolate of the empty correlation volume,
            # nets/pips.py:509 -> RuntimeError; recorded in tests/golden as edge/n0_error): same error type here
            raise RuntimeError("pips_b200.Pips: no particles (xys has N = 0); the reference raises here as well")
        if not rgbs.is_cuda:
            raise RuntimeError("pips_b200.Pips: the inference path is CUDA-only (sm_90a); move the model and "
                               "inputs to a CUDA device. There is no CPU fallback.")
        self._check_frames(S)
        with torch.no_grad():
            if self._shard is not None and self._shard[1] > 1 and self.shard_fnet and self.fnet_mode == "tc":
                from .sharding import encode_sharded
                fmaps = encode_sharded(self, rgbs)
            else:
                fmaps = self.encode(rgbs)
            if cuda_losses:
                return self.refine(xys, fmaps, coords_init=coords_init, feat_init=feat_init, iters=iters,
                                   return_feat=return_feat, trajs_g=trajs_g, vis_g=vis_g, valids=valids)
            return self.refine(xys, fmaps, coords_init=coords_init, feat_init=feat_init, iters=iters,
                               return_feat=return_feat)

    @torch.no_grad()
    def score_maps(self, xys, rgbs, particles, iters=3, coords_init=None, feat_init=None):
        """The dense score maps ``fcps`` of nets/pips.py:504-511,:565 for the chosen ``particles`` only
        (SURVEY.md section 8f-3): (B,S,iters,len(particles),H8,W8), i.e. ``fcps[:, :, :, particles]`` of the
        reference, without the all-pairs volume.  The reference's own consumers look at one particle
        (``fcps[0:1,:,:,0:1]``, nets/pips.py:572).  Also returns (coord_predictions, vis_e) of the same run."""
        if not rgbs.is_cuda:
            raise RuntimeError("pips_b200.Pips.score_maps is CUDA-only (sm_90a)")
        B, N, D = xys.shape
        assert (D == 2)
        S = rgbs.shape[1]
        self._check_frames(S)
        fmaps = self.encode(rgbs)
        stride = float(self.stride)
        if coords_init is None:
            coords = (xys.detach().float() / stride).reshape(B, 1, N, 2).repeat(1, S, 1, 1)
        else:
            coords = coords_init.detach().float() / stride
        sel = torch.as_tensor(particles, dtype=torch.int64, device=rgbs.device).flatten()
        H8, W8 = fmaps.shape[-2:]
        fcps = torch.empty(B, S, iters, sel.numel(), H8, W8, dtype=torch.float32, device=rgbs.device)
        preds, vis_e, _ = self._engine.refine(self, fmaps.float(), coords,
                                              None if feat_init is None else feat_init.detach().float(), iters, stride,
                                              heat_sel=sel, heat_out=fcps)
        return fcps, [preds[i] for i in range(iters)], vis_e

    def _check_frames(self, S: int) -> None:
        """The CUDA path's window: 2 <= S <= 16 frames, as many as the model was built for (its token mixing)."""
        from ._lib import PipsCudaError
        if not 2 <= S <= 16:
            raise PipsCudaError(f"pips_b200 CUDA path supports 2 <= S <= 16 frames per window (got S={S})")
        if S != self.S:
            raise PipsCudaError(f"pips_b200: the clip has S={S} frames, the model was built for S={self.S}")
        if S != 8 and self._shard is not None and self._shard[1] > 1:
            raise ValueError(f"pips_b200.Pips: particle-sharded models need S=8; this model has S={self.S}")

    def refine(self, xys, fmaps, coords_init=None, feat_init=None, iters=3, return_feat=False, trajs_g=None, vis_g=None,
               valids=None):
        """Everything after fnet (nets/pips.py:450-611) given precomputed feature maps.  With ground truth
        (trajs_g (B,S,N,2) in input pixels, vis_g and valids (B,S,N)) ``losses`` is the reference's
        (seq_loss, vis_loss, ce_loss) as 0-dim fp32 tensors (nets/pips.py:600-606), without gradients; the score-map
        loss comes from pips_scoremap_loss.  Not for particle-sharded models."""
        B, N, _ = xys.shape
        S = fmaps.shape[1]
        self._check_frames(S)
        stride = float(self.stride)
        loss_target = score = None
        if trajs_g is not None:
            from .torch_path import score_map_targets
            assert tuple(trajs_g.shape) == (B, S, N, 2), "trajs_g must be (B,S,N,2)"
            assert tuple(vis_g.shape) == (B, S, N) and tuple(valids.shape) == (B, S, N), "vis_g, valids must be (B,S,N)"
            if self._shard is not None and self._shard[1] > 1:
                raise RuntimeError("pips_b200.Pips: losses on the CUDA path are not available for particle-sharded models")
            H8, W8 = fmaps.shape[-2:]
            loss_target = score_map_targets(trajs_g / stride, vis_g, valids, H8, W8)      # :603
            score = torch.empty((), dtype=torch.float32, device=fmaps.device)
        xys_ = xys.detach().float() / stride                                            # :450
        if coords_init is None:
            coords = xys_.reshape(B, 1, N, 2).repeat(1, S, 1, 1)                        # :453
        else:
            coords = coords_init.detach().float() / self.stride                         # :455
        if feat_init is not None:
            feat_init = feat_init.detach().float()

        if self._shard is None or self._shard[1] == 1:
            preds, vis_e, ffeat = self._engine.refine(self, fmaps.float(), coords, feat_init, iters, stride,
                                                      loss_target=loss_target, loss_out=score)
        else:
            from .sharding import refine_sharded
            preds, vis_e, ffeat = refine_sharded(self, fmaps.float(), coords, feat_init, iters, stride)

        start = coords * stride
        coord_predictions = [preds[i] for i in range(iters)]                            # :538
        last = coord_predictions[-1] if iters > 0 else start
        coord_predictions2 = [start, start] + coord_predictions + [last, last]          # :474-475, :562-563
        losses = None
        if trajs_g is not None:                                                         # :600-604
            from .torch_path import balanced_ce_loss, sequence_loss
            losses = (sequence_loss(coord_predictions, trajs_g, vis_g, valids, 0.8),
                      balanced_ce_loss(vis_e, vis_g, valids)[0], score)
        if return_feat:
            return coord_predictions, coord_predictions2, vis_e, ffeat, losses
        return coord_predictions, coord_predictions2, vis_e, losses
