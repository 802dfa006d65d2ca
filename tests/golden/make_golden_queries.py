"""Queries at any frame (t, x, y), tracked forward and backward in time: the slice-and-flip composition of the
reference chain, and the golden it records from the UNMODIFIED reference (run in the build container only).

    python tests/golden/make_golden_queries.py          # needs /root/reference; writes reference_queries.npz

A query (t, x, y) in a clip of T frames is the chain of chain_demo.py:40-83 (``oracle.pips_oracle.chain_track``) on
rgbs[:, t:] from (x, y) for frames t..T-1, and the same chain on the time-reversed clip rgbs[:, t::-1] (frames t, t-1,
..., 0) from the same start for frames 0..t-1, read back in forward order; that chain also writes frame t, which comes
from the forward one.  The visibility of a frame is sigmoid(vis_e) of the window that last wrote it -- the overwrite
rule chain_demo.py:60-61 applies to the positions.  The clip is CHAIN_CASE's (make_golden.py); inputs are regenerated
from seeds by the tests, so only outputs are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import pips_oracle as po  # noqa: E402
from tests.golden.make_golden import CHAIN_CASE, chain_inputs  # noqa: E402

# The first and the last frame, and both sides of the first window boundary (frames 7 | 8).  The positions' seed is one
# whose chains pick varied skips (2, 3, 4, 5 and 7; up to 8 rounds).
QUERY_TIMES = [0, 1, 7, 9, 17, 18]
QUERY_SEED = 601
WIN = 8


def query_inputs(c):
    """CHAIN_CASE's clip and (1, 6, 3) queries (t, x, y) at QUERY_TIMES."""
    rgbs, _ = chain_inputs(c)
    xy = po.random_queries(1, len(QUERY_TIMES), c["H"], c["W"], seed=QUERY_SEED)
    t = torch.tensor(QUERY_TIMES, dtype=torch.float32).view(1, -1, 1)
    return rgbs, torch.cat([t, xy], dim=2)


def chain_track_vis(forward_fn, rgbs, xy0, iters=6):
    """oracle.pips_oracle.chain_track, plus vis (1,T,N): sigmoid(vis_e) of the window that last wrote each frame.
    chain_track calls the model particle by particle, window by window; its skips say where each window started."""
    T = rgbs.shape[1]
    seen = []

    def recording(xys, seq, feat_init):
        preds, vis_e, ffeat = forward_fn(xys, seq, feat_init)
        seen.append(torch.sigmoid(vis_e).reshape(WIN))                             # chain_demo.py:59
        return preds, vis_e, ffeat

    trajs, skips = po.chain_track(recording, rgbs, xy0, iters=iters)
    vis = torch.zeros(1, T, xy0.shape[1], dtype=torch.float32)
    k = 0
    for n, hist in enumerate(skips):
        cur = 0
        for si in hist:
            m = min(WIN, T - cur)                                                    # S_local truncation, :61
            vis[0, cur:cur + m, n] = seen[k][:m]
            cur, k = cur + si, k + 1
    assert k == len(seen)
    return trajs, skips, vis


def track_queries(forward_fn, rgbs, queries, iters=6):
    """queries (1,N,3) as (t, x, y), t integral in 0..T-1 -> trajs (1,T,N,2), vis (1,T,N) and per query
    (forward skips, backward skips -- [] when t == 0)."""
    B, T = rgbs.shape[:2]
    N = queries.shape[1]
    trajs = torch.zeros(B, T, N, 2, dtype=torch.float32)
    vis = torch.zeros(B, T, N, dtype=torch.float32)
    skips = []
    for n in range(N):
        t = int(queries[0, n, 0])
        xy = queries[:, n:n + 1, 1:3].float()
        tr, sk_f, vi = chain_track_vis(forward_fn, rgbs[:, t:], xy, iters)
        trajs[:, t:, n], vis[:, t:, n] = tr[:, :, 0], vi[:, :, 0]
        sk_b = [[]]
        if t > 0:
            tr, sk_b, vi = chain_track_vis(forward_fn, rgbs[:, :t + 1].flip(1), xy, iters)
            trajs[:, :t, n], vis[:, :t, n] = tr[:, 1:, 0].flip(1), vi[:, 1:, 0].flip(1)
        skips.append((sk_f[0], sk_b[0]))
    return trajs, vis, skips


def main():
    sys.path.insert(0, "/root/reference")
    torch.Tensor.cuda = lambda self, *a, **k: self                               # nets/pips.py:429, see make_golden.py
    from nets.pips import Pips  # the reference, unmodified

    torch.set_num_threads(min(16, os.cpu_count() or 1))
    c = CHAIN_CASE
    sd = po.init_state_dict(seed=c["seed"], head_scale=c["head_scale"])
    model = Pips(S=8, stride=c["stride"]).eval()
    model.load_state_dict(sd, strict=True)
    rgbs, queries = query_inputs(c)

    def ref_window(xys, seq, feat_init):
        with torch.no_grad():
            o = model(xys, seq, iters=c["iters"], feat_init=feat_init, return_feat=True)
        return o[0], o[2], o[3]

    trajs, vis, skips = track_queries(ref_window, rgbs, queries, iters=c["iters"])
    fwd, bwd = [f for f, _ in skips], [b for _, b in skips]
    out = {"trajs": trajs.numpy(), "vis": vis.numpy(),
           "skips_fwd": np.array([len(h) for h in fwd] + [s for h in fwd for s in h], dtype=np.int64),
           "skips_bwd": np.array([len(h) for h in bwd] + [s for h in bwd for s in h], dtype=np.int64)}
    print("query skips (forward, backward)", skips)
    path = os.path.join(HERE, "reference_queries.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
