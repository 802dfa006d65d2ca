"""On-disk weight pack (SURVEY.md section 8f-4): the kernel-layout weights of one checkpoint in one flat file.

The CUDA path does not read ``nn.Linear`` / ``nn.Conv2d`` parameters directly: dense weights are split into
bf16 (hi, lo) pairs, padded to whole TMA boxes (engine.PackedWeights) and the encoder's filters are
re-ordered tap-major / channel-padded for the implicit-GEMM kernel (encoder_fast._packed_weight).  A pack
file stores exactly those tensors so that

  * a process that loads ``model-000200000.pth`` (saverloader.py:25-66 in the reference) finds
    ``model-000200000.pack`` next to it and binds it without running the packing kernels, and
  * a C caller of include/pips_b200.h, which has no torch, can fill ``pips_weights`` from the file: every
    tensor is a named, 256-byte aligned, little-endian array described by a JSON manifest.

Layout:  bytes 0..15  magic "PIPSB200PACK\\0\\0\\0\\1";  16..23  u64 manifest length M;  24..31  u64 data origin D;
bytes 32..32+M  UTF-8 JSON {"fingerprint": hex, "abi": int, "tensors": [{"name", "dtype", "shape", "offset",
"nbytes"}]};  tensor ``name`` occupies file bytes D+offset .. D+offset+nbytes (D and offset multiples of 256).

The fingerprint is a BLAKE2b digest over the module's ``state_dict`` (names, shapes, raw bytes): a pack is
bound only to the parameters it was made from, anything else is re-packed from the module as usual.
"""
from __future__ import annotations

import hashlib
import json
import os
import struct
from typing import Dict, Optional

import numpy as np
import torch

MAGIC = b"PIPSB200PACK\0\0\0\1"
ALIGN = 256
HEADER = 32
_DT = {"float32": (torch.float32, np.float32), "bfloat16": (torch.bfloat16, np.int16)}


def fingerprint(module: torch.nn.Module) -> str:
    """BLAKE2b over (name, shape, bytes) of every state_dict entry, in key order."""
    h = hashlib.blake2b(digest_size=20)
    for name, v in sorted(module.state_dict().items()):
        a = v.detach().to("cpu", torch.float32).contiguous().numpy()
        h.update(name.encode())
        h.update(struct.pack("<%dq" % a.ndim, *a.shape))
        h.update(a.tobytes())
    return h.hexdigest()


def _collect(model) -> Dict[str, torch.Tensor]:
    """Every packed tensor of ``model`` (a pips_b200.Pips on a CUDA device), named.  Mixer / head tensors use
    the field names of ``pips_weights``; encoder filters are "fnet.<conv path>.w_hi" / ".w_lo" and their biases
    "fnet.<conv path>.b" (fp32), the fields of ``pips_encoder_weights``."""
    from . import encoder_fast as EF

    w = model.engine.weights(model)
    out = {"mixer." + k: v for k, v in w.t.items()}
    for name, conv in EF.packed_convs(model.fnet):
        hi, lo = EF.packed_filter(model.fnet, name, conv)
        out[f"fnet.{name}.w_hi"], out[f"fnet.{name}.w_lo"] = hi, lo
        if conv.bias is not None:
            out[f"fnet.{name}.b"] = conv.bias.detach().float().contiguous()
    return out


def write_tensors(path: str, tensors: Dict[str, torch.Tensor], fp: str, abi: int) -> str:
    """Write named tensors (fp32 / bf16, any device) as one pack file, atomically."""
    entries, blobs, off = [], [], 0
    for name, t in tensors.items():
        dt = str(t.dtype).replace("torch.", "")
        if dt not in _DT:
            raise ValueError(f"pack: tensor {name} has unsupported dtype {dt}")
        raw = t.detach().contiguous().cpu()
        raw = raw.view(torch.int16).numpy() if t.dtype == torch.bfloat16 else raw.numpy()
        entries.append({"name": name, "dtype": dt, "shape": list(t.shape), "offset": off, "nbytes": raw.nbytes})
        blobs.append(raw)
        off += (raw.nbytes + ALIGN - 1) // ALIGN * ALIGN
    hdr = json.dumps({"fingerprint": fp, "abi": abi, "tensors": entries}, separators=(",", ":")).encode()
    origin = (HEADER + len(hdr) + ALIGN - 1) // ALIGN * ALIGN
    tmp = path + ".tmp%d" % os.getpid()
    with open(tmp, "wb") as f:
        f.write(MAGIC)
        f.write(struct.pack("<QQ", len(hdr), origin))
        f.write(hdr)
        for e, raw in zip(entries, blobs):
            f.seek(origin + e["offset"])
            f.write(raw.tobytes())
        f.truncate(origin + off)
    os.replace(tmp, path)
    return path


def read_manifest(path: str) -> dict:
    """The JSON manifest plus "origin" (file offset the tensor offsets are relative to)."""
    with open(path, "rb") as f:
        if f.read(16) != MAGIC:
            raise ValueError(f"{path}: not a pips_b200 weight pack")
        n, origin = struct.unpack("<QQ", f.read(16))
        man = json.loads(f.read(n).decode())
    man["origin"] = origin
    return man


def read_tensors(path: str, device="cpu", manifest: Optional[dict] = None) -> Dict[str, torch.Tensor]:
    man = manifest if manifest is not None else read_manifest(path)
    size = os.path.getsize(path)
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    out: Dict[str, torch.Tensor] = {}
    for e in man["tensors"]:
        tdt, ndt = _DT[e["dtype"]]
        start = man["origin"] + e["offset"]
        count = 1
        for d in e["shape"]:
            count *= d
        if e["offset"] % ALIGN or start + e["nbytes"] > size or count * np.dtype(ndt).itemsize != e["nbytes"]:
            raise ValueError(f"{path}: tensor {e['name']} is inconsistent with the file")
        a = np.frombuffer(mm, dtype=ndt, count=count, offset=start)
        t = torch.from_numpy(a.copy()).to(device)
        out[e["name"]] = (t.view(torch.bfloat16) if tdt == torch.bfloat16 else t).reshape(e["shape"])
    return out


def save_pack(model, path: str) -> str:
    """Write the pack of ``model``'s current parameters to ``path``."""
    from . import _lib as L
    tensors = _collect(model)
    torch.cuda.synchronize()
    return write_tensors(path, tensors, fingerprint(model), L.ABI_VERSION)


def load_pack(model, path: str, expect_fingerprint: Optional[str] = None) -> bool:
    """Bind the pack at ``path`` to ``model`` if it was made from the parameters the model holds now.
    Returns False (and leaves the model untouched) on a fingerprint / ABI mismatch; raises on a corrupt file."""
    from . import _lib as L
    from . import encoder_fast as EF
    from .engine import PackedWeights

    man = read_manifest(path)
    fp = expect_fingerprint if expect_fingerprint is not None else fingerprint(model)
    if man.get("fingerprint") != fp or man.get("abi") != L.ABI_VERSION:
        return False
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise L.PipsCudaError("pips_b200: load_pack needs the module on a CUDA device")
    tensors = read_tensors(path, dev, man)
    mixer = {k[len("mixer."):]: v for k, v in tensors.items() if k.startswith("mixer.")}
    packed = PackedWeights(tensors=mixer)                       # validates names / devices before anything is adopted
    convs = EF.packed_convs(model.fnet)
    for name, _ in convs:
        if f"fnet.{name}.w_hi" not in tensors or f"fnet.{name}.w_lo" not in tensors:
            raise ValueError(f"{path}: no packed filter for fnet.{name}")
    model.engine.adopt_weights(model, packed)
    for name, conv in convs:
        EF.adopt_filter(model.fnet, name, conv, tensors[f"fnet.{name}.w_hi"], tensors[f"fnet.{name}.w_lo"])
    return True
