"""Deterministic synthetic RWKV weights in the reference's on-disk `.st` layout.

No RWKV checkpoints exist offline (SURVEY.md §0.4), so tests and bench.py use
random-init weights of the named architectures.  The file image written here
follows /root/reference/assets/scripts/convert_safetensors.py:22-101 exactly:
safetensors container, metadata {"format": "pt"}, every tensor float16, lower-case
keys after the `time_maa->time_mix` / `time_faaaa->time_first` renames, LoRA
matrices already transposed to [out, in].

Values come from a counter-based hash (murmur3 finaliser over the element index,
keyed by FNV-1a of the tensor name and the seed), so any element of any tensor
can be regenerated independently and bit-identically by NumPy here and by the
OpenMP C helper (csrc/synth_fill.c) that fills the 15 GB 7B image in seconds.
This module is bench/test tooling: the engine itself only ever sees `.st` bytes.
"""
from __future__ import annotations

import ctypes
import json
import os
import struct
from dataclasses import dataclass, field

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))


@dataclass
class Shape:
    version: int
    L: int
    C: int
    F: int
    V: int = 65536
    N: int = 64
    Dm: int = 32      # v6 time-mix LoRA rank
    Dd: int = 64      # v6 decay LoRA rank / v7 w rank
    Da: int = 64      # v7
    Dv: int = 32      # v7
    Dg: int = 128     # v7
    time_state: bool = False

    @property
    def H(self) -> int:
        return self.C // self.N


PRESETS = {
    # CI-sized
    "tiny6": Shape(6, 2, 256, 896, V=512, Dm=32, Dd=64),
    "tiny5": Shape(5, 2, 256, 896, V=512),
    "tiny7": Shape(7, 3, 256, 1024, V=512, Dd=32, Da=32, Dv=16, Dg=64),
    "small6": Shape(6, 4, 512, 1792, V=2048, Dm=32, Dd=64),
    "small5": Shape(5, 3, 512, 1792, V=2048),                                   # 8 heads: shards over 8 GPUs
    "small7": Shape(7, 3, 512, 2048, V=2048, Dd=32, Da=32, Dv=16, Dg=64),
    # BASELINE.json shapes (SURVEY.md §8a, last row)
    "v6-1b6": Shape(6, 24, 2048, 7168, Dm=32, Dd=64),
    "v6-3b": Shape(6, 32, 2560, 8960, Dm=32, Dd=64),
    "v6-7b": Shape(6, 32, 4096, 14336, Dm=64, Dd=128),
    "v7-2b9": Shape(7, 32, 2560, 10240, Dd=96, Da=96, Dv=64, Dg=320),
}


def _sq(c):
    return float(np.sqrt(3.0) / np.sqrt(c))    # uniform(-a,a) with std 1/sqrt(c)


def tensor_spec(s: Shape) -> list[tuple[str, tuple[int, ...], float, float]]:
    """[(name, shape, lo, hi)] in file order."""
    C, F, V, H, N, L = s.C, s.F, s.V, s.H, s.N, s.L
    out: list[tuple[str, tuple[int, ...], float, float]] = []

    def add(name, shape, lo, hi):
        out.append((name, tuple(shape), float(lo), float(hi)))

    def ln(prefix):
        add(prefix + ".weight", (C,), 0.9, 1.1)
        add(prefix + ".bias", (C,), -0.05, 0.05)

    add("emb.weight", (V, C), -1.0, 1.0)
    for l in range(L):
        b = f"blocks.{l}."
        if l == 0:
            ln(b + "ln0")
        ln(b + "ln1")
        ln(b + "ln2")
        a = b + "att."
        if s.version == 6:
            for n in ("x", "w", "k", "v", "r", "g"):
                add(a + f"time_mix_{n}", (1, 1, C), 0.0, 1.0)
            add(a + "time_mix_w1", (5 * s.Dm, C), -0.5 * _sq(C), 0.5 * _sq(C))
            add(a + "time_mix_w2", (5, C, s.Dm), -0.2 * _sq(s.Dm), 0.2 * _sq(s.Dm))
            add(a + "time_decay", (1, 1, C), -6.0, -1.0)
            add(a + "time_decay_w1", (s.Dd, C), -0.5 * _sq(C), 0.5 * _sq(C))
            add(a + "time_decay_w2", (C, s.Dd), -0.5 * _sq(s.Dd), 0.5 * _sq(s.Dd))
            add(a + "time_first", (H, N), -0.5, 0.5)
        elif s.version == 5:
            for n in ("k", "v", "r", "g"):
                add(a + f"time_mix_{n}", (1, 1, C), 0.0, 1.0)
            add(a + "time_decay", (H, N), -6.0, -1.0)
            add(a + "time_first", (H, N), -0.5, 0.5)
        else:
            for n in ("r", "w", "k", "v", "a", "g"):
                add(a + f"x_{n}", (1, 1, C), 0.0, 1.0)
            add(a + "w0", (1, 1, C), -3.0, 1.0)
            add(a + "w1", (s.Dd, C), -0.5 * _sq(C), 0.5 * _sq(C))
            add(a + "w2", (C, s.Dd), -1.0 * _sq(s.Dd), 1.0 * _sq(s.Dd))
            add(a + "a0", (1, 1, C), -1.0, 1.0)
            add(a + "a1", (s.Da, C), -0.5 * _sq(C), 0.5 * _sq(C))
            add(a + "a2", (C, s.Da), -1.0 * _sq(s.Da), 1.0 * _sq(s.Da))
            add(a + "v0", (1, 1, C), -1.0, 1.0)
            add(a + "v1", (s.Dv, C), -0.5 * _sq(C), 0.5 * _sq(C))
            add(a + "v2", (C, s.Dv), -1.0 * _sq(s.Dv), 1.0 * _sq(s.Dv))
            add(a + "g1", (s.Dg, C), -1.0 * _sq(C), 1.0 * _sq(C))
            # gate LoRA / output gains sized so that the synthetic model is as well conditioned as the RWKV-6 presets: with
            # gain 2 / 0.5 here the random RWKV-7 stack is chaotic (two f32 implementations that differ only in summation
            # order are 3e-3 apart after one token at 32 layers, f16 vs f32 operands 0.3), which
            # says nothing about an engine; trained RWKV-7 checkpoints initialise both near zero.
            add(a + "g2", (C, s.Dg), -1.0 * _sq(s.Dg), 1.0 * _sq(s.Dg))
            add(a + "k_k", (1, 1, C), 0.5, 1.2)
            add(a + "k_a", (1, 1, C), 0.0, 1.0)
            add(a + "r_k", (H, N), -0.3, 0.3)
        for n in ("receptance", "key", "value"):
            add(a + n + ".weight", (C, C), -_sq(C), _sq(C))
        if s.version != 7:
            add(a + "gate.weight", (C, C), -_sq(C), _sq(C))
        og = 0.25 if s.version == 7 else 0.5
        add(a + "output.weight", (C, C), -og * _sq(C), og * _sq(C))
        add(a + "ln_x.weight", (C,), 0.8, 1.2)
        add(a + "ln_x.bias", (C,), -0.05, 0.05)
        if s.time_state:
            add(a + "time_state", (H, N, N), -0.5, 0.5)
        f = b + "ffn."
        if s.version == 7:
            add(f + "x_k", (1, 1, C), 0.0, 1.0)
        else:
            add(f + "time_mix_k", (1, 1, C), 0.0, 1.0)
            add(f + "time_mix_r", (1, 1, C), 0.0, 1.0)
            add(f + "receptance.weight", (C, C), -_sq(C), _sq(C))
        add(f + "key.weight", (F, C), -_sq(C), _sq(C))
        add(f + "value.weight", (C, F), -0.5 * _sq(F), 0.5 * _sq(F))
    ln("ln_out")
    add("head.weight", (V, C), -2.0 * _sq(C), 2.0 * _sq(C))
    return out


def name_seed(name: str, seed: int) -> int:
    h = 0x811C9DC5
    for ch in name.encode("utf-8"):
        h = ((h ^ ch) * 0x01000193) & 0xFFFFFFFF
    return (h ^ ((seed * 0x9E3779B1) & 0xFFFFFFFF)) & 0xFFFFFFFF


def fill_numpy(dst: np.ndarray, seed32: int, lo: float, hi: float) -> None:
    """dst: flat float16 array.  Reference implementation of the fill."""
    n = dst.size
    chunk = 1 << 22
    lo32, span = np.float32(lo), np.float32(np.float32(hi) - np.float32(lo))
    for off in range(0, n, chunk):
        m = min(chunk, n - off)
        h = np.arange(off, off + m, dtype=np.uint64).astype(np.uint32)
        h = h * np.uint32(0x9E3779B1) + np.uint32(seed32)
        h ^= h >> np.uint32(16)
        h *= np.uint32(0x85EBCA6B)
        h ^= h >> np.uint32(13)
        h *= np.uint32(0xC2B2AE35)
        h ^= h >> np.uint32(16)
        u = (h >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
        dst[off:off + m] = (u * span + lo32).astype(np.float16)


_lib = None


def _fill_lib():
    global _lib
    if _lib is None:
        path = os.path.join(_HERE, "_synthfill.so")
        if os.path.exists(path):
            lib = ctypes.CDLL(path)
            lib.synth_fill_f16.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32,
                                           ctypes.c_float, ctypes.c_float]
            lib.synth_fill_f16.restype = None
            _lib = lib
        else:
            _lib = False
    return _lib


def fill(dst: np.ndarray, seed32: int, lo: float, hi: float, force_numpy: bool = False) -> None:
    lib = None if force_numpy else _fill_lib()
    if lib:
        lib.synth_fill_f16(dst.ctypes.data, dst.size, seed32, lo, hi)
    else:
        fill_numpy(dst, seed32, lo, hi)


def make_st(shape: Shape | str, seed: int = 0, force_numpy: bool = False) -> np.ndarray:
    """Build the `.st` file image (uint8 array) for `shape`."""
    if isinstance(shape, str):
        shape = PRESETS[shape]
    spec = tensor_spec(shape)
    header = {"__metadata__": {"format": "pt"}}
    off = 0
    for name, shp, _, _ in spec:
        nbytes = int(np.prod(shp)) * 2
        header[name] = {"dtype": "F16", "shape": list(shp), "data_offsets": [off, off + nbytes]}
        off += nbytes
    hjson = json.dumps(header, separators=(",", ":")).encode("utf-8")
    hjson += b" " * ((-len(hjson)) % 8)
    base = 8 + len(hjson)
    buf = np.empty(base + off, dtype=np.uint8)
    buf[:8] = np.frombuffer(struct.pack("<Q", len(hjson)), dtype=np.uint8)
    buf[8:base] = np.frombuffer(hjson, dtype=np.uint8)
    for name, shp, lo, hi in spec:
        b, e = header[name]["data_offsets"]
        view = buf[base + b:base + e].view(np.float16)
        fill(view, name_seed(name, seed), lo, hi, force_numpy)
    return buf


def pack_st(tensors: dict[str, np.ndarray]) -> np.ndarray:
    """safetensors image of a dict of arrays (F16 / F32), metadata {"format": "pt"}."""
    header = {"__metadata__": {"format": "pt"}}
    off, blobs = 0, []
    for name, a in tensors.items():
        a = np.ascontiguousarray(a)
        dt = {np.dtype(np.float16): "F16", np.dtype(np.float32): "F32"}[a.dtype]
        header[name] = {"dtype": dt, "shape": list(a.shape), "data_offsets": [off, off + a.nbytes]}
        blobs.append(a.tobytes())
        off += a.nbytes
    hjson = json.dumps(header, separators=(",", ":")).encode("utf-8")
    hjson += b" " * ((-len(hjson)) % 8)
    return np.frombuffer(struct.pack("<Q", len(hjson)) + hjson + b"".join(blobs), dtype=np.uint8).copy()


def make_lora_st(shape: Shape | str, rank: int = 8, seed: int = 1, targets=("att.key", "att.value", "att.output", "ffn.key", "ffn.value")) -> np.ndarray:
    """Synthetic LoRA file in the layout the reference's converter writes (assets/scripts/convert_safetensors.py:96-101):
    `<name>.lora.0` = lora_A transposed = [in, r], `<name>.lora.1` = lora_B = [out, r], float16, for every block and `head`."""
    if isinstance(shape, str):
        shape = PRESETS[shape]
    dims = {n: shp for n, shp, _, _ in tensor_spec(shape)}
    out = {}
    names = [f"blocks.{l}.{t}" for l in range(shape.L) for t in targets if f"blocks.{l}.{t}.weight" in dims] + ["head"]
    for base in names:
        o, i = dims[base + ".weight"]
        for idx, (rows, gain) in enumerate(((i, 1.0), (o, 1.0))):
            a = np.empty(rows * rank, np.float16)
            fill(a, name_seed(f"{base}.lora.{idx}", seed), -gain * _sq(rank) * 0.5, gain * _sq(rank) * 0.5, True)
            out[f"{base}.lora.{idx}"] = a.reshape(rows, rank)
    return pack_st(out)


def num_params(shape: Shape | str) -> int:
    if isinstance(shape, str):
        shape = PRESETS[shape]
    return sum(int(np.prod(shp)) for _, shp, _, _ in tensor_spec(shape))


def algorithmic_bytes_per_step(s: Shape | str, batch: int) -> int:
    """SURVEY.md §8(d) / BASELINE.md §3 figure: f16 weights streamed once per decode step,
    f32 state read + written once, embedding rows in, f32 logits out."""
    if isinstance(s, str):
        s = PRESETS[s]
    C, F, V, L, H, N = s.C, s.F, s.V, s.L, s.H, s.N
    if s.version == 7:
        p_layer = 4 * C * C + 2 * C * (s.Dd + s.Da + s.Dv + s.Dg) + 2 * C * F + 19 * C
    elif s.version == 6:
        p_layer = 5 * C * C + 2 * C * (5 * s.Dm + s.Dd) + 2 * C * F + C * C + 16 * C
    else:
        p_layer = 5 * C * C + 2 * C * F + C * C + 12 * C
    return 2 * (L * p_layer + V * C + 4 * C) + batch * (2 * L * (H * N * N + 2 * C) * 4 + 2 * C + 4 * V)
