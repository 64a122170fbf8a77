"""CPU oracle: NumPy restatement of the RWKV v5 / v6 / v7 forward pass.

TEST INFRASTRUCTURE ONLY.  Nothing on the product path (ai00_server_b200/, the
C-ABI library) may import this module; only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline leg use it, and only as the checker.

PARITY UNPINNED: the arithmetic of this path lives in the third-party crate
`web-rwkv = 0.10.18` (reference Cargo.toml:34-38, Cargo.lock:5530-5533), whose
source is not under /root/reference, and the reference ships no tests, golden
vectors or fixtures for it (SURVEY.md §0.3, §8c).  This file restates the
published RWKV algorithm that crate implements and is anchored on the
reference's own call sites and on-disk contract:

* weights: the `.st` layout written by
  /root/reference/assets/scripts/convert_safetensors.py:22-101 (lower-cased
  keys, f16, `time_maa->time_mix`, `time_faaaa->time_first`, last-two-dims
  transposes of the LoRA matrices so every matrix is [out, in]) and
  /root/reference/crates/converter/src/main.rs:8-22;
* forward contract: one f32 logits row of length `num_vocab` per requested token
  (reference crates/ai00-core/src/run.rs:675,694,730), `RnnOption::Last` vs
  `Full` (run.rs:812-822, 710-724);
* state contract: per-slot f32 tensor of web-rwkv shape [C, N+2, L, 1]
  (x-fastest) == numpy C-order (L, N+2, C) (run.rs:987, lib.rs:267-272):
  row 0 = time-mix token shift, rows 1..N = WKV state, row N+1 = channel-mix
  token shift;
* independent cross-checks committed under tests/golden/: flash-linear-attention's
  pure-torch naive recurrences (oracle/make_golden.py), its RWKV-6 / RWKV-7 layer
  forwards and its whole `RWKV6ForCausalLM` / `RWKV7ForCausalLM` models on the tiny
  synthetic weights (oracle/make_golden_fla_layers.py: logits 4e-7 from this file's).
  fla is a third-party implementation of the published architecture, not the
  reference's arithmetic, so the "unpinned" statement above stands.

Math follows BlinkDL's published inference code (rwkv pip `model.py`
att_one_v5_2/att_one_v6_0/ffn_one_v6 and RWKV-LM `rwkv_v7_demo_rnn.py`), as
restated in SURVEY.md App. A / App. B.

`act` selects the activation precision contract:
  "f32": every intermediate stays f32 (weights are f16 values up-converted).
  "f16": every vector that multiplies a weight matrix is first rounded to f16
         (the tensor-core / web-rwkv fp16 contract: f16 operands, f32 accumulate);
         everything else (LayerNorm, WKV state, residual, logits) stays f32.
"""
from __future__ import annotations

import json
import struct
from dataclasses import dataclass

import numpy as np

LN_EPS = 1e-5
GN_EPS = 64e-5          # GroupNorm over each head, eps = 1e-5 * 8^2 (v5.2 / v6 / v7)
L2_EPS = 1e-12          # torch.nn.functional.normalize default (v7 kk)
V7_DECAY_SCALE = -0.606531  # -exp(-0.5)


# --------------------------------------------------------------------------------------
# safetensors (.st) reader: header = u64 little-endian length + JSON; data follows.
# --------------------------------------------------------------------------------------
_ST_DTYPES = {"F16": np.float16, "F32": np.float32, "BF16": None}


def parse_st(buf) -> dict[str, np.ndarray]:
    """Parse a safetensors byte buffer into {name: ndarray view}."""
    mv = memoryview(buf)
    (hlen,) = struct.unpack("<Q", bytes(mv[:8]))
    header = json.loads(bytes(mv[8:8 + hlen]).decode("utf-8"))
    base = 8 + hlen
    out = {}
    for name, ent in header.items():
        if name == "__metadata__":
            continue
        dt = _ST_DTYPES[ent["dtype"]]
        if dt is None:
            raise ValueError(f"unsupported dtype {ent['dtype']} for {name}")
        b, e = ent["data_offsets"]
        arr = np.frombuffer(mv[base + b:base + e], dtype=dt).reshape(ent["shape"])
        out[name] = arr
    return out


def blend_lora(weights: dict[str, np.ndarray], lora: dict[str, np.ndarray], alpha: float) -> dict[str, np.ndarray]:
    """CPU restatement of the LoRA blend at load (reference lib.rs:466-485, `LoraBlend::full(alpha)`; tensor layout from the
    reference's converter, convert_safetensors.py:96-101): W <- f16(f32(W) + alpha * lora.1 [out, r] @ lora.0 [in, r]^T)."""
    out = dict(weights)
    for name in lora:
        if not name.endswith(".lora.0"):
            continue
        base = name[:-7]
        a, b = lora[name].astype(np.float32), lora[base + ".lora.1"].astype(np.float32)
        w = weights[base + ".weight"].astype(np.float32)
        out[base + ".weight"] = (w + np.float32(alpha) * (b @ a.T)).astype(np.float16)
    return out


@dataclass
class Info:
    version: int          # 5, 6 or 7
    num_layer: int
    num_emb: int
    num_hidden: int
    num_vocab: int
    num_head: int
    head_size: int
    time_mix_adapter: int = 0    # v6 Dm
    time_decay_adapter: int = 0  # v6 Dd / v7 Dw


def model_info(w: dict[str, np.ndarray]) -> Info:
    """Mirror of web-rwkv `Loader::info` as used at reference lib.rs:587: derive the
    model version and dimensions from tensor names/shapes only."""
    V, C = w["emb.weight"].shape
    L = 0
    while f"blocks.{L}.ln1.weight" in w:
        L += 1
    F = w["blocks.0.ffn.key.weight"].shape[0]
    if "blocks.0.att.r_k" in w:
        version = 7
        H, N = w["blocks.0.att.r_k"].shape
        return Info(7, L, C, F, V, H, N, 0, w["blocks.0.att.w1"].shape[0])
    if "blocks.0.att.time_mix_w1" in w:
        version = 6
        H, N = w["blocks.0.att.time_first"].shape
        return Info(6, L, C, F, V, H, N,
                    w["blocks.0.att.time_mix_w1"].shape[0] // 5,
                    w["blocks.0.att.time_decay_w1"].shape[0])
    if "blocks.0.att.ln_x.weight" in w and "blocks.0.att.gate.weight" in w:
        H, N = w["blocks.0.att.time_first"].shape
        return Info(5, L, C, F, V, H, N)
    raise ValueError("unsupported model (v4 and v5.0 are out of scope)")


# --------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------
def _f(a) -> np.ndarray:
    return np.asarray(a, dtype=np.float32)


def _vec(w, name) -> np.ndarray:
    return _f(w[name]).reshape(-1)


def layer_norm(x, weight, bias, eps=LN_EPS):
    x = _f(x)
    mean = x.mean(dtype=np.float32)
    var = np.mean((x - mean) ** 2, dtype=np.float32)
    return (x - mean) / np.sqrt(var + np.float32(eps)) * weight + bias


def group_norm(x, H, weight, bias, eps=GN_EPS):
    x = _f(x).reshape(H, -1)
    mean = x.mean(axis=1, keepdims=True, dtype=np.float32)
    var = np.mean((x - mean) ** 2, axis=1, keepdims=True, dtype=np.float32)
    y = (x - mean) / np.sqrt(var + np.float32(eps))
    return y.reshape(-1) * weight + bias


def sigmoid(x):
    return (1.0 / (1.0 + np.exp(-_f(x)))).astype(np.float32)


def silu(x):
    x = _f(x)
    return x * sigmoid(x)


class Oracle:
    """RWKV forward on one slot.  State layout: numpy (L, N+2, C) f32 ==
    web-rwkv [C, N+2, L, 1]."""

    def __init__(self, weights: dict[str, np.ndarray], act: str = "f16"):
        assert act in ("f16", "f32")
        self.w = weights
        self.act = act
        self.info = model_info(weights)
        self._mat_cache: dict[str, np.ndarray] = {}
        self.trace: dict | None = None      # set to {} to record per-layer intermediates of the last token

    def _tr(self, l, name, val):
        if self.trace is not None:
            self.trace[f"{l}.{name}"] = np.array(val, dtype=np.float32, copy=True)

    # ---- contract helpers -------------------------------------------------------------
    def _q(self, x):
        """Round a matmul input to f16 (saturating) in the "f16" contract."""
        x = _f(x)
        if self.act == "f16":
            return np.clip(x, -65504.0, 65504.0).astype(np.float16).astype(np.float32)
        return x

    def _mat(self, name):
        m = self._mat_cache.get(name)
        if m is None:
            m = _f(self.w[name])
            if m.size <= (1 << 24):      # keep small matrices converted
                self._mat_cache[name] = m
        return m

    def keep_all_matrices(self) -> "Oracle":
        """Convert every matrix to f32 once and keep it, large ones included: at the 7B layer shape the channel-mix
        matrices are otherwise converted again for every token, which costs far more than the products themselves.
        Costs 4 bytes per weight of host memory; the results are unchanged."""
        for name, m in self.w.items():
            if m.ndim == 2 and name != "emb.weight":
                self._mat_cache[name] = _f(m)
        return self

    def _mv(self, name, x):
        """y = W @ q(x); W stored [out, in]."""
        return self._mat(name) @ self._q(x)

    def state_init(self) -> np.ndarray:
        """`State::init()` (reference run.rs:477): zeros unless the model carries
        `blocks.{l}.att.time_state` [H, N, N] (state tuning, stored transposed by the
        converter: convert_safetensors.py:101)."""
        i = self.info
        st = np.zeros((i.num_layer, i.head_size + 2, i.num_emb), dtype=np.float32)
        for l in range(i.num_layer):
            key = f"blocks.{l}.att.time_state"
            if key in self.w:
                ts = _f(self.w[key])                      # [H, N(i), N(j)] after converter transpose
                # row 1+i, col h*N+j  <->  S[h][i][j]
                st[l, 1:1 + i.head_size, :] = ts.transpose(1, 0, 2).reshape(i.head_size, i.num_emb)
        return st

    # ---- forward ----------------------------------------------------------------------
    def run(self, tokens, state: np.ndarray, full: bool = False):
        """Feed `tokens` through the model on one slot.  Returns (logits, state):
        logits is [T, V] if `full` else [1, V] (last token); state is updated in a copy."""
        state = state.copy()
        outs = []
        T = len(tokens)
        for t, tok in enumerate(tokens):
            x = self._token(int(tok), state)
            if full or t == T - 1:
                outs.append(self._head(x))
        logits = np.stack(outs, 0) if outs else np.zeros((0, self.info.num_vocab), np.float32)
        return logits, state

    def hidden(self, tokens, state):
        """Residual stream after the last layer for each token (debug aid)."""
        state = state.copy()
        return np.stack([self._token(int(t), state) for t in tokens], 0), state

    def _head(self, x):
        w = self.w
        xo = layer_norm(x, _vec(w, "ln_out.weight"), _vec(w, "ln_out.bias"))
        return self._mv("head.weight", xo).astype(np.float32)

    def _token(self, tok, state):
        w, i = self.w, self.info
        x = layer_norm(_f(w["emb.weight"][tok]), _vec(w, "blocks.0.ln0.weight"), _vec(w, "blocks.0.ln0.bias"))
        v_first = None
        for l in range(i.num_layer):
            if i.version == 7:
                x, v_first = self._att_v7(l, x, state[l], v_first)
                x = self._ffn_v7(l, x, state[l])
            else:
                x = self._att_v56(l, x, state[l])
                x = self._ffn_v56(l, x, state[l])
        return x

    # ---- v5 / v6 ---------------------------------------------------------------------
    def _att_v56(self, l, x, st):
        w, i = self.w, self.info
        p = f"blocks.{l}.att."
        H, N, C = i.num_head, i.head_size, i.num_emb
        xx = layer_norm(x, _vec(w, f"blocks.{l}.ln1.weight"), _vec(w, f"blocks.{l}.ln1.bias"))
        prev = st[0]
        sx = prev - xx
        if i.version == 6:
            xxx = xx + sx * _vec(w, p + "time_mix_x")
            Dm = i.time_mix_adapter
            m = np.tanh(self._mv(p + "time_mix_w1", xxx)).reshape(5, Dm)      # w1: [5*Dm, C]
            w2 = self._mat(p + "time_mix_w2")                                   # [5, C, Dm]
            mm = np.stack([w2[j] @ self._q(m[j]) for j in range(5)], 0)         # order w,k,v,r,g
            xw = xx + sx * (_vec(w, p + "time_mix_w") + mm[0])
            xk = xx + sx * (_vec(w, p + "time_mix_k") + mm[1])
            xv = xx + sx * (_vec(w, p + "time_mix_v") + mm[2])
            xr = xx + sx * (_vec(w, p + "time_mix_r") + mm[3])
            xg = xx + sx * (_vec(w, p + "time_mix_g") + mm[4])
            d = np.tanh(self._mv(p + "time_decay_w1", xw))                      # [Dd]
            wd = _vec(w, p + "time_decay") + self._mv(p + "time_decay_w2", d)   # [C]
        else:
            # v5.1/5.2: x_* = xx*mix + prev*(1-mix)  (rwkv pip att_one_v5_2)
            def mix(name):
                mu = _vec(w, p + name)
                return xx * mu + prev * (1.0 - mu)
            xk, xv, xr, xg = mix("time_mix_k"), mix("time_mix_v"), mix("time_mix_r"), mix("time_mix_g")
            wd = _vec(w, p + "time_decay")                                      # [H,N] flattened
        decay = np.exp(-np.exp(_f(wd))).astype(np.float32)                      # (0,1)
        r = self._mv(p + "receptance.weight", xr)
        k = self._mv(p + "key.weight", xk)
        v = self._mv(p + "value.weight", xv)
        g = silu(self._mv(p + "gate.weight", xg))
        u = _vec(w, p + "time_first")
        for nm, val in (("x_in1", x), ("xx1", xx), ("sx1", sx), ("xk", xk), ("xv", xv), ("xr", xr), ("xg", xg),
                        ("r", r), ("k", k), ("v", v), ("g", g), ("w", decay)):
            self._tr(l, nm, val)
        S = st[1:1 + N].reshape(N, H, N).transpose(1, 0, 2)                     # S[h][i][j] (view)
        out = np.empty(C, np.float32)
        for h in range(H):
            sl = slice(h * N, (h + 1) * N)
            a = np.outer(k[sl], v[sl])                                          # a[i,j] = k[i] v[j]
            out[sl] = r[sl] @ (u[sl, None] * a + S[h])
            S[h] = a + decay[sl, None] * S[h]                                   # writes through to st
        out = group_norm(out, H, _vec(w, p + "ln_x.weight"), _vec(w, p + "ln_x.bias")) * g
        st[0] = xx
        att = self._mv(p + "output.weight", out)
        self._tr(l, "wkv_out", out)
        self._tr(l, "part_att", att)
        return x + att

    def _ffn_v56(self, l, x, st):
        w, i = self.w, self.info
        p = f"blocks.{l}.ffn."
        N = i.head_size
        xx = layer_norm(x, _vec(w, f"blocks.{l}.ln2.weight"), _vec(w, f"blocks.{l}.ln2.bias"))
        prev = st[N + 1]
        if i.version == 6:
            sx = prev - xx
            xk = xx + sx * _vec(w, p + "time_mix_k")
            xr = xx + sx * _vec(w, p + "time_mix_r")
        else:
            mk, mr = _vec(w, p + "time_mix_k"), _vec(w, p + "time_mix_r")
            xk = xx * mk + prev * (1.0 - mk)
            xr = xx * mr + prev * (1.0 - mr)
        rr = sigmoid(self._mv(p + "receptance.weight", xr))
        kk = np.maximum(self._mv(p + "key.weight", xk), 0.0) ** 2
        st[N + 1] = xx
        pf = self._mv(p + "value.weight", kk)
        for nm, val in (("x_in2", x), ("xx2", xx), ("fxk", xk), ("fxr", xr), ("rr", rr), ("kk", kk), ("part_ffn", pf)):
            self._tr(l, nm, val)
        return x + rr * pf

    # ---- v7 -------------------------------------------------------------------------
    def _att_v7(self, l, x, st, v_first):
        w, i = self.w, self.info
        p = f"blocks.{l}.att."
        H, N, C = i.num_head, i.head_size, i.num_emb
        xx = layer_norm(x, _vec(w, f"blocks.{l}.ln1.weight"), _vec(w, f"blocks.{l}.ln1.bias"))
        sx = st[0] - xx
        xr = xx + sx * _vec(w, p + "x_r")
        xw = xx + sx * _vec(w, p + "x_w")
        xk = xx + sx * _vec(w, p + "x_k")
        xv = xx + sx * _vec(w, p + "x_v")
        xa = xx + sx * _vec(w, p + "x_a")
        xg = xx + sx * _vec(w, p + "x_g")
        r = self._mv(p + "receptance.weight", xr)
        k = self._mv(p + "key.weight", xk)
        v = self._mv(p + "value.weight", xv)
        wl = _vec(w, p + "w0") + self._mv(p + "w2", np.tanh(self._mv(p + "w1", xw)))
        decay = np.exp(np.float32(V7_DECAY_SCALE) * sigmoid(wl)).astype(np.float32)
        a = sigmoid(_vec(w, p + "a0") + self._mv(p + "a2", self._mv(p + "a1", xa)))
        g = self._mv(p + "g2", sigmoid(self._mv(p + "g1", xg)))
        kk = (k * _vec(w, p + "k_k")).reshape(H, N)
        kk = (kk / np.maximum(np.sqrt((kk * kk).sum(axis=1, keepdims=True, dtype=np.float32)), L2_EPS)).reshape(C)
        k = k * (1.0 + (a - 1.0) * _vec(w, p + "k_a"))
        if l == 0:
            v_first = v
        else:
            nu = sigmoid(_vec(w, p + "v0") + self._mv(p + "v2", self._mv(p + "v1", xv)))
            v = v + (v_first - v) * nu
        S = st[1:1 + N].reshape(N, H, N).transpose(1, 0, 2)                     # S[h][i(value)][j(key)]
        out = np.empty(C, np.float32)
        for h in range(H):
            sl = slice(h * N, (h + 1) * N)
            sa = S[h] @ (-kk[sl])                                               # [N] over value index
            S[h] = S[h] * decay[sl][None, :] + np.outer(sa, kk[sl] * a[sl]) + np.outer(v[sl], k[sl])
            out[sl] = S[h] @ r[sl]
        out = group_norm(out, H, _vec(w, p + "ln_x.weight"), _vec(w, p + "ln_x.bias"))
        bonus = (r * k * _vec(w, p + "r_k")).reshape(H, N).sum(axis=1, keepdims=True, dtype=np.float32)
        out = out + (bonus * v.reshape(H, N)).reshape(C)
        st[0] = xx
        att = self._mv(p + "output.weight", out * g)
        for nm, val in (("x_in1", x), ("xx1", xx), ("xr", xr), ("xw", xw), ("xk", xk), ("xv", xv), ("xa", xa), ("xg", xg),
                        ("r", r), ("w", decay), ("a", a), ("g", g), ("wkv_out", out * g), ("part_att", att)):
            self._tr(l, nm, val)
        return x + att, v_first

    def _ffn_v7(self, l, x, st):
        w, i = self.w, self.info
        p = f"blocks.{l}.ffn."
        N = i.head_size
        xx = layer_norm(x, _vec(w, f"blocks.{l}.ln2.weight"), _vec(w, f"blocks.{l}.ln2.bias"))
        xk = xx + (st[N + 1] - xx) * _vec(w, p + "x_k")
        kk = np.maximum(self._mv(p + "key.weight", xk), 0.0) ** 2
        st[N + 1] = xx
        pf = self._mv(p + "value.weight", kk)
        for nm, val in (("x_in2", x), ("xx2", xx), ("fxk", xk), ("kk", kk), ("part_ffn", pf)):
            self._tr(l, nm, val)
        return x + pf


def softmax_rows(x: np.ndarray) -> np.ndarray:
    """`web_rwkv::runtime::softmax::softmax` contract (reference run.rs:1179): row-wise
    softmax over the vocabulary, f32."""
    x = _f(x)
    m = x.max(axis=-1, keepdims=True)
    e = np.exp(x - m)
    return (e / e.sum(axis=-1, keepdims=True, dtype=np.float32)).astype(np.float32)


# --------------------------------------------------------------------------------------
# stand-alone WKV recurrences (used to pin the oracle against fla's naive ops)
# --------------------------------------------------------------------------------------
def wkv6_seq(r, k, v, w_decay, u, S0):
    """r,k,v,w_decay: [T,H,N] (w_decay already exp(-exp(.))), u: [H,N], S0: [H,N,N] (i=key,j=value).
    Returns out [T,H,N], S [H,N,N]."""
    T, H, N = r.shape
    S = _f(S0).copy()
    out = np.zeros((T, H, N), np.float32)
    for t in range(T):
        for h in range(H):
            a = np.outer(k[t, h], v[t, h])
            out[t, h] = r[t, h] @ (u[h][:, None] * a + S[h])
            S[h] = a + w_decay[t, h][:, None] * S[h]
    return out, S


def wkv7_seq(r, k, v, w_decay, kk, a, S0):
    """Delta-rule recurrence.  r,k,v,w_decay,kk,a: [T,H,N]; S0: [H,N(value),N(key)]."""
    T, H, N = r.shape
    S = _f(S0).copy()
    out = np.zeros((T, H, N), np.float32)
    for t in range(T):
        for h in range(H):
            sa = S[h] @ (-kk[t, h])
            S[h] = S[h] * w_decay[t, h][None, :] + np.outer(sa, kk[t, h] * a[t, h]) + np.outer(v[t, h], k[t, h])
            out[t, h] = S[h] @ r[t, h]
    return out, S
