"""CPU oracle for the Falcon layouts beyond Falcon-7B's -- TEST INFRASTRUCTURE ONLY.

Restates HF transformers 5.5.0 models/falcon/modeling_falcon.py for every rotary, bias-free, parallel-residual
layout the Server engine loads:
  FalconAttention._split_heads   fused query_key_value rows, per kv group g of G = H / Hkv query heads:
                                 [q heads gG .. gG + G - 1 | k_g | v_g]. multi_query (Falcon-7B) is one group of
                                 G = H, multi_query=False is H groups of G = 1, new_decoder_architecture
                                 (Falcon-40B) num_kv_heads groups.
  FalconDecoderLayer.forward     h + attn(ln_attn(h)) + mlp(ln_mlp(h)) with num_ln_in_parallel_attn 2, else one
                                 input_layernorm feeds both
oracle/falcon_oracle.py is the falcon-7b layout alone; with num_kv_heads 1 and one norm this module computes what it
does. Pinned against FalconForCausalLM in tests/golden/falcon_tiny_layouts.npz and falcon_40b_width.npz
(tools/make_falcon_layout_goldens.py)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle.llama_oracle import apply_rope, causal_attention, rope_cos_sin


@dataclass
class Layout:
    vocab_size: int
    hidden_size: int
    num_layers: int
    num_heads: int
    head_dim: int = 64
    num_kv_heads: int = 1
    parallel_norms: bool = False
    ffn_hidden_size: int = 0
    layer_norm_epsilon: float = 1e-5
    rope_theta: float = 10000.0

    @property
    def ffn(self):
        return self.ffn_hidden_size or 4 * self.hidden_size

    @property
    def group(self):
        return self.num_heads // self.num_kv_heads

    def as_array(self) -> np.ndarray:
        return np.array([self.vocab_size, self.hidden_size, self.num_layers, self.num_heads, self.head_dim,
                         self.num_kv_heads, int(self.parallel_norms), self.ffn])

    @classmethod
    def from_array(cls, v) -> "Layout":
        V, d, L, H, dh, Hkv, two, f = (int(x) for x in v)
        return cls(V, d, L, H, dh, Hkv, bool(two), f)

    def hf_config(self, multi_query: bool | None = None) -> dict:
        """FalconConfig keywords of this layout. One kv head without two norms is Falcon-7B's multi_query layout,
        H kv heads the multi-head one (multi_query=False) unless multi_query is given; anything else, and every
        two-norm layout, is new_decoder_architecture."""
        H, Hkv = self.num_heads, self.num_kv_heads
        c = dict(vocab_size=self.vocab_size, hidden_size=self.hidden_size, num_hidden_layers=self.num_layers,
                 num_attention_heads=H, ffn_hidden_size=self.ffn, parallel_attn=True, bias=False, alibi=False,
                 layer_norm_epsilon=self.layer_norm_epsilon, max_position_embeddings=2048, tie_word_embeddings=True,
                 hidden_dropout=0.0, attention_dropout=0.0)
        if multi_query is None:
            multi_query = Hkv == 1
        if not self.parallel_norms and ((Hkv == 1 and multi_query) or (Hkv == H and not multi_query)):
            c.update(new_decoder_architecture=False, multi_query=multi_query)
        else:
            c.update(new_decoder_architecture=True, num_kv_heads=Hkv, num_ln_in_parallel_attn=2 if self.parallel_norms
                     else 1)
        return c


def qkv_hf_to_engine(w: np.ndarray, H: int, Hkv: int, dh: int) -> np.ndarray:
    """query_key_value [(H + 2 Hkv) dh, d] in HF's grouped row order -> [Q | K | V]."""
    G = H // Hkv
    g = w.reshape(Hkv, G + 2, dh, -1)
    return np.concatenate([g[:, :G].reshape(H * dh, -1), g[:, G].reshape(Hkv * dh, -1),
                           g[:, G + 1].reshape(Hkv * dh, -1)])


def qkv_engine_to_hf(w: np.ndarray, H: int, Hkv: int, dh: int) -> np.ndarray:
    """[Q | K | V] -> HF's grouped row order (the inverse of qkv_hf_to_engine)."""
    G, d = H // Hkv, w.shape[-1]
    q = w[:H * dh].reshape(Hkv, G, dh, d)
    k = w[H * dh:(H + Hkv) * dh].reshape(Hkv, 1, dh, d)
    v = w[(H + Hkv) * dh:].reshape(Hkv, 1, dh, d)
    return np.concatenate([q, k, v], axis=1).reshape(-1, d)


def param_shapes(a: Layout):
    d, dh, H, Hkv = a.hidden_size, a.head_dim, a.num_heads, a.num_kv_heads
    s = {"transformer.word_embeddings.weight": (a.vocab_size, d)}
    for l in range(a.num_layers):
        p = f"transformer.h.{l}."
        for ln in (("ln_attn", "ln_mlp") if a.parallel_norms else ("input_layernorm",)):
            s[p + ln + ".weight"] = (d,)
            s[p + ln + ".bias"] = (d,)
        s[p + "self_attention.query_key_value.weight"] = ((H + 2 * Hkv) * dh, d)
        s[p + "self_attention.dense.weight"] = (d, H * dh)
        s[p + "mlp.dense_h_to_4h.weight"] = (a.ffn, d)
        s[p + "mlp.dense_4h_to_h.weight"] = (d, a.ffn)
    s["transformer.ln_f.weight"] = (d,)
    s["transformer.ln_f.bias"] = (d,)
    return s


def seeded_params(a: Layout, seed: int, std: float) -> Dict[str, np.ndarray]:
    """bf16-representable fp32 parameters in HF's names and layout, drawn as float32 from one generator in
    param_shapes' order: norm weights 1 + 0.1 N, biases 0.05 N, the tied embedding 0.02 N, every projection std N.
    Layer matrices with std = 1 / sqrt(fan_in) keep a wide model's activations O(1)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shape in param_shapes(a).items():
        x = rng.standard_normal(shape, dtype=np.float32)
        if name.endswith("norm.weight") or name.endswith("ln_f.weight") or name.endswith(("ln_attn.weight",
                                                                                           "ln_mlp.weight")):
            x = 1.0 + np.float32(0.1) * x
        elif name.endswith(".bias"):
            x *= np.float32(0.05)
        elif "word_embeddings" in name:
            x *= np.float32(0.02)
        else:
            x *= np.float32(std)
        out[name] = torch.from_numpy(np.ascontiguousarray(x)).bfloat16().float().numpy()
    return out


def forward(params: Dict[str, torch.Tensor], ids: torch.Tensor, a: Layout) -> torch.Tensor:
    """ids [B, S] -> logits [B, S, V] (fp32, full causal forward, no cache)."""
    B, S = ids.shape
    H, Hkv, dh, d, G = a.num_heads, a.num_kv_heads, a.head_dim, a.hidden_size, a.group
    cos, sin = rope_cos_sin(S, dh, a.rope_theta)

    def ln(x, name):
        return F.layer_norm(x, (d,), params[name + ".weight"], params[name + ".bias"], a.layer_norm_epsilon)

    h = params["transformer.word_embeddings.weight"][ids]
    for l in range(a.num_layers):
        p = f"transformer.h.{l}."
        if a.parallel_norms:
            ln_a, ln_m = ln(h, p + "ln_attn"), ln(h, p + "ln_mlp")
        else:
            ln_a = ln_m = ln(h, p + "input_layernorm")
        qkv = F.linear(ln_a, params[p + "self_attention.query_key_value.weight"]).view(B, S, Hkv, G + 2, dh)
        q = qkv[:, :, :, :G].reshape(B, S, H, dh).transpose(1, 2)
        k = qkv[:, :, :, G].transpose(1, 2)
        v = qkv[:, :, :, G + 1].transpose(1, 2)
        q, k = apply_rope(q, cos, sin), apply_rope(k, cos, sin)
        att = causal_attention(q, k, v).transpose(1, 2).reshape(B, S, H * dh)
        att = F.linear(att, params[p + "self_attention.dense.weight"])
        mlp = F.linear(F.gelu(F.linear(ln_m, params[p + "mlp.dense_h_to_4h.weight"])),
                       params[p + "mlp.dense_4h_to_h.weight"])
        h = h + att + mlp
    h = ln(h, "transformer.ln_f")
    return F.linear(h, params["transformer.word_embeddings.weight"])
