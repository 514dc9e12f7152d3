"""Padding-free packing in the CPU oracle: oracle/llama_oracle.py's Llama forward and Trainer step with HF
position_ids that restart at 0 for each document of a packed row. TEST INFRASTRUCTURE, not product code.

What HF does with such position_ids (transformers 5.5, attention_mask=None and no cache):
masking_utils.find_packed_sequence_indices marks a new sequence wherever the position difference is not 1,
and the causal mask becomes block-diagonal, one block per document; RoPE rotates each token by its own
position_ids entry (modeling_llama.py LlamaRotaryEmbedding.forward). Both are restated here on top of the
oracle's ops; tests/golden/llama_tiny_packed.npz (tools/make_packed_golden.py) pins the result to the real
LlamaForCausalLM."""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import llama_oracle as O


def document_mask(positions) -> torch.Tensor:
    """positions [B, S] -> bool [B, 1, S, S]: query q sees key k iff doc_start[q] <= k <= q, where
    doc_start[q] = q - positions[q]."""
    pos = torch.as_tensor(np.asarray(positions), dtype=torch.int64)
    S = pos.shape[1]
    idx = torch.arange(S)
    start = idx[None, :] - pos                                   # [B, S]
    causal = idx[None, :] <= idx[:, None]                        # [q, k]
    return (causal[None] & (idx[None, None, :] >= start[:, :, None]))[:, None]


def rope_at(x: torch.Tensor, positions, dh: int, theta: float) -> torch.Tensor:
    """x [B, H, S, dh] rotated by positions [B, S] (the oracle's cos / sin table rows, gathered)."""
    pos = torch.as_tensor(np.asarray(positions), dtype=torch.int64)
    cos, sin = O.rope_cos_sin(int(pos.max()) + 1, dh, theta)
    cos, sin = cos[pos][:, None].to(x.dtype), sin[pos][:, None].to(x.dtype)
    return x * cos + O.rotate_half(x) * sin


def forward(params: Dict[str, torch.Tensor], ids: torch.Tensor, positions, a: O.Arch) -> torch.Tensor:
    """ids [B, S], positions [B, S] -> logits [B, S, V] (fp32): O.forward with per-document attention."""
    B, S = ids.shape
    H, Hkv, dh = a.num_heads, a.num_kv_heads, a.head_dim
    mask = document_mask(positions)
    h = F.embedding(ids, params["model.embed_tokens.weight"],
                    padding_idx=a.pad_token_id if a.pad_token_id >= 0 else None)
    for l in range(a.num_layers):
        p = f"model.layers.{l}."
        x = O.rmsnorm(h, params[p + "input_layernorm.weight"], a.rms_norm_eps)
        q = F.linear(x, params[p + "self_attn.q_proj.weight"]).view(B, S, H, dh).transpose(1, 2)
        k = F.linear(x, params[p + "self_attn.k_proj.weight"]).view(B, S, Hkv, dh).transpose(1, 2)
        v = F.linear(x, params[p + "self_attn.v_proj.weight"]).view(B, S, Hkv, dh).transpose(1, 2)
        q, k = rope_at(q, positions, dh, a.rope_theta), rope_at(k, positions, dh, a.rope_theta)
        k, v = k.repeat_interleave(H // Hkv, dim=1), v.repeat_interleave(H // Hkv, dim=1)
        s = torch.matmul(q, k.transpose(-1, -2)) * (dh ** -0.5)
        o = torch.matmul(torch.softmax(s.masked_fill(~mask, float("-inf")), dim=-1), v)
        h = h + F.linear(o.transpose(1, 2).reshape(B, S, H * dh), params[p + "self_attn.o_proj.weight"])
        x = O.rmsnorm(h, params[p + "post_attention_layernorm.weight"], a.rms_norm_eps)
        h = h + O.swiglu_mlp(x, params[p + "mlp.gate_proj.weight"], params[p + "mlp.up_proj.weight"],
                             params[p + "mlp.down_proj.weight"])
    h = O.rmsnorm(h, params["model.norm.weight"], a.rms_norm_eps)
    return F.linear(h, params["lm_head.weight"])


def forward_backward(params_np: Dict[str, np.ndarray], ids, labels, positions, a: O.Arch):
    """One Trainer forward / backward (loss = sum(nll) / num_items_in_batch): dict(loss, logits, grads)."""
    params = {k: torch.tensor(v, dtype=torch.float32, requires_grad=True) for k, v in params_np.items()}
    lab = torch.as_tensor(labels, dtype=torch.int64)
    logits = forward(params, torch.as_tensor(ids, dtype=torch.int64), positions, a)
    loss, _ = O.causal_lm_loss(logits, lab, O.trainer_num_items(lab))
    loss.backward()
    return dict(loss=float(loss.detach()), logits=logits.detach().numpy(),
                grads={k: p.grad.detach().numpy() for k, p in params.items()})
