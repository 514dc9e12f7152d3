"""The fp32 oracles with the fp8 KV cache's quantization: what the engine computes when its K/V come from an e4m3
pool (DESIGN §3.5). Query rows from `row0` on attend over K/V quantized per (position, head) from their bf16-rounded
values; earlier rows over the activations, as a cold prefill does. Test-only, next to the oracles it extends."""
import torch
import torch.nn.functional as F

from oracle import llama_oracle as LO
from oracle import opt_oracle as OO

_CAUSAL_ATTENTION = LO.causal_attention   # the unpatched one, whatever patch() has done since


def quantize(x):
    """x [..., dh] (bf16-representable) -> (e4m3 bytes uint8 [..., dh], fp32 scales [...]) as the engine stores them:
    scale = amax / 448, q = e4m3(x / scale), all zero where amax is 0."""
    x = x.float()
    amax = x.abs().amax(-1)
    scale = amax / 448
    q = (x / scale[..., None]).to(torch.float8_e4m3fn).view(torch.uint8)
    return torch.where(amax[..., None] > 0, q, torch.zeros_like(q)), scale


def dequantize(q, scale):
    return q.view(torch.float8_e4m3fn).float() * scale[..., None]


def fake_quant(x):
    """x [..., dh] -> the values an fp8 cache returns for it"""
    return dequantize(*quantize(x.bfloat16()))


def llama_attention(row0):
    """replacement for LO.causal_attention (also the Falcon oracle's)"""
    plain = _CAUSAL_ATTENTION

    def attn(q, k, v):
        out = plain(q, k, v)
        out[:, :, row0:] = plain(q, fake_quant(k), fake_quant(v))[:, :, row0:]
        return out
    return attn


def opt_attention(row0):
    """replacement for OO.attention: OPT's projections with biases, then the same split of the query rows"""

    def attention(x, P, pre, a):
        B, S, d = x.shape
        H, dh = a.num_heads, a.head_dim
        q = F.linear(x, P[pre + "q_proj.weight"], P[pre + "q_proj.bias"]) * dh ** -0.5
        k = F.linear(x, P[pre + "k_proj.weight"], P[pre + "k_proj.bias"])
        v = F.linear(x, P[pre + "v_proj.weight"], P[pre + "v_proj.bias"])
        q, k, v = (t.view(B, S, H, dh).transpose(1, 2) for t in (q, k, v))
        mask = torch.ones(S, S, dtype=torch.bool, device=x.device).tril()

        def core(k, v):
            s = (q @ k.transpose(-1, -2)).masked_fill(~mask, float("-inf"))
            return torch.softmax(s.float(), dim=-1).to(v.dtype) @ v
        o = core(k, v)
        o[:, :, row0:] = core(fake_quant(k), fake_quant(v))[:, :, row0:]
        o = o.transpose(1, 2).reshape(B, S, d)
        return F.linear(o, P[pre + "out_proj.weight"], P[pre + "out_proj.bias"])
    return attention


def patch(monkeypatch, module, row0):
    """make `module`'s forward (LO, FO or OO) read quantized K/V from query row row0 on"""
    if module is OO:
        monkeypatch.setattr(OO, "attention", opt_attention(row0))
    else:
        monkeypatch.setattr(module, "causal_attention", llama_attention(row0))
