"""Host side of the Server decode path: `InferEngine` wraps the b200w_infer_* C ABI; `Generator`
turns it into a continuously-batched greedy generator (one cache slot per request, one token per
slot per step — prompt ingestion and generation are the same step)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Tuple

import numpy as np

from . import _lib
from ._lib import B200WError, InferArch as _CArch
from .engine import Engine

FAMILY = {"llama": 0, "falcon": 1, "opt": 2}


@dataclass
class ServeArch:
    family: str
    vocab_size: int
    hidden_size: int
    intermediate_size: int
    num_layers: int
    num_heads: int
    num_kv_heads: int
    head_dim: int
    max_ctx: int = 2048
    norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    tie_embeddings: bool = False
    max_positions: int = 0        # OPT: max_position_embeddings (learned table, +2 rows)

    @classmethod
    def falcon_7b(cls, max_ctx: int = 2048) -> "ServeArch":
        return cls("falcon", 65024, 4544, 18176, 32, 71, 1, 64, max_ctx, 1e-5, 10000.0, True)

    @classmethod
    def from_hf_config(cls, cfg: dict, max_ctx: Optional[int] = None) -> "ServeArch":
        mt = cfg.get("model_type")
        if mt == "falcon":
            if cfg.get("alibi") or cfg.get("bias") or cfg.get("new_decoder_architecture") or not cfg.get(
                    "parallel_attn", True):
                raise ValueError("only the falcon-7b layout (rotary, bias-free, parallel_attn, 1 layernorm) is supported")
            heads = cfg["num_attention_heads"]
            d = cfg["hidden_size"]
            kv = 1 if cfg.get("multi_query", True) else heads
            return cls("falcon", cfg["vocab_size"], d, cfg.get("ffn_hidden_size") or 4 * d,
                       cfg["num_hidden_layers"], heads, kv, d // heads,
                       max_ctx or min(2048, cfg.get("max_position_embeddings", 2048)),
                       cfg.get("layer_norm_epsilon", 1e-5), float(cfg.get("rope_theta", 10000.0)),
                       bool(cfg.get("tie_word_embeddings", True)))
        if mt == "llama":
            heads = cfg["num_attention_heads"]
            rope = cfg.get("rope_parameters") or {}
            from .engine import LlamaArch
            LlamaArch.from_hf_config(cfg)              # same rejections as the trainer (rope scaling, biases, ...)
            return cls("llama", cfg["vocab_size"], cfg["hidden_size"], cfg["intermediate_size"],
                       cfg["num_hidden_layers"], heads, cfg.get("num_key_value_heads") or heads,
                       cfg.get("head_dim") or cfg["hidden_size"] // heads,
                       max_ctx or min(4096, cfg.get("max_position_embeddings", 4096)),
                       cfg.get("rms_norm_eps", 1e-6), float(cfg.get("rope_theta") or rope.get("rope_theta") or 1e4),
                       bool(cfg.get("tie_word_embeddings", False)))
        if mt == "opt":
            from .engine import OptArch
            o = OptArch.from_hf_config(cfg)            # rejects the variants that are not built
            ctx = min(max_ctx or o.max_positions, o.max_positions)
            return cls("opt", o.vocab_size, o.hidden_size, o.intermediate_size, o.num_layers, o.num_heads,
                       o.num_heads, o.head_dim, ctx, o.layer_norm_eps, 10000.0, True, o.max_positions)
        raise ValueError(f"unsupported model_type {mt!r} (falcon, llama, opt)")


KV_PAGE = 128   # positions per page of the paged KV cache (one key block of the decode attention)


def kv_page_bytes(arch: ServeArch) -> int:
    """Device bytes of one page: K and V, every layer, 128 positions of num_kv_heads * head_dim bf16."""
    return 2 * arch.num_layers * KV_PAGE * arch.num_kv_heads * arch.head_dim * 2


def pages_for(n_tokens: int) -> int:
    return (n_tokens + KV_PAGE - 1) // KV_PAGE


class CacheFull(RuntimeError):
    """The paged KV cache has too few free pages for a request right now (it fits the pool once others end)."""


class InferEngine(Engine):
    kv_pages: Optional[int] = None   # pages in the pool; None: the contiguous max_batch x max_ctx cache

    def init_infer(self, arch: ServeArch, max_batch: int = 32, kv_pages: Optional[int] = None,
                   prefill_tokens: Optional[int] = None):
        """kv_pages: serve from a pool of that many 128-position pages shared by all slots (b200w_infer_init_paged)
        instead of reserving max_ctx positions per slot; arch.max_ctx is then the longest single request.
        prefill_tokens: the most tokens (n_seqs * padded length) one prefill call takes in paged mode."""
        ca = _CArch(FAMILY[arch.family], arch.vocab_size, arch.hidden_size, arch.intermediate_size,
                    arch.num_layers, arch.num_heads, arch.num_kv_heads, arch.head_dim, arch.max_ctx,
                    arch.norm_eps, arch.rope_theta, 1 if arch.tie_embeddings else 0, arch.max_positions)
        if kv_pages is None:
            self._check(self._lib.b200w_infer_init(self._h, C.byref(ca), max_batch))
        else:
            if prefill_tokens is None:
                prefill_tokens = max(16384, pages_for(arch.max_ctx) * KV_PAGE)
            self._check(self._lib.b200w_infer_init_paged(self._h, C.byref(ca), max_batch, kv_pages, prefill_tokens))
            self.kv_pages, self.prefill_tokens = kv_pages, prefill_tokens
        self.serve_arch, self.max_batch = arch, max_batch

    def reserve(self, slot: int, n_tokens: int):
        """Give `slot` the pages for positions [0, n_tokens) (releasing what it held); B200WError with status
        B200W_ERR_OOM (-5) when too few pages are free."""
        self._check(self._lib.b200w_infer_reserve(self._h, slot, n_tokens))

    def release(self, slot: int):
        self._check(self._lib.b200w_infer_release(self._h, slot))

    def kv_pages_free(self) -> int:
        free = C.c_int64()
        self._check(self._lib.b200w_infer_kv_pages(self._h, None, C.byref(free)))
        return free.value

    def slot_pages(self, slot: int) -> List[int]:
        out = np.empty(self.kv_pages, dtype=np.int32)
        n = self._lib.b200w_infer_slot_pages(self._h, slot, out.ctypes.data, out.size)
        if n < 0:
            self._check(n)
        return out[:n].tolist()

    def infer_params(self) -> Iterable[Tuple[str, Tuple[int, ...]]]:
        n = C.c_int64()
        self._check(self._lib.b200w_infer_param_count(self._h, C.byref(n), None))
        buf = C.create_string_buffer(256)
        r, c = C.c_int64(), C.c_int64()
        for i in range(n.value):
            self._check(self._lib.b200w_infer_param_info(self._h, i, buf, 256, C.byref(r), C.byref(c)))
            name = buf.value.decode()
            one_d = r.value == 1      # norm weights, LayerNorm parameters, biases
            yield name, ((c.value,) if one_d else (r.value, c.value))

    def infer_load_tensor(self, name: str, arr: np.ndarray):
        arr = np.ascontiguousarray(arr)
        dt = _lib.BF16 if arr.dtype == np.uint16 else _lib.F32
        if dt == _lib.F32:
            arr = arr.astype(np.float32, copy=False)
        self._check(self._lib.b200w_infer_load_tensor(self._h, name.encode(), arr.ctypes.data, dt, arr.size))

    def infer_load_state_dict(self, sd: Dict[str, np.ndarray]):
        for name, _ in self.infer_params():
            if name not in sd:
                raise KeyError(f"state dict lacks {name}")
            self.infer_load_tensor(name, sd[name])

    def infer_init_random(self, seed: int = 0, std: float = 0.02):
        self._check(self._lib.b200w_infer_init_random(self._h, seed, std))

    def step(self, tokens, positions, slots, want_logits: bool = False):
        tok = np.ascontiguousarray(tokens, dtype=np.int32)
        pos = np.ascontiguousarray(positions, dtype=np.int32)
        sl = np.ascontiguousarray(slots, dtype=np.int32)
        n = tok.size
        nxt = np.empty(n, dtype=np.int32)
        logits = np.empty((n, self.serve_arch.vocab_size), dtype=np.float32) if want_logits else None
        self._check(self._lib.b200w_infer_step(self._h, tok.ctypes.data, pos.ctypes.data, sl.ctypes.data, n,
                                               nxt.ctypes.data, logits.ctypes.data if want_logits else None))
        return nxt, logits


    def prefill(self, prompts: List[List[int]], slots: List[int], want_logits: bool = False):
        """One pass over whole prompts (b200w_infer_prefill): K/V of every prompt position goes to its
        cache slot; returns (greedy token after each prompt, logits [n, V] or None)."""
        n = len(prompts)
        longest = max(len(p) for p in prompts)
        S = ((longest + 127) // 128) * 128
        tok = np.zeros((n, S), dtype=np.int32)
        for i, p in enumerate(prompts):
            tok[i, :len(p)] = p
        lens = np.array([len(p) for p in prompts], dtype=np.int32)
        sl = np.ascontiguousarray(slots, dtype=np.int32)
        nxt = np.empty(n, dtype=np.int32)
        logits = np.empty((n, self.serve_arch.vocab_size), dtype=np.float32) if want_logits else None
        self._check(self._lib.b200w_infer_prefill(self._h, tok.ctypes.data, lens.ctypes.data, sl.ctypes.data, n, S,
                                                  nxt.ctypes.data, logits.ctypes.data if want_logits else None))
        return nxt, logits


def sample_token(logits: np.ndarray, temperature: float, top_p: float, rng: np.random.Generator) -> int:
    """Host-side sampling of one row (the engine itself is greedy): softmax(logits / T) restricted to the
    smallest prefix of the sorted distribution whose mass reaches top_p (nucleus sampling)."""
    z = logits.astype(np.float64) / max(temperature, 1e-6)
    z -= z.max()
    p = np.exp(z)
    p /= p.sum()
    if top_p < 1.0:
        order = np.argsort(-p)
        keep = np.searchsorted(np.cumsum(p[order]), top_p) + 1
        mask = np.zeros_like(p)
        mask[order[:keep]] = 1.0
        p = p * mask
        p /= p.sum()
    return int(rng.choice(len(p), p=p))


@dataclass
class _Req:
    prompt: List[int]
    max_tokens: int
    out: List[int]
    fed: int = 0          # tokens fed so far (prompt + generated)
    slot: int = -1
    done: bool = False
    temperature: float = 0.0
    top_p: float = 1.0
    rng: Optional[np.random.Generator] = None

    @property
    def greedy(self) -> bool:
        return self.temperature <= 0.0


class Generator:
    """Continuous batching over the engine's cache slots. A request's prompt is ingested in one prefill
    pass when it is admitted (engines without `prefill`, i.e. the CPU test stubs, feed it one token per
    step through the decode path); from then on every active request advances one token per step."""

    def __init__(self, engine: InferEngine, eos_id: Optional[int] = None, use_prefill: bool = True):
        self.e, self.eos = engine, eos_id
        self.free = list(range(engine.max_batch))
        self.active: List[_Req] = []
        self.use_prefill = use_prefill and hasattr(engine, "prefill")
        self._deferred: List[_Req] = []
        # paged KV cache: a request holds pages for len(prompt) + max_tokens positions from admission to its end
        self.kv_pages = getattr(engine, "kv_pages", None)

    def add(self, prompt: List[int], max_tokens: int, temperature: float = 0.0, top_p: float = 1.0,
            seed: Optional[int] = None, defer_prefill: bool = False) -> _Req:
        """defer_prefill: only register the request; flush_prefill() then ingests every deferred prompt of the
        same padded length in ONE prefill call (what the scheduler does when several requests are admitted in
        the same round)."""
        if not prompt:
            raise ValueError("empty prompt")
        V = self.e.serve_arch.vocab_size
        bad = [t for t in prompt if not 0 <= int(t) < V]
        if bad:   # a per-request error (HTTP 400), never an engine failure that would take the server down
            raise ValueError(f"token id {bad[0]} outside the model vocabulary ({V})")
        if len(prompt) + max_tokens > self.e.serve_arch.max_ctx:
            raise ValueError("prompt + max_tokens exceeds the KV cache length")
        if self.kv_pages is not None and pages_for(len(prompt) + max_tokens) > self.kv_pages:
            raise ValueError(f"prompt + max_tokens needs {pages_for(len(prompt) + max_tokens)} KV pages, "
                             f"the cache holds {self.kv_pages}")
        if not self.free:
            raise RuntimeError("no free cache slot")
        if self.kv_pages is not None:
            if pages_for(len(prompt) + max_tokens) > self.e.kv_pages_free():
                raise CacheFull("KV cache full: too few free pages for this request now")
            self.e.reserve(self.free[-1], len(prompt) + max_tokens)
        r = _Req(list(prompt), max_tokens, [], 0, self.free.pop(), False, float(temperature), float(top_p),
                 np.random.default_rng(seed) if temperature > 0 else None)
        self.active.append(r)
        if self.use_prefill and len(prompt) > 1:
            self._deferred.append(r)
            if not defer_prefill:
                self.flush_prefill()
        return r

    def flush_prefill(self):
        """One prefill call per group of deferred prompts that pad to the same multiple of 128 tokens."""
        pend, self._deferred = self._deferred, []
        groups: Dict[int, List[_Req]] = {}
        for r in pend:
            groups.setdefault((len(r.prompt) + 127) // 128, []).append(r)
        calls = []
        for blocks, rs in sorted(groups.items()):
            # paged: a call's n_seqs * padded_len stays within the prefill workspace the engine allocated
            per_call = max(1, self.e.prefill_tokens // (blocks * 128)) if self.kv_pages is not None else len(rs)
            calls += [rs[i:i + per_call] for i in range(0, len(rs), per_call)]
        for rs in calls:
            need_logits = any(not r.greedy for r in rs)
            nxt, lg = self.e.prefill([r.prompt for r in rs], [r.slot for r in rs], want_logits=need_logits)
            if need_logits and lg is None:
                raise ValueError("sampling (temperature > 0) needs an engine that returns logits")
            for i, r in enumerate(rs):
                r.fed = len(r.prompt)
                self._emit(r, int(nxt[i]) if r.greedy else sample_token(lg[i], r.temperature, r.top_p, r.rng))
        self._retire()

    def _emit(self, r: _Req, t: int):
        r.out.append(t)
        if len(r.out) >= r.max_tokens or (self.eos is not None and t == self.eos):
            r.done = True

    def cancel(self, r: _Req):
        """Stop a request now (stop string hit, client gone): its slot is free for the next admission."""
        if r in self.active:
            r.done = True
            self.active.remove(r)
            self._free_slot(r)

    def _free_slot(self, r: _Req):
        self.free.append(r.slot)
        if self.kv_pages is not None:
            self.e.release(r.slot)

    def _retire(self):
        for r in [r for r in self.active if r.done]:
            self.active.remove(r)
            self._free_slot(r)

    def step(self):
        """One engine step for every active request."""
        if not self.active:
            return
        toks = [(r.prompt[r.fed] if r.fed < len(r.prompt) else r.out[-1]) for r in self.active]
        need_logits = any(not r.greedy for r in self.active)
        nxt, lg = self.e.step(toks, [r.fed for r in self.active], [r.slot for r in self.active],
                              want_logits=need_logits)
        if need_logits and lg is None:
            raise ValueError("sampling (temperature > 0) needs an engine that returns logits")
        for i, (r, t) in enumerate(zip(self.active, nxt)):
            r.fed += 1
            if r.fed >= len(r.prompt):        # the token just fed was the last known one
                self._emit(r, int(t) if r.greedy else sample_token(lg[i], r.temperature, r.top_p, r.rng))
        self._retire()

    def generate(self, prompts: List[List[int]], max_tokens: int) -> List[List[int]]:
        reqs = [self.add(p, max_tokens) for p in prompts]
        while self.active:
            self.step()
        return [r.out for r in reqs]
