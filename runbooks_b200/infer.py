"""Host side of the Server decode path: `InferEngine` wraps the b200w_infer_* C ABI; `Generator`
turns it into a continuously-batched generator (one cache slot per request, one token per slot per step —
prompt ingestion and generation are the same step), greedy or sampled on the device (`InferEngine.sample`), with
penalties and logit bias applied on the device before the draw (`InferEngine.sample_penalized`)."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
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
    parallel_norms: bool = False  # Falcon: ln_attn + ln_mlp per layer instead of one input_layernorm

    @classmethod
    def falcon_7b(cls, max_ctx: int = 2048) -> "ServeArch":
        return cls("falcon", 65024, 4544, 18176, 32, 71, 1, 64, max_ctx, 1e-5, 10000.0, True)

    @classmethod
    def from_hf_config(cls, cfg: dict, max_ctx: Optional[int] = None) -> "ServeArch":
        mt = cfg.get("model_type")
        if mt == "falcon":
            if cfg.get("alibi") or cfg.get("bias") or not cfg.get("parallel_attn", True):
                raise ValueError("only rotary, bias-free Falcon layouts with parallel_attn are supported")
            heads = cfg["num_attention_heads"]
            d = cfg["hidden_size"]
            if "n_head_kv" in cfg and "num_kv_heads" not in cfg:   # transformers reads no such key: it would be lost
                raise ValueError("the config names its kv heads n_head_kv; FalconConfig reads num_kv_heads")
            n_ln = cfg.get("num_ln_in_parallel_attn")
            if n_ln not in (None, 1, 2):
                raise ValueError(f"num_ln_in_parallel_attn must be 1 or 2, got {n_ln!r}")
            # the kv heads as FalconAttention counts them; the grouped row order of query_key_value follows from them
            # (the engine loads it for every layout, b200w.h)
            if cfg.get("new_decoder_architecture"):
                kv = cfg.get("num_kv_heads") or heads
                two = (n_ln or 2) == 2
            else:
                if n_ln == 2:
                    raise ValueError("num_ln_in_parallel_attn 2 needs new_decoder_architecture")
                kv, two = (1 if cfg.get("multi_query", True) else heads), False
            if heads % kv:
                raise ValueError(f"num_attention_heads {heads} is not a multiple of num_kv_heads {kv}")
            return cls("falcon", cfg["vocab_size"], d, cfg.get("ffn_hidden_size") or 4 * d,
                       cfg["num_hidden_layers"], heads, kv, d // heads,
                       max_ctx or min(2048, cfg.get("max_position_embeddings", 2048)),
                       cfg.get("layer_norm_epsilon", 1e-5), float(cfg.get("rope_theta", 10000.0)),
                       bool(cfg.get("tie_word_embeddings", True)), parallel_norms=two)
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


KV_DTYPES = {"bf16": 0, "fp8": 1}   # b200w_kv_dtype: bf16, or e4m3 with one fp32 scale per (position, kv head)
# B200W_WEIGHTS_*: int4 / int8 = group-quantized projections (DESIGN §3.5)
WEIGHT_DTYPES = {"bf16": 0, "int4": 1, "int8": 2}


def kv_page_bytes(arch: ServeArch, kv_dtype: str = "bf16") -> int:
    """Device bytes of one page: K and V, every layer, 128 positions of num_kv_heads * head_dim bf16 values, or of
    as many e4m3 bytes plus one fp32 scale per kv head (kv_dtype "fp8")."""
    if kv_dtype not in KV_DTYPES:
        raise ValueError(f"kv_dtype must be one of {sorted(KV_DTYPES)}, got {kv_dtype!r}")
    kd = arch.num_kv_heads * arch.head_dim
    row = 2 * kd if kv_dtype == "bf16" else kd + 4 * arch.num_kv_heads
    return 2 * arch.num_layers * KV_PAGE * row


def pages_for(n_tokens: int) -> int:
    return (n_tokens + KV_PAGE - 1) // KV_PAGE


class CacheFull(RuntimeError):
    """The paged KV cache has too few free pages for a request right now (it fits the pool once others end)."""


class InferEngine(Engine):
    kv_pages: Optional[int] = None   # pages in the pool; None: the contiguous max_batch x max_ctx cache
    kv_dtype: str = "bf16"

    def init_infer(self, arch: ServeArch, max_batch: int = 32, kv_pages: Optional[int] = None,
                   prefill_tokens: Optional[int] = None, kv_dtype: str = "bf16", max_rows: Optional[int] = None,
                   weight_dtype: str = "bf16"):
        """kv_pages: serve from a pool of that many 128-position pages shared by all slots (b200w_infer_init_paged)
        instead of reserving max_ctx positions per slot; arch.max_ctx is then the longest single request.
        prefill_tokens: the most tokens (n_seqs * padded length) one prefill call takes in paged mode.
        kv_dtype: "bf16", or "fp8" (paged only): K/V stored as e4m3 with per-(position, kv head) scales, about half
        the bytes per page (DESIGN §3.5).
        max_rows (max_batch..128; None: max_batch): rows one step may hold, for steps that verify drafted tokens
        (b200w_infer_set_step_rows).
        weight_dtype: "bf16", "int4" or "int8": every projection stored as int4 / int8 with one bf16 scale per row
        and 64 input columns, about a quarter / half of the bytes; the engine computes exactly what the bf16 engine
        does on the dequantized weights (read_weight). int8 is weight-only round-to-nearest, not bitsandbytes'
        LLM.int8: the activations stay bf16 and there is no outlier decomposition."""
        if weight_dtype not in WEIGHT_DTYPES:
            raise ValueError(f"weight_dtype must be one of {sorted(WEIGHT_DTYPES)}, got {weight_dtype!r}")
        if kv_dtype not in KV_DTYPES:
            raise ValueError(f"kv_dtype must be one of {sorted(KV_DTYPES)}, got {kv_dtype!r}")
        if kv_dtype != "bf16" and kv_pages is None:
            raise ValueError("an fp8 KV cache must be paged (kv_pages)")
        ca = _CArch(FAMILY[arch.family], arch.vocab_size, arch.hidden_size, arch.intermediate_size,
                    arch.num_layers, arch.num_heads, arch.num_kv_heads, arch.head_dim, arch.max_ctx,
                    arch.norm_eps, arch.rope_theta, 1 if arch.tie_embeddings else 0, arch.max_positions,
                    WEIGHT_DTYPES[weight_dtype])
        ca.reserved[1] = 1 if arch.parallel_norms else 0   # parallel_norms
        if kv_pages is None:
            self._check(self._lib.b200w_infer_init(self._h, C.byref(ca), max_batch))
        else:
            if prefill_tokens is None:
                prefill_tokens = max(16384, pages_for(arch.max_ctx) * KV_PAGE)
            self._check(self._lib.b200w_infer_init_paged_kv(self._h, C.byref(ca), max_batch, kv_pages, prefill_tokens,
                                                            KV_DTYPES[kv_dtype]))
            self.kv_pages, self.prefill_tokens = kv_pages, prefill_tokens
        if max_rows is not None:
            self._check(self._lib.b200w_infer_set_step_rows(self._h, max_rows))
        self.serve_arch, self.max_batch, self.kv_dtype, self.weight_dtype = arch, max_batch, kv_dtype, weight_dtype
        self.max_rows = max_batch if max_rows is None else max_rows

    def kv_read(self, layer: int, slot: int, pos0: int, n: int):
        """The raw cache rows of positions [pos0, pos0 + n) of `slot` (b200w_infer_kv_read): (k, v) as bf16 bit
        patterns (uint16 [n, Hkv * dh]), or on an fp8 cache (k, v, k_scale, v_scale) with e4m3 bytes (uint8) and
        fp32 scales [n, Hkv]."""
        a = self.serve_arch
        kd = a.num_kv_heads * a.head_dim
        dt = np.uint8 if self.kv_dtype == "fp8" else np.uint16
        k, v = np.empty((n, kd), dtype=dt), np.empty((n, kd), dtype=dt)
        ks, vs = (np.empty((n, a.num_kv_heads), dtype=np.float32) for _ in range(2))
        self._check(self._lib.b200w_infer_kv_read(self._h, layer, slot, pos0, n, k.ctypes.data, v.ctypes.data,
                                                  ks.ctypes.data, vs.ctypes.data))
        return (k, v, ks, vs) if self.kv_dtype == "fp8" else (k, v)

    def reserve(self, slot: int, n_tokens: int):
        """Give `slot` the pages for positions [0, n_tokens) (releasing what it held); B200WError with status
        B200W_ERR_OOM (-5) when too few pages are free."""
        self._check(self._lib.b200w_infer_reserve(self._h, slot, n_tokens))

    def reserve_shared(self, slot: int, n_tokens: int, shared_pages: List[int]):
        """reserve, with the slot's first len(shared_pages) pages being those (already referenced) pages; the slot
        may then write K/V only from position 128 * len(shared_pages) on (b200w_infer_reserve_shared)."""
        sp = np.ascontiguousarray(shared_pages, dtype=np.int32)
        self._check(self._lib.b200w_infer_reserve_shared(self._h, slot, n_tokens, sp.ctypes.data if sp.size else None,
                                                         sp.size))

    def retain_pages(self, pages: List[int], delta: int):
        """The host prefix index's references: +1 retains pages that hold a reference, -1 drops retained ones."""
        pg = np.ascontiguousarray(pages, dtype=np.int32)
        self._check(self._lib.b200w_infer_retain_pages(self._h, pg.ctypes.data if pg.size else None, pg.size, delta))

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

    def weight_bytes(self) -> int:
        """Device bytes the weights are stored in (b200w_infer_weight_bytes): the bf16 parameters and, with int4
        or int8 weights, the projections' images."""
        return self._lib.b200w_infer_weight_bytes(self._h)

    def read_weight(self, name: str, shape) -> np.ndarray:
        """The values the engine computes with for parameter `name` as bf16 bit patterns (uint16 of `shape`): the
        dequantized weights for a projection of an int4 or int8 engine, the loaded ones otherwise."""
        out = np.empty(shape, dtype=np.uint16)
        self._check(self._lib.b200w_infer_read_weight(self._h, name.encode(), out.ctypes.data, out.size))
        return out

    def _outputs(self, n: int, want_logits: bool):
        """The next tokens [n] and, with want_logits, fp32 logits [n, V] a step or prefill call writes."""
        return (np.empty(n, dtype=np.int32),
                np.empty((n, self.serve_arch.vocab_size), dtype=np.float32) if want_logits else None)

    def _step_args(self, tokens, positions, slots, want_logits: bool):
        """-> the int32 arguments of a step call (tokens, positions, slots) and its outputs (next tokens, logits)."""
        tok, pos, sl = (np.ascontiguousarray(x, dtype=np.int32) for x in (tokens, positions, slots))
        return (tok, pos, sl) + self._outputs(tok.size, want_logits)

    @staticmethod
    def _padded(prompts, starts=None):
        """The prompts, or their suffixes prompts[i][starts[i]:], zero-padded into [n, S] int32 with S the longest
        rounded up to a multiple of 128 -> (that array, the int32 lengths of the whole prompts)."""
        if starts is None:
            starts = [0] * len(prompts)
        S = ((max(len(p) - s for p, s in zip(prompts, starts)) + 127) // 128) * 128
        tok = np.zeros((len(prompts), S), dtype=np.int32)
        for i, (p, s) in enumerate(zip(prompts, starts)):
            tok[i, :len(p) - s] = p[s:]
        return tok, np.array([len(p) for p in prompts], dtype=np.int32)

    def step(self, tokens, positions, slots, want_logits: bool = False):
        tok, pos, sl, nxt, logits = self._step_args(tokens, positions, slots, want_logits)
        self._check(self._lib.b200w_infer_step(self._h, tok.ctypes.data, pos.ctypes.data, sl.ctypes.data, tok.size,
                                               nxt.ctypes.data, logits.ctypes.data if want_logits else None))
        return nxt, logits

    def prefill(self, prompts: List[List[int]], slots: List[int], want_logits: bool = False):
        """One pass over whole prompts (b200w_infer_prefill): K/V of every prompt position goes to its
        cache slot; returns (greedy token after each prompt, logits [n, V] or None)."""
        tok, lens = self._padded(prompts)
        sl = np.ascontiguousarray(slots, dtype=np.int32)
        nxt, logits = self._outputs(len(prompts), want_logits)
        self._check(self._lib.b200w_infer_prefill(self._h, tok.ctypes.data, lens.ctypes.data, sl.ctypes.data,
                                                  *tok.shape, nxt.ctypes.data,
                                                  logits.ctypes.data if want_logits else None))
        return nxt, logits

    def prefill_cached(self, prompts: List[List[int]], starts: List[int], slots: List[int], want_logits: bool = False):
        """prefill of whole prompts whose positions [0, starts[i]) already have their K/V in the slot's (shared)
        pages: only prompts[i][starts[i]:] is computed (b200w_infer_prefill_cached)."""
        tok, lens = self._padded(prompts, starts)
        st = np.ascontiguousarray(starts, dtype=np.int32)
        sl = np.ascontiguousarray(slots, dtype=np.int32)
        nxt, logits = self._outputs(len(prompts), want_logits)
        self._check(self._lib.b200w_infer_prefill_cached(self._h, tok.ctypes.data, st.ctypes.data, lens.ctypes.data,
                                                         sl.ctypes.data, *tok.shape, nxt.ctypes.data,
                                                         logits.ctypes.data if want_logits else None))
        return nxt, logits

    def step_logprobs(self, tokens, positions, slots, top_k: int, want_logits: bool = False):
        """step, plus the log-probabilities of each row's next-token distribution (b200w_infer_step_logprobs):
        -> (next tokens, logits or None, TokenLogprobs)."""
        tok, pos, sl, nxt, logits = self._step_args(tokens, positions, slots, want_logits)
        lp, s = TokenLogprobs.alloc(tok.size, top_k)
        self._check(self._lib.b200w_infer_step_logprobs(self._h, tok.ctypes.data, pos.ctypes.data, sl.ctypes.data,
                                                        tok.size, nxt.ctypes.data,
                                                        logits.ctypes.data if want_logits else None, C.byref(s)))
        return nxt, logits, lp

    def prefill_logprobs(self, prompts: List[List[int]], slots: List[int], top_k: int, want_logits: bool = False,
                         score_prompts: bool = True):
        """prefill (cold), plus the next-token log-probabilities and, with score_prompts, every prompt position's
        (b200w_infer_prefill_logprobs): -> (next tokens, logits or None, TokenLogprobs, prompt) where prompt[i] is
        None or (lp [len], top_ids [len, top_k], top_lp [len, top_k]) of prompts[i]; lp[p] = log P(prompt[p] |
        prompt[:p]) and position 0 has none (0, ids -1)."""
        tok, lens = self._padded(prompts)
        n, S = tok.shape
        sl = np.ascontiguousarray(slots, dtype=np.int32)
        nxt, logits = self._outputs(n, want_logits)
        lp, s = TokenLogprobs.alloc(n, top_k)
        if score_prompts:
            plp = np.empty((n, S), dtype=np.float32)
            pids = np.empty((n, S, top_k), dtype=np.int32)
            ptop = np.empty((n, S, top_k), dtype=np.float32)
        self._check(self._lib.b200w_infer_prefill_logprobs(
            self._h, tok.ctypes.data, lens.ctypes.data, sl.ctypes.data, n, S, nxt.ctypes.data,
            logits.ctypes.data if want_logits else None, C.byref(s), plp.ctypes.data if score_prompts else None,
            pids.ctypes.data if score_prompts and top_k else None, ptop.ctypes.data if score_prompts and top_k else None))
        prompt = [(plp[i, :len(p)], pids[i, :len(p)], ptop[i, :len(p)]) if score_prompts else None
                  for i, p in enumerate(prompts)]
        return nxt, logits, lp, prompt

    def sample(self, n: int, temperature, top_p, top_k, seeds, draws, want_logit: bool = False):
        """One token per row of the logits the step / prefill call just before left on the device
        (b200w_infer_sample; n is that call's row count): softmax(logits / temperature) cut by top_k (0: off), then
        top_p, drawn with the uniform number Philox4x32-10 gives for (seeds[i], draws[i]). Rows with temperature <= 0
        get the greedy token. -> (tokens, the tokens' logits as fp32 or None)."""
        t = np.ascontiguousarray(temperature, dtype=np.float32)
        p = np.ascontiguousarray(top_p, dtype=np.float32)
        k = np.ascontiguousarray(top_k, dtype=np.int32)
        sd = np.ascontiguousarray(seeds, dtype=np.uint64)
        dr = np.ascontiguousarray(draws, dtype=np.uint64)
        if not t.size == p.size == k.size == sd.size == dr.size == n:
            raise ValueError("sample: one temperature, top_p, top_k, seed and draw index per row")
        s = _lib.Sampling(0, t.ctypes.data, p.ctypes.data, k.ctypes.data, sd.ctypes.data, dr.ctypes.data)
        tok = np.empty(n, dtype=np.int32)
        lg = np.empty(n, dtype=np.float32) if want_logit else None
        self._check(self._lib.b200w_infer_sample(self._h, n, C.byref(s), tok.ctypes.data,
                                                 lg.ctypes.data if want_logit else None))
        return tok, lg

    def sample_penalized(self, n: int, temperature, top_p, top_k, seeds, draws, penalties: "Penalties",
                         want_logit: bool = False):
        """sample on the rows after their presence, frequency and repetition penalties and logit bias
        (b200w_infer_sample_penalized; DESIGN §3.5). Rows with temperature <= 0 get the argmax of the penalized row.
        -> (tokens, the tokens' raw logits as fp32 or None)."""
        t = np.ascontiguousarray(temperature, dtype=np.float32)
        p = np.ascontiguousarray(top_p, dtype=np.float32)
        k = np.ascontiguousarray(top_k, dtype=np.int32)
        sd = np.ascontiguousarray(seeds, dtype=np.uint64)
        dr = np.ascontiguousarray(draws, dtype=np.uint64)
        if not t.size == p.size == k.size == sd.size == dr.size == penalties.presence.size == n:
            raise ValueError("sample_penalized: one temperature, top_p, top_k, seed, draw index and penalty per row")
        s = _lib.Sampling(0, t.ctypes.data, p.ctypes.data, k.ctypes.data, sd.ctypes.data, dr.ctypes.data)
        pen = penalties.c_struct()
        tok = np.empty(n, dtype=np.int32)
        lg = np.empty(n, dtype=np.float32) if want_logit else None
        self._check(self._lib.b200w_infer_sample_penalized(self._h, n, C.byref(s), C.byref(pen), tok.ctypes.data,
                                                           lg.ctypes.data if want_logit else None))
        return tok, lg


@dataclass
class Penalties:
    """The b200w_penalties of one call: per row presence, frequency and repetition, and the rows' entries in CSR form
    (row i's are [offsets[i], offsets[i + 1])): distinct ids, how often each occurs in the request's output, whether
    it occurs in its prompt, and its logit bias."""
    presence: np.ndarray     # float32 [n]
    frequency: np.ndarray    # float32 [n]
    repetition: np.ndarray   # float32 [n]
    offsets: np.ndarray      # int32 [n + 1]
    ids: np.ndarray          # int32 [entries]
    out_count: np.ndarray    # int32 [entries]
    in_prompt: np.ndarray    # int32 [entries]
    bias: np.ndarray         # float32 [entries]

    @classmethod
    def pack(cls, rows: List[Optional["RequestPenalties"]]) -> "Penalties":
        """One call's arrays from each row's RequestPenalties (None: a row without penalties)."""
        live = [r for r in rows if r is not None]
        counts = [r.n if r is not None else 0 for r in rows]
        offsets = np.zeros(len(rows) + 1, np.int32)
        np.cumsum(counts, out=offsets[1:])

        def cat(field, dt):
            return np.concatenate([getattr(r, field)[:r.n] for r in live]) if live else np.zeros(0, dt)
        return cls(np.array([r.presence if r else 0.0 for r in rows], np.float32),
                   np.array([r.frequency if r else 0.0 for r in rows], np.float32),
                   np.array([r.repetition if r else 1.0 for r in rows], np.float32), offsets,
                   cat("ids", np.int32), cat("out_count", np.int32), cat("in_prompt", np.int32),
                   cat("bias", np.float32))

    def c_struct(self) -> _lib.Penalties:
        arrs = [np.ascontiguousarray(getattr(self, f), dtype=dt) for f, dt in (
            ("presence", np.float32), ("frequency", np.float32), ("repetition", np.float32), ("offsets", np.int32),
            ("ids", np.int32), ("out_count", np.int32), ("in_prompt", np.int32), ("bias", np.float32))]
        s = _lib.Penalties(0, *(a.ctypes.data for a in arrs))
        s._keep = arrs   # the struct holds raw pointers: keep the arrays alive with it
        return s


class RequestPenalties:
    """A request's penalties and its entries, kept as it generates: the distinct ids of its prompt (only when
    repetition != 1: they matter to nothing else), of its logit_bias and of its output so far, with the output counts,
    the prompt flags and the biases. emit() counts a generated token; a step packs these arrays as they stand."""

    def __init__(self, prompt: List[int], presence: float, frequency: float, repetition: float,
                 logit_bias: Dict[int, float]):
        self.presence, self.frequency, self.repetition = float(presence), float(frequency), float(repetition)
        ids = list(dict.fromkeys((list(prompt) if self.repetition != 1.0 else []) + list(logit_bias)))
        self.pos = {t: i for i, t in enumerate(ids)}
        self.n = len(ids)
        cap = max(16, 2 * self.n)
        self.ids, self.out_count, self.in_prompt = (np.zeros(cap, np.int32) for _ in range(3))
        self.bias = np.zeros(cap, np.float32)
        self.ids[:self.n] = ids
        if self.repetition != 1.0:
            self.in_prompt[[self.pos[t] for t in set(prompt)]] = 1
        for t, b in logit_bias.items():
            self.bias[self.pos[t]] = b

    def after(self, tokens: List[int]) -> "RequestPenalties":
        """A copy with `tokens` counted as emitted: the entries of a step row that follows drafted tokens."""
        c = RequestPenalties.__new__(RequestPenalties)
        c.presence, c.frequency, c.repetition, c.n = self.presence, self.frequency, self.repetition, self.n
        c.pos = dict(self.pos)
        c.ids, c.out_count, c.in_prompt, c.bias = (a.copy() for a in (self.ids, self.out_count, self.in_prompt,
                                                                       self.bias))
        for t in tokens:
            c.emit(t)
        return c

    def emit(self, t: int):
        i = self.pos.get(t)
        if i is None:
            if self.n == self.ids.size:
                for f in ("ids", "out_count", "in_prompt", "bias"):
                    a = getattr(self, f)
                    setattr(self, f, np.concatenate([a, np.zeros_like(a)]))
            i = self.pos[t] = self.n
            self.ids[i] = t
            self.n += 1
        self.out_count[i] += 1


@dataclass
class TokenLogprobs:
    """Host arrays of a b200w_logprobs: per row the log-sum-exp of the next-token logits, the log-probability of the
    greedy token and the top_k largest logits' ids and log-probabilities (descending, ties to the smaller id)."""
    lse: np.ndarray
    token_lp: np.ndarray
    top_ids: np.ndarray
    top_lp: np.ndarray

    @classmethod
    def alloc(cls, n: int, top_k: int):
        if not 0 <= top_k <= _lib.MAX_TOP_LOGPROBS:
            raise ValueError(f"top_k must be in 0..{_lib.MAX_TOP_LOGPROBS}, got {top_k}")
        lp = cls(np.empty(n, np.float32), np.empty(n, np.float32), np.empty((n, top_k), np.int32),
                 np.empty((n, top_k), np.float32))
        return lp, _lib.Logprobs(top_k, 0, lp.lse.ctypes.data, lp.token_lp.ctypes.data, lp.top_ids.ctypes.data,
                                 lp.top_lp.ctypes.data)


def sample_token(logits: np.ndarray, temperature: float, top_p: float, rng: np.random.Generator) -> int:
    """Host-side sampling of one row, for engines without `sample`: softmax(logits / T) restricted to the
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


class NgramProposer:
    """Prompt lookup (HF generate(prompt_lookup_num_tokens=...), vLLM's ngram speculation) over a request's ids, the
    prompt as fed and then its output: the draft is what followed the latest earlier occurrence of the ids' last n
    tokens, n = 3, then 2, then 1. An index from each n-gram to the end of its latest occurrence is built over the
    prompt when the request is admitted and grows as ids are appended, so a step's proposal costs O(n + d) however
    long the request is."""
    N = 3

    def __init__(self, ids: Iterable[int] = ()):
        self.ids: List[int] = list(ids)
        self.latest: List[Dict[Tuple[int, ...], int]] = [{} for _ in range(self.N + 1)]
        self.indexed = 0     # n-grams that end at positions <= indexed are in the index
        self._index()

    def append(self, t: int):
        self.ids.append(t)

    def _index(self):
        """Every n-gram that ends before the last id (the suffix a proposal looks up ends there) into the index."""
        ids, L = self.ids, len(self.ids)
        for e in range(self.indexed + 1, L):
            for n in range(1, min(self.N, e) + 1):
                self.latest[n][tuple(ids[e - n:e])] = e
        self.indexed = max(self.indexed, L - 1)

    def propose(self, d: int) -> List[int]:
        """At most d tokens: ids[e : e + d] for the end e < len(ids) of the latest earlier occurrence of the longest
        suffix n-gram that has one; [] when none has."""
        self._index()
        ids, L = self.ids, len(self.ids)
        if d <= 0:
            return []
        for n in range(min(self.N, L - 1), 0, -1):
            e = self.latest[n].get(tuple(ids[L - n:]))
            if e is not None:
                return ids[e:e + d]
        return []


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
    rng: Optional[np.random.Generator] = None                 # host sampling only (an engine without `sample`)
    cached_tokens: int = 0                                    # prompt positions whose K/V came from the prefix index
    nodes: List["_Node"] = field(default_factory=list)        # index nodes whose page the slot holds
    entered: List["_Node"] = field(default_factory=list)      # of those, the ones this request's prefill fills
    # log-probabilities: `logprobs` top entries per token (None: not asked). out_lp[i] = (log-probability of out[i],
    # [(id, log-probability)] of the top entries); prompt_lp the same per prompt position, None at position 0
    logprobs: Optional[int] = None
    prompt_logprobs: bool = False
    out_lp: List[Tuple[float, List[Tuple[int, float]]]] = field(default_factory=list)
    prompt_lp: Optional[List[Optional[Tuple[float, List[Tuple[int, float]]]]]] = None
    # sampling on the device: draw i of the request uses the uniform number of (seed, i), i = len(out)
    top_k: int = 0
    seed: int = 0
    pen: Optional[RequestPenalties] = None                    # None: no penalty and no logit_bias
    error: Optional[str] = None                               # set when the request failed on its own (done too)
    lookup: Optional[NgramProposer] = None                    # speculation: the n-gram index of prompt + output

    @property
    def greedy(self) -> bool:
        return self.temperature <= 0.0

    @property
    def step_token(self) -> bool:
        """Whether the token it emits is the step's own greedy token (not drawn, and nothing to penalize)."""
        return self.greedy and self.pen is None

    @property
    def scores_prompt(self) -> bool:
        return self.prompt_logprobs and len(self.prompt) > 1


class _Node:
    """A full prompt page in the prefix index: the K/V of the KV_PAGE tokens `key` that follow the tokens of its
    ancestors. A page's K/V depend on every token before it, and the path from the root spells exactly those."""
    __slots__ = ("parent", "key", "page", "children", "users", "last_use")

    def __init__(self, parent: Optional["_Node"], key: Tuple[int, ...], page: int):
        self.parent, self.key, self.page = parent, key, page
        self.children: Dict[Tuple[int, ...], "_Node"] = {}
        self.users = 0          # active requests whose slot holds the page
        self.last_use = 0


class Generator:
    """Continuous batching over the engine's cache slots. A request's prompt is ingested in one prefill
    pass when it is admitted (engines without `prefill`, i.e. the CPU test stubs, feed it one token per
    step through the decode path); from then on every active request advances one token per step, or with
    speculation up to 1 + speculative_tokens."""

    def __init__(self, engine: InferEngine, eos_id: Optional[int] = None, use_prefill: bool = True,
                 prefix_cache: bool = False, speculative_tokens: int = 0):
        """prefix_cache (paged KV cache only): requests whose prompts share leading full pages share those pages and
        prefill only the rest. An index of the prompt pages served keeps them (one retained reference each) until
        pages run short, then gives back the least recently used ones.
        speculative_tokens (0..7; 0: off): a request past its prompt feeds its last token and up to that many drafted
        tokens (`propose`, prompt lookup by default) at consecutive positions in one step, and emits the step's
        tokens while they match the drafts (DESIGN §3.5). Its tokens are the same as without speculation; the step's
        rows stay within the engine's max_rows."""
        if isinstance(speculative_tokens, bool) or not isinstance(speculative_tokens, int) or \
                not 0 <= speculative_tokens <= 7:
            raise ValueError(f"speculative_tokens must be an integer in 0..7, got {speculative_tokens!r}")
        self.spec = speculative_tokens
        self.max_rows = getattr(engine, "max_rows", engine.max_batch)
        self.e, self.eos = engine, eos_id
        self.free = list(range(engine.max_batch))
        self.active: List[_Req] = []
        self.use_prefill = use_prefill and hasattr(engine, "prefill")
        self._deferred: List[_Req] = []
        # paged KV cache: a request holds pages for len(prompt) + max_tokens positions from admission to its end
        self.kv_pages = getattr(engine, "kv_pages", None)
        self.prefix_cache = prefix_cache
        if prefix_cache and (self.kv_pages is None or not self.use_prefill):
            raise ValueError("prefix caching needs the paged KV cache and an engine that prefills")
        self._root = _Node(None, (), -1)
        self._nodes: Dict[_Node, None] = {}     # every node of the index, in insertion order
        self._tick = 0
        self.device_sampling = hasattr(engine, "sample")   # else the logits come to the host (sample_token)

    def add(self, prompt: List[int], max_tokens: int, temperature: float = 0.0, top_p: float = 1.0,
            seed: Optional[int] = None, defer_prefill: bool = False, logprobs: Optional[int] = None,
            prompt_logprobs: bool = False, top_k: int = 0, presence_penalty: float = 0.0,
            frequency_penalty: float = 0.0, repetition_penalty: float = 1.0,
            logit_bias: Optional[Dict[int, float]] = None) -> _Req:
        """defer_prefill: only register the request; flush_prefill() then ingests every deferred prompt of the
        same padded length in ONE prefill call (what the scheduler does when several requests are admitted in
        the same round).
        logprobs (0..5): record the log-probability of every generated token and its `logprobs` top entries
        (req.out_lp); prompt_logprobs: the same for every prompt position after the first (req.prompt_lp), computed
        by the prefill. Both are the engine's raw log-softmax (temperature 1, no top_p), and a request that asks for
        either borrows no prefix-cache pages: their hidden states are needed and were never computed.
        top_k (0: off; at or above the vocabulary size keeps everything): sample among the top_k largest logits only,
        before top_p; needs an engine that samples on the device. seed (None: from OS entropy): with it the
        request's tokens are a function of its logits alone.
        presence_penalty, frequency_penalty, repetition_penalty (> 0; 1 is off) and logit_bias ({token id: bias}):
        applied to the logits on the device before the draw, greedy rows included (DESIGN §3.5), with the counts of
        this request's own output; needs an engine that samples on the device. Log-probabilities stay raw."""
        if not prompt:
            raise ValueError("empty prompt")
        V = self.e.serve_arch.vocab_size
        pen = self._penalties(prompt, presence_penalty, frequency_penalty, repetition_penalty, logit_bias, V)
        if not (isinstance(top_k, int) and top_k >= 0):
            raise ValueError(f"top_k must be 0 (off) or a positive integer, got {top_k!r}")
        if top_k and not self.device_sampling:
            raise ValueError("top_k needs an engine that samples on the device")
        if logprobs is not None and not (isinstance(logprobs, int) and 0 <= logprobs <= _lib.MAX_TOP_LOGPROBS):
            raise ValueError(f"logprobs must be in 0..{_lib.MAX_TOP_LOGPROBS}, got {logprobs!r}")
        if logprobs is not None and not hasattr(self.e, "step_logprobs"):
            raise ValueError("log-probabilities need an engine that computes them")
        if prompt_logprobs and not (self.use_prefill and hasattr(self.e, "prefill_logprobs")):
            raise ValueError("prompt log-probabilities need an engine that prefills")
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
        matched, entered = [], []
        if self.prefix_cache:
            matched, entered = self._admit(list(prompt), len(prompt) + max_tokens, self.free[-1],
                                           borrow=logprobs is None and not prompt_logprobs)
        elif self.kv_pages is not None:
            if pages_for(len(prompt) + max_tokens) > self.e.kv_pages_free():
                raise CacheFull("KV cache full: too few free pages for this request now")
            self.e.reserve(self.free[-1], len(prompt) + max_tokens)
        r = _Req(list(prompt), max_tokens, [], 0, self.free.pop(), False, float(temperature), float(top_p),
                 np.random.default_rng(seed) if temperature > 0 and not self.device_sampling else None,
                 len(matched) * KV_PAGE, matched + entered, entered, logprobs, bool(prompt_logprobs))
        if self.device_sampling and not r.greedy:
            r.top_k = 0 if top_k >= V else top_k
            r.seed = (int(seed) if seed is not None else int.from_bytes(os.urandom(8), "little")) % 2 ** 64
        r.pen = pen
        if self.spec:
            r.lookup = NgramProposer(r.prompt)
        if r.prompt_logprobs and not r.scores_prompt:
            r.prompt_lp = [None]          # one token: nothing to score
        self.active.append(r)
        if self.use_prefill and len(prompt) > 1:
            self._deferred.append(r)
            if not defer_prefill:
                self.flush_prefill()
        return r

    def _penalties(self, prompt, presence, frequency, repetition, logit_bias, V) -> Optional[RequestPenalties]:
        """A request's RequestPenalties, None when every penalty is neutral; ValueError on a value out of range. The
        values are checked as the float32 the engine receives: one the engine would refuse fails this request alone,
        never a whole step's batch."""
        with np.errstate(over="ignore", under="ignore"):
            presence, frequency, repetition = (float(np.float32(x)) for x in (presence, frequency, repetition))
            if not all(np.isfinite(x) for x in (presence, frequency, repetition)) or not repetition > 0:
                raise ValueError("presence_penalty and frequency_penalty must be finite, repetition_penalty finite and "
                                 "> 0 (as float32)")
            bias = {}
            for t, b in (logit_bias or {}).items():
                if isinstance(t, bool) or not isinstance(t, (int, np.integer)) or not 0 <= t < V:
                    raise ValueError(f"logit_bias token id {t!r} outside the model vocabulary ({V})")
                if not np.isfinite(np.float32(b)):
                    raise ValueError(f"logit_bias of token {t} must be finite (as float32)")
                bias[int(t)] = float(np.float32(b))
        if presence == 0 and frequency == 0 and repetition == 1 and not bias:
            return None
        if not hasattr(self.e, "sample_penalized"):
            raise ValueError("presence, frequency and repetition penalties and logit_bias need an engine that samples "
                             "on the device")
        return RequestPenalties(prompt, presence, frequency, repetition, bias)

    def _admit(self, prompt: List[int], n_tokens: int, slot: int, borrow: bool = True):
        """Prefix cache admission into `slot`: the longest chain of indexed pages that prefixes the prompt (at most
        (len - 1) // 128, so that at least one prompt token is computed for the next-token logits) is shared; the
        request's own full prompt pages beyond it enter the index at once, so that requests admitted later in the
        same round share them too. borrow=False shares nothing (a request whose every position is computed).
        -> (matched nodes, entered nodes)."""
        matched: List[_Node] = []
        node = self._root
        for k in range((len(prompt) - 1) // KV_PAGE if borrow else 0):
            node = node.children.get(tuple(prompt[k * KV_PAGE:(k + 1) * KV_PAGE]))
            if node is None:
                break
            matched.append(node)
        short = pages_for(n_tokens) - len(matched) - self.e.kv_pages_free()
        if short > 0:
            keep = set(matched)
            if short > sum(1 for n in self._nodes if n.users == 0 and n not in keep):
                raise CacheFull("KV cache full: too few free or evictable pages for this request now")
            for _ in range(short):   # least recently used leaves that no request holds (each frees its page)
                self._drop(min((n for n in self._nodes if not n.children and n.users == 0 and n not in keep),
                               key=lambda n: n.last_use))
        self.e.reserve_shared(slot, n_tokens, [n.page for n in matched])
        self._tick += 1
        for n in matched:
            n.users += 1
            n.last_use = self._tick
        entered: List[_Node] = []
        parent = matched[-1] if matched else self._root
        if len(prompt) // KV_PAGE > len(matched):
            pages = self.e.slot_pages(slot)
            for k in range(len(matched), len(prompt) // KV_PAGE):
                key = tuple(prompt[k * KV_PAGE:(k + 1) * KV_PAGE])
                if key in parent.children:   # the last page of an indexed prompt of the same length (the cap above)
                    break
                node = _Node(parent, key, pages[k])
                node.users, node.last_use = 1, self._tick
                parent.children[key] = node
                self._nodes[node] = None
                entered.append(node)
                parent = node
            if entered:
                self.e.retain_pages([n.page for n in entered], +1)
        return matched, entered

    def _drop(self, node: _Node):
        """Takes `node` and everything below it out of the prefix index, with the index's references."""
        gone, stack = [], [node]
        while stack:
            n = stack.pop()
            gone.append(n)
            stack.extend(n.children.values())
        del node.parent.children[node.key]
        for n in gone:
            del self._nodes[n]
        self.e.retain_pages([n.page for n in gone], -1)

    def clear_prefix_cache(self):
        """Drops every index entry; a page returns to the free list once no request holds it either."""
        for n in list(self._root.children.values()):
            self._drop(n)

    def flush_prefill(self):
        """One prefill call per group of deferred prompts with the same cached prefix that pad to the same multiple of
        128 tokens. Cold prompts (no cached prefix) go first, then the others in ascending prefix length: a request
        shares only pages that a request with a shorter prefix fills, so those are written by an earlier call."""
        pend, self._deferred = self._deferred, []
        groups: Dict[Tuple[int, int, bool], List[_Req]] = {}
        for r in pend:   # prompts to score go through their own calls: a plain prompt never pays for scoring
            groups.setdefault((r.cached_tokens, pages_for(len(r.prompt) - r.cached_tokens), r.scores_prompt),
                              []).append(r)
        calls = []
        for (start, blocks, score), rs in sorted(groups.items()):
            # paged: a call's n_seqs * padded_len stays within the prefill workspace the engine allocated
            per_call = max(1, self.e.prefill_tokens // (blocks * 128)) if self.kv_pages is not None else len(rs)
            calls += [(start, score, rs[i:i + per_call]) for i in range(0, len(rs), per_call)]
        for ci, (start, score, rs) in enumerate(calls):
            need_logits = not self.device_sampling and any(not r.greedy for r in rs)
            top_k = max((r.logprobs for r in rs if r.logprobs is not None), default=None)
            lp = prompt = None
            try:
                if start:
                    nxt, lg = self.e.prefill_cached([r.prompt for r in rs], [start] * len(rs), [r.slot for r in rs],
                                                    want_logits=need_logits)
                elif score or top_k is not None:
                    nxt, lg, lp, prompt = self.e.prefill_logprobs([r.prompt for r in rs], [r.slot for r in rs],
                                                                  top_k or 0, want_logits=need_logits,
                                                                  score_prompts=score)
                else:
                    nxt, lg = self.e.prefill([r.prompt for r in rs], [r.slot for r in rs], want_logits=need_logits)
            except Exception:
                # the pages this call and the calls after it were to fill hold no K/V: out of the index
                for _, _, later in calls[ci:]:
                    for r in later:
                        for n in r.entered:
                            if n in self._nodes:
                                self._drop(n)
                raise
            if need_logits and lg is None:
                raise ValueError("sampling (temperature > 0) needs an engine that returns logits")
            drawn = self._sample(rs, [True] * len(rs))
            for i, r in enumerate(rs):
                r.fed = len(r.prompt)
                if score:
                    plp, pids, ptop = prompt[i]
                    k = r.logprobs or 0
                    r.prompt_lp = [None] + [(float(plp[p]), list(zip(pids[p, :k].tolist(), ptop[p, :k].tolist())))
                                            for p in range(1, len(r.prompt))]
                self._emit_token(r, i, nxt, lg, lp, drawn)
        self._retire()

    def _sample(self, rs: List[_Req], emits: List[bool], ahead: Optional[List[List[int]]] = None):
        """Right after the step / prefill call over the rows `rs`: one engine.sample call for them when a row that
        emits a token samples (the others go as greedy rows), or one engine.sample_penalized call when such a row
        is penalized (the others go without entries) -> (tokens, their raw logits or None), or None.
        ahead[i] (speculation): the drafted tokens row i follows; its draw is len(out) + len(ahead[i]), and its
        penalties count them as emitted."""
        ahead = ahead or [[]] * len(rs)
        on = [e and not r.greedy for r, e in zip(rs, emits)]
        pen = [e and r.pen is not None for r, e in zip(rs, emits)]
        if not (self.device_sampling and (any(on) or any(pen))):
            return None
        args = (len(rs), [r.temperature if s else 0.0 for r, s in zip(rs, on)], [r.top_p for r in rs],
                [r.top_k for r in rs], [r.seed for r in rs], [len(r.out) + len(a) for r, a in zip(rs, ahead)])
        want_logit = any((s or p) and r.logprobs is not None for r, s, p in zip(rs, on, pen))
        if any(pen):
            return self.e.sample_penalized(*args, Penalties.pack([(r.pen.after(a) if a else r.pen) if p else None
                                                                  for r, p, a in zip(rs, pen, ahead)]),
                                           want_logit=want_logit)
        return self.e.sample(*args, want_logit=want_logit)

    def _emit_token(self, r: _Req, i: int, nxt, lg, lp: Optional[TokenLogprobs], drawn=None):
        """Emits row i's token for r: the greedy one, or one drawn from its (penalized) logits (`drawn`, what _sample
        returned, or on the host from lg); with its log-probability when r asks for it (the greedy token's from the
        engine, any other's from its raw logit and the row's lse)."""
        if r.step_token:
            t = int(nxt[i])
        elif drawn is not None:
            t = int(drawn[0][i])
        else:
            t = sample_token(lg[i], r.temperature, r.top_p, r.rng)
        if not 0 <= t < self.e.serve_arch.vocab_size:   # e.g. a row of infinite logits: fail r, not the batch
            r.error = f"no token could be drawn from this request's logits (got id {t})"
            r.done = True
            return
        if r.logprobs is not None:
            x = (lp.token_lp[i] if r.step_token
                 else (drawn[1][i] if drawn is not None else np.float32(lg[i][t])) - lp.lse[i])
            k = r.logprobs
            r.out_lp.append((float(x), list(zip(lp.top_ids[i, :k].tolist(), lp.top_lp[i, :k].tolist()))))
        self._emit(r, t)

    def _emit(self, r: _Req, t: int):
        r.out.append(t)
        if r.pen is not None:
            r.pen.emit(t)
        if r.lookup is not None:
            r.lookup.append(t)
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
        self._tick += 1
        for n in r.nodes:
            n.users -= 1
            n.last_use = self._tick
        if self.kv_pages is not None:
            self.e.release(r.slot)

    def _retire(self):
        for r in [r for r in self.active if r.done]:
            self.active.remove(r)
            self._free_slot(r)

    def propose(self, r: _Req, d: int) -> List[int]:
        """Up to d drafted tokens to follow r's ids (prompt lookup); a test may replace this."""
        return r.lookup.propose(d)

    def _drafts(self) -> List[List[int]]:
        """Each active request's drafts for this step. Only a request past its prompt drafts, at most
        min(speculative_tokens, max_tokens - len(out) - 1) tokens (its last position stays inside what admission
        reserved), and the step's rows stay within max_rows: requests take the spare rows in the order they are
        active. A request sampled on the host drafts nothing (its generator has state)."""
        spare = self.max_rows - len(self.active)
        drafts = []
        for r in self.active:
            d = min(self.spec, r.max_tokens - len(r.out) - 1, spare)
            if r.fed < len(r.prompt) or (r.rng is not None) or d <= 0:
                drafts.append([])
                continue
            dr = [int(t) for t in self.propose(r, d)[:d]]
            spare -= len(dr)
            drafts.append(dr)
        return drafts

    def step(self):
        """One engine step for every active request: its next token's row, then one row per drafted token."""
        if not self.active:
            return
        drafts = self._drafts() if self.spec else [[] for _ in self.active]
        rs, toks, pos, ahead = [], [], [], []
        for r, dr in zip(self.active, drafts):
            for j, t in enumerate([r.prompt[r.fed] if r.fed < len(r.prompt) else r.out[-1]] + dr):
                rs.append(r)
                toks.append(t)
                pos.append(r.fed + j)
                ahead.append(dr[:j])
        slots = [r.slot for r in rs]
        need_logits = not self.device_sampling and any(not r.greedy for r in self.active)
        top_k = max((r.logprobs for r in self.active if r.logprobs is not None), default=None)
        lp = None
        if top_k is None:
            nxt, lg = self.e.step(toks, pos, slots, want_logits=need_logits)
        else:
            nxt, lg, lp = self.e.step_logprobs(toks, pos, slots, top_k, want_logits=need_logits)
        if need_logits and lg is None:
            raise ValueError("sampling (temperature > 0) needs an engine that returns logits")
        drawn = self._sample(rs, [r.fed + 1 + len(a) >= len(r.prompt) for r, a in zip(rs, ahead)],
                             ahead if self.spec else None)
        i = 0
        for r, dr in zip(self.active, drafts):
            r.fed += 1
            if r.fed >= len(r.prompt):        # the token just fed was the last known one
                # row j's token is right while every draft before it was: emit until the first mismatch
                for j in range(len(dr) + 1):
                    self._emit_token(r, i + j, nxt, lg, lp, drawn)
                    if r.done or j == len(dr) or r.out[-1] != dr[j]:
                        break
                    r.fed += 1
            i += 1 + len(dr)
        self._retire()

    def generate(self, prompts: List[List[int]], max_tokens: int) -> List[List[int]]:
        reqs = [self.add(p, max_tokens) for p in prompts]
        while self.active:
            self.step()
        return [r.out for r in reqs]
