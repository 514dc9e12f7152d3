"""Python host over the C ABI (include/b200w.h): one `Engine` = one b200w context on one GPU.

This is the layer the worker (runbooks_b200/worker.py — the container-contract entry point) and
bench.py drive. It holds no arithmetic; every number comes out of libb200w.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Iterable, Optional, Tuple

import numpy as np

from . import _lib
from ._lib import Arch as _CArch, HParams as _CHParams, B200WError


FAMILY_LLAMA, FAMILY_FALCON, FAMILY_OPT = 0, 1, 2


def _reject(cond: bool, what: str):
    """An unimplemented setting that changes the arithmetic must fail the Job, never be ignored
    (same policy as contract.load_params)."""
    if cond:
        raise ValueError(f"unsupported checkpoint config: {what}")


@dataclass
class LlamaArch:
    """Subset of the HF LlamaConfig the kernels need (config.json keys in comments)."""
    vocab_size: int
    hidden_size: int
    intermediate_size: int
    num_layers: int            # num_hidden_layers
    num_heads: int             # num_attention_heads
    num_kv_heads: int          # num_key_value_heads
    head_dim: int = 128
    max_seq_len: int = 4096    # sequences are packed to this length
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    pad_token_id: int = -1     # nn.Embedding(padding_idx): that row gets no lookup gradient; -1 = None
    family = FAMILY_LLAMA
    max_positions = 0

    @classmethod
    def llama2_7b(cls, seq_len: int = 4096) -> "LlamaArch":
        return cls(32000, 4096, 11008, 32, 32, 32, 128, seq_len, 1e-5, 10000.0)

    @classmethod
    def from_hf_config(cls, cfg: dict, seq_len: Optional[int] = None) -> "LlamaArch":
        if cfg.get("model_type", "llama") != "llama":
            raise ValueError(f"unsupported model_type {cfg.get('model_type')!r} (llama / opt)")
        heads = cfg["num_attention_heads"]
        rope = cfg.get("rope_parameters") or {}
        scaling = cfg.get("rope_scaling") or {}
        rope_type = rope.get("rope_type") or scaling.get("rope_type") or scaling.get("type") or "default"
        _reject(rope_type != "default", f"rope_type {rope_type!r} (only the default rotary embedding is built)")
        _reject(bool(cfg.get("attention_bias")), "attention_bias=true")
        _reject(bool(cfg.get("mlp_bias")), "mlp_bias=true")
        _reject(cfg.get("hidden_act", "silu") != "silu", f"hidden_act {cfg.get('hidden_act')!r}")
        _reject(bool(cfg.get("tie_word_embeddings")), "tie_word_embeddings=true for a Llama checkpoint")
        _reject(cfg.get("sliding_window") not in (None, 0), "sliding_window attention")
        pad = cfg.get("pad_token_id")
        return cls(
            vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
            intermediate_size=cfg["intermediate_size"], num_layers=cfg["num_hidden_layers"],
            num_heads=heads, num_kv_heads=cfg.get("num_key_value_heads") or heads,
            head_dim=cfg.get("head_dim") or cfg["hidden_size"] // heads,
            max_seq_len=seq_len or cfg.get("max_position_embeddings", 4096),
            rms_norm_eps=cfg.get("rms_norm_eps", 1e-6),
            rope_theta=float(cfg.get("rope_theta") or rope.get("rope_theta") or 10000.0),
            pad_token_id=-1 if pad is None else int(pad),
        )

    def to_hf_config(self) -> dict:
        cfg = {
            "architectures": ["LlamaForCausalLM"], "model_type": "llama",
            "vocab_size": self.vocab_size, "hidden_size": self.hidden_size,
            "intermediate_size": self.intermediate_size, "num_hidden_layers": self.num_layers,
            "num_attention_heads": self.num_heads, "num_key_value_heads": self.num_kv_heads,
            "head_dim": self.head_dim, "max_position_embeddings": self.max_seq_len,
            "rms_norm_eps": self.rms_norm_eps, "rope_theta": self.rope_theta,
            "hidden_act": "silu", "tie_word_embeddings": False, "attention_bias": False,
            "mlp_bias": False, "torch_dtype": "bfloat16",
        }
        if self.pad_token_id >= 0:
            cfg["pad_token_id"] = self.pad_token_id
        return cfg

    def c_fields(self) -> dict:
        return dict(vocab_size=self.vocab_size, hidden_size=self.hidden_size,
                    intermediate_size=self.intermediate_size, num_layers=self.num_layers,
                    num_heads=self.num_heads, num_kv_heads=self.num_kv_heads, head_dim=self.head_dim,
                    max_seq_len=self.max_seq_len, rms_norm_eps=self.rms_norm_eps, rope_theta=self.rope_theta,
                    family=self.family, pad_token_id=self.pad_token_id, max_positions=self.max_positions)


@dataclass
class OptArch:
    """facebook/opt-125m family (HF models/opt/modeling_opt.py; the reference's config #1,
    examples/facebook-opt-125m/finetuned-model.yaml): learned positions at +2, pre-LayerNorm with bias,
    biased projections, ReLU MLP, lm_head tied to the token embedding."""
    vocab_size: int
    hidden_size: int
    intermediate_size: int     # ffn_dim
    num_layers: int
    num_heads: int
    max_positions: int = 2048  # max_position_embeddings (the table holds 2 more rows)
    max_seq_len: int = 2048    # packed sequence length, <= max_positions, multiple of 128
    layer_norm_eps: float = 1e-5
    pad_token_id: int = 1
    family = FAMILY_OPT

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_heads

    @property
    def num_kv_heads(self) -> int:
        return self.num_heads

    @classmethod
    def opt_125m(cls, seq_len: int = 2048) -> "OptArch":
        return cls(50272, 768, 3072, 12, 12, 2048, seq_len)

    @classmethod
    def from_hf_config(cls, cfg: dict, seq_len: Optional[int] = None) -> "OptArch":
        if cfg.get("model_type") != "opt":
            raise ValueError(f"unsupported model_type {cfg.get('model_type')!r}")
        d = cfg["hidden_size"]
        _reject(not cfg.get("do_layer_norm_before", True), "do_layer_norm_before=false (opt-350m layout)")
        _reject(cfg.get("word_embed_proj_dim", d) != d, "word_embed_proj_dim != hidden_size (project_in/out)")
        _reject(cfg.get("activation_function", "relu") != "relu", f"activation_function {cfg.get('activation_function')!r}")
        _reject(not cfg.get("enable_bias", True), "enable_bias=false")
        _reject(not cfg.get("layer_norm_elementwise_affine", True), "layer_norm_elementwise_affine=false")
        _reject(cfg.get("_remove_final_layer_norm", False), "_remove_final_layer_norm")
        _reject(not cfg.get("tie_word_embeddings", True), "untied lm_head for an OPT checkpoint")
        _reject((d // cfg["num_attention_heads"]) not in (64, 128), "head_dim other than 64 / 128")
        maxpos = cfg.get("max_position_embeddings", 2048)
        s = seq_len or maxpos
        pad = cfg.get("pad_token_id", 1)
        return cls(cfg["vocab_size"], d, cfg.get("ffn_dim", 4 * d), cfg["num_hidden_layers"],
                   cfg["num_attention_heads"], maxpos, min(s, maxpos), 1e-5, -1 if pad is None else int(pad))

    def to_hf_config(self) -> dict:
        return {
            "architectures": ["OPTForCausalLM"], "model_type": "opt", "vocab_size": self.vocab_size,
            "hidden_size": self.hidden_size, "ffn_dim": self.intermediate_size,
            "num_hidden_layers": self.num_layers, "num_attention_heads": self.num_heads,
            "max_position_embeddings": self.max_positions, "word_embed_proj_dim": self.hidden_size,
            "do_layer_norm_before": True, "activation_function": "relu", "enable_bias": True,
            "layer_norm_elementwise_affine": True, "tie_word_embeddings": True, "dropout": 0.0,
            "attention_dropout": 0.0, "layerdrop": 0.0, "pad_token_id": self.pad_token_id,
            "bos_token_id": 2, "eos_token_id": 2, "torch_dtype": "bfloat16",
        }

    def c_fields(self) -> dict:
        return dict(vocab_size=self.vocab_size, hidden_size=self.hidden_size,
                    intermediate_size=self.intermediate_size, num_layers=self.num_layers,
                    num_heads=self.num_heads, num_kv_heads=self.num_heads, head_dim=self.head_dim,
                    max_seq_len=self.max_seq_len, rms_norm_eps=self.layer_norm_eps, rope_theta=0.0,
                    family=self.family, pad_token_id=self.pad_token_id, max_positions=self.max_positions)


@dataclass
class FalconArch:
    """tiiuae/falcon-7b family (HF models/falcon/modeling_falcon.py; the reference serves it from
    examples/falcon-7b-instruct/): multi-query attention (H query heads, one key/value head), parallel
    attention + MLP after one LayerNorm, rotate_half RoPE, exact GeLU, no biases, tied lm_head."""
    vocab_size: int
    hidden_size: int
    intermediate_size: int     # ffn_hidden_size (4 x hidden_size)
    num_layers: int
    num_heads: int
    max_seq_len: int = 2048
    layer_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    pad_token_id: int = -1
    num_kv_heads: int = 1
    family = FAMILY_FALCON

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_heads

    @classmethod
    def falcon_7b(cls, seq_len: int = 2048) -> "FalconArch":
        return cls(65024, 4544, 18176, 32, 71, seq_len)

    @classmethod
    def from_hf_config(cls, cfg: dict, seq_len: Optional[int] = None) -> "FalconArch":
        if cfg.get("model_type") != "falcon":
            raise ValueError(f"unsupported model_type {cfg.get('model_type')!r}")
        d, heads = cfg["hidden_size"], cfg["num_attention_heads"]
        _reject(cfg.get("alibi", False), "alibi positions")
        _reject(cfg.get("bias", False), "bias=true")
        _reject(cfg.get("new_decoder_architecture", False), "new_decoder_architecture (falcon-40b layout)")
        _reject(not cfg.get("parallel_attn", True), "parallel_attn=false")
        _reject(not cfg.get("multi_query", True), "multi_query=false")
        _reject(cfg.get("activation", "gelu") != "gelu", f"activation {cfg.get('activation')!r}")
        _reject(not cfg.get("tie_word_embeddings", True), "untied lm_head for a Falcon checkpoint")
        _reject((cfg.get("rope_scaling") or {}).get("rope_type", "default") != "default", "rope scaling")
        _reject((d // heads) not in (64, 128), "head_dim other than 64 / 128")
        rope = cfg.get("rope_parameters") or {}
        _reject(rope.get("rope_type", "default") != "default", "rope scaling")
        maxpos = cfg.get("max_position_embeddings", 2048)
        # FalconModel builds nn.Embedding(vocab, d) WITHOUT padding_idx (modeling_falcon.py:680): the pad row
        # gets its lookup gradient like every other row, whatever config.pad_token_id says
        return cls(cfg["vocab_size"], d, cfg.get("ffn_hidden_size") or 4 * d, cfg["num_hidden_layers"], heads,
                   min(seq_len or maxpos, maxpos), cfg.get("layer_norm_epsilon", 1e-5),
                   float(rope.get("rope_theta", cfg.get("rope_theta", 10000.0))), -1)

    def to_hf_config(self) -> dict:
        return {
            "architectures": ["FalconForCausalLM"], "model_type": "falcon", "vocab_size": self.vocab_size,
            "hidden_size": self.hidden_size, "ffn_hidden_size": self.intermediate_size,
            "num_hidden_layers": self.num_layers, "num_attention_heads": self.num_heads, "multi_query": True,
            "parallel_attn": True, "new_decoder_architecture": False, "bias": False, "alibi": False,
            "activation": "gelu", "layer_norm_epsilon": self.layer_norm_eps, "rope_theta": self.rope_theta,
            "max_position_embeddings": self.max_seq_len, "tie_word_embeddings": True, "hidden_dropout": 0.0,
            "attention_dropout": 0.0, "bos_token_id": 11, "eos_token_id": 11, "torch_dtype": "bfloat16",
        }

    def c_fields(self) -> dict:
        return dict(vocab_size=self.vocab_size, hidden_size=self.hidden_size,
                    intermediate_size=self.intermediate_size, num_layers=self.num_layers,
                    num_heads=self.num_heads, num_kv_heads=self.num_kv_heads, head_dim=self.head_dim,
                    max_seq_len=self.max_seq_len, rms_norm_eps=self.layer_norm_eps, rope_theta=self.rope_theta,
                    family=self.family, pad_token_id=self.pad_token_id, max_positions=0)


def arch_from_hf_config(cfg: dict, seq_len: Optional[int] = None):
    """config.json -> LlamaArch | OptArch | FalconArch; anything else (or any unimplemented variant) raises."""
    mt = cfg.get("model_type", "llama")
    if mt == "llama":
        return LlamaArch.from_hf_config(cfg, seq_len)
    if mt == "opt":
        return OptArch.from_hf_config(cfg, seq_len)
    if mt == "falcon":
        return FalconArch.from_hf_config(cfg, seq_len)
    raise ValueError(f"unsupported model_type {mt!r}: the fine-tune engine builds llama, opt and falcon")


def _as_i32(a) -> np.ndarray:
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.int32)


class Engine:
    """Owns a b200w context. Raises B200WError on any failure (no CPU fallback exists)."""

    def __init__(self, device: int = 0):
        self._lib = _lib.load()
        h = _lib.c_ctx()
        st = self._lib.b200w_create(device, C.byref(h))
        if st != 0:
            raise B200WError(st, (self._lib.b200w_last_error(None) or b"").decode())
        self._h = h
        self.arch = None   # LlamaArch | OptArch
        self.micro_batch = 0

    # -- plumbing -----------------------------------------------------------------------------
    def _check(self, st: int):
        if st != 0:
            raise B200WError(st, (self._lib.b200w_last_error(self._h) or b"").decode())

    @property
    def handle(self):
        return self._h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b200w_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        self._check(self._lib.b200w_sync(self._h))

    # -- model --------------------------------------------------------------------------------
    def init_model(self, arch, micro_batch: int = 1, training: bool = True,
                   max_grad_norm: float = 1.0, weight_decay: float = 0.0,
                   betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, shard_state: bool = False,
                   recompute: bool = False):
        """shard_state: keep fp32 master / Adam moments for 1/nranks of the parameters only (ZeRO-style;
        needs comm_init() first). Results equal the replicated mode.
        recompute: keep only every layer's input through the forward and re-run the layer in the backward
        (B200W_TRAIN_RECOMPUTE, Llama family): bit-identical results, ~10x less activation memory."""
        ca = _CArch(**arch.c_fields())
        hp = _CHParams()
        self._lib.b200w_default_hparams(C.byref(hp))
        hp.max_grad_norm, hp.weight_decay = max_grad_norm, weight_decay
        hp.beta1, hp.beta2, hp.eps = betas[0], betas[1], eps
        self._check(self._lib.b200w_model_init(self._h, C.byref(ca), C.byref(hp), micro_batch,
                                               ((2 if shard_state else 1) | (4 if recompute else 0)) if training else 0))
        self.arch, self.micro_batch = arch, micro_batch

    def params(self) -> Iterable[Tuple[str, Tuple[int, ...]]]:
        n = C.c_int64()
        self._check(self._lib.b200w_param_count(self._h, C.byref(n), None))
        buf = C.create_string_buffer(256)
        r, c = C.c_int64(), C.c_int64()
        for i in range(n.value):
            self._check(self._lib.b200w_param_info(self._h, i, buf, 256, C.byref(r), C.byref(c)))
            name = buf.value.decode()
            one_d = r.value == 1 or c.value == 1      # norm weights, LayerNorm parameters, biases
            yield name, ((r.value * c.value,) if one_d else (r.value, c.value))

    def load_tensor(self, name: str, arr: np.ndarray):
        """arr: float32, or uint16 holding raw bf16 bits."""
        arr = np.ascontiguousarray(arr)
        if arr.dtype == np.uint16:
            dt = _lib.BF16
        else:
            arr = arr.astype(np.float32, copy=False)
            dt = _lib.F32
        self._check(self._lib.b200w_load_tensor(self._h, name.encode(), arr.ctypes.data, dt, arr.size))

    def load_state_dict(self, sd: Dict[str, np.ndarray]):
        names = {n for n, _ in self.params()}
        missing = names - set(sd)
        if missing:
            raise KeyError(f"state dict lacks {sorted(missing)[:4]}... ({len(missing)} tensors)")
        for n in names:
            self.load_tensor(n, sd[n])

    def read_tensor(self, name: str, shape, bf16_bits: bool = False) -> np.ndarray:
        out = np.empty(shape, dtype=np.uint16 if bf16_bits else np.float32)
        self._check(self._lib.b200w_read_tensor(self._h, name.encode(), out.ctypes.data,
                                                _lib.BF16 if bf16_bits else _lib.F32, out.size))
        return out

    def read_state(self, name: str, shape, kind: str) -> np.ndarray:
        out = np.empty(shape, dtype=np.float32)
        k = {"master": 0, "grad": 1, "m": 2, "v": 3}[kind]
        self._check(self._lib.b200w_read_state(self._h, name.encode(), k, out.ctypes.data, out.size))
        return out

    def state_dict(self, bf16_bits: bool = False) -> Dict[str, np.ndarray]:
        return {n: self.read_tensor(n, s, bf16_bits) for n, s in self.params()}

    def init_random(self, seed: int = 0, std: float = 0.02):
        self._check(self._lib.b200w_init_random(self._h, seed, std))

    # -- data parallel ------------------------------------------------------------------------
    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(128)
        st = self._lib.b200w_comm_unique_id(buf)
        if st != 0:
            raise B200WError(st, (self._lib.b200w_last_error(None) or b"").decode())
        return buf.raw

    def comm_init(self, rank: int, nranks: int, uid: bytes):
        buf = C.create_string_buffer(uid, 128)
        self._check(self._lib.b200w_comm_init(self._h, rank, nranks, buf))

    # -- the hot path -------------------------------------------------------------------------
    def train_step(self, ids, labels, lr: float = 5e-5, positions=None) -> Tuple[float, float]:
        """ids/labels: [n_seqs, seq_len] host integer arrays (labels unshifted, -100 ignored).
        positions (optional, same shape): HF position_ids of packed documents (contract.pack_documents); each
        document then attends only to itself (b200w_train_step_docs).
        Runs fwd + loss + bwd + all-reduce + clip + AdamW; returns (loss, grad_norm)."""
        ids, labels = _as_i32(ids), _as_i32(labels)
        assert ids.shape == labels.shape and ids.shape[1] == self.arch.max_seq_len
        loss, gn = C.c_float(), C.c_float()
        if positions is None:
            self._check(self._lib.b200w_train_step(self._h, ids.ctypes.data, labels.ctypes.data,
                                                   ids.shape[0], lr, C.byref(loss), C.byref(gn)))
        else:
            pos = _as_i32(positions)
            assert pos.shape == ids.shape
            self._check(self._lib.b200w_train_step_docs(self._h, ids.ctypes.data, labels.ctypes.data,
                                                        pos.ctypes.data, ids.shape[0], lr, C.byref(loss),
                                                        C.byref(gn)))
        return loss.value, gn.value

    def train_step_resident(self, ids_dev_ptr: int, labels_dev_ptr: int, n_seqs: int, n_valid: int,
                            lr: float = 5e-5):
        """The same step on a batch already in HBM (raw device addresses); no host sync."""
        self._check(self._lib.b200w_train_step_resident(self._h, ids_dev_ptr, labels_dev_ptr, n_seqs,
                                                        n_valid, lr))

    def read_scalars(self) -> Tuple[float, float]:
        loss, gn = C.c_float(), C.c_float()
        self._check(self._lib.b200w_read_scalars(self._h, C.byref(loss), C.byref(gn)))
        return loss.value, gn.value

    def timer_start(self):
        self._check(self._lib.b200w_timer_start(self._h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        self._check(self._lib.b200w_timer_stop(self._h, C.byref(ms)))
        return ms.value

    def profile_gemm(self, enable: bool):
        self._check(self._lib.b200w_profile_gemm(self._h, 1 if enable else 0))

    def profile_read(self) -> Tuple[float, float, int]:
        ms, fl, n = C.c_double(), C.c_double(), C.c_int64()
        self._check(self._lib.b200w_profile_read(self._h, C.byref(ms), C.byref(fl), C.byref(n)))
        return ms.value, fl.value, n.value

    def forward_backward(self, ids, labels, positions=None) -> float:
        ids, labels = _as_i32(ids), _as_i32(labels)
        loss = C.c_float()
        if positions is None:
            self._check(self._lib.b200w_forward_backward(self._h, ids.ctypes.data, labels.ctypes.data,
                                                         ids.shape[0], C.byref(loss)))
        else:
            pos = _as_i32(positions)
            assert pos.shape == ids.shape
            self._check(self._lib.b200w_forward_backward_docs(self._h, ids.ctypes.data, labels.ctypes.data,
                                                              pos.ctypes.data, ids.shape[0], C.byref(loss)))
        return loss.value

    def forward(self, ids, labels=None, want_logits: bool = True, positions=None):
        """Returns (logits [T,V] float32 or None, nll [T] or None, loss or None)."""
        ids = _as_i32(ids)
        T = ids.size
        logits = np.empty((T, self.arch.vocab_size), dtype=np.float32) if want_logits else None
        lab = _as_i32(labels) if labels is not None else None
        nll = np.empty(T, dtype=np.float32) if lab is not None else None
        loss = C.c_float()
        outs = (logits.ctypes.data if want_logits else None, nll.ctypes.data if nll is not None else None,
                C.byref(loss))
        if positions is None:
            self._check(self._lib.b200w_forward(
                self._h, ids.ctypes.data, lab.ctypes.data if lab is not None else None, ids.shape[0], *outs))
        else:
            pos = _as_i32(positions)
            assert pos.shape == ids.shape
            self._check(self._lib.b200w_forward_docs(
                self._h, ids.ctypes.data, lab.ctypes.data if lab is not None else None, pos.ctypes.data,
                ids.shape[0], *outs))
        return logits, nll, (loss.value if lab is not None else None)

    def launch_count(self) -> int:
        return int(self._lib.b200w_launch_count(self._h))

    def device_bytes(self) -> int:
        return int(self._lib.b200w_device_bytes(self._h))
