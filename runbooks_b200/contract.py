"""Host-side halves of the substratus container contract that touch no GPU: parameters, the
dataset → packed-sequence path, and HF-format checkpoint I/O (SURVEY.md §8 rows a1, a2, a13).

Contract (reference): docs/container-contract.md —
  WORKDIR /content (:7); /content/data, /content/model, /content/artifacts (:27-32);
  /content/params.json + PARAM_<UPPER> env (:36-48).
What the controller really mounts: internal/controller/model_controller.go:344 (params),
:348-357 (artifacts RW), :359-370 (dataset RO), :372-383 (base model RO);
params.json is json.MarshalIndent of spec.params or `{}` (params_reconciler.go:28-68) and its
values are int-or-string (api/v1/model_types.go:35).
"""
from __future__ import annotations

import glob
import json
import math
import os
import shutil
from dataclasses import dataclass, field
from typing import Dict, Iterable, Iterator, List, Optional, Tuple

import numpy as np

CONTENT = os.environ.get("B200W_CONTENT_DIR", "/content")


# ------------------------------------------------------------------------------------------------
# parameters
# ------------------------------------------------------------------------------------------------
@dataclass
class TrainParams:
    """Names follow transformers.TrainingArguments, which the reference's examples point at
    (examples/llama2-7b/finetuned-model.yaml:11-16); defaults are the TrainingArguments defaults
    (SURVEY.md §8 a12). `epochs` is the alias examples/facebook-opt-125m/finetuned-model.yaml uses."""
    num_train_epochs: float = 3.0
    max_steps: int = -1
    per_device_train_batch_size: int = 8
    gradient_accumulation_steps: int = 1
    learning_rate: float = 5e-5
    weight_decay: float = 0.0
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_epsilon: float = 1e-8
    max_grad_norm: float = 1.0
    lr_scheduler_type: str = "linear"
    warmup_steps: float = 0.0         # >= 1: exact steps; in [0, 1): ratio of the total (training_args.py:789, :2068-2075)
    optim: str = "adamw_torch_fused"   # the default with torch >= 2.8 (training_args.py:797-806); same AdamW formula as adamw_torch
    label_smoothing_factor: float = 0.0
    average_tokens_across_devices: str = "true"
    gradient_checkpointing: str = "false"   # TrainingArguments.gradient_checkpointing: activation recomputation (same results)
    padding_free: str = "false"       # TRL SFTConfig.padding_free: each packed record attends only to itself (pack_documents)
    save_steps: int = 500
    logging_steps: int = 1
    seed: int = 42
    max_seq_length: int = 0           # 0: min(4096, model max_position_embeddings), multiple of 128
    prompt_template: str = "{prompt}{completion}"
    extra: Dict[str, object] = field(default_factory=dict)

    # warmup_ratio: deprecated TrainingArguments alias that is assigned into warmup_steps (training_args.py:1472-1474)
    ALIASES = {"epochs": "num_train_epochs", "lr": "learning_rate", "batch_size": "per_device_train_batch_size",
               "warmup_ratio": "warmup_steps"}


def _coerce(value, target_type):
    """params.json values are JSON numbers OR strings (intstr.IntOrString)."""
    if target_type is str:
        return str(value)
    if isinstance(value, str):
        value = value.strip()
        return target_type(float(value)) if target_type is int else target_type(value)
    return target_type(value)


def load_params(path: Optional[str] = None, environ: Optional[Dict[str, str]] = None) -> TrainParams:
    """/content/params.json first, PARAM_<UPPER> environment variables override
    (container-contract.md:36-48; the controller of this reference version only writes the file)."""
    path = path or os.path.join(CONTENT, "params.json")
    environ = os.environ if environ is None else environ
    raw: Dict[str, object] = {}
    if os.path.exists(path):
        with open(path) as f:
            txt = f.read().strip()
        raw = json.loads(txt) if txt else {}
        if not isinstance(raw, dict):
            raise ValueError(f"{path} must hold a JSON object, got {type(raw).__name__}")
    for k, v in environ.items():
        if k.startswith("PARAM_") and len(k) > 6:
            raw[k[6:].lower()] = v
    p = TrainParams()
    fields = {f for f in p.__dataclass_fields__ if f != "extra"}
    for k, v in raw.items():
        k2 = TrainParams.ALIASES.get(k, k)
        if k2 in fields:
            try:
                setattr(p, k2, _coerce(v, type(getattr(p, k2))))
            except (TypeError, ValueError) as e:
                raise ValueError(f"param {k!r}: cannot read {v!r} as {type(getattr(p, k2)).__name__}") from e
        else:
            p.extra[k] = v
    # TrainingArguments that change the arithmetic and are not implemented must fail the Job (exit 1 is the
    # whole protocol) instead of training something else and reporting success; everything else that is
    # unknown lands in `extra` and is listed in the worker's start event.
    if p.lr_scheduler_type != "linear":
        raise ValueError("only lr_scheduler_type=linear (the TrainingArguments default) is implemented")
    if p.optim not in ("adamw_torch", "adamw_torch_fused"):
        raise ValueError(f"optim={p.optim!r} is not implemented (AdamW, the TrainingArguments default, is)")
    if p.label_smoothing_factor != 0.0:
        raise ValueError("label_smoothing_factor != 0 is not implemented")
    if str(p.average_tokens_across_devices).strip().lower() not in ("true", "1"):
        raise ValueError("average_tokens_across_devices=false is not implemented: the N-rank step always "
                         "normalises by the global target count (the TrainingArguments default)")
    if str(p.gradient_checkpointing).strip().lower() not in ("true", "false", "1", "0"):
        raise ValueError(f"gradient_checkpointing={p.gradient_checkpointing!r}: expected true or false")
    if str(p.padding_free).strip().lower() not in ("true", "false", "1", "0"):
        raise ValueError(f"padding_free={p.padding_free!r}: expected true or false")
    if p.warmup_steps < 0:
        raise ValueError("warmup_steps must be >= 0")
    if p.gradient_accumulation_steps < 1 or p.per_device_train_batch_size < 1:
        raise ValueError("batch sizes must be >= 1")
    return p


def wants_recompute(p: TrainParams) -> bool:
    return str(p.gradient_checkpointing).strip().lower() in ("true", "1")


def wants_padding_free(p: TrainParams) -> bool:
    return str(p.padding_free).strip().lower() in ("true", "1")


def warmup_steps_for(total_steps: int, warmup_steps: float) -> int:
    """TrainingArguments.get_warmup_steps (training_args.py:2068-2075)."""
    return int(warmup_steps) if warmup_steps >= 1 else int(math.ceil(total_steps * warmup_steps))


def linear_lr(step_index: int, total_steps: int, base_lr: float, warmup: int = 0) -> float:
    """transformers.get_linear_schedule_with_warmup lambda, evaluated for optimizer step
    `step_index` (0-based)."""
    if step_index < warmup:
        return base_lr * step_index / max(1, warmup)
    return base_lr * max(0.0, (total_steps - step_index) / max(1, total_steps - warmup))


# ------------------------------------------------------------------------------------------------
# dataset: jsonl {prompt, completion} -> template -> tokens -> packed [n, S] sequences
# ------------------------------------------------------------------------------------------------
def iter_records(data_dir: str) -> Iterator[Dict[str, str]]:
    """Every *.jsonl / *.json file under /content/data (the dataset loader's artifacts dir,
    examples/datasets/k8s-instructions.yaml:6-7)."""
    files = sorted(glob.glob(os.path.join(data_dir, "**", "*.jsonl"), recursive=True) +
                   glob.glob(os.path.join(data_dir, "**", "*.json"), recursive=True))
    if not files:
        raise FileNotFoundError(f"no .jsonl/.json dataset files under {data_dir}")
    for fn in files:
        with open(fn) as f:
            head = f.read(1)
            f.seek(0)
            if head == "[":
                for rec in json.load(f):
                    yield rec
            else:
                for line in f:
                    line = line.strip()
                    if line:
                        yield json.loads(line)


def render(rec: Dict[str, str], template: str) -> str:
    """`{prompt}` / `{completion}` substitution
    (examples/falcon-7b-instruct/finetuned-model-custom-prompt.yaml:15-20). Records with a single
    `text` field pass through unchanged."""
    if "text" in rec and "prompt" not in rec:
        return str(rec["text"])
    return template.replace("{prompt}", str(rec.get("prompt", ""))).replace(
        "{completion}", str(rec.get("completion", "")))


class Tokenizer:
    """tokenizer.json (HF `tokenizers`) from the model directory; nothing else is needed to turn
    text into ids, so `transformers` is not imported by the worker."""

    def __init__(self, model_dir: str):
        from tokenizers import Tokenizer as _T

        path = os.path.join(model_dir, "tokenizer.json")
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} not found (only tokenizer.json tokenizers are supported)")
        self.tok = _T.from_file(path)
        self.eos_id = self._special(model_dir, "eos_token", ("</s>", "<|endoftext|>"))
        self.bos_id = self._special(model_dir, "bos_token", ("<s>",))

    def _special(self, model_dir, key, fallbacks):
        names = []
        cfg = os.path.join(model_dir, "tokenizer_config.json")
        if os.path.exists(cfg):
            v = json.load(open(cfg)).get(key)
            if isinstance(v, dict):
                v = v.get("content")
            if v:
                names.append(v)
        for n in names + list(fallbacks):
            i = self.tok.token_to_id(n)
            if i is not None:
                return i
        return None

    def encode(self, text: str) -> List[int]:
        return self.tok.encode(text, add_special_tokens=False).ids

    def decode(self, ids: Iterable[int]) -> str:
        return self.tok.decode(list(ids))


def pack_sequences(docs: Iterable[List[int]], seq_len: int, bos_id: Optional[int],
                   eos_id: Optional[int]) -> Tuple[np.ndarray, np.ndarray]:
    """Concatenate [bos] doc [eos] streams and cut them into rows of exactly `seq_len` tokens
    (the metric's "packed 4096-token sequences"). labels = ids (train on all tokens — the HF
    causal-LM default); the ragged tail is padded with eos and its labels set to -100."""
    stream: List[int] = []
    for d in docs:
        if bos_id is not None:
            stream.append(bos_id)
        stream.extend(d)
        if eos_id is not None:
            stream.append(eos_id)
    if not stream:
        raise ValueError("dataset is empty after tokenisation")
    n = (len(stream) + seq_len - 1) // seq_len
    ids = np.full(n * seq_len, eos_id if eos_id is not None else 0, dtype=np.int32)
    labels = np.full(n * seq_len, -100, dtype=np.int32)
    ids[: len(stream)] = stream
    labels[: len(stream)] = stream
    return ids.reshape(n, seq_len), labels.reshape(n, seq_len)


def pack_documents(docs: Iterable[List[int]], seq_len: int, bos_id: Optional[int],
                   eos_id: Optional[int]) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Padding-free packing (HF DataCollatorWithFlattening, TRL padding_free): the token stream and row cut of
    pack_sequences, plus position_ids that restart at 0 at every document start, which makes each document attend
    only to itself (b200w_train_step_docs). A document cut by a row end continues in the next row as a new
    document, so every position is < seq_len. As the collator does, the label of every document start (row starts
    included) is -100. The eos padding of the last row is one more document, with labels -100.
    Returns (ids, labels, positions), each int32 [n, seq_len]."""
    stream: List[int] = []
    starts: List[int] = []
    for d in docs:
        piece = ([bos_id] if bos_id is not None else []) + list(d) + ([eos_id] if eos_id is not None else [])
        if piece:
            starts.append(len(stream))
            stream.extend(piece)
    if not stream:
        raise ValueError("dataset is empty after tokenisation")
    n = (len(stream) + seq_len - 1) // seq_len
    total = n * seq_len
    ids = np.full(total, eos_id if eos_id is not None else 0, dtype=np.int32)
    ids[: len(stream)] = stream
    is_start = np.zeros(total, dtype=bool)
    is_start[starts] = True
    is_start[::seq_len] = True
    if len(stream) < total:
        is_start[len(stream)] = True
    labels = ids.copy()
    labels[len(stream):] = -100
    labels[is_start] = -100
    idx = np.arange(total)
    positions = (idx - np.maximum.accumulate(np.where(is_start, idx, 0))).astype(np.int32)
    return ids.reshape(n, seq_len), labels.reshape(n, seq_len), positions.reshape(n, seq_len)


# ------------------------------------------------------------------------------------------------
# HF-format checkpoints (safetensors): /content/model in, /content/artifacts out
# ------------------------------------------------------------------------------------------------
def read_hf_config(model_dir: str) -> dict:
    with open(os.path.join(model_dir, "config.json")) as f:
        return json.load(f)


def iter_safetensors(model_dir: str) -> Iterator[Tuple[str, np.ndarray]]:
    """Yields (name, array) with bf16 tensors as uint16 bit patterns and everything else as
    float32, one tensor at a time (a 7B checkpoint is never fully resident on the host)."""
    import torch
    from safetensors import safe_open

    files = sorted(glob.glob(os.path.join(model_dir, "*.safetensors")))
    if not files:
        raise FileNotFoundError(f"no *.safetensors under {model_dir}")
    for fn in files:
        with safe_open(fn, framework="pt", device="cpu") as f:
            for name in f.keys():
                t = f.get_tensor(name)
                if t.dtype == torch.bfloat16:
                    yield name, t.contiguous().view(torch.uint16).numpy()
                else:
                    yield name, t.float().contiguous().numpy()


def canonical_tensor_name(name: str, hf_config: dict) -> str:
    """Checkpoint key -> the key of the *ForCausalLM state dict. OPT checkpoints saved from the bare
    OPTModel (and the original metaseq conversions) lack the leading "model."."""
    if hf_config.get("model_type") == "opt" and name.startswith("decoder."):
        return "model." + name
    return name


def is_ignorable_tensor(name: str, hf_config: dict) -> bool:
    """Tensors a checkpoint may hold that carry no trainable arithmetic: rotary inv_freq buffers, and
    the duplicate lm_head.weight of a tied model."""
    if name.endswith("rotary_emb.inv_freq"):
        return True
    tied = hf_config.get("tie_word_embeddings", hf_config.get("model_type") in ("opt", "falcon"))
    return bool(tied) and name == "lm_head.weight"


MAX_SHARD_BYTES = 5 * 1000 ** 3  # save_pretrained's default max_shard_size="5GB"


def plan_shards(sizes: Dict[str, int]) -> List[List[str]]:
    """save_pretrained's greedy sharding over the tensors in order: a new shard starts when the next
    tensor would take the current one past MAX_SHARD_BYTES."""
    shards: List[List[str]] = [[]]
    cur = 0
    for name, nbytes in sizes.items():
        if cur and cur + nbytes > MAX_SHARD_BYTES:
            shards.append([])
            cur = 0
        shards[-1].append(name)
        cur += nbytes
    return shards


def save_hf_checkpoint(out_dir: str, hf_config: dict, tensors: Iterable[Tuple[str, np.ndarray]],
                       copy_from: Optional[str] = None, sizes: Optional[Dict[str, int]] = None) -> List[str]:
    """Writes config.json + bf16 safetensors shards (+ model.safetensors.index.json when there is
    more than one) in the layout `save_pretrained` produces, so that the Server the controller
    later points at this directory (server_controller.go:184-193) — or AutoModelForCausalLM —
    can load it. `tensors` yields (name, uint16 bf16-bit array) in the order of `sizes` (name ->
    bytes); with `sizes` every shard is written as soon as its last tensor has arrived, so at most
    one 5 GB shard is resident on the host. Tokenizer files are copied through from the base
    model directory."""
    import torch
    from safetensors.torch import save_file

    os.makedirs(out_dir, exist_ok=True)
    if sizes is None:
        tensors = list(tensors)
        sizes = {n: a.size * 2 for n, a in tensors}
    plan = plan_shards(sizes)
    written: List[str] = []
    weight_map: Dict[str, str] = {}
    it = iter(tensors)
    for i, names in enumerate(plan):
        shard: Dict[str, "torch.Tensor"] = {}
        for want in names:
            name, arr = next(it)
            assert name == want, f"tensor order differs from the shard plan: {name} != {want}"
            assert arr.dtype == np.uint16, "checkpoints are written in bf16"
            shard[name] = torch.from_numpy(np.ascontiguousarray(arr)).view(torch.bfloat16)
        fn = "model.safetensors" if len(plan) == 1 else f"model-{i + 1:05d}-of-{len(plan):05d}.safetensors"
        save_file(shard, os.path.join(out_dir, fn), metadata={"format": "pt"})
        written.append(fn)
        weight_map.update({k: fn for k in shard})
        del shard
    if len(plan) > 1:
        with open(os.path.join(out_dir, "model.safetensors.index.json"), "w") as f:
            json.dump({"metadata": {"total_size": int(sum(sizes.values()))}, "weight_map": weight_map}, f, indent=2)
    cfg = dict(hf_config)
    cfg["torch_dtype"] = "bfloat16"
    with open(os.path.join(out_dir, "config.json"), "w") as f:
        json.dump(cfg, f, indent=2)
    if copy_from:
        for pat in ("tokenizer*", "special_tokens_map.json", "generation_config.json", "vocab.*", "merges.txt"):
            for src in glob.glob(os.path.join(copy_from, pat)):
                if os.path.isfile(src):
                    shutil.copy2(src, os.path.join(out_dir, os.path.basename(src)))
    return written
