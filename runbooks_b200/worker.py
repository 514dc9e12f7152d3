"""Container entry point of the H100 fine-tune worker — what the trainer Job's container "model"
runs (internal/controller/model_controller.go:330-337: image + command from the Model spec).

    python -m runbooks_b200.worker train         # ENTRYPOINT of the trainer image

Contract honoured (docs/container-contract.md; SURVEY.md §8b):
  in   /content/params.json (+ PARAM_* env), /content/model (HF dir, RO), /content/data (RO)
  out  /content/artifacts/{config.json, model*.safetensors, tokenizer files, checkpoint-N/...}
  exit 0 => Job Complete => Model.status.ready (internal/controller/utils.go:37-49);
  any failure => non-zero exit => JobFailed, no retry for GPU jobs (model_controller.go:294-303)
  logs: one JSON line per optimiser step on stdout (what `sub run` tails).

All N GPUs of the Pod arrive in this one container (internal/resources/resources.go:45-46), so
the worker forks one rank per visible GPU itself; ranks shard the batch and meet in a single
NCCL gradient all-reduce per step inside libb200w.so.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time
import traceback
from typing import List

import numpy as np

from . import contract
from .contract import TrainParams


def log(**kv):
    print(json.dumps(kv), flush=True)


def visible_gpus() -> int:
    env = os.environ.get("B200W_NUM_GPUS")
    if env:
        return int(env)
    cvd = os.environ.get("CUDA_VISIBLE_DEVICES")
    if cvd is not None and cvd.strip() != "":
        return len([x for x in cvd.split(",") if x.strip()])
    import glob
    return max(1, len(glob.glob("/dev/nvidia[0-9]*")))


def _records(params: TrainParams, model_dir: str, data_dir: str):
    tok = contract.Tokenizer(model_dir)
    docs = (tok.encode(contract.render(r, params.prompt_template)) for r in contract.iter_records(data_dir))
    return docs, tok


def build_dataset(params: TrainParams, model_dir: str, data_dir: str, seq_len: int):
    docs, tok = _records(params, model_dir, data_dir)
    return contract.pack_sequences(docs, seq_len, tok.bos_id, tok.eos_id)


def build_documents(params: TrainParams, model_dir: str, data_dir: str, seq_len: int):
    """padding_free: (ids, labels, positions) of contract.pack_documents."""
    docs, tok = _records(params, model_dir, data_dir)
    return contract.pack_documents(docs, seq_len, tok.bos_id, tok.eos_id)


def plan_steps(n_seqs: int, params: TrainParams, world: int):
    per_step = params.per_device_train_batch_size * params.gradient_accumulation_steps * world
    steps_per_epoch = max(1, n_seqs // per_step)   # drop_last, as HF's sampler does for DP shards
    total = params.max_steps if params.max_steps > 0 else int(math.ceil(params.num_train_epochs * steps_per_epoch))
    return per_step, steps_per_epoch, max(1, total)


def train_rank(rank: int, world: int, uid: bytes, content: str) -> None:
    from .engine import Engine, LlamaArch, arch_from_hf_config

    model_dir, data_dir = os.path.join(content, "model"), os.path.join(content, "data")
    out_dir = os.path.join(content, "artifacts")
    params = contract.load_params(os.path.join(content, "params.json"))
    hf_cfg = contract.read_hf_config(model_dir)
    seq_len = params.max_seq_length or min(4096, int(hf_cfg.get("max_position_embeddings", 4096)))
    seq_len = min(seq_len, int(hf_cfg.get("max_position_embeddings", seq_len)))
    if seq_len % 128:
        raise ValueError(f"max_seq_length {seq_len} must be a multiple of 128")
    arch = arch_from_hf_config(hf_cfg, seq_len)   # llama | opt; unimplemented variants raise
    padding_free = contract.wants_padding_free(params)
    if padding_free and not isinstance(arch, LlamaArch):
        raise ValueError(f"padding_free is implemented for the Llama family only, not {hf_cfg.get('model_type')!r}")

    t0 = time.time()
    eng = Engine(rank)
    eng.init_model(arch, micro_batch=1, training=True, max_grad_norm=params.max_grad_norm,
                   weight_decay=params.weight_decay, betas=(params.adam_beta1, params.adam_beta2),
                   eps=params.adam_epsilon, recompute=contract.wants_recompute(params))   # Llama family; others raise
    wanted = {n for n, _ in eng.params()}
    seen, unused = set(), []
    t_load, load_bytes = time.time(), 0
    for name, arr in contract.iter_safetensors(model_dir):
        name = contract.canonical_tensor_name(name, hf_cfg)
        if name in wanted:
            eng.load_tensor(name, arr)
            seen.add(name)
            load_bytes += arr.nbytes
        elif not contract.is_ignorable_tensor(name, hf_cfg):
            unused.append(name)
    if wanted - seen:
        raise KeyError(f"checkpoint lacks {sorted(wanted - seen)[:3]} ... ({len(wanted - seen)} tensors)")
    if unused:
        # a tensor the engine does not consume (a bias on a "bias-free" layer, an adapter, ...) means the
        # checkpoint's arithmetic is not the one that would be trained: fail the Job instead
        raise ValueError(f"checkpoint holds tensors this engine does not use: {sorted(unused)[:4]} "
                         f"({len(unused)} tensors)")
    load_seconds = time.time() - t_load
    if world > 1:
        eng.comm_init(rank, world, uid)

    if padding_free:
        ids, labels, positions = build_documents(params, model_dir, data_dir, seq_len)
    else:
        (ids, labels), positions = build_dataset(params, model_dir, data_dir, seq_len), None
    per_step, steps_per_epoch, total_steps = plan_steps(len(ids), params, world)
    if len(ids) < per_step:  # tiny datasets: repeat rows so that one full step exists
        reps = (per_step + len(ids) - 1) // len(ids)
        ids, labels = np.tile(ids, (reps, 1)), np.tile(labels, (reps, 1))
        if positions is not None:
            positions = np.tile(positions, (reps, 1))
    per_rank = per_step // world
    warmup = contract.warmup_steps_for(total_steps, params.warmup_steps)
    if rank == 0:
        log(event="start", model=hf_cfg.get("_name_or_path", hf_cfg.get("model_type", "llama")),
            params=int(sum(np.prod(s) for _, s in eng.params())),
            checkpoint_read_gb_per_s=round(load_bytes / 1e9 / max(load_seconds, 1e-9), 3),
            sequences=int(len(ids)), seq_len=seq_len, world_size=world, total_steps=total_steps,
            global_batch=per_step, load_seconds=round(time.time() - t0, 2), device_gb=round(eng.device_bytes() / 1e9, 2),
            warmup_steps=warmup, ignored_params=sorted(params.extra), padding_free=padding_free,
            documents=int((positions == 0).sum()) if positions is not None else None)

    rng = np.random.default_rng(params.seed)
    order: List[int] = []
    step = 0
    t_last = time.time()
    while step < total_steps:
        if len(order) < per_step:
            order = list(rng.permutation(len(ids)))       # same permutation on every rank (same seed)
        batch, order = order[:per_step], order[per_step:]
        mine = batch[rank::world]                           # SURVEY.md §8e: rank r takes sequences [r::N]
        lr = contract.linear_lr(step, total_steps, params.learning_rate, warmup)
        if positions is None:
            loss, gnorm = eng.train_step(ids[mine], labels[mine], lr=lr)
        else:
            loss, gnorm = eng.train_step(ids[mine], labels[mine], lr=lr, positions=positions[mine])
        step += 1
        if rank == 0 and step % max(1, params.logging_steps) == 0:
            now = time.time()
            log(step=step, loss=round(loss, 5), grad_norm=round(gnorm, 5), learning_rate=lr,
                epoch=round(step / steps_per_epoch, 4),
                tokens_per_second=round(per_step * seq_len * max(1, params.logging_steps) / max(now - t_last, 1e-9), 1))
            t_last = now
        if not math.isfinite(loss):
            raise FloatingPointError(f"loss is {loss} at step {step}")
        if rank == 0 and params.save_steps > 0 and step % params.save_steps == 0 and step < total_steps:
            save(eng, hf_cfg, os.path.join(out_dir, f"checkpoint-{step}"), model_dir, step)
    if rank == 0:
        save(eng, hf_cfg, out_dir, model_dir, step)
        log(event="done", steps=step, seconds=round(time.time() - t0, 2))
    eng.close()


def save(eng, hf_cfg, out_dir, model_dir, step):
    t = time.time()
    plist = list(eng.params())
    sizes = {n: int(np.prod(s)) * 2 for n, s in plist}
    files = contract.save_hf_checkpoint(
        out_dir, hf_cfg, ((n, eng.read_tensor(n, s, bf16_bits=True)) for n, s in plist), copy_from=model_dir,
        sizes=sizes)
    with open(os.path.join(out_dir, "trainer_state.json"), "w") as f:
        json.dump({"global_step": step}, f)
    secs = time.time() - t
    log(event="save", dir=out_dir, files=files, seconds=round(secs, 2),
        write_gb_per_s=round(sum(sizes.values()) / 1e9 / max(secs, 1e-9), 3))


def _rank_main(rank, world, uid, content, q):
    try:
        train_rank(rank, world, uid, content)
        q.put((rank, 0, ""))
    except BaseException:  # noqa: BLE001 — the exit code is the whole failure protocol
        q.put((rank, 1, traceback.format_exc()))
        # deliver the report, then leave WITHOUT interpreter teardown: destructors would shut NCCL /
        # CUDA down on a dead context and can block while the peers sit in a collective
        q.close()
        q.join_thread()
        os._exit(1)


def train(content: str) -> int:
    world = visible_gpus()
    if world == 1:
        train_rank(0, 1, b"", content)
        return 0
    import multiprocessing as mp

    from .engine import Engine  # noqa: F401  (fail early if the library is missing)
    from . import _lib
    import ctypes as C

    buf = C.create_string_buffer(128)
    if _lib.load().b200w_comm_unique_id(buf) != 0:
        raise RuntimeError("NCCL unique id: " + (_lib.load().b200w_last_error(None) or b"").decode())
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(r, world, buf.raw, content, q)) for r in range(world)]
    for p in procs:
        p.start()
    return supervise(procs, q)


def supervise(procs, q, poll: float = 0.25, grace: float = 10.0) -> int:
    """Waits for every rank's (rank, code, traceback) report. One rank down means that the
    collective can never complete, so the others are terminated at once -- also when a rank died
    WITHOUT reporting (device fault in a C call, OOM kill): its exit code is the report. Ranks
    that ignore SIGTERM (blocked in a driver call) are killed after `grace` seconds."""
    import queue as queue_mod

    reported, failed = set(), 0
    while len(reported) < len(procs) and not failed:
        try:
            rank, code, tb = q.get(timeout=poll)
            reported.add(rank)
            if code:
                failed += 1
                sys.stderr.write(f"[rank {rank}] failed:\n{tb}\n")
        except queue_mod.Empty:
            for r, p in enumerate(procs):
                if r not in reported and p.exitcode is not None:  # gone without a word
                    reported.add(r)
                    if p.exitcode != 0:
                        failed += 1
                        sys.stderr.write(f"[rank {r}] died with exit code {p.exitcode} and no report\n")
    if failed:
        for p in procs:
            if p.is_alive():
                p.terminate()
    deadline = time.time() + grace
    for p in procs:
        p.join(max(0.0, deadline - time.time()) if failed else None)
        if p.is_alive():
            p.kill()
            p.join()
    return 1 if failed or any(p.exitcode for p in procs) else 0


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="runbooks_b200.worker")
    ap.add_argument("mode", choices=["train"], help="train: the Model (trainer) Job")
    ap.add_argument("--content", default=contract.CONTENT, help="contract root (default /content)")
    a = ap.parse_args(argv)
    try:
        return train(a.content)
    except BaseException:  # noqa: BLE001
        traceback.print_exc()
        log(event="failed", error=traceback.format_exc().strip().splitlines()[-1])
        return 1


if __name__ == "__main__":
    sys.exit(main())
