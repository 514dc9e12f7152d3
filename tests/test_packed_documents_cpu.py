"""Padding-free packing on the host (no GPU): contract.pack_documents against the real HF
DataCollatorWithFlattening, the padding_free parameter, the worker's refusal of families without document
attention, and the position-aware CPU oracle against tests/golden/llama_tiny_packed.npz (the real
LlamaForCausalLM, tools/make_packed_golden.py)."""
import json

import numpy as np
import pytest
import torch

from runbooks_b200 import contract, worker
from tests.test_contract import _tiny_model_dir
from tests.test_worker_host_cpu import CALLS, StubEngine
from util import rel_err

BOS, EOS = 1, 2


def _docs(lengths, seed=0):
    rng = np.random.default_rng(seed)
    return [list(rng.integers(3, 100, size=n)) for n in lengths]


def test_pack_documents_matches_data_collator_with_flattening():
    """Documents that fit in a row: input_ids, labels and position_ids are the collator's, row by row."""
    from transformers import DataCollatorWithFlattening

    S = 64
    # rows of exactly S tokens: [bos] doc [eos] pieces of 20 + 30 + 14, then 40 + 24
    docs = _docs([18, 28, 12, 38, 22], seed=1)
    ids, labels, pos = contract.pack_documents(docs, S, BOS, EOS)
    assert ids.shape == labels.shape == pos.shape == (2, S)
    coll = DataCollatorWithFlattening(return_tensors="np")
    pieces = [[BOS] + d + [EOS] for d in docs]
    for r, row in enumerate((pieces[:3], pieces[3:])):
        want = coll([{"input_ids": p, "labels": p} for p in row])
        assert np.array_equal(ids[r], want["input_ids"][0])
        assert np.array_equal(labels[r], want["labels"][0])
        assert np.array_equal(pos[r], want["position_ids"][0])


def test_row_cut_documents_restart_and_tail_padding_is_ignored():
    S = 32
    docs = _docs([10, 40, 5], seed=2)               # pieces of 12, 42, 7 tokens: 61 of 64
    ids, labels, pos = contract.pack_documents(docs, S, BOS, EOS)
    flat_pos, flat_lab = pos.reshape(-1), labels.reshape(-1)
    starts = [0, 12, 32, 54, 61]                    # documents, the row cut at 32, the eos padding at 61
    assert list(np.flatnonzero(flat_pos == 0)) == starts
    assert (flat_lab[starts] == -100).all()
    assert (flat_lab[61:] == -100).all() and (ids.reshape(-1)[61:] == EOS).all()
    assert pos.max() < S
    # every position is 0 or the previous one + 1, and each row starts at 0
    assert (pos[:, 0] == 0).all()
    d = np.diff(pos, axis=1)
    assert ((d == 1) | (pos[:, 1:] == 0)).all()
    # the same token stream and row cut as pack_sequences, whose output keeps its meaning
    ids_s, labels_s = contract.pack_sequences(docs, S, BOS, EOS)
    assert np.array_equal(ids, ids_s)
    stream = np.concatenate([[BOS] + d + [EOS] for d in docs])
    assert np.array_equal(labels_s.reshape(-1)[:61], stream) and (labels_s.reshape(-1)[61:] == -100).all()
    # outside document starts and padding, the labels are the ids, as with pack_sequences
    keep = flat_lab != -100
    assert np.array_equal(flat_lab[keep], labels_s.reshape(-1)[keep])


def test_padding_free_param(tmp_path):
    for value, want in (("true", True), (True, True), ("1", True), ("false", False), (False, False)):
        (tmp_path / "params.json").write_text(json.dumps({"padding_free": value}))
        p = contract.load_params(str(tmp_path / "params.json"), environ={})
        assert contract.wants_padding_free(p) is want and "padding_free" not in p.extra
    assert not contract.wants_padding_free(contract.load_params(str(tmp_path / "none.json"), environ={}))
    (tmp_path / "params.json").write_text(json.dumps({"padding_free": "maybe"}))
    with pytest.raises(ValueError, match="padding_free"):
        contract.load_params(str(tmp_path / "params.json"), environ={})


@pytest.fixture()
def content(tmp_path, monkeypatch):
    CALLS.clear()
    _tiny_model_dir(tmp_path)
    (tmp_path / "data").mkdir()
    rng = np.random.default_rng(4)
    with open(tmp_path / "data" / "train.jsonl", "w") as f:
        for _ in range(60):
            w = [f"w{i}" for i in rng.integers(0, 250, size=int(rng.integers(4, 40)))]
            f.write(json.dumps({"prompt": " ".join(w[:3]), "completion": " ".join(w[3:])}) + "\n")
    import runbooks_b200.engine as eng_mod
    monkeypatch.setattr(eng_mod, "Engine", StubEngine)
    return tmp_path


def test_worker_trains_padding_free_with_positions(content, capsys, monkeypatch):
    steps = []

    def train_step(self, ids, labels, lr=0.0, positions=None):
        steps.append((np.array(ids), np.array(labels), positions))
        return 2.0, 1.0

    monkeypatch.setattr(StubEngine, "train_step", train_step)
    (content / "params.json").write_text(json.dumps(dict(max_steps=2, per_device_train_batch_size=2,
                                                         max_seq_length=128, save_steps=0, padding_free="true")))
    worker.train_rank(0, 1, b"", str(content))
    assert len(steps) == 2
    for ids, labels, pos in steps:
        assert pos is not None and pos.shape == ids.shape == (2, 128)
        assert (labels[pos == 0] == -100).all()
    start = [json.loads(l) for l in capsys.readouterr().out.splitlines() if l.startswith("{")][0]
    assert start["event"] == "start" and start["padding_free"] is True and start["documents"] >= 60


@pytest.mark.parametrize("family", ["opt", "falcon"])
def test_worker_refuses_padding_free_without_document_attention(content, family):
    from runbooks_b200.engine import FalconArch, OptArch
    arch = OptArch(256, 256, 1024, 2, 2, 2048, 128) if family == "opt" else FalconArch(256, 256, 1024, 2, 2, 128)
    (content / "model" / "config.json").write_text(json.dumps(arch.to_hf_config()))
    (content / "params.json").write_text(json.dumps(dict(max_steps=1, max_seq_length=128, padding_free=True)))
    with pytest.raises(ValueError, match="padding_free"):
        worker.train_rank(0, 1, b"", str(content))
    assert not CALLS   # failed before any engine existed


def test_oracle_with_positions_reproduces_hf_packed_golden():
    import packed_oracle as P
    from oracle import llama_oracle as O

    fx = np.load("tests/golden/llama_tiny_packed.npz")
    a = O.Arch(*[int(x) for x in fx["arch"]], *[float(x) for x in fx["arch_f"]])
    params = O.seeded_params(a, int(fx["seed"]))
    r = P.forward_backward(params, fx["ids"], fx["labels"], fx["positions"], a)
    rows, stride = fx["logit_rows"], int(fx["sample_stride"])
    assert rel_err(r["logits"].reshape(-1, a.vocab_size)[rows], fx["logits"]) < 1e-5
    assert abs(r["loss"] - float(fx["loss"])) < 1e-5 * float(fx["loss"])
    for name, g in r["grads"].items():
        assert rel_err(g.reshape(-1)[::stride], fx["grad/" + name]) < 1e-4, name
    # and the document mask is what made the difference: plain causal attention is far off
    causal = O.forward({k: torch.tensor(v) for k, v in params.items()}, torch.as_tensor(fx["ids"]), a)
    assert rel_err(causal.detach().reshape(-1, a.vocab_size)[rows], fx["logits"]) > 1e-2
