"""Container entry point of the Server Deployment's container "serve"
(internal/controller/server_controller.go:114-205):

    python -m runbooks_b200.server            # ENTRYPOINT of the server image

Contract (docs/container-contract.md:50-55; server_controller.go:156-173): listen on :8080,
`GET /` answers 200 once the model in /content/model is loaded (readiness probe), and — what
test/system.sh:73-78 and the basaran image speak — `POST /v1/completions {"prompt", "max_tokens"}`
returns an OpenAI-style completion; `"stream": true` answers with server-sent events (one `data:` JSON
chunk per text delta, then `data: [DONE]`), as basaran does. Accepted and honoured: temperature / top_p /
top_k (sampled on the GPU from the step's logits; default temperature 0 = greedy), stop, n, echo, seed, a prompt of
token ids, logprobs up to the server's max_logprobs (0 by default: logprobs > 0 is then a 400), and, when the
server runs with penalties on (off by default: they are then a 400, a repetition_penalty other than 1 included),
presence_penalty / frequency_penalty /
repetition_penalty / logit_bias (applied on the GPU before the draw, greedy requests included); anything else
that would change the result (best_of, suffix) is a 400. Prompts are ingested in one
prefill pass; continuous batching over the engine's cache slots (one scheduler thread owns the GPU,
HTTP handler threads only queue requests); a full admission queue answers 503 + Retry-After.
"""
from __future__ import annotations

import argparse
import json
import os
import queue
import sys
import threading
import time
import traceback
import uuid
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer

from . import contract


FATAL_STATUSES = (-2, -3)   # B200W_ERR_CUDA, B200W_ERR_NCCL: the context is dead, the Pod must restart


class Scheduler(threading.Thread):
    """Owns the GPU: admits queued requests into free cache slots (prompt prefill happens at admission),
    advances every active request by one token per engine step, and feeds each request's event queue
    (text deltas for streaming clients, one final record for everybody)."""

    def __init__(self, engine, tokenizer, max_queue: int = 0, prefix_cache: bool = False, max_logprobs: int = 0,
                 penalties: bool = False, speculative_tokens: int = 0):
        """max_logprobs (0..5): the most top entries a request may ask for with `logprobs`; 0 refuses them.
        penalties: accept presence_penalty, frequency_penalty, repetition_penalty and logit_bias (else a 400).
        speculative_tokens (0..7): tokens drafted by prompt lookup and verified per request and step (Generator)."""
        super().__init__(daemon=True)
        from .infer import Generator
        self.gen = Generator(engine, eos_id=tokenizer.eos_id, prefix_cache=prefix_cache,
                             speculative_tokens=speculative_tokens)
        self.tok, self.q = tokenizer, queue.Queue()
        self.max_queue = max_queue or 4 * engine.max_batch
        self.max_logprobs = max_logprobs
        self.penalties = penalties
        self.ready = threading.Event()
        self.failed: str | None = None

    def submit(self, prompt, max_tokens: int, temperature: float = 0.0, top_p: float = 1.0, stop=(),
               seed=None, logprobs=None, echo: bool = False, top_k: int = 0, penalties=None):
        """prompt: text, or token ids fed as given. logprobs (None: not asked): log-probabilities of the completion
        tokens with that many top entries, and with echo of the prompt tokens too. penalties (None: none): the
        presence_penalty, frequency_penalty, repetition_penalty and logit_bias arguments of Generator.add.
        -> item (dict) or None when the admission queue is full (the caller answers 503)."""
        if self.q.qsize() >= self.max_queue:
            return None
        item = {"prompt": prompt, "max_tokens": max_tokens, "temperature": temperature, "top_p": top_p,
                "stop": tuple(stop), "seed": seed, "events": queue.Queue(), "cancelled": False,
                "logprobs": logprobs, "echo": echo, "top_k": top_k, "penalties": dict(penalties or {})}
        if isinstance(prompt, list):
            item["ids"] = list(prompt)
        self.q.put(item)
        return item

    # ---- log-probabilities in the OpenAI completions shape (scheduler thread only) ----
    def _detok(self, ids, st):
        """Extends st["strs"] to one string per id by incremental decoding: a token's string is the text it completes
        given the tokens before it ("" while it only starts a character, e.g. part of a UTF-8 sequence)."""
        strs = st.setdefault("strs", [])
        for i in range(len(strs), len(ids)):
            p, r = st.get("p", 0), st.get("r", 0)
            prev = self.tok.decode(ids[p:r])
            new = self.tok.decode(ids[p:i + 1])
            if len(new) > len(prev) and not new.endswith("\ufffd"):
                strs.append(new[len(prev):])
                st["p"], st["r"] = r, i + 1
            else:
                strs.append("")
        return strs

    def _lp_entries(self, strs, lps, base, first, last, offset0):
        """{"tokens", "token_logprobs", "top_logprobs", "text_offset"} of tokens [first, last): offset0 is the text
        offset of token `first`; lps[i] is (log-probability, [(id, log-probability)]) or None (no distribution)."""
        e = {"tokens": [], "token_logprobs": [], "top_logprobs": [], "text_offset": []}
        off = offset0
        for i in range(first, last):
            e["tokens"].append(strs[i])
            e["text_offset"].append(base + off)
            off += len(strs[i])
            if lps[i] is None:
                e["token_logprobs"].append(None)
                e["top_logprobs"].append(None)
                continue
            lp, top = lps[i]
            d = {self.tok.decode([t]): v for t, v in top}
            d[strs[i]] = lp          # the chosen token is always listed
            e["token_logprobs"].append(lp)
            e["top_logprobs"].append(d)
        return e

    def _prompt_entries(self, req):
        """The echoed prompt's text and entries: every prompt token as the engine saw it, the first without a
        log-probability."""
        strs = self._detok(req.prompt, {})
        return "".join(strs), self._lp_entries(strs, req.prompt_lp, 0, 0, len(strs), 0)

    # ---- per-request bookkeeping (scheduler thread only) ----
    def _progress(self, req, item, n_prompt, state):
        """Push the text produced since the last call; finish the request on EOS / length / stop string, or with an
        error when the Generator failed it on its own. A step that emitted several tokens (speculation) is taken one
        token at a time, so that a stop string ends the request at the token that completed it."""
        if getattr(req, "error", None):
            item["events"].put(("error", req.error))
            return True
        n0 = state.get("n", 0)
        for n in range(min(n0 + 1, len(req.out)), len(req.out) + 1):
            state["n"] = n
            if self._progress_upto(req, item, n_prompt, state, n):
                return True
        return False

    def _progress_upto(self, req, item, n_prompt, state, n):
        """_progress as it stands after the request's first n tokens."""
        out = req.out[:n]
        done = req.done and n == len(req.out)
        eos_hit = self.tok.eos_id is not None and out and out[-1] == self.tok.eos_id
        text = self.tok.decode(out[:-1] if eos_hit else out)
        finish, cut = None, False
        for st in item["stop"]:
            k = text.find(st)
            if k >= 0:
                text, finish, cut = text[:k], "stop", True
                break
        if finish is None and done:
            finish = "stop" if eos_hit else "length"
        # hold back a tail that could still turn into a stop string or an incomplete UTF-8 sequence
        safe = len(text)
        if finish is None:
            hold = max((len(st) - 1 for st in item["stop"]), default=0)
            safe = max(state["sent"], len(text) - hold)
            if text.endswith("\ufffd"):
                safe = min(safe, len(text) - 1)
        if item["logprobs"] is not None:
            # the entries of the tokens whose text starts in the text sent so far (EOS adds none and is not listed);
            # at the end every token, or after a stop string those that start before the cut
            strs = self._detok(out[:-1] if eos_hit else out, state["detok"])
            i0 = i = state["lp_n"]
            off = state["lp_off"]
            while i < len(strs) and (off < safe or (finish is not None and not cut)):
                off += len(strs[i])
                i += 1
            if i > i0:
                e = self._lp_entries(strs, req.out_lp, state["base"], i0, i, state["lp_off"])
                for key, vals in e.items():
                    state["lp"][key] += vals
                item["events"].put(("logprobs", e))
                state["lp_n"], state["lp_off"] = i, off
        if safe > state["sent"]:
            item["events"].put(("delta", text[state["sent"]:safe]))
            state["sent"] = safe
        if finish is not None:
            if not req.done:            # stopped by a stop string: free the slot now
                self.gen.cancel(req)
            done = {"text": text, "prompt_tokens": n_prompt, "completion_tokens": len(out),
                    "cached_tokens": req.cached_tokens, "finish_reason": finish}
            if item["logprobs"] is not None:
                done["logprobs"] = state["lp"]
            item["events"].put(("done", done))
            return True
        return False

    def run(self):
        from ._lib import B200WError
        from .infer import CacheFull
        self.ready.set()
        pending = {}
        held = None     # paged KV cache: the head of the line, waiting for pages that running requests hold
        try:
            while True:
                # admit as many queued requests as there are free slots; their prompts are then ingested together
                # (one prefill call per padded length) before the next decode step
                block = not self.gen.active and held is None
                admitted = []
                while self.gen.free:
                    if held is not None:
                        item, held = held, None
                    else:
                        try:
                            item = self.q.get(timeout=0.5 if block else 0)
                        except queue.Empty:
                            break
                    block = False
                    if item["cancelled"]:
                        continue
                    try:
                        if "ids" not in item:
                            ids = self.tok.encode(item["prompt"])
                            item["ids"] = [self.tok.bos_id] + ids if self.tok.bos_id is not None else ids
                        ids = item["ids"]
                        req = self.gen.add(ids, item["max_tokens"], item["temperature"], item["top_p"], item["seed"],
                                           defer_prefill=True, logprobs=item["logprobs"],
                                           prompt_logprobs=item["echo"] and item["logprobs"] is not None,
                                           top_k=item["top_k"], **(item.get("penalties") or {}))
                        admitted.append((req, item, len(ids)))
                    except CacheFull:       # fits the pool, not now: keep its place, retry after the next step
                        held = item
                        break
                    except Exception as e:  # noqa: BLE001 — per-request failure, the server lives on
                        item["events"].put(("error", str(e)))
                if admitted:
                    try:
                        self.gen.flush_prefill()
                    except Exception as e:  # noqa: BLE001
                        if isinstance(e, B200WError) and e.status in FATAL_STATUSES:
                            raise
                        for req, item, _ in admitted:
                            self.gen.cancel(req)
                            item["events"].put(("error", f"{type(e).__name__}: {e}"))
                        admitted = []
                    for req, item, n_ids in admitted:
                        state = {"sent": 0}
                        if item["logprobs"] is not None:
                            state.update(detok={}, lp_n=0, lp_off=0, base=0,
                                         lp={"tokens": [], "token_logprobs": [], "top_logprobs": [], "text_offset": []})
                            if item["echo"]:   # completion offsets count from the start of the echoed prompt
                                echo, state["lp"] = self._prompt_entries(req)
                                state["base"] = len(echo)
                                item["events"].put(("prompt", (echo, state["lp"])))
                                state["lp"] = {k: list(v) for k, v in state["lp"].items()}
                        if not self._progress(req, item, n_ids, state):
                            pending[id(req)] = (req, item, n_ids, state)
                try:
                    self.gen.step()
                except Exception as e:  # noqa: BLE001
                    if isinstance(e, B200WError) and e.status in FATAL_STATUSES:
                        raise           # CUDA / NCCL: the context is dead, the Pod must restart
                    # a rejected batch (bad argument, an engine without logits asked to sample): fail the
                    # requests that were in it, keep serving
                    for req, item, _, _ in pending.values():
                        self.gen.cancel(req)
                        item["events"].put(("error", f"{type(e).__name__}: {e}"))
                    pending.clear()
                    continue
                for key in list(pending):
                    req, item, n_prompt, state = pending[key]
                    if item["cancelled"]:
                        self.gen.cancel(req)
                        del pending[key]
                    elif self._progress(req, item, n_prompt, state):
                        del pending[key]
        except BaseException:  # noqa: BLE001 — a CUDA failure is fatal: fail readiness, exit non-zero
            self.failed = traceback.format_exc()
            sys.stderr.write(self.failed)
            os._exit(1)


def _is_token_ids(x) -> bool:
    return isinstance(x, list) and len(x) > 0 and all(isinstance(t, int) and not isinstance(t, bool) for t in x)


MAX_LOGIT_BIAS = 300   # entries per request, OpenAI's limit
REPETITION_RANGE = (0.01, 100.0)   # far beyond what clients use (1 to 2), and exact enough as float32


def _parse_penalties(req: dict) -> dict:
    """presence_penalty and frequency_penalty in [-2, 2], repetition_penalty in [0.01, 100] (absent or null: 1) and
    logit_bias (up to 300 entries, token ids as strings or integers, biases in [-100, 100]) -> Generator.add's
    arguments."""
    def num(key, default):
        v = req.get(key)
        if v is None:
            return default
        if isinstance(v, bool) or not isinstance(v, (int, float)):
            raise ValueError(f"{key} must be a number")
        return float(v)
    presence, frequency = num("presence_penalty", 0.0), num("frequency_penalty", 0.0)
    repetition = num("repetition_penalty", 1.0)
    if not (-2 <= presence <= 2 and -2 <= frequency <= 2):
        raise ValueError("presence_penalty and frequency_penalty must be in [-2, 2]")
    if not REPETITION_RANGE[0] <= repetition <= REPETITION_RANGE[1]:
        raise ValueError(f"repetition_penalty must be in [{REPETITION_RANGE[0]}, {REPETITION_RANGE[1]:g}]")
    raw = req.get("logit_bias") or {}
    if not isinstance(raw, dict) or len(raw) > MAX_LOGIT_BIAS:
        raise ValueError(f"logit_bias must map up to {MAX_LOGIT_BIAS} token ids to biases")
    bias = {}
    for k, v in raw.items():
        if isinstance(k, str) and k.strip().lstrip("-").isdigit():
            k = int(k)
        if isinstance(k, bool) or not isinstance(k, int) or k < 0:
            raise ValueError(f"logit_bias key {k!r} is not a token id")
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not -100 <= v <= 100:
            raise ValueError(f"logit_bias of token {k} must be a number in [-100, 100]")
        bias[k] = float(v)
    return dict(presence_penalty=presence, frequency_penalty=frequency, repetition_penalty=repetition,
                logit_bias=bias)


def parse_completion_request(req: dict, max_logprobs: int = 0, penalties: bool = False) -> dict:
    """The OpenAI / basaran `/v1/completions` fields. Everything that is accepted is honoured; a value this
    server does not implement is a 400, never a silent fallback to something else.
    prompt: a string, a list of token ids (fed as given, no BOS added), or a list holding one of either.
    logprobs: refused above 0 unless the server was started with max_logprobs >= 1; then 0..max_logprobs.
    presence_penalty, frequency_penalty, repetition_penalty, logit_bias: refused unless the server was started with
    penalties on; then in the ranges of _parse_penalties."""
    prompt = req["prompt"]
    if isinstance(prompt, list) and not _is_token_ids(prompt):
        if len(prompt) != 1:
            raise ValueError("exactly one prompt per request")
        prompt = prompt[0]
    if not (isinstance(prompt, str) or _is_token_ids(prompt)):
        raise ValueError("prompt must be a string or a list of token ids")
    max_tokens = int(req.get("max_tokens", 16))
    if max_tokens < 1:
        raise ValueError("max_tokens must be >= 1")
    def num(key, default):            # JSON null means "default"; 0 is a value
        v = req.get(key)
        return default if v is None else float(v)
    temperature = num("temperature", 0.0)   # this server's default is greedy
    top_p = num("top_p", 1.0)
    if temperature < 0 or not 0 < top_p <= 1:
        raise ValueError("temperature must be >= 0 and top_p in (0, 1]")
    top_k = req.get("top_k")       # absent, null, 0 or -1: off (the vLLM convention)
    if top_k in (None, -1):
        top_k = 0
    if isinstance(top_k, bool) or not isinstance(top_k, int) or top_k < 0:
        raise ValueError("top_k must be a positive integer, or 0 / -1 / null for off")
    n = int(num("n", 1))
    if n < 1 or n > 8:
        raise ValueError("n must be in 1..8")
    stop = req.get("stop") or []
    if isinstance(stop, str):
        stop = [stop]
    if not all(isinstance(x, str) and x for x in stop) or len(stop) > 4:
        raise ValueError("stop must be a string or a list of up to 4 non-empty strings")
    stream = bool(req.get("stream", False))
    if stream and n != 1:
        raise ValueError("stream with n > 1 is not implemented")
    logprobs = req.get("logprobs")
    if max_logprobs >= 1 and logprobs is not None:
        if isinstance(logprobs, bool) or not isinstance(logprobs, int) or not 0 <= logprobs <= max_logprobs:
            raise ValueError(f"logprobs must be an integer in 0..{max_logprobs}")
    else:
        logprobs = None
    for key, default in (("logprobs", None), ("best_of", None), ("suffix", None), ("logit_bias", None)):
        if (key == "logprobs" and max_logprobs >= 1) or (key == "logit_bias" and penalties):
            continue
        if req.get(key, default) not in (default, 0 if key == "logprobs" else default, 1 if key == "best_of" else default):
            raise ValueError(f"{key} is not implemented")
    if penalties:
        pen = _parse_penalties(req)
    else:
        for key in ("presence_penalty", "frequency_penalty"):
            if float(req.get(key, 0) or 0) != 0:
                raise ValueError(f"{key} is not implemented")
        if req.get("repetition_penalty") not in (None, 1):
            raise ValueError("repetition_penalty is not implemented")
        pen = {}
    seed = req.get("seed")
    return dict(prompt=prompt, max_tokens=max_tokens, temperature=temperature, top_p=top_p, n=n, stop=stop,
                stream=stream, echo=bool(req.get("echo", False)), seed=None if seed is None else int(seed),
                logprobs=logprobs, top_k=top_k, penalties=pen)


def make_handler(sched: Scheduler, model_name: str, request_timeout_s: float = 600.0):
    class H(BaseHTTPRequestHandler):
        protocol_version = "HTTP/1.1"

        def _send(self, code, obj, headers=()):
            body = json.dumps(obj).encode()
            self.send_response(code)
            self.send_header("Content-Type", "application/json")
            self.send_header("Content-Length", str(len(body)))
            for k, v in headers:
                self.send_header(k, v)
            self.end_headers()
            self.wfile.write(body)

        def log_message(self, fmt, *args):  # one JSON line per request on stdout
            print(json.dumps({"event": "http", "msg": fmt % args}), flush=True)

        def do_GET(self):
            if self.path in ("/", "/healthz"):
                ok = sched.ready.is_set() and not sched.failed
                self._send(200 if ok else 503, {"status": "ok" if ok else "loading", "model": model_name})
            elif self.path == "/v1/models":
                self._send(200, {"object": "list", "data": [{"id": model_name, "object": "model"}]})
            else:
                self._send(404, {"error": "not found"})

        def _chunk(self, cid, created, text, finish, logprobs=None):
            return {"id": cid, "object": "text_completion", "created": created, "model": model_name,
                    "choices": [{"index": 0, "text": text, "logprobs": logprobs, "finish_reason": finish}]}

        def do_POST(self):
            if self.path != "/v1/completions":
                return self._send(404, {"error": "not found"})
            try:
                n = int(self.headers.get("Content-Length", "0"))
                r = parse_completion_request(json.loads(self.rfile.read(n) or b"{}"), sched.max_logprobs,
                                             sched.penalties)
            except Exception as e:  # noqa: BLE001
                return self._send(400, {"error": f"bad request: {e}"})
            # the echoed prompt: a token-id prompt's decoding; with log-probabilities, the prompt tokens' strings
            echo = r["prompt"] if isinstance(r["prompt"], str) else sched.tok.decode(r["prompt"])
            items = []
            for i in range(r["n"]):
                seed = None if r["seed"] is None else r["seed"] + i
                it = sched.submit(r["prompt"], r["max_tokens"], r["temperature"], r["top_p"], r["stop"], seed,
                                  r["logprobs"], r["echo"], r["top_k"], r["penalties"])
                if it is None:          # back-pressure: every slot busy and the admission queue full
                    for x in items:
                        x["cancelled"] = True
                    return self._send(503, {"error": "server busy: all cache slots and the admission queue are full"},
                                      headers=(("Retry-After", "1"),))
                items.append(it)
            cid, created = "cmpl-" + uuid.uuid4().hex[:24], int(time.time())
            deadline = time.time() + request_timeout_s
            if r["stream"]:
                return self._stream(items[0], r, echo, cid, created, deadline)
            choices, usage_p, usage_c, cached = [], 0, 0, 0
            for i, it in enumerate(items):
                final = None
                while final is None:
                    try:
                        kind, val = it["events"].get(timeout=max(0.0, deadline - time.time()))
                    except queue.Empty:
                        for x in items:
                            x["cancelled"] = True
                        return self._send(504, {"error": f"request timed out after {request_timeout_s:.0f} s"})
                    if kind == "error":
                        for x in items:
                            x["cancelled"] = True
                        return self._send(400, {"error": val})
                    if kind == "prompt":
                        echo = val[0]
                    if kind == "done":
                        final = val
                text = (echo if r["echo"] else "") + final["text"]
                choices.append({"index": i, "text": text, "logprobs": final.get("logprobs"),
                                "finish_reason": final["finish_reason"]})
                usage_p, usage_c = final["prompt_tokens"], usage_c + final["completion_tokens"]
                # the prompt is counted once, as prompt_tokens is: its tokens that the best-served copy found cached
                cached = max(cached, final["cached_tokens"])
            usage = {"prompt_tokens": usage_p, "completion_tokens": usage_c, "total_tokens": usage_p + usage_c}
            if sched.gen.prefix_cache:
                usage["prompt_tokens_details"] = {"cached_tokens": cached}
            self._send(200, {"id": cid, "object": "text_completion", "created": created, "model": model_name,
                             "choices": choices, "usage": usage})

        def _stream(self, item, r, echo, cid, created, deadline):
            """Server-sent events, the OpenAI / basaran streaming shape: one `data: {json}` per text delta,
            a final chunk carrying finish_reason, then `data: [DONE]`. With logprobs, each chunk carries the entries of
            the tokens whose text starts in it (the echo chunk the prompt's), and the final chunk any left."""
            self.send_response(200)
            self.send_header("Content-Type", "text/event-stream")
            self.send_header("Cache-Control", "no-cache")
            self.send_header("Connection", "close")
            self.end_headers()
            self.close_connection = True

            def emit(obj):
                self.wfile.write(b"data: " + (obj if isinstance(obj, bytes) else json.dumps(obj).encode()) + b"\n\n")
                self.wfile.flush()
            lp = r["logprobs"] is not None
            empty = {"tokens": [], "token_logprobs": [], "top_logprobs": [], "text_offset": []}
            try:
                if r["echo"] and not lp:
                    emit(self._chunk(cid, created, echo, None))
                entries = empty
                while True:
                    try:
                        kind, val = item["events"].get(timeout=max(0.0, deadline - time.time()))
                    except queue.Empty:
                        item["cancelled"] = True
                        emit({"error": "request timed out"})
                        break
                    if kind == "prompt":
                        emit(self._chunk(cid, created, val[0], None, val[1]))
                    elif kind == "logprobs":
                        entries = {k: entries[k] + val[k] for k in empty}
                    elif kind == "delta":
                        emit(self._chunk(cid, created, val, None, entries if lp else None))
                        entries = empty
                    elif kind == "error":
                        emit({"error": val})
                        break
                    else:
                        emit(self._chunk(cid, created, "", val["finish_reason"], entries if lp else None))
                        break
                emit(b"[DONE]")
            except (BrokenPipeError, ConnectionResetError):
                item["cancelled"] = True    # the client went away: free the slot at the next step

    return H


def server_params(content: str, max_batch: int | None = None, kv_cache_gb: float | None = None,
                  environ=None) -> tuple:
    """(max_batch, kv_cache_gb) of the Server. A command-line value wins; otherwise the container contract's
    params (/content/params.json, PARAM_<UPPER> overriding it, merged by contract.load_params); otherwise 32 slots
    and the contiguous cache (kv_cache_gb None)."""
    extra = contract.load_params(os.path.join(content, "params.json"), environ).extra

    def pick(cli, key, typ):
        if cli is not None or key not in extra:
            return cli
        try:
            return contract._coerce(extra[key], typ)
        except (TypeError, ValueError) as e:
            raise ValueError(f"param {key!r}: cannot read {extra[key]!r} as {typ.__name__}") from e
    max_batch = pick(max_batch, "max_batch", int)
    max_batch = 32 if max_batch is None else max_batch
    kv_cache_gb = pick(kv_cache_gb, "kv_cache_gb", float)
    if not 1 <= max_batch <= 128:
        raise ValueError(f"max_batch must be in 1..128, got {max_batch}")
    if kv_cache_gb is not None and not (kv_cache_gb > 0 and kv_cache_gb < float("inf")):
        raise ValueError(f"kv_cache_gb must be a positive number of GB, got {kv_cache_gb}")
    return max_batch, kv_cache_gb


def prefix_cache_param(content: str, prefix_cache: bool | None = None, environ=None) -> bool:
    """Whether the Server shares the K/V pages of repeated prompt prefixes: --prefix-cache, else the params'
    prefix_cache (params.json, PARAM_PREFIX_CACHE over it: true / false, 1 / 0, yes / no), else off."""
    return _bool_param(content, "prefix_cache", prefix_cache, environ)


def penalties_param(content: str, penalties: bool | None = None, environ=None) -> bool:
    """Whether the Server accepts presence_penalty, frequency_penalty, repetition_penalty and logit_bias: --penalties,
    else the params' penalties (params.json, PARAM_PENALTIES over it: true / false, 1 / 0, yes / no), else off (they
    are then a 400)."""
    return _bool_param(content, "penalties", penalties, environ)


def _bool_param(content: str, key: str, cli: bool | None, environ) -> bool:
    if cli is not None:
        return bool(cli)
    extra = contract.load_params(os.path.join(content, "params.json"), environ).extra
    return _as_bool(f"param {key!r}", extra.get(key, False))


def _as_bool(what: str, v) -> bool:
    """true / false, 1 / 0, yes / no (any case, as a bool, a number or a string); anything else is a ValueError"""
    if isinstance(v, bool) or v in (0, 1):
        return bool(v)
    if isinstance(v, str) and v.strip().lower() in ("true", "1", "yes", "false", "0", "no"):
        return v.strip().lower() in ("true", "1", "yes")
    raise ValueError(f"{what}: cannot read {v!r} as a boolean")


def load_in_4bit_param(load_in_4bit: bool | None = None, environ=None) -> bool:
    """Whether the Server asks for int4 projections (weight_dtype "int4"): --load-in-4bit, else the environment's
    MODEL_LOAD_IN_4BIT (true / false, 1 / 0, yes / no; anything else is an error), else off. MODEL_LOAD_IN_8BIT is
    load_in_8bit_param's; weight_dtype_param refuses both on."""
    if load_in_4bit is not None:
        return bool(load_in_4bit)
    environ = os.environ if environ is None else environ
    return _as_bool("MODEL_LOAD_IN_4BIT", environ.get("MODEL_LOAD_IN_4BIT", False))


def load_in_8bit_param(load_in_8bit: bool | None = None, environ=None) -> bool:
    """Whether the Server asks for int8 projections (weight_dtype "int8"): --load-in-8bit, else the environment's
    MODEL_LOAD_IN_8BIT (true / false, 1 / 0, yes / no; anything else is an error), else off."""
    if load_in_8bit is not None:
        return bool(load_in_8bit)
    environ = os.environ if environ is None else environ
    return _as_bool("MODEL_LOAD_IN_8BIT", environ.get("MODEL_LOAD_IN_8BIT", False))


def weight_dtype_param(load_in_4bit: bool | None = None, load_in_8bit: bool | None = None, environ=None) -> str:
    """The engine's weight_dtype: "int4" (load_in_4bit_param), "int8" (load_in_8bit_param) or "bf16". Both on is a
    ValueError, as transformers refuses load_in_4bit together with load_in_8bit."""
    w4, w8 = load_in_4bit_param(load_in_4bit, environ), load_in_8bit_param(load_in_8bit, environ)
    if w4 and w8:
        raise ValueError("load_in_4bit and load_in_8bit are both on (MODEL_LOAD_IN_4BIT / MODEL_LOAD_IN_8BIT or "
                         "--load-in-4bit / --load-in-8bit): choose one")
    return "int4" if w4 else "int8" if w8 else "bf16"


def speculative_tokens_param(content: str, speculative_tokens: int | None = None, environ=None) -> int:
    """Tokens drafted (prompt lookup) and verified per request and step, 0..7: --speculative-tokens, else the params'
    speculative_tokens (params.json, PARAM_SPECULATIVE_TOKENS over it), else 0 (off)."""
    if speculative_tokens is None:
        extra = contract.load_params(os.path.join(content, "params.json"), environ).extra
        v = speculative_tokens = extra.get("speculative_tokens", 0)
        if isinstance(v, str):
            try:
                speculative_tokens = int(v.strip())
            except ValueError as e:
                raise ValueError(f"param 'speculative_tokens': cannot read {v!r} as an integer") from e
    if isinstance(speculative_tokens, bool) or not isinstance(speculative_tokens, int) or \
            not 0 <= speculative_tokens <= 7:
        raise ValueError(f"speculative_tokens must be an integer in 0..7, got {speculative_tokens!r}")
    return speculative_tokens


def max_logprobs_param(content: str, max_logprobs: int | None = None, environ=None) -> int:
    """The most top entries a request may ask for with `logprobs` (vLLM's max_logprobs), 0..5: --max-logprobs, else
    the params' max_logprobs (params.json, PARAM_MAX_LOGPROBS over it), else 0, which refuses logprobs > 0."""
    if max_logprobs is None:
        extra = contract.load_params(os.path.join(content, "params.json"), environ).extra
        v = max_logprobs = extra.get("max_logprobs", 0)
        if isinstance(v, str):
            try:
                max_logprobs = int(v.strip())
            except ValueError as e:
                raise ValueError(f"param 'max_logprobs': cannot read {v!r} as an integer") from e
    if isinstance(max_logprobs, bool) or not isinstance(max_logprobs, int) or not 0 <= max_logprobs <= 5:
        raise ValueError(f"max_logprobs must be an integer in 0..5, got {max_logprobs!r}")
    return max_logprobs


KV_CACHE_DTYPES = {"auto": "bf16", "bf16": "bf16", "fp8": "fp8", "fp8_e4m3": "fp8"}


def kv_cache_dtype_param(content: str, kv_cache_dtype: str | None = None, environ=None) -> str:
    """The element type of the paged KV cache, "bf16" or "fp8": --kv-cache-dtype, else the params' kv_cache_dtype
    (params.json, PARAM_KV_CACHE_DTYPE over it), else bf16. auto / bf16 and fp8 / fp8_e4m3 are accepted."""
    if kv_cache_dtype is None:
        extra = contract.load_params(os.path.join(content, "params.json"), environ).extra
        kv_cache_dtype = extra.get("kv_cache_dtype", "auto")
    v = kv_cache_dtype.strip().lower() if isinstance(kv_cache_dtype, str) else kv_cache_dtype
    if v not in KV_CACHE_DTYPES:
        raise ValueError(f"param 'kv_cache_dtype' must be one of {sorted(KV_CACHE_DTYPES)}, got {kv_cache_dtype!r}")
    return KV_CACHE_DTYPES[v]


def kv_pages_for_gb(arch, kv_cache_gb: float, kv_dtype: str = "bf16") -> int:
    """Pages of a paged KV cache of kv_cache_gb * 10^9 bytes; ValueError when that cannot hold one max_ctx request."""
    from .infer import kv_page_bytes, pages_for
    page = kv_page_bytes(arch, kv_dtype)
    pages = int(kv_cache_gb * 1e9 // page)
    if pages < pages_for(arch.max_ctx):
        raise ValueError(f"kv_cache_gb {kv_cache_gb} holds {pages} pages of {page / 1e6:.1f} MB; one "
                         f"request of max_ctx {arch.max_ctx} needs {pages_for(arch.max_ctx)}")
    return pages


def load_engine(model_dir: str, max_batch: int, max_ctx: int | None, kv_cache_gb: float | None = None,
                kv_dtype: str = "bf16", speculative_tokens: int = 0, load_in_4bit: bool | None = None,
                load_in_8bit: bool | None = None):
    """speculative_tokens > 0: a step holds up to min(128, max_batch * (1 + speculative_tokens)) rows.
    load_in_4bit / load_in_8bit: int4 / int8 projections (None: MODEL_LOAD_IN_4BIT / MODEL_LOAD_IN_8BIT,
    weight_dtype_param)."""
    from .infer import InferEngine, ServeArch

    cfg = contract.read_hf_config(model_dir)
    arch = ServeArch.from_hf_config(cfg, max_ctx)
    kv_pages = None if kv_cache_gb is None else kv_pages_for_gb(arch, kv_cache_gb, kv_dtype)
    e = InferEngine(int(os.environ.get("B200W_DEVICE", "0")))
    e.init_infer(arch, max_batch=max_batch, kv_pages=kv_pages, kv_dtype=kv_dtype,
                 max_rows=min(128, max_batch * (1 + speculative_tokens)) if speculative_tokens else None,
                 weight_dtype=weight_dtype_param(load_in_4bit, load_in_8bit))
    wanted = {n for n, _ in e.infer_params()}
    seen, unused = set(), []
    for name, arr in contract.iter_safetensors(model_dir):
        name = contract.canonical_tensor_name(name, cfg)
        if name in wanted:
            e.infer_load_tensor(name, arr)
            seen.add(name)
        elif not contract.is_ignorable_tensor(name, cfg):
            unused.append(name)
    if wanted - seen:
        raise KeyError(f"checkpoint lacks {sorted(wanted - seen)[:3]} ... ({len(wanted - seen)} tensors)")
    if unused:   # same policy as the trainer: a tensor we would silently drop means different arithmetic
        raise ValueError(f"checkpoint holds tensors this engine does not use: {sorted(unused)[:4]} ({len(unused)})")
    return e, cfg


def serve(content: str, port: int, max_batch: int | None, max_ctx: int | None, kv_cache_gb: float | None = None,
          prefix_cache: bool | None = None, kv_cache_dtype: str | None = None, max_logprobs: int | None = None,
          penalties: bool | None = None, speculative_tokens: int | None = None, load_in_4bit: bool | None = None,
          load_in_8bit: bool | None = None):
    max_batch, kv_cache_gb = server_params(content, max_batch, kv_cache_gb)
    weight_dtype = weight_dtype_param(load_in_4bit, load_in_8bit)
    load_in_4bit, load_in_8bit = weight_dtype == "int4", weight_dtype == "int8"
    speculative_tokens = speculative_tokens_param(content, speculative_tokens)
    prefix_cache = prefix_cache_param(content, prefix_cache)
    kv_dtype = kv_cache_dtype_param(content, kv_cache_dtype)
    max_logprobs = max_logprobs_param(content, max_logprobs)
    penalties = penalties_param(content, penalties)
    if prefix_cache and kv_cache_gb is None:
        raise ValueError("prefix_cache shares pages of the paged KV cache: it needs kv_cache_gb")
    if kv_dtype != "bf16" and kv_cache_gb is None:
        raise ValueError("an fp8 KV cache is paged: kv_cache_dtype fp8 needs kv_cache_gb")
    model_dir = os.path.join(content, "model")
    t0 = time.time()
    engine, cfg = load_engine(model_dir, max_batch, max_ctx, kv_cache_gb, kv_dtype, speculative_tokens, load_in_4bit,
                              load_in_8bit)
    tok = contract.Tokenizer(model_dir)
    sched = Scheduler(engine, tok, prefix_cache=prefix_cache, max_logprobs=max_logprobs, penalties=penalties,
                      speculative_tokens=speculative_tokens)
    sched.start()
    name = cfg.get("_name_or_path") or cfg.get("model_type", "model")
    httpd = ThreadingHTTPServer(("0.0.0.0", port), make_handler(sched, name))
    ready = {"event": "ready", "port": port, "model": name, "load_seconds": round(time.time() - t0, 2),
             "max_batch": max_batch, "max_logprobs": max_logprobs, "penalties": penalties,
             "speculative_tokens": speculative_tokens, "weight_dtype": engine.weight_dtype,
             "weight_gb": round(engine.weight_bytes() / 1e9, 3)}
    if engine.kv_pages is not None:
        from .infer import kv_page_bytes
        ready.update(kv_pages=engine.kv_pages, kv_page_mb=round(kv_page_bytes(engine.serve_arch, kv_dtype) / 1e6, 2),
                     kv_cache_dtype=kv_dtype, prefix_cache=prefix_cache)
    print(json.dumps(ready), flush=True)
    httpd.serve_forever()


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="runbooks_b200.server")
    ap.add_argument("--content", default=contract.CONTENT)
    ap.add_argument("--port", type=int, default=8080)       # server_controller.go:156-161
    ap.add_argument("--max-batch", type=int, default=None, help="cache slots (default: param max_batch, else 32)")
    ap.add_argument("--max-ctx", type=int, default=None)
    ap.add_argument("--kv-cache-gb", type=float, default=None,
                    help="serve from a paged KV cache of this many GB (default: param kv_cache_gb, else a "
                         "contiguous max_batch x max_ctx cache)")
    ap.add_argument("--prefix-cache", action="store_true", default=None,
                    help="share the KV pages of repeated prompt prefixes (needs the paged cache; default: param "
                         "prefix_cache, else off)")
    ap.add_argument("--kv-cache-dtype", default=None,
                    help="element type of the paged KV cache: auto / bf16, or fp8 / fp8_e4m3 (needs kv_cache_gb; "
                         "default: param kv_cache_dtype, else bf16)")
    ap.add_argument("--max-logprobs", type=int, default=None,
                    help="the most top entries a request may ask for with logprobs, 0..5 (default: param "
                         "max_logprobs, else 0: logprobs > 0 is refused)")
    ap.add_argument("--penalties", action="store_true", default=None,
                    help="accept presence_penalty, frequency_penalty, repetition_penalty and logit_bias (default: "
                         "param penalties, else off: they are refused)")
    ap.add_argument("--speculative-tokens", type=int, default=None,
                    help="tokens drafted by prompt lookup and verified per request and step, 0..7 (default: param "
                         "speculative_tokens, else 0: off)")
    ap.add_argument("--load-in-4bit", action="store_true", default=None,
                    help="store the projections as int4, one bf16 scale per row and 64 inputs (default: env "
                         "MODEL_LOAD_IN_4BIT, else bf16)")
    ap.add_argument("--load-in-8bit", action="store_true", default=None,
                    help="store the projections as int8, one bf16 scale per row and 64 inputs; weight-only, no "
                         "outlier decomposition (default: env MODEL_LOAD_IN_8BIT, else bf16)")
    a = ap.parse_args(argv)
    try:
        serve(a.content, a.port, a.max_batch, a.max_ctx, a.kv_cache_gb, a.prefix_cache, a.kv_cache_dtype,
              a.max_logprobs, a.penalties, a.speculative_tokens, a.load_in_4bit, a.load_in_8bit)
        return 0
    except BaseException:  # noqa: BLE001
        traceback.print_exc()
        return 1


if __name__ == "__main__":
    sys.exit(main())
