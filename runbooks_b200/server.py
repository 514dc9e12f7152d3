"""Container entry point of the Server Deployment's container "serve"
(internal/controller/server_controller.go:114-205):

    python -m runbooks_b200.server            # ENTRYPOINT of the server image

Contract (docs/container-contract.md:50-55; server_controller.go:156-173): listen on :8080,
`GET /` answers 200 once the model in /content/model is loaded (readiness probe), and — what
test/system.sh:73-78 and the basaran image speak — `POST /v1/completions {"prompt", "max_tokens"}`
returns an OpenAI-style completion; `"stream": true` answers with server-sent events (one `data:` JSON
chunk per text delta, then `data: [DONE]`), as basaran does. Accepted and honoured: temperature / top_p
(host-side nucleus sampling over the engine's logits; default 0 = greedy), stop, n, echo, seed; anything
else that would change the result (logprobs, penalties, best_of) is a 400. Prompts are ingested in one
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

    def __init__(self, engine, tokenizer, max_queue: int = 0):
        super().__init__(daemon=True)
        from .infer import Generator
        self.gen = Generator(engine, eos_id=tokenizer.eos_id)
        self.tok, self.q = tokenizer, queue.Queue()
        self.max_queue = max_queue or 4 * engine.max_batch
        self.ready = threading.Event()
        self.failed: str | None = None

    def submit(self, prompt: str, max_tokens: int, temperature: float = 0.0, top_p: float = 1.0, stop=(),
               seed=None):
        """-> item (dict) or None when the admission queue is full (the caller answers 503)."""
        if self.q.qsize() >= self.max_queue:
            return None
        item = {"prompt": prompt, "max_tokens": max_tokens, "temperature": temperature, "top_p": top_p,
                "stop": tuple(stop), "seed": seed, "events": queue.Queue(), "cancelled": False}
        self.q.put(item)
        return item

    # ---- per-request bookkeeping (scheduler thread only) ----
    def _progress(self, req, item, n_prompt, state):
        """Push the text produced since the last call; finish the request on EOS / length / stop string."""
        out = req.out
        eos_hit = self.tok.eos_id is not None and out and out[-1] == self.tok.eos_id
        text = self.tok.decode(out[:-1] if eos_hit else out)
        finish = None
        for st in item["stop"]:
            k = text.find(st)
            if k >= 0:
                text, finish = text[:k], "stop"
                break
        if finish is None and req.done:
            finish = "stop" if eos_hit else "length"
        # hold back a tail that could still turn into a stop string or an incomplete UTF-8 sequence
        safe = len(text)
        if finish is None:
            hold = max((len(st) - 1 for st in item["stop"]), default=0)
            safe = max(state["sent"], len(text) - hold)
            if text.endswith("\ufffd"):
                safe = min(safe, len(text) - 1)
        if safe > state["sent"]:
            item["events"].put(("delta", text[state["sent"]:safe]))
            state["sent"] = safe
        if finish is not None:
            if not req.done:            # stopped by a stop string: free the slot now
                self.gen.cancel(req)
            item["events"].put(("done", {"text": text, "prompt_tokens": n_prompt, "completion_tokens": len(out),
                                         "finish_reason": finish}))
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
                                           defer_prefill=True)
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


def parse_completion_request(req: dict) -> dict:
    """The OpenAI / basaran `/v1/completions` fields. Everything that is accepted is honoured; a value this
    server does not implement is a 400, never a silent fallback to something else."""
    prompt = req["prompt"]
    if isinstance(prompt, list):
        if len(prompt) != 1:
            raise ValueError("exactly one prompt per request")
        prompt = prompt[0]
    if not isinstance(prompt, str):
        raise ValueError("prompt must be a string")
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
    for key, default in (("logprobs", None), ("best_of", None), ("suffix", None), ("logit_bias", None)):
        if req.get(key, default) not in (default, 0 if key == "logprobs" else default, 1 if key == "best_of" else default):
            raise ValueError(f"{key} is not implemented")
    for key in ("presence_penalty", "frequency_penalty"):
        if float(req.get(key, 0) or 0) != 0:
            raise ValueError(f"{key} is not implemented")
    seed = req.get("seed")
    return dict(prompt=prompt, max_tokens=max_tokens, temperature=temperature, top_p=top_p, n=n, stop=stop,
                stream=stream, echo=bool(req.get("echo", False)), seed=None if seed is None else int(seed))


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

        def _chunk(self, cid, created, text, finish):
            return {"id": cid, "object": "text_completion", "created": created, "model": model_name,
                    "choices": [{"index": 0, "text": text, "logprobs": None, "finish_reason": finish}]}

        def do_POST(self):
            if self.path != "/v1/completions":
                return self._send(404, {"error": "not found"})
            try:
                n = int(self.headers.get("Content-Length", "0"))
                r = parse_completion_request(json.loads(self.rfile.read(n) or b"{}"))
            except Exception as e:  # noqa: BLE001
                return self._send(400, {"error": f"bad request: {e}"})
            items = []
            for i in range(r["n"]):
                seed = None if r["seed"] is None else r["seed"] + i
                it = sched.submit(r["prompt"], r["max_tokens"], r["temperature"], r["top_p"], r["stop"], seed)
                if it is None:          # back-pressure: every slot busy and the admission queue full
                    for x in items:
                        x["cancelled"] = True
                    return self._send(503, {"error": "server busy: all cache slots and the admission queue are full"},
                                      headers=(("Retry-After", "1"),))
                items.append(it)
            cid, created = "cmpl-" + uuid.uuid4().hex[:24], int(time.time())
            deadline = time.time() + request_timeout_s
            if r["stream"]:
                return self._stream(items[0], r, cid, created, deadline)
            choices, usage_p, usage_c = [], 0, 0
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
                    if kind == "done":
                        final = val
                text = (r["prompt"] if r["echo"] else "") + final["text"]
                choices.append({"index": i, "text": text, "logprobs": None, "finish_reason": final["finish_reason"]})
                usage_p, usage_c = final["prompt_tokens"], usage_c + final["completion_tokens"]
            self._send(200, {"id": cid, "object": "text_completion", "created": created, "model": model_name,
                             "choices": choices,
                             "usage": {"prompt_tokens": usage_p, "completion_tokens": usage_c,
                                       "total_tokens": usage_p + usage_c}})

        def _stream(self, item, r, cid, created, deadline):
            """Server-sent events, the OpenAI / basaran streaming shape: one `data: {json}` per text delta,
            a final chunk carrying finish_reason, then `data: [DONE]`."""
            self.send_response(200)
            self.send_header("Content-Type", "text/event-stream")
            self.send_header("Cache-Control", "no-cache")
            self.send_header("Connection", "close")
            self.end_headers()
            self.close_connection = True

            def emit(obj):
                self.wfile.write(b"data: " + (obj if isinstance(obj, bytes) else json.dumps(obj).encode()) + b"\n\n")
                self.wfile.flush()
            try:
                if r["echo"]:
                    emit(self._chunk(cid, created, r["prompt"], None))
                while True:
                    try:
                        kind, val = item["events"].get(timeout=max(0.0, deadline - time.time()))
                    except queue.Empty:
                        item["cancelled"] = True
                        emit({"error": "request timed out"})
                        break
                    if kind == "delta":
                        emit(self._chunk(cid, created, val, None))
                    elif kind == "error":
                        emit({"error": val})
                        break
                    else:
                        emit(self._chunk(cid, created, "", val["finish_reason"]))
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


def kv_pages_for_gb(arch, kv_cache_gb: float) -> int:
    """Pages of a paged KV cache of kv_cache_gb * 10^9 bytes; ValueError when that cannot hold one max_ctx request."""
    from .infer import kv_page_bytes, pages_for
    pages = int(kv_cache_gb * 1e9 // kv_page_bytes(arch))
    if pages < pages_for(arch.max_ctx):
        raise ValueError(f"kv_cache_gb {kv_cache_gb} holds {pages} pages of {kv_page_bytes(arch) / 1e6:.1f} MB; one "
                         f"request of max_ctx {arch.max_ctx} needs {pages_for(arch.max_ctx)}")
    return pages


def load_engine(model_dir: str, max_batch: int, max_ctx: int | None, kv_cache_gb: float | None = None):
    from .infer import InferEngine, ServeArch

    cfg = contract.read_hf_config(model_dir)
    arch = ServeArch.from_hf_config(cfg, max_ctx)
    kv_pages = None if kv_cache_gb is None else kv_pages_for_gb(arch, kv_cache_gb)
    e = InferEngine(int(os.environ.get("B200W_DEVICE", "0")))
    e.init_infer(arch, max_batch=max_batch, kv_pages=kv_pages)
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


def serve(content: str, port: int, max_batch: int | None, max_ctx: int | None, kv_cache_gb: float | None = None):
    max_batch, kv_cache_gb = server_params(content, max_batch, kv_cache_gb)
    model_dir = os.path.join(content, "model")
    t0 = time.time()
    engine, cfg = load_engine(model_dir, max_batch, max_ctx, kv_cache_gb)
    tok = contract.Tokenizer(model_dir)
    sched = Scheduler(engine, tok)
    sched.start()
    name = cfg.get("_name_or_path") or cfg.get("model_type", "model")
    httpd = ThreadingHTTPServer(("0.0.0.0", port), make_handler(sched, name))
    ready = {"event": "ready", "port": port, "model": name, "load_seconds": round(time.time() - t0, 2),
             "max_batch": max_batch}
    if engine.kv_pages is not None:
        from .infer import kv_page_bytes
        ready.update(kv_pages=engine.kv_pages, kv_page_mb=round(kv_page_bytes(engine.serve_arch) / 1e6, 2))
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
    a = ap.parse_args(argv)
    try:
        serve(a.content, a.port, a.max_batch, a.max_ctx, a.kv_cache_gb)
        return 0
    except BaseException:  # noqa: BLE001
        traceback.print_exc()
        return 1


if __name__ == "__main__":
    sys.exit(main())
