"""Failure protocol of the N-rank launchers (CPU, no GPU): one rank down must end the job in
seconds with exit code 1 -- the reference's Job has backoffLimit 0 for GPU workloads
(internal/controller/model_controller.go:294-303), so a hung trainer is a hung Model.
Motivated by a multi-GPU run in which a rank that failed but did not exit kept seven GPUs
spinning in a collective for ten minutes."""
import multiprocessing as mp
import os
import signal
import subprocess
import sys
import time

from runbooks_b200 import worker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ok(rank, q):
    q.put((rank, 0, ""))


def _reports_failure(rank, q):
    q.put((rank, 1, "Traceback: boom"))
    q.close()
    q.join_thread()
    os._exit(1)


def _dies_silently(rank, q):
    os._exit(3)          # device fault inside a C call, OOM kill: no report


def _stuck_in_collective(rank, q):
    time.sleep(600)      # a healthy rank waiting for a peer that is gone


def _ignores_sigterm(rank, q):
    signal.signal(signal.SIGTERM, signal.SIG_IGN)   # blocked in a driver call
    ready = os.environ.get("B200W_TEST_READY_FILE")
    if ready:
        open(ready, "w").close()                    # the handler is installed: the peer may die now
    time.sleep(600)


def _dies_silently_once_the_peer_ignores_sigterm(rank, q):
    # a spawned child needs a second or more to import its modules; a SIGTERM that arrives before the peer has
    # installed SIG_IGN would kill it the ordinary way and the grace-period path would not be exercised
    ready = os.environ["B200W_TEST_READY_FILE"]
    t0 = time.time()
    while not os.path.exists(ready) and time.time() - t0 < 60:
        time.sleep(0.05)
    os._exit(3)


def _run(targets, grace=2.0):
    ctx = mp.get_context("spawn")   # not fork: the pytest process is multi-threaded by the time this runs
    q = ctx.Queue()
    procs = [ctx.Process(target=t, args=(r, q)) for r, t in enumerate(targets)]
    for p in procs:
        p.start()
    t0 = time.time()
    code = worker.supervise(procs, q, poll=0.05, grace=grace)
    return code, time.time() - t0, procs


def test_all_ranks_succeed():
    code, secs, procs = _run([_ok, _ok, _ok])
    assert code == 0 and all(p.exitcode == 0 for p in procs)


def test_reported_failure_terminates_the_peers():
    code, secs, procs = _run([_stuck_in_collective, _reports_failure])
    assert code == 1 and secs < 5 and not any(p.is_alive() for p in procs)


def test_silent_death_is_detected_by_exit_code():
    code, secs, procs = _run([_stuck_in_collective, _dies_silently, _stuck_in_collective])
    assert code == 1 and secs < 5 and not any(p.is_alive() for p in procs)


def test_rank_that_ignores_sigterm_is_killed_after_the_grace_period(tmp_path, monkeypatch):
    monkeypatch.setenv("B200W_TEST_READY_FILE", str(tmp_path / "ready"))
    code, secs, procs = _run([_ignores_sigterm, _dies_silently_once_the_peer_ignores_sigterm], grace=1.0)
    assert code == 1 and secs < 60 and not any(p.is_alive() for p in procs)
    assert procs[0].exitcode == -signal.SIGKILL


def test_bench_exits_nonzero_at_once_without_a_json_line_when_it_cannot_run():
    """No GPU here: bench.py (our arm) must fail loudly -- exit code != 0, nothing on stdout -- and do
    so through os._exit, i.e. without hanging in teardown. (There is no CPU fallback to fall into.)"""
    t0 = time.time()
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "3", "--no-cpu"],
                       capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert p.returncode != 0
    assert p.stdout.strip() == "", p.stdout[:300]
    assert "Traceback" in p.stderr or "b200w" in p.stderr or "CUDA" in p.stderr
    assert time.time() - t0 < 240
