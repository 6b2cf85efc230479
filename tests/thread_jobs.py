"""Runs jobs on several host threads at once, for the concurrency tests (test_threads_cpu.py,
test_gpu_threads.py, test_zz_flight_threads_gpu.py)."""
import random
import threading
import time

import pytest

TIMEOUT = 600  # seconds for a whole run: generous, so that only a hang reaches it


def run_threads(per_thread, rounds, seed=0, timeout=TIMEOUT):
    """per_thread[t] is thread t's list of (name, fn).  The threads start together on a barrier; thread t then runs
    its jobs `rounds` times, each round in its own seeded shuffle.  Every fn checks its own result.  The first
    failure is re-raised with the thread, round and job named; if threads are still running at the timeout the
    test fails naming their jobs.  The threads are daemons, so that a hung one cannot keep the process alive."""
    T = len(per_thread)
    barrier = threading.Barrier(T)
    current = ["not started"] * T
    errors = [None] * T

    def worker(t):
        rng = random.Random(1000 * seed + t)
        try:
            barrier.wait(timeout=120)
            for r in range(rounds):
                jobs = list(per_thread[t])
                rng.shuffle(jobs)
                for name, fn in jobs:
                    current[t] = f"thread {t} round {r}: {name}"
                    fn()
        except BaseException as e:  # noqa: BLE001  (re-raised on the main thread)
            errors[t] = (current[t], e)
        current[t] = None

    threads = [threading.Thread(target=worker, args=(t,), daemon=True) for t in range(T)]
    for th in threads:
        th.start()
    deadline = time.monotonic() + timeout
    for th in threads:
        th.join(max(0.0, deadline - time.monotonic()))
    stuck = [current[t] for t in range(T) if threads[t].is_alive()]
    if stuck:
        pytest.fail(f"still running after {timeout} s: {stuck}")
    for err in errors:
        if err is not None:
            where, e = err
            raise AssertionError(f"{where}: {type(e).__name__}: {e}") from e
