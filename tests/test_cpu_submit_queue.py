"""The asynchronous submission queue without a GPU: libde265_b200/csrc/submit_queue.cuh (the queue behind
b200_engine_submit_picture_async), compiled for the host by tests/submit_queue_emul.cu with stand-in plan and issue steps.
Checks its contract with 1, 3 and 8 planner threads: commands are issued in submission order whatever order their plans finish
in, tickets, wait(ticket), per-slot tickets (waiting for a slot is not a flush), queued errors reported once by the next wait
with the failing thread's message, back-pressure, and shutdown with commands still queued.  Each check runs in a child
process with a time limit, so that a queue that hangs fails the check instead of the run."""
import ctypes as C
import os
import re
import subprocess
import sys
import time

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libsubmit_queue_emul.so")
SRC = os.path.join(HERE, "submit_queue_emul.cu")
CSRC = os.path.join(ROOT, "libde265_b200", "csrc")

PICTURE, READ = 0, 1
FAIL_PLAN, FAIL_ISSUE = 1, 2
B200_ERR_INVALID, B200_ERR_CUDA = -1, -2
THREADS = [1, 3, 8]
u64 = C.c_ulonglong


def build_emulator():
    deps = [SRC, os.path.join(CSRC, "submit_queue.cuh"), os.path.join(ROOT, "include", "b200hevc.h")]
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden,-pthread", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", SO, SRC])


def load():
    lib = C.CDLL(SO)
    lib.sq_create.restype = C.c_void_p
    lib.sq_create.argtypes = [C.c_int]
    for f in ("sq_destroy", "sq_stop"):
        getattr(lib, f).argtypes = [C.c_void_p]
    lib.sq_picture.restype = lib.sq_read.restype = lib.sq_last_ticket.restype = lib.sq_slot_ticket.restype = u64
    lib.sq_picture.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.sq_read.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.sq_wait.argtypes = [C.c_void_p, u64]
    lib.sq_last_ticket.argtypes = [C.c_void_p]
    lib.sq_slot_ticket.argtypes = [C.c_void_p, C.c_int]
    lib.sq_open_gate.argtypes = [C.c_void_p, C.c_int]
    lib.sq_last_error.restype = C.c_char_p
    for f in ("sq_thread_starts", "sq_live_threads", "sq_max_queued", "sq_gate_timeouts"):
        getattr(lib, f).argtypes = [C.c_void_p]
    lib.sq_log.argtypes = [C.c_void_p, C.POINTER(u64), C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int]
    lib.sq_plan_order.argtypes = [C.c_void_p, C.POINTER(u64), C.c_int]
    return lib


class Queue:
    """One SubmitQueue with `n` planner threads; picture() / read() return the ticket."""

    def __init__(self, lib, n):
        self.lib, self.n = lib, n
        self.h = lib.sq_create(n)
        assert self.h

    def picture(self, slot, plan_us=0, fail=0, gate=0, hold_until=0):
        return self.lib.sq_picture(self.h, slot, plan_us, fail, gate, hold_until)

    def read(self, slot, fail=0):
        return self.lib.sq_read(self.h, slot, fail)

    def wait(self, ticket):
        rc = self.lib.sq_wait(self.h, ticket)
        return rc, self.lib.sq_last_error().decode()

    def flush(self):
        return self.wait(self.lib.sq_last_ticket(self.h))

    def log(self):
        cap = 4096
        t, k, s = (u64 * cap)(), (C.c_int * cap)(), (C.c_int * cap)()
        n = self.lib.sq_log(self.h, t, k, s, cap)
        return [(t[i], k[i], s[i]) for i in range(n)]

    def tickets(self):
        return [e[0] for e in self.log()]

    def plan_order(self):
        cap = 4096
        t = (u64 * cap)()
        return list(t[:self.lib.sq_plan_order(self.h, t, cap)])

    def close(self):
        if self.h:
            self.lib.sq_destroy(self.h)
            self.h = None


@pytest.fixture(scope="module")
def emulator():
    build_emulator()


def isolated(check, n, queue_env=None, limit=60):
    """Runs check(n) of this module in a child process; fails if it fails or does not finish within `limit` seconds."""
    env = {k: v for k, v in os.environ.items() if k not in ("B200_ASYNC_QUEUE", "B200_HOST_PROF")}
    if queue_env:
        env["B200_ASYNC_QUEUE"] = queue_env
    code = f"import test_cpu_submit_queue as t; t.{check}({n})"
    try:
        r = subprocess.run([sys.executable, "-c", code], cwd=HERE, env=env, capture_output=True, text=True, timeout=limit)
    except subprocess.TimeoutExpired:
        pytest.fail(f"{check}({n}) did not finish within {limit} s: the queue hangs")
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("n", THREADS)
def test_issue_order_is_submission_order(emulator, n):
    isolated("check_issue_order", n)


def check_issue_order(n):
    q = Queue(load(), n)
    # pictures and read-backs interleaved; every plan takes longer than the next one, so plans finish in reverse order
    kinds = [PICTURE, PICTURE, READ, PICTURE, READ, PICTURE, PICTURE, READ, PICTURE, PICTURE, READ, PICTURE]
    n_pic = kinds.count(PICTURE)
    want, i_pic = [], 0
    for i, k in enumerate(kinds):
        slot = i % 5
        if k == PICTURE:
            t = q.picture(slot, plan_us=12000 * (n_pic - i_pic))
            i_pic += 1
        else:
            t = q.read(slot)
        want.append((t, k, slot))
    assert [w[0] for w in want] == list(range(1, len(kinds) + 1))  # one ticket sequence across both kinds
    assert q.lib.sq_last_ticket(q.h) == len(kinds)
    assert q.flush()[0] == 0
    assert q.log() == want
    order = q.plan_order()
    assert sorted(order) == [w[0] for w in want if w[1] == PICTURE]
    if n > 1:
        assert order != sorted(order), "no plan finished before an earlier one: the order check proved nothing"
    q.close()


@pytest.mark.parametrize("n", THREADS)
def test_wait_ticket(emulator, n):
    isolated("check_wait_ticket", n)


def check_wait_ticket(n):
    q = Queue(load(), n)
    assert q.wait(0)[0] == 0  # nothing queued yet
    ts = [q.picture(i, plan_us=20000) for i in range(6)]
    assert q.wait(ts[2])[0] == 0
    assert q.tickets()[:3] == ts[:3]  # every command up to the ticket has been issued
    assert q.wait(10**12)[0] == 0  # a ticket never handed out: everything queued so far
    assert q.tickets() == ts
    q.close()


@pytest.mark.parametrize("n", THREADS)
def test_slot_ticket_is_not_a_flush(emulator, n):
    isolated("check_slot_ticket", n)


def check_slot_ticket(n):
    q = Queue(load(), n)
    assert q.lib.sq_slot_ticket(q.h, 0) == 0
    t1 = q.picture(0)
    t2 = q.read(0)
    t3 = q.picture(1, gate=1)  # held until the gate opens
    t4 = q.picture(2)
    assert [q.lib.sq_slot_ticket(q.h, s) for s in (0, 1, 2, 5)] == [t2, t3, t4, 0]  # last picture writing / read-back of the slot
    assert q.wait(q.lib.sq_slot_ticket(q.h, 0))[0] == 0
    # returned while the later picture's plan is still held: waiting for slot 0 did not wait for it
    assert q.lib.sq_gate_timeouts(q.h) == 0
    assert q.tickets() == [t1, t2]
    q.lib.sq_open_gate(q.h, 1)
    assert q.flush()[0] == 0
    assert q.tickets() == [t1, t2, t3, t4]
    t5 = q.picture(0)
    t6 = q.read(1)
    assert (q.lib.sq_slot_ticket(q.h, 0), q.lib.sq_slot_ticket(q.h, 1)) == (t5, t6)
    assert q.flush()[0] == 0
    assert q.lib.sq_gate_timeouts(q.h) == 0
    q.close()


# A wait reports the first queued error whichever command it came from: wait(t) may report the error of a command after t when
# the sequencer has already retired it.  That is the engine's contract too (b200_engine_wait_ticket); these checks do not pin it.
@pytest.mark.parametrize("n", THREADS)
def test_errors_reported_once_by_the_next_wait(emulator, n):
    isolated("check_errors", n)


def check_errors(n):
    q = Queue(load(), n)
    ts = [q.picture(i, plan_us=5000, fail=FAIL_PLAN if i == 2 else 0) for i in range(5)]
    rc, msg = q.flush()
    assert rc == B200_ERR_INVALID
    m = re.fullmatch(r"plan of ticket (\d+) failed on planner (\d+)", msg)  # set on a planner thread, reported on this one
    assert m and int(m.group(1)) == ts[2] and int(m.group(2)) < n, msg
    assert q.tickets() == [ts[0], ts[1], ts[3], ts[4]]  # skipped; its neighbours issued
    assert q.flush()[0] == 0  # cleared
    assert q.wait(ts[4])[0] == 0

    us = [q.picture(5), q.read(5, fail=FAIL_ISSUE), q.picture(6, plan_us=5000), q.read(6)]
    rc, msg = q.flush()
    assert (rc, msg) == (B200_ERR_CUDA, f"issue of ticket {us[1]} failed")
    assert q.tickets()[-3:] == [us[0], us[2], us[3]]
    assert q.flush()[0] == 0
    q.close()


@pytest.mark.parametrize("n", THREADS)
@pytest.mark.parametrize("queue_env", [None, "3"])
def test_back_pressure_pictures(emulator, n, queue_env):
    isolated("check_back_pressure_pictures", n, queue_env)


def check_back_pressure_pictures(n):
    queue_env = os.environ.get("B200_ASYNC_QUEUE")
    depth = int(queue_env) if queue_env else min(32, n + 8)
    q = Queue(load(), n)
    # the first plan is held until `depth` pictures are in and the caller is blocked queueing the next (or got it in)
    q.picture(0, hold_until=depth)
    for i in range(1, 3 * depth):
        q.picture(i % 8, plan_us=1000)
    assert q.flush()[0] == 0
    assert q.lib.sq_gate_timeouts(q.h) == 0
    assert q.lib.sq_max_queued(q.h) == depth
    assert len(q.tickets()) == 3 * depth
    q.close()


@pytest.mark.parametrize("n", THREADS)
def test_back_pressure_read_backs(emulator, n):
    isolated("check_back_pressure_read_backs", n, queue_env="2")


def check_back_pressure_read_backs(n):
    q = Queue(load(), n)
    total = q.lib.sq_total_limit()
    # read-backs do not count towards the depth of 2 pictures, but the queue holds `total` commands at most
    q.picture(0, hold_until=total)
    for i in range(total + 40):
        q.read(i % 8)
    assert q.flush()[0] == 0
    assert q.lib.sq_gate_timeouts(q.h) == 0
    assert q.lib.sq_max_queued(q.h) == total
    assert len(q.tickets()) == total + 41
    q.close()


def live_threads(q, expect):
    """The queue's threads that have started and not yet exited, once it reaches `expect` (threads start asynchronously)."""
    for _ in range(500):
        n = q.lib.sq_live_threads(q.h)
        if n == expect:
            return n
        time.sleep(0.01)
    return n


@pytest.mark.parametrize("n", THREADS)
def test_stop_issues_what_is_queued_and_joins(emulator, n):
    isolated("check_stop", n)


def check_stop(n):
    lib = load()
    q = Queue(lib, n)
    assert live_threads(q, n + 1) == n + 1
    ts = []
    for i in range(20):
        ts.append(q.picture(i % 8, plan_us=3000))
        if i % 3 == 0:
            ts.append(q.read(i % 8))
    lib.sq_stop(q.h)  # with commands still queued
    assert q.tickets() == ts
    assert lib.sq_live_threads(q.h) == 0  # every thread joined: none is left behind
    assert lib.sq_thread_starts(q.h) == n + 1  # every planner and the sequencer ran the start step, once
    q.close()
