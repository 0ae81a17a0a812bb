"""The stage drivers' ordered worker thread (particlesfm_b200._stage.Worker), which writes the flow, depth and database
files: order, the first failure kept and later calls skipped, how join(), close() and a with block hand that failure
back, and the bounded queue, all without a device."""
import threading

import pytest

from particlesfm_b200._stage import Worker


def _fail(msg):
    raise OSError(msg)


def test_calls_run_in_submit_order_on_one_thread():
    seen = []
    w = Worker("test-worker")
    for i in range(50):
        w.submit(lambda i: seen.append((i, threading.get_ident())), i)
    assert w.join() is None
    assert [i for i, _ in seen] == list(range(50))
    assert len({t for _, t in seen}) == 1 and seen[0][1] != threading.get_ident()
    assert w.seconds >= 0.0


def test_no_call_runs_after_a_failure():
    seen = []
    w = Worker("test-worker")
    w.submit(seen.append, 0)
    w.submit(_fail, "first")
    w.submit(seen.append, 1)
    w.submit(_fail, "second")
    w.submit(seen.append, 2)
    e = w.join()
    assert isinstance(e, OSError) and str(e) == "first"
    assert seen == [0]


def test_join_returns_the_failure_and_close_raises_it():
    w = Worker("test-worker")
    w.submit(_fail, "kept")
    assert str(w.join()) == "kept"
    assert str(w.join()) == "kept"          # a second join does not wait again
    with pytest.raises(OSError, match="kept"):
        w.close()
    ok = Worker("test-worker")
    ok.submit(lambda: None)
    ok.close()


def test_with_raises_the_failure_on_a_clean_exit():
    with pytest.raises(OSError, match="kept"):
        with Worker("test-worker") as w:
            w.submit(_fail, "kept")


def test_with_does_not_replace_an_exception_in_flight():
    with pytest.raises(KeyError, match="in flight"):
        with Worker("test-worker") as w:
            w.submit(_fail, "kept")
            raise KeyError("in flight")
    assert str(w.error) == "kept"


def test_no_thread_is_alive_after_join():
    before = set(threading.enumerate())
    w = Worker("test-worker")
    w.submit(_fail, "x")
    w.submit(lambda: None)
    w.join()
    assert set(threading.enumerate()) == before
    with Worker("test-worker") as w:
        w.submit(lambda: None)
    assert set(threading.enumerate()) == before


def test_a_bounded_queue_blocks_the_submitter_at_its_bound():
    started, gate = threading.Event(), threading.Event()

    def hold():
        started.set()
        gate.wait()

    w = Worker("test-worker", maxsize=1)
    w.submit(hold)
    assert started.wait(10)                 # the thread holds the first call
    w.submit(lambda: None)                  # fills the one waiting slot
    third = threading.Thread(target=w.submit, args=(lambda: None,))
    third.start()
    third.join(0.2)
    assert third.is_alive()                 # blocked at the bound
    gate.set()
    third.join(10)
    assert not third.is_alive()
    w.close()
