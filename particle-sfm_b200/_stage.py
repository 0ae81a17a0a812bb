"""The host plumbing the frame-based stage drivers share (optical_flow, midas, sfm; DESIGN.md §4.14): an ordered worker
thread, the sink that writes a stage's batches on one, the frame reader, the checkpoint loader and key checks, and the
device checks."""
import ctypes
import os
import queue
import threading
import time
from collections import OrderedDict
from concurrent.futures import ThreadPoolExecutor

from . import _abi, _lib


def stream():
    """torch's current CUDA stream as the C ABI takes it."""
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_device(what):
    """PsfmError PSFM_ERR_NO_DEVICE naming the stage `what` when no CUDA device is visible."""
    from . import device_count
    if device_count() <= 0:
        raise _lib.PsfmError("%s: no CUDA device (the product has no CPU path)" % what, _abi.PSFM_ERR_NO_DEVICE)


# ----------------------------------------------------------------------------- weights

def load_checkpoint(path):
    """torch.load(path, weights_only=True) on the host; ValueError naming the file when it does not exist or cannot be
    read as a checkpoint."""
    import torch
    if not os.path.isfile(path):
        raise ValueError("%s: no such weights file" % path)
    try:
        return torch.load(path, map_location="cpu", weights_only=True)
    except Exception as e:
        raise ValueError("%s: not a readable checkpoint (%s)" % (path, e)) from None


def check_keys(sd, shapes, what):
    """ValueError naming the key for the first key of the state dict sd that shapes {key: shape} does not hold or whose
    value is not a tensor of that shape, then for the first key of shapes that sd lacks."""
    import torch
    for k, v in sd.items():
        if k not in shapes:
            raise ValueError("%s: unexpected key %r" % (what, k))
        if not isinstance(v, torch.Tensor) or tuple(v.shape) != shapes[k]:
            raise ValueError("%s: key %r has shape %s, expected %s" % (what, k, tuple(getattr(v, "shape", ())), shapes[k]))
    for k in shapes:
        if k not in sd:
            raise ValueError("%s: missing key %r" % (what, k))


# ----------------------------------------------------------------------------- threads

class Worker:
    """One thread that runs the submitted calls in order.  The first exception a call raises is kept and every later
    call is skipped; submit() does not raise it, so the caller can finish its own work and collect the failure at the
    end.  maxsize bounds the calls waiting (0: no bound), and submit() blocks while that many wait.  seconds: the
    thread's time in calls.

    join() ends the thread once the calls submitted so far have run (or been skipped) and returns the kept exception
    or None; close() joins and raises it.  As a context manager the worker joins on exit, and raises the kept exception
    only when no other exception is already propagating."""

    def __init__(self, name, maxsize=0):
        self.error, self.seconds = None, 0.0
        self._q = queue.Queue(maxsize)
        self._thread = threading.Thread(target=self._run, name=name, daemon=True)
        self._thread.start()

    def submit(self, fn, *args):
        self._q.put((fn, args))

    def _run(self):
        while True:
            item = self._q.get()
            if item is None:
                return
            if self.error is None:
                t0 = time.perf_counter()
                try:
                    item[0](*item[1])
                except BaseException as e:          # handed to the calling thread by join()
                    self.error = e
                self.seconds += time.perf_counter() - t0

    def join(self):
        if self._thread is not None:
            self._q.put(None)
            self._thread.join()
            self._thread = None
        return self.error

    def close(self):
        if self.join() is not None:
            raise self.error

    def __enter__(self):
        return self

    def __exit__(self, kind, value, tb):
        if self.join() is not None and kind is None:
            raise self.error


class PinnedSink(Worker):
    """A stage's sink, sink(meta, *device tensors), that writes each batch on its worker thread while the next batch
    runs: the tensors are copied into new pinned host buffers on torch's current stream, and once that copy is done the
    thread calls self.write(meta, *host tensors), which a subclass defines.  A failed write is also raised by the next
    call.  At most 2 batches wait, which caps the pinned host memory held."""

    def __init__(self, name):
        super().__init__(name, maxsize=2)

    def __call__(self, meta, *tensors):
        import torch
        if self.error is not None:
            raise self.error
        host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in tensors]
        for h, t in zip(host, tensors):
            h.copy_(t, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self.submit(self._write_copied, ev, meta, host)

    def _write_copied(self, ev, meta, host):
        ev.synchronize()
        self.write(meta, *host)


# ----------------------------------------------------------------------------- frames

class FrameReader:
    """Decodes the frames a run needs, in order, on host threads into pinned [H][W][3] uint8 tensors, a few ahead of
    their use; upload(i) copies frame i on the copy stream and returns the device tensor, ordered before torch's
    current stream.  decode(path) gives a frame as an [H][W][3] uint8 RGB array."""

    AHEAD = 6

    def __init__(self, paths, order, decode):
        import torch
        self.paths, self.order, self.next, self.decode = paths, list(order), 0, decode
        self.pool = ThreadPoolExecutor(max_workers=4, thread_name_prefix="psfm-frame-reader")
        self.pending = OrderedDict()
        self.copy = torch.cuda.Stream()
        self._fill()

    def _decode(self, i):
        import torch
        a = self.decode(self.paths[i])
        t = torch.empty(a.shape, dtype=torch.uint8, pin_memory=True)
        t.numpy()[...] = a
        return t

    def _fill(self):
        while self.next < len(self.order) and len(self.pending) < self.AHEAD:
            i = self.order[self.next]
            self.pending[i] = self.pool.submit(self._decode, i)
            self.next += 1

    def upload(self, i):
        import torch
        host = self.pending.pop(i).result()
        self._fill()
        with torch.cuda.stream(self.copy):
            dev = host.to("cuda", non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy)
        torch.cuda.current_stream().wait_event(ev)
        dev.record_stream(torch.cuda.current_stream())
        ev.synchronize()            # the pinned buffer may be freed once the copy has left it
        return dev

    def close(self):
        for f in self.pending.values():
            f.cancel()
        self.pool.shutdown(wait=True)
