"""Data parallelism: one process per GPU (torchrun), the batch sharded over ranks (SURVEY 8(e)).

The reference is single-device; reproducing ITS function on a sharded batch needs two exchanges:

* **BatchNorm batch statistics** (conv4_1 / conv4_2, network.py:177-178): 2 x 512 f64 sums per layer, forward and backward.
  They are exchanged INSIDE the BN finalize kernel over NVLink peer memory (csrc/peer.cu: P2P stores into every rank's inbox,
  release/acquire flags at system scope, fixed-order summation -> bit-identical statistics on all ranks, no collective launch);
  ``setup_peer_memory`` creates the inboxes (cudaMalloc + CUDA IPC, handles exchanged through torch.distributed).  Without peer
  memory the C library calls back into ``_allreduce_cb`` (an NCCL all-reduce of the 8 KB buffer).
* **Gradients**: SUM over ranks of the flat f32 buffer (7 158 592 floats, 28.6 MB), then the configured solver's step
  (``CrnnModel.apply_gradients(grad_mul=1/world, wd_mul=world)``: Adam, Momentum or RMSProp) -- the global-norm clip sees the
  reduced gradient (train.py:81-83).  ``crnn_backward`` announces each contiguous
  range of the buffer as soon as it is final (LSTM+logits first, conv1+conv2 last); ``GradBuckets`` all-reduces every range
  on a side stream while the rest of the backward pass runs, and ``finish()`` makes the compute stream wait for them.
"""
import ctypes

import numpy as np
import torch
import torch.distributed as dist

from . import _lib


def is_initialized():
    return dist.is_available() and dist.is_initialized()


def world_size():
    return dist.get_world_size() if is_initialized() else 1


def rank():
    return dist.get_rank() if is_initialized() else 0


def allreduce_sum_(flat):
    """In-place SUM all-reduce of a flat tensor (no-op for world size 1)."""
    if world_size() > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    return flat


def broadcast_(flat, src=0):
    if world_size() > 1:
        dist.broadcast(flat, src=src)
    return flat


def shard_batch(data, labels, label_len, time_step_len, rank_, world):
    """Contiguous sample shard of one global batch (data-layer tuple, gen.py:67): returns this rank's
    (data, flat_labels, label_len, time_step_len).  N must be divisible by world."""
    data = np.asarray(data); labels = np.asarray(labels); label_len = np.asarray(label_len); time_step_len = np.asarray(time_step_len)
    N = data.shape[0]
    if N % world != 0:
        raise ValueError(f"global batch {N} is not divisible by world size {world}")
    per = N // world
    lo, hi = rank_ * per, (rank_ + 1) * per
    offs = np.concatenate([[0], np.cumsum(label_len)])
    return data[lo:hi], labels[offs[lo]:offs[hi]], label_len[lo:hi], time_step_len[lo:hi]


def bucket_ranges(table, total):
    """The 7 ranges crnn_backward announces, in announcement order (mirrors csrc/backward.cu): (offset, count) pairs that tile
    [0, total) exactly once.  `table`: OrderedDict name -> (offset, shape) as CrnnModel.table holds it."""
    off = lambda n: table[n][0]
    marks = [("logits/bidirectional_rnn/fw/lstm_cell/weights", None), ("conv5/weights", "logits/bidirectional_rnn/fw/lstm_cell/weights"),
             ("conv4_2/weights", "conv5/weights"), ("conv4_1/weights", "conv4_2/weights"), ("conv3_2/weights", "conv4_1/weights"),
             ("conv3_1/weights", "conv3_2/weights"), ("conv1/weights", "conv3_1/weights")]
    return [(off(a), (off(b) if b else total) - off(a)) for a, b in marks]


class GradBuckets(object):
    """Overlap of the gradient all-reduce with the backward pass: registered as the model's grad-ready callback.

    The announced ranges arrive in descending address order and are contiguous, so they are merged until `min_bucket_bytes` are
    ready; each bucket is all-reduced on a side stream.  `sm_reserve` SMs are left free by the persistent backward kernels so the
    collective's CTAs do not delay the tail of a full-GPU grid (without the reserve every NCCL kernel displaces persistent CTAs
    for its whole duration)."""

    def __init__(self, eng, min_bucket_bytes=8 << 20, sm_reserve=8):
        self.eng = eng
        self.stream = torch.cuda.Stream(device=eng.device)
        self.pending = []
        self.error = None
        self.enabled = True
        self.seen = []
        self.min_bucket_bytes = int(min_bucket_bytes)
        self.ready = None                                          # merged (offset, count) not yet launched
        self.launched = 0
        _lib.check(eng.lib.crnn_model_set_backward_sm_reserve(eng.handle, int(sm_reserve)))
        self._cb = _lib.GRAD_READY_FN(self._on_ready)             # keep the ctypes thunk alive
        _lib.check(eng.lib.crnn_model_set_grad_ready_callback(eng.handle, ctypes.cast(self._cb, ctypes.c_void_p), None))

    def _on_ready(self, user, offset, count, stream):
        try:
            self.seen.append((int(offset), int(count)))
            if not self.enabled or world_size() <= 1:
                return
            if self.ready is not None and offset + count == self.ready[0]:
                self.ready = (int(offset), self.ready[1] + int(count))          # contiguous with the range announced before it
            else:
                self._launch()
                self.ready = (int(offset), int(count))
            if self.ready[1] * 4 >= self.min_bucket_bytes:
                self._launch()
        except Exception as e:                                     # exceptions cannot cross the C frame: re-raised by finish()
            self.error = e

    def _launch(self):
        if self.ready is None:
            return
        offset, count = self.ready
        self.ready = None
        ev = torch.cuda.Event()
        ev.record()                                                # everything enqueued so far produced this range
        self.stream.wait_event(ev)
        with torch.cuda.stream(self.stream):
            self.pending.append(dist.all_reduce(self.eng.grads[offset:offset + count], op=dist.ReduceOp.SUM, async_op=True))
        self.launched += 1

    def finish(self):
        """Make the current (compute) stream wait for every bucket's all-reduce; returns the ranges seen this step."""
        if self.enabled and world_size() > 1 and self.error is None:
            self._launch()                                         # the remainder (conv1 + conv2: the only exposed exchange)
        for w in self.pending:
            w.wait()
        self.pending = []
        seen, self.seen = self.seen, []
        if self.error is not None:
            e, self.error = self.error, None
            raise e
        return seen

    def close(self):
        try:
            _lib.check(self.eng.lib.crnn_model_set_grad_ready_callback(self.eng.handle, None, None))
            _lib.check(self.eng.lib.crnn_model_set_backward_sm_reserve(self.eng.handle, 0))
        except Exception:
            pass


class DataParallel(object):
    """Everything a rank needs around one CrnnModel: parameter broadcast, global-batch BatchNorm, overlapped gradient exchange.

        dp = DataParallel(eng)                # after dist.init_process_group, once
        ... eng.forward / ctc_loss / eng.backward ...
        dp.step(lr, step)                     # gradient all-reduce, then clip + Adam on the reduced gradient

    `overlap=True` reduces merged gradient buckets on a side stream while the backward still runs (GradBuckets).  Every
    overlapped NCCL kernel displaces CTAs of the persistent full-GPU GEMM grids for its duration while the exchange itself is a
    small part of the step, so the default is ONE all-reduce of the flat buffer after the backward.
    """

    def __init__(self, eng, sync_bn=True, overlap=False, peer_memory=True, min_bucket_bytes=8 << 20, sm_reserve=8):
        self.eng = eng
        self.rank, self.world = rank(), world_size()
        self.sync_bn, self.peer = bool(sync_bn), False
        self._inbox = None
        self._opened = []
        self._xcb = None
        self.buckets = GradBuckets(eng, min_bucket_bytes=min_bucket_bytes, sm_reserve=sm_reserve) if overlap else None
        if self.world > 1:
            broadcast_(eng.params)
            _lib.check(eng.lib.crnn_model_params_changed(eng.handle))
            self._xcb = _lib.ALLREDUCE_FN(self._allreduce_cb)
            _lib.check(eng.lib.crnn_model_set_data_parallel(eng.handle, self.rank, self.world, ctypes.cast(self._xcb, ctypes.c_void_p), None))
            if peer_memory:
                self.peer = self.setup_peer_memory()
            if not self.sync_bn:
                self.set_sync_bn(False)

    # ---- fallback exchange of the BN sums: an NCCL all-reduce issued from the callback --------------------------------
    def _allreduce_cb(self, user, dev_ptr, count, is_f64, stream):
        try:
            eng = self.eng
            base = eng._ws.data_ptr()
            off = int(dev_ptr) - base
            if off < 0 or off + count * 8 > eng._ws.numel():
                return 1
            view = eng._ws[off:off + count * (8 if is_f64 else 4)].view(torch.float64 if is_f64 else torch.float32)
            dist.all_reduce(view, op=dist.ReduceOp.SUM)
            return 0
        except Exception:
            return 1

    # ---- peer-memory inboxes -------------------------------------------------------------------------------------------
    def setup_peer_memory(self):
        lib = self.eng.lib
        ptr = _lib.c_void_p()
        handle = (ctypes.c_ubyte * 64)()
        ok = lib.crnn_peer_inbox_create(ctypes.byref(ptr), handle) == 0
        blob = bytes(handle) if ok else None
        blobs = [None] * self.world
        dist.all_gather_object(blobs, blob)
        if any(b is None for b in blobs):
            return False
        ptrs = (ctypes.c_void_p * self.world)()
        good = True
        for r in range(self.world):
            if r == self.rank:
                ptrs[r] = ptr.value
                continue
            p = _lib.c_void_p()
            h = (ctypes.c_ubyte * 64).from_buffer_copy(blobs[r])
            if lib.crnn_peer_inbox_open(h, ctypes.byref(p)) != 0:
                good = False
                break
            ptrs[r] = p.value
            self._opened.append(p.value)
        flags = [None] * self.world
        dist.all_gather_object(flags, good)
        if not all(flags):
            return False
        self._inbox = ptr.value
        _lib.check(lib.crnn_model_set_peers(self.eng.handle, self.rank, self.world, ptrs))
        torch.cuda.synchronize(self.eng.device)
        dist.barrier()                                             # every inbox is zeroed and mapped before the first exchange
        return True

    def set_sync_bn(self, flag):
        """Switch the BN layers between GLOBAL-batch statistics (training semantics of the single-device reference) and
        per-replica statistics (independent inference replicas).  The peer inboxes / callback stay registered."""
        if self.world <= 1:
            return
        cb = ctypes.cast(self._xcb, ctypes.c_void_p) if self._xcb is not None else None
        _lib.check(self.eng.lib.crnn_model_set_data_parallel(self.eng.handle, self.rank if flag else 0, self.world if flag else 1, cb, None))
        self.sync_bn = bool(flag)

    def peer_error(self):
        e = _lib.c_int()
        _lib.check(self.eng.lib.crnn_peer_error(self.eng.handle, e))
        return int(e.value)

    # ---- optimizer step on the reduced gradient -----------------------------------------------------------------------
    def reduce_gradients(self):
        if self.world <= 1:
            if self.buckets is not None:
                self.buckets.finish()
            return
        if self.buckets is not None and self.buckets.enabled:
            seen = self.buckets.finish()
            if sum(c for _, c in seen) != self.eng.total:          # backward did not announce the whole buffer: reduce it all
                allreduce_sum_(self.eng.grads)
        else:
            if self.buckets is not None:
                self.buckets.finish()
            allreduce_sum_(self.eng.grads)

    def step(self, lr, step, clip=10.0):
        self.reduce_gradients()
        self.eng.apply_gradients(lr, step, clip=clip, grad_mul=1.0 / self.world, wd_mul=float(self.world))

    def close(self):
        if self.buckets is not None:
            self.buckets.close()
        lib = self.eng.lib
        if self._inbox is not None:
            torch.cuda.synchronize(self.eng.device)
            try:
                lib.crnn_model_set_peers(self.eng.handle, 0, 1, None)
                for p in self._opened:
                    lib.crnn_peer_inbox_close(p)
                if is_initialized():
                    dist.barrier()
                lib.crnn_peer_inbox_destroy(self._inbox)
            except Exception:
                pass
            self._inbox, self._opened = None, []
