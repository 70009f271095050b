"""``Session.run(fetches, feed_dict)`` -- the call the reference's solver makes every iteration
(lib/lstm/train.py:129-130,160; lib/lstm/test.py:77), evaluated by the sm_90a engine.

Per run: feed_dict numpy arrays -> pinned host staging -> async H2D on the current stream ->
crnn_forward -> crnn_ctc_loss / crnn_total_loss / crnn_ctc_greedy as the fetches require -> D2H of
exactly the fetched values."""
import numpy as np
import torch

from . import engine
from ._lib import CrnnError
from .lib.networks.network import Fetch, Placeholder

_NP2T = {np.dtype("float32"): torch.float32, np.dtype("int32"): torch.int32, np.dtype("uint8"): torch.uint8}
LOSS_KINDS = ("loss", "ctc_costs", "train_op", "ctc_grad")


class _Pinned(object):
    """Host->device staging.  Default: copy into reusable pinned staging buffers, then async DMA.  A LARGE C-contiguous
    numpy input that is fed again from the same buffer (a feeder reusing its batch buffers) is page-locked IN PLACE on its
    second sighting (cudaHostRegister) and DMA'd directly from then on.  The registry keeps a reference to every registered
    array, so its memory cannot be freed or reused while it is pinned; the oldest entry is unregistered on overflow."""
    REGISTER_MIN_BYTES = 8 << 20
    MAX_REGISTERED = 16

    def __init__(self):
        self.bufs = {}
        self.events = {}              # staging buffer name -> event recorded after its last H2D copy
        self.pending = []             # events of copies that read the CALLER's memory in place
        self.registered = {}          # (ptr, nbytes) -> array (keeps the memory alive), insertion-ordered
        self.seen_once = {}           # (ptr, nbytes) -> True, bounded
        from . import _lib
        self._is_pinned = _lib.load().crnn_host_is_pinned

    def _registered(self, arr):
        key = (arr.ctypes.data, arr.nbytes)
        if key in self.registered:
            return True
        if key not in self.seen_once:
            if len(self.seen_once) > 64:
                self.seen_once.pop(next(iter(self.seen_once)))
            self.seen_once[key] = True
            return False
        rt = torch.cuda.cudart()
        if len(self.registered) >= self.MAX_REGISTERED:
            old = next(iter(self.registered))
            rt.cudaHostUnregister(old[0])
            del self.registered[old]
        if int(rt.cudaHostRegister(arr.ctypes.data, arr.nbytes, 0)) != 0:
            return False
        self.registered[key] = arr
        self.seen_once.pop(key, None)
        return True

    def is_page_locked(self, arr):
        """True when `arr` lives in page-locked memory: registered in place by stage(), or allocated pinned by the caller
        (e.g. a PrefetchFeeder ring slot) -- asked of the driver through crnn_host_is_pinned."""
        return (arr.ctypes.data, arr.nbytes) in self.registered or bool(self._is_pinned(arr.ctypes.data))

    def wait_pending(self):
        for ev in self.pending:
            ev.synchronize()
        self.pending = []

    def close(self):
        rt = torch.cuda.cudart()
        for (ptr, _n) in list(self.registered):
            rt.cudaHostUnregister(ptr)
        self.registered.clear()

    def stage_ints(self, arrays, device, name="_ints"):
        """The small int32 feeds of one run (time_step_len, labels, labels_len) through ONE pinned staging buffer and ONE async
        copy; returns {name: device view}.  Sub-arrays start on 256-byte boundaries."""
        offs, tot = {}, 0
        for k, a in arrays.items():
            offs[k] = tot
            tot += (max(a.size, 1) + 63) // 64 * 64
        t = self.bufs.get(name)
        if t is None or t.numel() < tot:
            t = self.bufs[name] = torch.empty(max(tot, 4096), dtype=torch.int32).pin_memory()
            self.events.pop(name, None)
        ev = self.events.get(name)
        if ev is not None:
            ev.synchronize()          # the previous run's DMA out of this staging buffer must be done before it is rewritten
        tn = t.numpy()
        for k, a in arrays.items():
            tn[offs[k]:offs[k] + a.size] = a.reshape(-1)
        d = t[:tot].to(device, non_blocking=True)
        if ev is None:
            ev = self.events[name] = torch.cuda.Event()
        ev.record()
        return {k: d[offs[k]:offs[k] + a.size].view(a.shape) for k, a in arrays.items()}

    def staging_for(self, name, numel, dtype=torch.float32):
        """Page-locked staging buffer `name` of `dtype` (f32, or uint8 for pixel batches) with room for `numel` elements, safe to
        overwrite (the previous DMA out of it has completed), and the event the caller must record after issuing the next DMA out
        of it."""
        t = self.bufs.get(name)
        if t is None or t.numel() < numel or t.dtype != dtype:
            t = self.bufs[name] = torch.empty(max(numel, 1), dtype=dtype).pin_memory()
            self.events.pop(name, None)
        ev = self.events.get(name)
        if ev is not None:
            ev.synchronize()
        else:
            ev = self.events[name] = torch.cuda.Event()
        return t, ev

    def stage(self, name, arr, device):
        arr = np.ascontiguousarray(arr)
        tdt = _NP2T[arr.dtype]
        if arr.nbytes >= self.REGISTER_MIN_BYTES and arr.flags.owndata and self._registered(arr):
            d = torch.from_numpy(arr).to(device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            self.pending.append(ev)   # DMA straight out of the caller's array: run() waits for it before returning
            return d
        t = self.bufs.get(name)
        if t is None or t.numel() < arr.size or t.dtype != tdt:
            t = torch.empty(max(arr.size, 1), dtype=tdt).pin_memory()
            self.bufs[name] = t
            self.events.pop(name, None)
        ev = self.events.get(name)
        if ev is not None:
            ev.synchronize()          # the previous run's DMA out of this staging buffer must be done before it is rewritten
        v = t[:arr.size].view(arr.shape)
        v.copy_(torch.from_numpy(arr))
        d = v.to(device, non_blocking=True)
        if ev is None:
            ev = self.events[name] = torch.cuda.Event()
        ev.record()
        return d


class Session(object):
    def __init__(self, device=None):
        if not torch.cuda.is_available():
            raise CrnnError("Session needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self._engines = {}
        self._pinned = _Pinned()
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        self.last_feed_path = None    # "page-locked in place" (chunked crnn_forward_host) | "staged" (copy into pinned staging first)
        import os
        self.h2d_chunks = int(os.environ.get("CRNN_H2D_CHUNKS", "4"))   # image ranges of the overlapped host->device feed (1 = copy, then compute)
        self.pageable_pool = not os.environ.get("CRNN_NO_PAGEABLE_POOL")   # large pageable batches through crnn_forward_pageable (else: torch copy into staging, then copy-then-compute)
        self.host_copy_threads = int(os.environ.get("CRNN_HOST_COPY_THREADS", str(min(8, os.cpu_count() or 1))))   # pageable -> pinned staging copies
        # device prefetch (attach_feeder): the NEXT batch of a PrefetchFeeder is copied host->device on a side stream while the
        # current step computes -- what tf.data's prefetch_to_device does for a TF input pipeline
        self._feeder = None
        self._ahead = None                      # (feeder sequence number, host ptr, nbytes, device tensor, copy-done event, buffer index)
        self._ahead_bufs = [None, None]
        self._ahead_free = [None, None]         # per buffer: event recorded on the compute stream after the last step that read it
        self._ahead_idx = 0
        self._ahead_stream = None
        self.ahead_hits = 0

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def close(self):
        torch.cuda.synchronize(self.device)
        self._feeder = None
        self._ahead = None
        self._ahead_bufs = [None, None]
        self._pinned.close()
        self._engines.clear()

    # ---- device prefetch ------------------------------------------------------------------
    def attach_feeder(self, feeder):
        """``feeder``: a PrefetchFeeder (anything with ``peek()`` and ``delivered``) whose batches are fed to ``run`` in order.
        From then on every ``run`` starts the host->device copy of the feeder's NEXT batch on a side stream before it waits for
        its own results, and the next ``run`` finds its input already resident (the copy is still one H2D per step, issued
        from the page-locked ring slot; it just overlaps the previous step instead of preceding its own).  ``None`` detaches."""
        self._feeder = feeder if (feeder is not None and hasattr(feeder, "peek") and hasattr(feeder, "delivered")) else None
        self._ahead = None

    def _stage_ahead(self):
        f = self._feeder
        if f is None or self._ahead is not None:
            return
        try:
            nxt = f.peek()
        except StopIteration:
            return
        data = nxt[0]
        if not (isinstance(data, np.ndarray) and data.dtype in (np.float32, np.uint8) and data.flags.c_contiguous and data.ndim == 3
                and self._pinned.is_page_locked(data)):
            return
        i = self._ahead_idx
        buf = self._ahead_bufs[i]
        if buf is None or tuple(buf.shape) != tuple(data.shape) or buf.dtype != _NP2T[data.dtype]:
            buf = self._ahead_bufs[i] = torch.empty(data.shape, dtype=_NP2T[data.dtype], device=self.device)
            self._ahead_free[i] = None
        if self._ahead_stream is None:
            self._ahead_stream = torch.cuda.Stream(device=self.device)
        st = self._ahead_stream
        if self._ahead_free[i] is not None:
            st.wait_event(self._ahead_free[i])   # the step that last read this device buffer has finished with it
        # the small integer feeds of that batch too (validated here, off the critical path); run() re-uses them when the arrays it
        # is fed compare equal
        ints = None
        try:
            h = {"labels": np.ascontiguousarray(nxt[1], dtype=np.int32), "llen": np.ascontiguousarray(nxt[2], dtype=np.int32),
                 "tsl": np.ascontiguousarray(nxt[3], dtype=np.int32)}
            self.validate_feed(data, h["tsl"], h["labels"], h["llen"])
        except Exception:
            h = None                            # run() will validate what it is actually fed and raise there
        with torch.cuda.stream(st):
            buf.copy_(torch.from_numpy(data), non_blocking=True)
            if h is not None:
                ints = (h, self._pinned.stage_ints(h, self.device, name="_ints_ahead%d" % i))
            ev = torch.cuda.Event()
            ev.record(st)
        self._ahead = (f.delivered, data.ctypes.data, data.nbytes, buf, ev, i, ints)   # f.delivered == sequence number of the peeked batch
        self._ahead_idx = i ^ 1

    def _take_ahead(self, data):
        """Device copy of `data` if it is the batch staged ahead (same feeder sequence number, same ring slot), else None."""
        a, f = self._ahead, self._feeder
        if a is None or f is None:
            return None
        self._ahead = None
        seq, ptr, nbytes, buf, ev, i, ints = a
        if (seq != f.delivered - 1 or ptr != data.ctypes.data or nbytes != data.nbytes or tuple(buf.shape) != tuple(data.shape)
                or buf.dtype != _NP2T[data.dtype]):
            return None
        torch.cuda.current_stream(self.device).wait_event(ev)
        self._pinned.pending.append(ev)        # the ring slot must not be recycled before this DMA is done (it is, long before)
        return buf, i, ints

    # ---- variables ------------------------------------------------------------------------
    def engine_for(self, net):
        eng = self._engines.get(id(net))
        if eng is None:
            from .lib.lstm.config import cfg
            # evaluation networks run in cfg.TEST.COMPUTE_DTYPE ("bf16" or "fp8") and normalise conv4_x with cfg.TEST.BN_STATS
            # ("batch" or "moving"); training networks ignore both keys
            test = type(net).__name__ == "LSTM_test"
            dt = str(cfg.TEST.get("COMPUTE_DTYPE", "bf16")) if test else "bf16"
            if dt not in ("bf16", "fp8"):
                raise ValueError(f"cfg.TEST.COMPUTE_DTYPE must be 'bf16' or 'fp8', got {dt!r}")
            bn = str(cfg.TEST.get("BN_STATS", "batch")) if test else "batch"
            if bn not in ("batch", "moving"):
                raise ValueError(f"cfg.TEST.BN_STATS must be 'batch' or 'moving', got {bn!r}")
            eng = engine.CrnnModel(weight_decay=float(getattr(net, "_wd", cfg.TRAIN.WEIGHT_DECAY)), device=self.device,
                                   compute_dtype=dt)
            eng.set_bn_statistics(bn)
            self._engines[id(net)] = eng
        return eng

    def assign(self, net, state_dict, ignore_missing=False):
        eng = self.engine_for(net)
        full = eng.state_dict()
        for k in full:
            if k in state_dict:
                full[k] = np.asarray(state_dict[k], dtype=np.float32).reshape(full[k].shape)
            elif not ignore_missing:
                raise KeyError(k)
        eng.load_params(full)
        # moving statistics under their TF names (engine.BN_MOVING_KEYS) when given; required by an engine that evaluates with them
        if all(k in state_dict for k in engine.BN_MOVING_KEYS):
            eng.load_bn_moving(state_dict)
        elif eng.bn_statistics == "moving" and not ignore_missing:
            raise KeyError("cfg.TEST.BN_STATS is 'moving' but no moving statistics were given ({})".format(", ".join(engine.BN_MOVING_KEYS)))
        self.params_loaded(net)

    def params_loaded(self, net):
        """Call after a network's parameters were (re)loaded -- assign and checkpoint restores do.  An fp8 engine gets its
        activation scales here: a parameter change invalidates them."""
        eng = self.engine_for(net)
        if eng.compute_dtype == 4:
            self._calibrate_fp8(eng)

    FP8_CALIBRATION_LINES, FP8_CALIBRATION_WIDTH = 256, 256

    def _calibrate_fp8(self, eng):
        """An fp8 engine's activation scales from a fixed calibration set the package renders itself: 256 lines of the data
        path's default stream (seed cfg.RNG_SEED) drawn in Pillow's embedded font (whatever fonts the machine has), padded to
        256 px.  The scales depend on the weights (and the Pillow version) alone, never on the lines being evaluated, so a
        line evaluated in a packed batch still computes as if alone."""
        import random
        from .lib.lstm.config import cfg
        from .lib.lstm.utils import gen
        if getattr(self, "_fp8_cal", None) is None:
            rng = random.Random(int(cfg.RNG_SEED))
            font = gen.embedded_font(42)
            labels = [gen.gen_rand(rng) for _ in range(self.FP8_CALIBRATION_LINES)]
            imgs, _, _, tsl = gen.groupBatch([gen.render_line(t, rng=rng, font=font) for t in labels], labels,
                                             pad_to=self.FP8_CALIBRATION_WIDTH)
            self._fp8_cal = (torch.tensor(np.stack(imgs), device=self.device), torch.tensor(np.asarray(tsl, np.int32), device=self.device))
        eng.calibrate_fp8(*self._fp8_cal)

    def variables(self, net):
        return self.engine_for(net).state_dict()

    # ---- run ------------------------------------------------------------------------------
    @staticmethod
    def validate_feed(data, tsl, labels, labels_len, line_width=None):
        """Host-side checks the C ABI cannot do without a device sync (SURVEY §8(b): invalid lengths).  With `line_width` (packed
        evaluation) every W_i must be a multiple of 4 in [8, W] and time_step_len[i] at most W_i/4 - 1."""
        if data.ndim != 3 or data.shape[2] != 32:
            raise ValueError(f"data must be [N, W, 32], got {data.shape}")
        N, W, _ = data.shape
        if W % 4 != 0 or W < 8:
            raise ValueError("padded width must be a multiple of POOL_SCALE=4 (gen.py:58) and >= 8")
        T = W // 4 - 1
        if tsl.shape != (N,):
            raise ValueError("time_step_len must be [N]")
        if tsl.min() < 0 or tsl.max() > T:
            raise ValueError(f"time_step_len must lie in [0, {T}] (conv output has W/4-1 frames)")
        if labels is not None:
            if labels_len.shape != (N,) or labels_len.min() < 0:
                raise ValueError("labels_len must be [N], non-negative")
            if int(labels_len.sum()) != labels.size:
                raise ValueError("sum(labels_len) != len(labels)")
            if labels.size and (labels.min() < 1 or labels.max() > 62):
                raise ValueError("label ids must lie in 1..62 (0 is the CTC blank, 63 the decoder blank)")
            if labels_len.size and int(labels_len.max()) > engine.CTC_MAX_LABEL_LEN:
                raise ValueError(f"a label of {int(labels_len.max())} ids is longer than the {engine.CTC_MAX_LABEL_LEN} the CTC kernels "
                                 "support")
        if line_width is not None:
            if line_width.shape != (N,):
                raise ValueError("line_width must be [N]")
            if line_width.min() < 8 or line_width.max() > W or (line_width % 4).any():
                raise ValueError(f"line_width must hold multiples of 4 in [8, {W}] (each line's padded width)")
            if (tsl > line_width // 4 - 1).any():
                raise ValueError("time_step_len[i] must be <= line_width[i]/4 - 1 (frames past a line are not defined)")

    @staticmethod
    def _data_feed(feeds):
        """The fed batch: `data` widened to f32 as a TF float placeholder casts it, or `data_u8` kept as uint8 pixels (the engine's
        u8 entry points divide by 255 on the device).  Feeding both is ambiguous and refused.  `data_u8` may also be a batch
        already on the device (gen.DeviceLineRenderer): a contiguous [N, W, 32] uint8 CUDA tensor, used in place (run checks
        that it is on the session's device)."""
        if "data_u8" in feeds:
            if "data" in feeds:
                raise ValueError("feed either data or data_u8, not both")
            d = feeds["data_u8"]
            if torch.is_tensor(d):
                if not (d.is_cuda and d.dtype == torch.uint8 and d.dim() == 3 and d.is_contiguous()):
                    raise ValueError(f"a tensor fed as data_u8 must be a contiguous [N, W, 32] uint8 CUDA tensor, got "
                                     f"{d.dtype} {tuple(d.shape)} on {d.device}")
                return d
            return np.asarray(d, dtype=np.uint8)
        return np.asarray(feeds["data"], dtype=np.float32)

    def run(self, fetches, feed_dict=None):
        single = not isinstance(fetches, (list, tuple))
        flist = [fetches] if single else list(fetches)
        feed_dict = feed_dict or {}
        net = None
        for f in flist:
            if isinstance(f, Fetch):
                net = f.net
        if net is None:
            raise ValueError("nothing to run: fetches must come from a network (build_loss / get_output)")
        feeds = {}
        for k, v in feed_dict.items():
            if not isinstance(k, Placeholder):
                raise TypeError("feed_dict keys must be the network's placeholders")
            feeds[k.name] = v
        kinds = [f.kind for f in flist]
        need_loss = any(k in LOSS_KINDS for k in kinds)
        need_labels = need_loss or "label_alignment" in kinds
        if "images" in feeds:
            clash = [k for k in ("data", "data_u8", "line_width", "time_step_len") if k in feeds]
            if clash:
                raise ValueError(f"images carries the lines, their widths and time_step_len: do not feed it with {', '.join(clash)}")
            images = self._images_feed(feeds["images"])
        data = self._data_feed(feeds) if "images" not in feeds else None
        tsl = np.asarray(feeds["time_step_len"], dtype=np.int32) if "images" not in feeds else None
        labels = np.asarray(feeds["labels"], dtype=np.int32) if need_labels else None
        llen = np.asarray(feeds["labels_len"], dtype=np.int32) if need_labels else None
        eng = self.engine_for(net)
        if eng.compute_dtype == 4 and not eng.fp8_calibrated:
            self._calibrate_fp8(eng)        # parameters loaded straight into the engine (not through assign / a restore)
        if "images" in feeds:
            return self._run_images(flist, single, eng, images, labels, llen)
        dev = self.device
        if feeds.get("line_width") is not None:
            if torch.is_tensor(data):
                raise ValueError("line_width (packed evaluation) takes host batches: feed data_u8 as a numpy array")
            return self._run_lines(flist, single, net, eng, data, tsl, labels, llen, np.asarray(feeds["line_width"], dtype=np.int32))
        # training mode is sticky: its forward is a superset (it also saves what the backward needs), and switching back
        # and forth would re-plan the multi-GB workspace
        if any(k == "train_op" for k in kinds) and not eng.training:
            eng.set_training(True)
        on_device = torch.is_tensor(data)
        if on_device and data.device != dev:
            raise ValueError(f"data_u8 is on {data.device}, the session runs on {dev}")
        if not on_device:
            data = np.ascontiguousarray(data)
        ahead = self._take_ahead(data) if not on_device else None
        d_ints = None
        if ahead is not None and ahead[2] is not None:
            h, dv = ahead[2]
            if np.array_equal(h["tsl"], tsl) and (not need_labels or (np.array_equal(h["labels"], labels) and np.array_equal(h["llen"], llen))):
                d_ints = dv                     # validated and copied while the previous step was running
        if d_ints is None:
            self.validate_feed(data, tsl, labels, llen)
            ints = {"tsl": tsl}
            if need_labels:
                ints["labels"], ints["llen"] = labels, llen
            d_ints = self._pinned.stage_ints(ints, dev)
        d_tsl = d_ints["tsl"]
        self.h2d_bytes = (0 if on_device else data.nbytes) + tsl.nbytes
        used_ahead = None
        if on_device:
            d_data = data
            logits = eng.forward(d_data, d_tsl)
            self.last_feed_path = "device-resident"
        elif ahead is not None:
            d_data, used_ahead = ahead[0], ahead[1]
            logits = eng.forward(d_data, d_tsl)
            self.last_feed_path = "page-locked in place, copied during the previous step (device prefetch)"
            self.ahead_hits += 1
        elif self.h2d_chunks > 1 and (self._pinned.is_page_locked(data) or
                                      (data.nbytes >= self._pinned.REGISTER_MIN_BYTES and data.flags.owndata and self._pinned._registered(data))):
            # page-locked batch buffer (a feeder's ring slot, or a large array fed a second time and registered in place now):
            # chunked H2D overlapped with the conv front end
            logits, d_data = eng.forward_host(data, d_tsl, chunks=self.h2d_chunks)
            self.last_feed_path = "page-locked in place"
        elif self.pageable_pool and self.h2d_chunks > 1 and data.nbytes >= self._pinned.REGISTER_MIN_BYTES:
            # large batch in ordinary memory (the reference's np.array(...) per step): the library's host threads move it into
            # page-locked staging range by range while the GPU copies / computes the previous range (crnn_forward_pageable)
            pin, ev = self._pinned.staging_for("data" + engine._feed_suffix(data.dtype), data.size, _NP2T[data.dtype])
            logits, d_data, cst = eng.forward_pageable(data, pin, d_tsl, chunks=self.h2d_chunks, host_threads=self.host_copy_threads)
            ev.record(cst)
            self.last_feed_path = "staged"
        else:
            d_data = self._pinned.stage("data" + engine._feed_suffix(data.dtype), data, dev)
            logits = eng.forward(d_data, d_tsl)
            self.last_feed_path = "staged"
        costs = grad = loss = d_lab = d_ll = None
        if need_labels:
            d_lab, d_ll = d_ints["labels"], d_ints["llen"]
            self.h2d_bytes += labels.nbytes + llen.nbytes
        if need_loss:
            N = data.shape[0]
            # warp-ctc computes the gradient inside its forward op; so does this kernel (one launch)
            costs, grad = engine.ctc_loss(logits, d_lab, d_ll, d_tsl, want_grad=True, grad_scale=1.0 / N,
                                          max_label_len=int(llen.max()) if llen.size else 0, workspace="auto")
            loss = eng.total_loss(costs)
        has_train = any(k == "train_op" for k in kinds)
        if not has_train:
            self._stage_ahead()                # everything of this step is enqueued: start the next batch's copy before waiting for results
        out = self._fetch(flist, eng, logits, d_tsl, data.shape[0], data.shape[1], loss, costs, grad, d_lab, d_ll, llen,
                          train=lambda f: f.step_fn(eng, logits, grad, d_data, d_tsl))
        if used_ahead is not None:
            ev = self._ahead_free[used_ahead]
            if ev is None:
                ev = self._ahead_free[used_ahead] = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.device))
        self._pinned.wait_pending()
        return out[0] if single else out

    @staticmethod
    def _check_lines(kinds, eng, what):
        if "train_op" in kinds:
            raise ValueError(f"{what} (packed evaluation) cannot be fed with train_op: training uses whole-batch statistics")
        if eng.training:
            raise ValueError(f"{what} (packed evaluation) needs a model that has not been switched to training")

    def _run_lines(self, flist, single, net, eng, data, tsl, labels, llen, line_width):
        """Packed evaluation (``line_width`` fed): the batch is staged to the device and every line is evaluated as if it were run
        alone (engine.CrnnModel.forward_lines).  Evaluation fetches only."""
        self._check_lines([f.kind for f in flist], eng, "line_width")
        data = np.ascontiguousarray(data)
        self.validate_feed(data, tsl, labels, llen, line_width)
        ints = {"tsl": tsl, "lw": line_width}
        if labels is not None:
            ints["labels"], ints["llen"] = labels, llen
        d_ints = self._pinned.stage_ints(ints, self.device)
        d_data = self._pinned.stage("data" + engine._feed_suffix(data.dtype), data, self.device)
        self.h2d_bytes = data.nbytes + tsl.nbytes + line_width.nbytes + (labels.nbytes + llen.nbytes if labels is not None else 0)
        self.last_feed_path = "staged"
        return self._eval_lines(flist, single, eng, d_data, d_ints, llen)

    @staticmethod
    def _images_feed(images):
        """The `images` feed checked on the host: a non-empty sequence of lines, each a 2-D uint8 array or the bytes of a PNG or JPEG
        file, of 1 .. engine.RESIZE_MAX_HEIGHT rows and at least one column (a PNG's size read from its IHDR, at most
        engine.PNG_MAX_WIDTH columns; a JPEG's from its first SOF segment).  Nothing is converted: a line of another dtype is refused
        rather than cast."""
        if isinstance(images, np.ndarray) and images.dtype != object:
            raise ValueError("images must be a sequence of 2-D uint8 arrays or PNG / JPEG file bytes (one per line), not one array")
        images = list(images)
        if not images:
            raise ValueError("images: no lines")
        for i, im in enumerate(images):
            if isinstance(im, (bytes, bytearray)):
                size = engine.png_size(im)
                if size is None:
                    size = engine.jpeg_size(im)
                    if size is None:
                        raise ValueError(f"images[{i}] is {len(im)} bytes that start with neither a PNG signature and IHDR nor "
                                         "JPEG marker segments up to an SOF")
                elif size[1] > engine.PNG_MAX_WIDTH:
                    raise ValueError(f"images[{i}] is a PNG {size[1]} columns wide: the device decoder reads at most {engine.PNG_MAX_WIDTH}")
                h, w = size
            elif not isinstance(im, np.ndarray) or im.ndim != 2 or im.dtype != np.uint8:
                raise ValueError(f"images[{i}] must be a 2-D uint8 array (a gray line) or PNG / JPEG file bytes, got "
                                 f"{getattr(im, 'dtype', type(im).__name__)} {getattr(im, 'shape', '')}")
            else:
                h, w = im.shape
            if not 1 <= h <= engine.RESIZE_MAX_HEIGHT or w < 1:
                raise ValueError(f"images[{i}] is {h} x {w}: lines need 1 .. {engine.RESIZE_MAX_HEIGHT} rows and at least one column")
        return images

    def _run_images(self, flist, single, eng, images, labels, llen):
        """Packed evaluation of native-size lines (``images`` fed, checked by _images_feed): the raw bytes go to the device in one
        copy, crnn_resize_lines_u8 resizes and packs them into the uint8 batch that prepare_line + pack_lines build on the host, and
        from forward_lines on the run is _run_lines'.  Evaluation fetches only.  PNG and JPEG entries travel encoded, and
        crnn_png_decode_gray_u8 / crnn_jpeg_decode_gray_u8 decode them in front of the resize with lib/lstm/test.py gray_rule().
        Files they refuse raise engine.PngDecodeError (PNG entries only), engine.JpegDecodeError (JPEG entries only) or
        engine.ImageDecodeError (both) naming the entries, and the run returns nothing."""
        from .lib.lstm.test import gray_rule, line_size
        self._check_lines([f.kind for f in flist], eng, "images")
        N = len(images)
        coded = [i for i, im in enumerate(images) if not isinstance(im, np.ndarray)]
        png = [i for i in coded if engine.png_size(images[i]) is not None]
        jpeg = [i for i in coded if i not in set(png)]
        hw = [im.shape if isinstance(im, np.ndarray) else engine.png_size(im) or engine.jpeg_size(im) for im in images]
        src_h = np.array([s[0] for s in hw], np.int32)
        src_w = np.array([s[1] for s in hw], np.int32)
        size = np.array([line_size(h, w) for h, w in zip(src_h, src_w)], np.int32).reshape(N, 3)
        out_w, lw, tsl = (np.ascontiguousarray(size[:, k]) for k in range(3))
        W = int(lw.max())
        # what travels: the arrays' pixels and the files' bytes; the decoded lines follow them in the same device buffer
        nbytes = np.array([len(im) if not isinstance(im, np.ndarray) else im.size for im in images], np.int64)
        offs = np.zeros(N, np.int64)
        np.cumsum(nbytes[:-1], out=offs[1:])
        tot = int(nbytes.sum())
        # labels checked as for any packed batch (a zero-stride stand-in has the batch's shape and no memory)
        self.validate_feed(np.broadcast_to(np.uint8(0), (N, W, 32)), tsl, labels, llen, lw)
        pin, ev = self._pinned.staging_for("images", tot, torch.uint8)
        pn = pin.numpy()
        for im, o in zip(images, offs):
            if isinstance(im, np.ndarray):
                pn[o:o + im.size].reshape(im.shape)[...] = im
            else:
                pn[o:o + len(im)] = np.frombuffer(im, np.uint8)
        src_offset = offs
        if coded:
            dec = src_h[coded].astype(np.int64) * src_w[coded]
            dec_off = np.zeros(len(coded), np.int64)
            np.cumsum(dec[:-1], out=dec_off[1:])
            dec_off += tot
            src_offset = offs.copy()
            src_offset[coded] = dec_off
            d_src = torch.empty(tot + int(dec.sum()), dtype=torch.uint8, device=self.device)
            d_src[:tot].copy_(pin[:tot], non_blocking=True)
        else:
            d_src = pin[:tot].to(self.device, non_blocking=True)
        ev.record()
        ints = {"off": src_offset.view(np.int32), "h": src_h, "w": src_w, "ow": out_w, "tsl": tsl, "lw": lw}
        rule = gray_rule()
        if png:
            ihdr = np.stack([np.frombuffer(images[i], np.uint8, 13, 16) for i in png])
            ws_offset, ws_bytes = engine.png_plan(ihdr, nbytes[png])
            ints.update({"foff": offs[png].view(np.int32), "flen": nbytes[png].view(np.int32), "doff": src_offset[png].view(np.int32),
                         "ws": ws_offset.view(np.int32), "ph": src_h[png], "pw": src_w[png]})
        if jpeg:
            jws_offset, jws_bytes = engine.jpeg_plan(engine.jpeg_sof_records([images[i] for i in jpeg]), nbytes[jpeg], rule)
            ints.update({"jfoff": offs[jpeg].view(np.int32), "jflen": nbytes[jpeg].view(np.int32),
                         "jdoff": src_offset[jpeg].view(np.int32), "jws": jws_offset.view(np.int32), "jh": src_h[jpeg],
                         "jw": src_w[jpeg]})
        if labels is not None:
            ints["labels"], ints["llen"] = labels, llen
        d_ints = self._pinned.stage_ints(ints, self.device)
        i64 = lambda k: d_ints[k].view(torch.int64)   # noqa: E731
        statuses = []                                  # (feed entries, pinned status, event, error class)
        if png:
            _, d_status = engine.decode_png_gray(d_src, i64("foff"), i64("flen"), d_ints["ph"], d_ints["pw"], i64("doff"), i64("ws"),
                                                 rule, out=d_src,
                                                 workspace=torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=self.device))
            status, sev = self._pinned.staging_for("png_status", len(png), torch.int32)
            status[:len(png)].copy_(d_status, non_blocking=True)
            sev.record()
            statuses.append((png, status, sev, engine.PngDecodeError))
        if jpeg:
            _, d_status = engine.decode_jpeg_gray(d_src, i64("jfoff"), i64("jflen"), d_ints["jh"], d_ints["jw"], i64("jdoff"),
                                                  i64("jws"), rule, out=d_src,
                                                  workspace=torch.empty(max(jws_bytes, 1), dtype=torch.uint8, device=self.device))
            status, sev = self._pinned.staging_for("jpeg_status", len(jpeg), torch.int32)
            status[:len(jpeg)].copy_(d_status, non_blocking=True)
            sev.record()
            statuses.append((jpeg, status, sev, engine.JpegDecodeError))
        d_data = engine.resize_lines_u8(d_src, d_ints["off"].view(torch.int64), d_ints["h"], d_ints["w"], d_ints["ow"], W,
                                        int(src_h.max()))
        self.h2d_bytes = tot + sum(a.nbytes for a in ints.values())
        self.last_feed_path = "native-size lines, resized on the device"
        out = self._eval_lines(flist, single, eng, d_data, d_ints, llen)
        refused = []                                   # (error class, entries, codes) per codec with refused files
        for entries, status, sev, err in statuses:
            sev.synchronize()
            st = status[:len(entries)].numpy()
            bad = np.flatnonzero(st)
            if bad.size:
                refused.append((err, [entries[k] for k in bad], st[bad].tolist()))
        if len(refused) == 1:
            err, entries, codes = refused[0]
            raise err(entries, codes)
        if refused:
            raise engine.ImageDecodeError.mixed([(e, c, "PNG" if err is engine.PngDecodeError else "JPEG")
                                                 for err, es, cs in refused for e, c in zip(es, cs)])
        return out

    def _eval_lines(self, flist, single, eng, d_data, d_ints, llen):
        """The fetches of a packed batch already on the device: d_data [N, W, 32], d_ints["lw"] / ["tsl"] (and ["labels"] /
        ["llen"] with labels)."""
        kinds = [f.kind for f in flist]
        N, W = d_data.shape[0], d_data.shape[1]
        d_tsl = d_ints["tsl"]
        logits = eng.forward_lines(d_data, d_ints["lw"], d_tsl)
        costs = grad = loss = None
        if any(k in LOSS_KINDS for k in kinds):
            costs, grad = engine.ctc_loss(logits, d_ints["labels"], d_ints["llen"], d_tsl, want_grad="ctc_grad" in kinds,
                                          grad_scale=1.0 / N, max_label_len=int(llen.max()) if llen.size else 0,
                                          workspace="auto")
            loss = eng.total_loss(costs)
        out = self._fetch(flist, eng, logits, d_tsl, N, W, loss, costs, grad, d_ints.get("labels"), d_ints.get("llen"), llen)
        self._pinned.wait_pending()
        return out[0] if single else out

    def _fetch(self, flist, eng, logits, d_tsl, N, W, loss, costs, grad, d_lab, d_ll, llen, train=None):
        """The values of the fetches, counting the bytes they bring to the host in d2h_bytes.  `train(f)` runs a train_op fetch (the
        whole-batch path only: packed feeds refuse it)."""
        out = []
        self.d2h_bytes = 0
        for f in flist:
            k = f.kind
            if k == "loss":
                v = loss.cpu().numpy()[0]
            elif k == "ctc_costs":
                v = costs.cpu().numpy()
            elif k == "ctc_grad":
                v = grad.cpu().numpy()
            elif k == "logits":
                v = logits.cpu().numpy()
            elif k == "dense_decoded":
                v = self._decode(logits, d_tsl)
            elif k == "read_alignment":
                v = self._read_alignment(logits, d_tsl)
            elif k == "label_alignment":
                v = self._label_alignment(logits, d_tsl, d_lab, d_ll, llen)
            elif k == "lexicon_decoded":
                v = self._lexicon_decoded(logits, d_tsl)
            elif k == "beam_decoded":
                v = self._beam_decoded(logits, d_tsl)
            elif k == "train_op" and train is not None:
                v = train(f)
                self._stage_ahead()
            elif k.startswith("layer:"):
                name = k.split(":", 1)[1]
                tapname = {"pool1": "conv1", "pool2": "conv3_2", "pool3": "conv4_2", "reshaped_layer": "conv5"}.get(name, name)
                v = eng.tap(tapname, N, W).cpu().numpy()
            else:
                raise ValueError(f"unknown fetch {f}")
            if isinstance(v, np.ndarray):
                self.d2h_bytes += v.nbytes
            elif isinstance(v, dict):
                self.d2h_bytes += sum(a.nbytes for a in v.values())
            elif isinstance(v, (np.floating, float)):
                self.d2h_bytes += 4
            out.append(v)
        return out

    @staticmethod
    def _decode_device(logits, d_tsl):
        """(out [N,T], out_len [N]) on the device, decoded with cfg.DECODER (greedy, or the reference's beam search)."""
        from .lib.lstm.config import cfg
        if str(cfg.get("DECODER", "greedy")) == "beam":
            # the reference's own decoder (network.py:656): prefix beam search, width 100, blank 63, on the device
            o, ol, _ = engine.ctc_beam_search_device(logits, d_tsl, beam_width=int(cfg.get("BEAM_WIDTH", 100)), merge_repeated=True)
        else:
            o, ol = engine.ctc_greedy(logits, d_tsl)
        return o, ol

    @staticmethod
    def _decode(logits, d_tsl):
        """dense_decoded of device logits with cfg.DECODER (greedy, or the reference's beam search on the device)."""
        return engine.dense_decoded(*Session._decode_device(logits, d_tsl)).cpu().numpy()

    @staticmethod
    def _read_alignment(logits, d_tsl):
        """"read_alignment": the best alignment (blank 0) of the read dense_decoded returns, as engine.alignment_dict."""
        o, ol = Session._decode_device(logits, d_tsl)
        dense = engine.dense_decoded(o, ol)
        r = engine.ctc_align(logits, dense, ol, d_tsl, blank=0, max_label_len=dense.shape[1])
        return engine.alignment_dict(dense.cpu().numpy(), *(a.cpu().numpy() for a in r))

    def _lexicon_decoded(self, logits, d_tsl):
        """"lexicon_decoded": each line read against cfg.TEST.LEXICON (engine.lexicon_decode, blank 0) from the read dense_decoded
        returns (cfg.DECODER applies).  The word list is loaded once per path and device and stays on the device."""
        from .lib.lstm.config import cfg
        path = str(cfg.TEST.get("LEXICON", ""))
        if not path:
            raise ValueError('the "lexicon_decoded" fetch needs cfg.TEST.LEXICON (a word-list file)')
        cache = self.__dict__.setdefault("_lexicons", {})
        key = (path, str(logits.device))
        if key not in cache:
            from .lib.lstm.lexicon import load_lexicon
            cache[key] = engine.Lexicon(load_lexicon(path), device=logits.device)
        o, ol = Session._decode_device(logits, d_tsl)
        return engine.lexicon_decode(logits, d_tsl, engine.dense_decoded(o, ol), ol, cache[key],
                                     max_edit=int(cfg.TEST.get("LEXICON_MAX_EDIT", 3)),
                                     max_candidates=int(cfg.TEST.get("LEXICON_CANDIDATES", 64)))

    @staticmethod
    def _beam_decoded(logits, d_tsl):
        """"beam_decoded": the cfg.TEST.TOP_PATHS best reads of the beam search (width cfg.BEAM_WIDTH, on the device, whatever
        cfg.DECODER says), engine.ctc_beam_search_topk_device: {"labels" [N,K,L] (L the longest read, zero padded), "len" [N,K],
        "log_prob" [N,K], "num_paths" [N]}."""
        from .lib.lstm.config import cfg
        o, ol, lp, npaths = engine.ctc_beam_search_topk_device(logits, d_tsl, beam_width=int(cfg.get("BEAM_WIDTH", 100)),
                                                               top_paths=int(cfg.TEST.get("TOP_PATHS", 1)), merge_repeated=True)
        ol = ol.cpu().numpy()
        L = int(ol.max()) if ol.size else 0
        return {"labels": o[:, :, :L].cpu().numpy(), "len": ol, "log_prob": lp.cpu().numpy(), "num_paths": npaths.cpu().numpy()}

    @staticmethod
    def _label_alignment(logits, d_tsl, d_lab, d_ll, llen):
        """"label_alignment": the best alignment (blank 0) of the fed flat labels, laid out [N, max(labels_len)] as
        engine.alignment_dict (label 0, span -1 and peak 0 past each length)."""
        N = llen.size
        M = int(llen.max()) if N else 0
        r = [a.cpu().numpy() for a in engine.ctc_align(logits, d_lab, d_ll, d_tsl, blank=0, max_label_len=M)]
        rows = np.repeat(np.arange(N), llen)
        cols = np.arange(llen.sum()) - np.repeat(np.cumsum(llen) - llen, llen)
        out = []
        for flat, fill, dt in ((d_lab.cpu().numpy(), 0, np.int32), (r[0], -1, np.int32), (r[1], -1, np.int32), (r[2], 0, np.float32)):
            a = np.full((N, M), fill, dt)
            a[rows, cols] = flat
            out.append(a)
        return engine.alignment_dict(out[0], out[1], out[2], out[3], r[3])
