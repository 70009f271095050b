"""Device-side engine behind the reference-facing API.  PyTorch tensors are used purely as
device-memory containers and for the current CUDA stream; every kernel on this path lives in
libcrnnctc.so (hand-written sm_90a CUDA, see csrc/)."""
import ctypes
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from ._lib import CrnnConfig, CrnnError, check

NCLASSES = 64
TF_BLANK = NCLASSES - 1

# solver -> (checkpoint key prefix, slot buffer) pairs; the keys are TF-style slot names, the buffers those bound as adam_m / adam_v
SOLVER_SLOTS = {"Adam": (("adam_m", "adam_m"), ("adam_v", "adam_v")),
                "Momentum": (("momentum", "adam_m"),),
                "RMS": (("rms", "adam_v"), ("rms_momentum", "adam_m"))}
# tf.train.RMSPropOptimizer defaults: the reference constructs it with the learning rate alone (lib/lstm/train.py:75)
RMS_DECAY, RMS_MOMENTUM, RMS_EPSILON = 0.9, 0.0, 1e-10
# the five e4m3 GEMMs of compute_dtype "fp8": layer -> (K, Cout) of its [Cout][K] weight operand
# moving BatchNorm statistics of conv4_1 / conv4_2 under their TF names (buffer [layer][mean, variance][512]), tracked with
# tf.contrib.layers.batch_norm's default decay
BN_MOVING_KEYS = ("conv4_1/conv4_1/moving_mean", "conv4_1/conv4_1/moving_variance",
                  "conv4_2/conv4_2/moving_mean", "conv4_2/conv4_2/moving_variance")
BN_MOVING_DECAY = 0.999
FP8_WEIGHTS = OrderedDict([("conv3_1", (1152, 256)), ("conv3_2", (2304, 256)), ("conv4_1", (2304, 512)), ("conv4_2", (4608, 512)),
                           ("conv5", (2048, 512))])


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _feed_suffix(dtype):
    """Entry-point suffix of a batch's element type: f32 data -> "", uint8 pixels (x = u / 255, include/crnn_ctc.h) -> "_u8"."""
    if dtype in (torch.float32, np.float32):
        return ""
    if dtype in (torch.uint8, np.uint8):
        return "_u8"
    raise CrnnError(f"data must be float32 or uint8 pixels, got {dtype}")


class CrnnModel:
    """Owns the flat f32 parameter buffer (TF variable names/layouts) and the C model handle."""

    def __init__(self, weight_decay=1e-5, bn_eps=1e-3, device=None, compute_dtype="bf16"):
        if not torch.cuda.is_available():
            raise CrnnError("lstm_ctc_ocr_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        torch.cuda.set_device(self.device)
        # "bf16": bf16 operands / f32 accumulate (throughput path); "f32": split-bf16 operands, f32-class (BASELINE configs[1]);
        # "tf32": tf32 operands, same forward-only orchestration as "f32"; "fp8": e4m3 operands in conv3_1 .. conv5, inference
        # only, after calibrate_fp8 / set_fp8_scales
        self.compute_dtype = {"bf16": 1, "f32": 2, "tf32": 3, "fp8": 4, 1: 1, 2: 2, 3: 3, 4: 4}[compute_dtype]
        cfg = CrnnConfig(32, NCLASSES, 512, bn_eps, weight_decay, self.compute_dtype)
        h = _lib.c_void_p()
        check(self.lib.crnn_model_create(cfg, h))
        self.handle = h
        self.weight_decay = weight_decay
        self.total = int(self.lib.crnn_param_count(h))
        self.table = OrderedDict()
        for i in range(self.lib.crnn_num_tensors(h)):
            name = _lib.c_char_p(); off = _lib.c_int64(); shp = (_lib.c_int64 * 4)(); nd = _lib.c_int()
            check(self.lib.crnn_param_info(h, i, name, off, shp, nd))
            self.table[name.value.decode()] = (int(off.value), tuple(int(shp[k]) for k in range(nd.value)))
        self.params = torch.zeros(self.total, dtype=torch.float32, device=self.device)
        self.grads = None
        self.adam_m = None
        self.adam_v = None
        self.solver = "Adam"
        self.momentum = 0.9
        self._bind()
        # moving statistics (bf16 and fp8 models): always bound, so every training step tracks them; evaluation uses them after
        # set_bn_statistics("moving")
        self.bn_statistics = "batch"
        self.bn_moving = None
        if self.compute_dtype in (1, 4):
            self.bn_moving = torch.empty((2, 2, 512), dtype=torch.float32, device=self.device)
            self.bn_moving[:, 0].zero_()
            self.bn_moving[:, 1].fill_(1.0)
            check(self.lib.crnn_model_bind_bn_moving(h, self.bn_moving.data_ptr(), BN_MOVING_DECAY))
        self._ws = None
        self._ws_key = None
        self._ws_lines = False
        self.training = False
        self.fp8_calibrated = False     # fp8: activation scales valid for the loaded parameters (load_params invalidates them)

    # ---- training --------------------------------------------------------------------------
    def set_training(self, flag=True):
        """Allocate the gradient / solver-slot buffers (flat f32, same layout as params), initialised for the recorded solver,
        and switch the forward to the variant that saves what the backward pass needs."""
        if flag and self.grads is None:
            self.grads = torch.zeros_like(self.params)
            self.adam_m = torch.zeros_like(self.params)
            self.adam_v = torch.zeros_like(self.params)
            self.reset_slots()
            self._bind()
        check(self.lib.crnn_model_set_training(self.handle, 1 if flag else 0))
        self.training = bool(flag)
        self._ws_key = None

    def set_solver(self, name, momentum=0.9):
        """Record the optimizer apply_gradients runs and reset its slots as TensorFlow initialises them.  `name` is one of
        "Adam" (m = v = 0), "Momentum" (accum = 0 in the adam_m buffer) and "RMS" (mom = 0 in adam_m, ms = 1 in adam_v).
        `momentum` is MomentumOptimizer's coefficient; RMSProp runs with TF's defaults (decay 0.9, momentum 0, epsilon 1e-10)."""
        if name not in SOLVER_SLOTS:
            raise CrnnError(f"unknown solver {name!r}: expected one of {sorted(SOLVER_SLOTS)}")
        self.solver, self.momentum = name, float(momentum)
        self.reset_slots()

    def reset_slots(self):
        """Slots as TF's slot initialisers leave them: zeros, except RMSProp's mean square (adam_v), which starts at 1.0."""
        if self.adam_m is not None:
            self.adam_m.zero_()
            self.adam_v.fill_(1.0 if self.solver == "RMS" else 0.0)

    def apply_gradients(self, lr, step, clip=10.0, grad_mul=1.0, wd_mul=1.0):
        """Gradient finish (L2 term, global norm), clip by global norm and one update of the recorded solver.  `step` is the
        1-based global step (only Adam's bias correction reads it); grad_mul / wd_mul as in clip_adam_step."""
        if self.solver == "Adam":
            self.clip_adam_step(lr, step, clip=clip, grad_mul=grad_mul, wd_mul=wd_mul)
        elif self.solver == "Momentum":
            check(self.lib.crnn_clip_momentum_step(self.handle, float(lr), self.momentum, float(clip), float(grad_mul), float(wd_mul),
                                                   _stream()))
        else:
            check(self.lib.crnn_clip_rmsprop_step(self.handle, float(lr), RMS_DECAY, RMS_MOMENTUM, RMS_EPSILON, float(clip), float(grad_mul),
                                                  float(wd_mul), _stream()))

    def solver_slots(self):
        """{checkpoint key prefix: flat slot buffer} of the recorded solver."""
        return {prefix: getattr(self, buf) for prefix, buf in SOLVER_SLOTS[self.solver]}

    def grad_tensor(self, name):
        off, shp = self.table[name]
        return self.grads[off:off + int(np.prod(shp))].view(*shp)

    def backward(self, data, time_step_len, dlogits):
        """dlogits [T,N,64] f32 = d loss / d logits (e.g. the CTC gradient scaled by 1/N) -> fills self.grads.  `data` is the
        batch the training forward read: f32, or uint8 pixels (crnn_backward_u8)."""
        N, W, _ = data.shape
        ws, nbytes = self._workspace(N, W)
        fn = getattr(self.lib, "crnn_backward" + _feed_suffix(data.dtype))
        check(fn(self.handle, data.data_ptr(), time_step_len.data_ptr(), dlogits.data_ptr(), N, W, ws, nbytes,
                                     _stream()))

    def clip_adam_step(self, lr, step, clip=10.0, grad_mul=1.0, wd_mul=1.0):
        check(self.lib.crnn_clip_adam_step(self.handle, float(lr), float(clip), int(step), float(grad_mul), float(wd_mul), _stream()))

    def last_grad_norm(self, grad_mul=1.0):
        out = _lib.c_float()
        check(self.lib.crnn_last_grad_norm(self.handle, float(grad_mul), out, _stream()))
        return float(out.value)

    def _bind(self):
        check(self.lib.crnn_model_bind(self.handle, _ptr(self.params), _ptr(self.grads), _ptr(self.adam_m), _ptr(self.adam_v)))
        self.fp8_calibrated = False     # a bind invalidates the fp8 scales, as a parameter change does

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                torch.cuda.synchronize(self.device)
                self.lib.crnn_model_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # ---- parameters, addressable by TF variable name --------------------------------------
    def tensor(self, name):
        off, shp = self.table[name]
        n = int(np.prod(shp))
        return self.params[off:off + n].view(*shp)

    def load_params(self, params):
        for name in self.table:
            v = params[name]
            v = torch.as_tensor(np.asarray(v, dtype=np.float32)) if not torch.is_tensor(v) else v.detach().float().cpu()
            self.tensor(name).copy_(v.to(self.device))
        check(self.lib.crnn_model_params_changed(self.handle))
        self.fp8_calibrated = False

    def state_dict(self):
        return OrderedDict((k, self.tensor(k).detach().cpu().numpy().copy()) for k in self.table)

    # ---- moving BatchNorm statistics ----------------------------------------------------------
    def _moving_buffer(self):
        if self.bn_moving is None:
            raise CrnnError("moving BatchNorm statistics exist on the bf16 and fp8 models only")
        return self.bn_moving

    def bn_moving_state(self):
        """{TF name (BN_MOVING_KEYS): float32 [512]} of the moving statistics; synchronises the device."""
        b = self._moving_buffer().detach().cpu().numpy()
        return OrderedDict((k, b[i // 2, i % 2].copy()) for i, k in enumerate(BN_MOVING_KEYS))

    def load_bn_moving(self, state=None):
        """Set the moving statistics from {TF name: [512]} (all four BN_MOVING_KEYS), or, with None, to TF's initial values
        (mean 0, variance 1).  Invalidates fp8 scales, as a parameter change does."""
        b = self._moving_buffer()
        if state is None:
            b[:, 0].zero_()
            b[:, 1].fill_(1.0)
        else:
            missing = [k for k in BN_MOVING_KEYS if k not in state]
            if missing:
                raise KeyError(f"moving statistics missing: {missing}")
            for i, k in enumerate(BN_MOVING_KEYS):
                b[i // 2, i % 2].copy_(torch.as_tensor(np.asarray(state[k], dtype=np.float32).reshape(512)).to(self.device))
        check(self.lib.crnn_model_params_changed(self.handle))
        self.fp8_calibrated = False

    def set_bn_statistics(self, mode):
        """"batch" (default, the reference): conv4_1 / conv4_2 normalise with the statistics of the evaluated batch (each line's
        own in forward_lines).  "moving": evaluation forwards normalise with the moving statistics training tracked, folded into
        the conv weights and bias; training forwards always use batch statistics.  A change invalidates fp8 scales."""
        if mode not in ("batch", "moving"):
            raise CrnnError(f"BN statistics must be 'batch' or 'moving', got {mode!r}")
        check(self.lib.crnn_model_set_bn_statistics(self.handle, 1 if mode == "moving" else 0))
        if mode != self.bn_statistics:
            self.fp8_calibrated = False
            self._ws_key = None            # a packed-evaluation workspace has a mode-dependent size
        self.bn_statistics = mode

    # ---- forward ----------------------------------------------------------------------------
    def _workspace(self, N, W, lines=False):
        # a packed-evaluation workspace holds the inference plan too, so it serves both forwards (and the taps after either)
        key = (N, W, self.training, self.bn_statistics)
        if self._ws_key != key or (lines and not self._ws_lines):
            nbytes = _lib.c_size_t()
            if lines:
                check(self.lib.crnn_lines_workspace_size(self.handle, N, W, nbytes))
            else:
                check(self.lib.crnn_model_workspace_size(self.handle, N, W, 1 if self.training else 0, nbytes))
            self._ws = None
            self._ws = torch.empty(nbytes.value + 1024, dtype=torch.uint8, device=self.device)
            self._ws_key = key
            self._ws_lines = lines
        base = self._ws.data_ptr()
        aligned = (base + 1023) // 1024 * 1024
        return aligned, self._ws.numel() - (aligned - base)

    def forward(self, data, time_step_len, out=None):
        """data [N,W,32] f32 cuda, or uint8 pixels (crnn_forward_u8: x = u / 255), time_step_len [N] i32 cuda -> logits [T,N,64]
        f32 (time-major)."""
        fn = getattr(self.lib, "crnn_forward" + _feed_suffix(data.dtype))
        assert data.is_cuda and data.is_contiguous()
        assert time_step_len.is_cuda and time_step_len.dtype == torch.int32
        N, W, Hh = data.shape
        if Hh != 32:
            raise CrnnError("data must be [N, W, 32] (cfg.NUM_FEATURES = 32)")
        T = W // 4 - 1
        if out is None:
            out = torch.empty((T, N, NCLASSES), dtype=torch.float32, device=self.device)
        ws, nbytes = self._workspace(N, W)
        check(fn(self.handle, data.data_ptr(), time_step_len.data_ptr(), N, W, out.data_ptr(), ws,
                                    nbytes, _stream()))
        return out

    # ---- fp8 scales (compute_dtype "fp8") -----------------------------------------------------
    def calibrate_fp8(self, data, time_step_len):
        """Set the five activation scales of an fp8 model from a calibration batch (data [N,W,32] f32 cuda, time_step_len [N]
        i32 cuda; or uint8 pixels): the bf16 front end runs on it and each scale becomes 2^ceil(log2(amax / 448)).  Asynchronous,
        on the device."""
        fn = getattr(self.lib, "crnn_model_calibrate_fp8" + _feed_suffix(data.dtype))
        assert data.is_cuda and data.is_contiguous()
        assert time_step_len.is_cuda and time_step_len.dtype == torch.int32
        N, W, Hh = data.shape
        if Hh != 32:
            raise CrnnError("data must be [N, W, 32] (cfg.NUM_FEATURES = 32)")
        ws, nbytes = self._workspace(N, W)
        check(fn(self.handle, data.data_ptr(), time_step_len.data_ptr(), N, W, ws, nbytes, _stream()))
        self.fp8_calibrated = True

    def fp8_scales(self):
        """The five activation scales (a2, a3, a3p, a4a, a4b) as a float32 numpy array; synchronises the device."""
        out = np.zeros(5, dtype=np.float32)
        check(self.lib.crnn_model_get_fp8_scales(self.handle, out.ctypes.data))
        return out

    def set_fp8_scales(self, scales):
        """Set the five activation scales (powers of two, else CrnnError with CRNN_INVALID_VALUE)."""
        s = np.ascontiguousarray(np.asarray(scales, dtype=np.float32).reshape(5))
        check(self.lib.crnn_model_set_fp8_scales(self.handle, s.ctypes.data))
        self.fp8_calibrated = True

    def forward_lines(self, data, line_width, time_step_len, out=None):
        """Packed evaluation: data [N,W,32] f32 cuda holding line i in columns [0, W_i), line_width [N] i32 cuda (W_i, a multiple
        of 4 in [8, W]), time_step_len [N] i32 cuda (<= W_i/4 - 1) -> logits [W/4-1,N,64] f32, each line's frames t < W_i/4 - 1
        as forward() computes them for that line fed alone as [1, W_i, 32] (per-line BatchNorm statistics and width boundaries).
        Evaluation only: a model in training mode is refused.  uint8 pixels (crnn_forward_lines_u8) are accepted as data."""
        fn = getattr(self.lib, "crnn_forward_lines" + _feed_suffix(data.dtype))
        assert data.is_cuda and data.is_contiguous()
        assert line_width.is_cuda and line_width.dtype == torch.int32 and time_step_len.is_cuda and time_step_len.dtype == torch.int32
        N, W, Hh = data.shape
        if Hh != 32:
            raise CrnnError("data must be [N, W, 32] (cfg.NUM_FEATURES = 32)")
        if self.training:
            raise CrnnError("forward_lines is evaluation only: the model is in training mode (training uses whole-batch statistics)")
        T = W // 4 - 1
        if out is None:
            out = torch.empty((T, N, NCLASSES), dtype=torch.float32, device=self.device)
        ws, nbytes = self._workspace(N, W, lines=True)
        check(fn(self.handle, data.data_ptr(), line_width.data_ptr(), time_step_len.data_ptr(), N, W,
                                          out.data_ptr(), ws, nbytes, _stream()))
        return out

    def forward_host(self, host_data, time_step_len, chunks=4, out=None, wait_copy=True):
        """host_data: C-contiguous f32 (or uint8 pixel) numpy array [N,W,32] in PAGE-LOCKED memory.  The H2D copy is cut into
        `chunks` image ranges on a side stream and overlapped with the conv front end (crnn_forward_host / _u8).  Returns
        (logits, device data): the device staging of the batch's dtype."""
        N, W, Hh = host_data.shape
        if Hh != 32:
            raise CrnnError("data must be [N, W, 32] (cfg.NUM_FEATURES = 32)")
        fn = getattr(self.lib, "crnn_forward_host" + _feed_suffix(host_data.dtype))
        assert host_data.flags.c_contiguous
        T = W // 4 - 1
        if out is None:
            out = torch.empty((T, N, NCLASSES), dtype=torch.float32, device=self.device)
        stage = self._staging(N, W, host_data.dtype)
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        ws, nbytes = self._workspace(N, W)
        check(fn(self.handle, host_data.ctypes.data, stage.data_ptr(), time_step_len.data_ptr(), N, W,
                                         out.data_ptr(), ws, nbytes, int(chunks), _stream(), self._copy_stream.cuda_stream))
        if wait_copy:
            # the caller may rewrite `host_data` as soon as this returns (a feeder recycling its ring slot): wait for the DMA --
            # not for the compute, which keeps running on the main stream
            self._copy_stream.synchronize()
        return out, stage

    def _staging(self, N, W, dtype):
        """Device staging [N,W,32] of the host feeds, one per element type (f32, uint8)."""
        dt = torch.uint8 if _feed_suffix(dtype) else torch.float32
        if getattr(self, "_stage", None) is None:
            self._stage = {}
        st = self._stage.get(dt)
        if st is None or st.shape != (N, W, 32):
            st = self._stage[dt] = torch.empty((N, W, 32), dtype=dt, device=self.device)
        return st

    def forward_pageable(self, host_data, pinned, time_step_len, chunks=4, host_threads=8, out=None):
        """host_data: C-contiguous f32 (or uint8 pixel) numpy array [N,W,32] in ORDINARY memory (the reference's np.array(...) per
        step); `pinned`: a page-locked torch tensor with at least N*W*32 elements of the same element size.  Range by range the
        library's host threads move the batch into `pinned`, DMA it and run the conv front end (crnn_forward_pageable / _u8).
        Returns (logits, device data, copy stream)."""
        N, W, Hh = host_data.shape
        if Hh != 32:
            raise CrnnError("data must be [N, W, 32] (cfg.NUM_FEATURES = 32)")
        fn = getattr(self.lib, "crnn_forward_pageable" + _feed_suffix(host_data.dtype))
        assert (host_data.flags.c_contiguous and pinned.is_pinned() and pinned.element_size() == host_data.itemsize
                and pinned.numel() >= host_data.size)
        T = W // 4 - 1
        if out is None:
            out = torch.empty((T, N, NCLASSES), dtype=torch.float32, device=self.device)
        stage = self._staging(N, W, host_data.dtype)
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        ws, nbytes = self._workspace(N, W)
        check(fn(self.handle, host_data.ctypes.data, pinned.data_ptr(), stage.data_ptr(),
                                             time_step_len.data_ptr(), N, W, out.data_ptr(), ws, nbytes, int(chunks), int(host_threads),
                                             _stream(), self._copy_stream.cuda_stream))
        return out, stage, self._copy_stream

    def tap(self, name, N, W):
        """Intermediate of the last forward (or, for the backward buffers, the last backward) as f32 NHWC (tests only)."""
        H1, H2 = W // 2, W // 4
        Npad, T = (N + 127) // 128 * 128, H2 - 1
        shapes = {"conv1": (N, H1, 16, 64), "conv2": (N, H2, 8, 128), "conv3_1": (N, H2, 8, 256),
                  "conv3_2": (N, H2, 4, 256), "conv4_1": (N, H2, 4, 512), "conv4_2": (N, H2, 2, 512),
                  "conv5": (N, H2, 512), "lstm_out": (N, H2, 512), "xproj": (N, H2, 2048),
                  "a4a_pre": (N, H2, 4, 512), "a4b_pre": (N, H2, 4, 512),
                  # training only; gates: [dir * Npad/128 + tile][step][gate i,j,f,o][unit / 8][row][unit % 8]
                  "gates": (2 * Npad // 128, T, 4, 32, 128, 8), "dl_rows": (N, H2, 64), "d_lstm_out": (N, H2, 512),
                  "dz_all": (N, H2, 2048), "d_a5": (N, H2, 512), "d_a4b": (N, H2, 2, 512), "d_pre4b": (N, H2, 4, 512),
                  "d_pre4a": (N, H2, 4, 512), "d_a3p": (N, H2, 4, 256), "d_pre32": (N, H2, 8, 256),
                  "d_pre31": (N, H2, 8, 256), "d_a2": (N, H2, 8, 128), "d_pre2": (N, H1, 16, 128), "d_a1": (N, H1, 16, 64)}
        shp = shapes[name]
        dst = torch.empty(shp, dtype=torch.float32, device=self.device)
        ws, _ = self._workspace(N, W)
        check(self.lib.crnn_debug_tap(self.handle, name.encode(), dst.data_ptr(), dst.numel(), ws, _stream()))
        return dst

    def tap_raw(self, name, N, W, lines=False):
        """Non-bf16 workspace buffer of the last forward, byte for byte (tests only): "bn" f32 [2][4][512] (scale, shift,
        mean, invstd per BN layer), "stats" f64 [2][2][512]; bf16 path, training only: "am1" / "am2" / "am3" u8 pool window
        index (dy*2+dx) in the pooled NHWC shape, "csave" f32 [dir * Npad/128 + tile][step][unit / 4][row][unit % 4].
        f32-class paths: "cst" f32 [2][Npad][256] (final cell state) and the stored activations "conv1" .. "conv5",
        "lstm_out": "f32" (split) bf16 [..., 2 (hi, lo), C] per position, conv4_2 [N, H2, 2 (hi, lo), 2 positions, 512]
        (rows of G = 2 positions); "tf32" f32 in the tap shape.  lines=True (after forward_lines): per-line "bn" f32 [2][N][4][512]
        and "stats" f64 [2][N][2][512].  "fp8": the e4m3 operands "conv2" .. "conv4_2" as u8 bytes in the tap shape, "fp8_scales"
        f32 [5], "fp8_wscale" / "fp8_colscale" f32 [5][512], "fp8_w_<layer>" u8 [Cout][K] (FP8_WEIGHTS)."""
        H1, H2 = W // 2, W // 4
        Npad, T = (N + 127) // 128 * 128, H2 - 1
        shapes = {"bn": ((2, 4, 512), torch.float32), "stats": ((2, 2, 512), torch.float64)}
        if lines:
            shapes = {"bn": ((2, N, 4, 512), torch.float32), "stats": ((2, N, 2, 512), torch.float64)}
        # folded operands of the moving statistics (bf16 and fp8 models): W' [Cout][K] bf16, b' [2][512] f32
        shapes.update({"moving_w_conv4_1": ((512, 2304), torch.bfloat16), "moving_w_conv4_2": ((512, 4608), torch.bfloat16),
                       "moving_bias": ((2, 512), torch.float32), "fp8_colscale_moving": ((2, 512), torch.float32)})
        if self.compute_dtype == 1:
            shapes.update({"am1": ((N, H1, 16, 64), torch.uint8), "am2": ((N, H2, 8, 128), torch.uint8),
                           "am3": ((N, H2, 4, 256), torch.uint8), "csave": ((2 * Npad // 128, T, 64, 128, 4), torch.float32)})
        elif self.compute_dtype == 4:
            # fp8: the e4m3 operands as stored, the activation scales, per-layer weight scales and colscale ([5][512]), e4m3 weights
            shapes.update({"conv2": ((N, H2, 8, 128), torch.uint8), "conv3_1": ((N, H2, 8, 256), torch.uint8),
                           "conv3_2": ((N, H2, 4, 256), torch.uint8), "conv4_1": ((N, H2, 4, 512), torch.uint8),
                           "conv4_2": ((N, H2, 2, 512), torch.uint8), "fp8_scales": ((5,), torch.float32),
                           "fp8_wscale": ((5, 512), torch.float32), "fp8_colscale": ((5, 512), torch.float32)})
            for k, (K, co) in FP8_WEIGHTS.items():
                shapes["fp8_w_" + k] = ((co, K), torch.uint8)
        else:
            acts = {"conv1": (N, H1, 16), "conv2": (N, H2, 8), "conv3_1": (N, H2, 8), "conv3_2": (N, H2, 4),
                    "conv4_1": (N, H2, 4), "conv4_2": (N, H2), "conv5": (N, H2), "lstm_out": (N, H2)}
            chans = {"conv1": 64, "conv2": 128, "conv3_1": 256, "conv3_2": 256}
            shapes["cst"] = ((2, Npad, 256), torch.float32)
            for k, lead in acts.items():
                C = chans.get(k, 512)
                if self.compute_dtype == 3:
                    shapes[k] = (lead + ((2,) if k == "conv4_2" else ()) + (C,), torch.float32)
                else:
                    shapes[k] = (lead + (2,) + ((2,) if k == "conv4_2" else ()) + (C,), torch.bfloat16)
        # a name this path does not have goes to the library as well, which refuses it with CRNN_INVALID_VALUE
        shp, dt = shapes.get(name, ((1,), torch.uint8))
        dst = torch.empty(shp, dtype=dt, device=self.device)
        ws, _ = self._workspace(N, W)
        check(self.lib.crnn_debug_tap_raw(self.handle, name.encode(), dst.data_ptr(), dst.numel() * dst.element_size(), ws,
                                          _stream()))
        return dst

    # ---- loss / decode ------------------------------------------------------------------------
    def total_loss(self, costs):
        loss = torch.empty(1, dtype=torch.float32, device=self.device)
        check(self.lib.crnn_total_loss(self.handle, costs.data_ptr(), costs.numel(), loss.data_ptr(), _stream()))
        return loss


CTC_MAX_LABEL_LEN = 639       # the workspace kernel's limit (S = 2L+1 <= 1279 states), warp-ctc's on the GPU
_ctc_ws = {}                  # device -> workspace tensor of the largest size asked for so far, reused call to call


def ctc_workspace_bytes(T, N, C, max_label_len):
    """Bytes of device workspace crnn_ctc_loss needs for this shape: 0 where a shared-memory kernel serves it at any alignment
    (max_label_len <= 63 and T within 517 / 259 / 130), else the workspace kernel's size.  CrnnError (CRNN_UNSUPPORTED) above
    max_label_len 639 or when the size overflows.  No CUDA call."""
    nbytes = _lib.c_size_t()
    check(_lib.load().crnn_ctc_workspace_size(int(T), int(N), int(C), int(max_label_len), nbytes))
    return int(nbytes.value)


def _auto_ctc_workspace(T, N, C, max_label_len, device):
    nbytes = ctc_workspace_bytes(T, N, C, max_label_len)
    if nbytes == 0:
        return None
    ws = _ctc_ws.get(device)
    if ws is None or ws.numel() < nbytes:
        _ctc_ws.pop(device, None)
        ws = _ctc_ws[device] = torch.empty(nbytes, dtype=torch.uint8, device=device)
    return ws


def ctc_loss(logits, flat_labels, label_len, input_len, blank=0, want_grad=False, grad_scale=1.0, max_label_len=None,
             costs=None, grad=None, validate=False, workspace=None):
    """logits [T,N,64] f32 cuda; integer tensors i32 cuda.  Returns (costs [N], grad [T,N,64] | None).
    workspace: None passes none (shapes beyond the shared-memory kernels fail with CRNN_UNSUPPORTED); "auto" sizes it with
    ctc_workspace_bytes and reuses a per-device buffer; a uint8 cuda tensor is passed as given.  Shapes a shared-memory kernel
    serves give the same bits with or without a workspace."""
    lib = _lib.load()
    assert logits.is_cuda and logits.dtype == torch.float32 and logits.is_contiguous()
    T, N, C = logits.shape
    if label_len.numel() != N or input_len.numel() != N:
        raise CrnnError("ctc_loss: label_len and input_len must hold one entry per utterance")
    if validate:         # host-synchronising checks (the kernel itself rejects bad ids per sample: cost NaN, zero gradient)
        ll = label_len.cpu()
        if int(ll.min()) < 0 or int(ll.sum()) != flat_labels.numel():
            raise CrnnError("ctc_loss: label_len must be non-negative and sum to len(flat_labels)")
        if flat_labels.numel() and (int(flat_labels.min()) < 0 or int(flat_labels.max()) >= C or bool((flat_labels == blank).any())):
            raise CrnnError(f"ctc_loss: label ids must lie in [0, {C}) and differ from the blank ({blank})")
    if max_label_len is None:
        max_label_len = int(label_len.max().item()) if label_len.numel() else 0      # host sync; pass it to avoid
    if costs is None:
        costs = torch.empty(N, dtype=torch.float32, device=logits.device)
    if want_grad and grad is None:
        grad = torch.empty_like(logits)
    if isinstance(workspace, str):
        if workspace != "auto":
            raise CrnnError(f"ctc_loss: workspace must be None, 'auto' or a cuda tensor, got {workspace!r}")
        workspace = _auto_ctc_workspace(T, N, C, max_label_len, logits.device)
    ws_ptr, ws_bytes = 0, 0
    if workspace is not None:
        if not (torch.is_tensor(workspace) and workspace.is_cuda and workspace.is_contiguous()):
            raise CrnnError("ctc_loss: workspace must be a contiguous cuda tensor")
        ws_ptr, ws_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
    check(lib.crnn_ctc_loss(logits.data_ptr(), _ptr(grad) if want_grad else 0, flat_labels.data_ptr(),
                            label_len.data_ptr(), input_len.data_ptr(), T, N, C, blank, int(max_label_len),
                            float(grad_scale), costs.data_ptr(), ws_ptr, ws_bytes, _stream()))
    return costs, (grad if want_grad else None)


_align_ws = {}                # device -> workspace tensor of crnn_ctc_align, the largest size asked for so far


def ctc_align_workspace_bytes(T, N, C, max_label_len):
    """Bytes of device workspace crnn_ctc_align needs for this shape.  CrnnError (CRNN_UNSUPPORTED) for C != 64 or max_label_len
    above 639.  No CUDA call."""
    nbytes = _lib.c_size_t()
    check(_lib.load().crnn_ctc_align_workspace_size(int(T), int(N), int(C), int(max_label_len), nbytes))
    return int(nbytes.value)


def ctc_align(logits, labels, label_len, input_len, blank=0, max_label_len=None, workspace="auto"):
    """CTC forced alignment (crnn_ctc_align): the best path of each utterance's GIVEN labelling.  logits [T,N,64] f32 cuda;
    labels i32 cuda, 2-D [N, M] dense rows (the decoders' layout: row n holds label_len[n] ids) or 1-D flat (crnn_ctc_loss's
    layout); label_len, input_len [N] i32 cuda.  Returns device (start, end, peak, path_logprob): start / end i32 and peak f32
    shaped like `labels` -- label k occupies frames [start, end) of the best path (input columns [4*start, 4*end + 4)), peak is
    its largest posterior over them; dense entries past label_len[n] are -1 / -1 / 0 -- and path_logprob [N] f32 (natural log).
    Infeasible labellings give -inf and spans -1, invalid ones (ids outside [0,64) or equal to the blank, label_len negative or
    above max_label_len) NaN and spans -1.  max_label_len: None takes the row width for dense labels and label_len.max() for
    flat ones (one host sync).  workspace: "auto" reuses a per-device buffer; a contiguous uint8 cuda tensor is passed as given.
    No host fallback: CPU tensors raise CrnnError."""
    tensors = (logits, labels, label_len, input_len)
    if not all(torch.is_tensor(t) and t.is_cuda for t in tensors):
        raise CrnnError("ctc_align needs CUDA tensors (sm_90a); there is no CPU fallback")
    if logits.dtype != torch.float32 or logits.dim() != 3 or any(t.dtype != torch.int32 for t in tensors[1:]):
        raise CrnnError("ctc_align: logits must be [T,N,64] f32 and labels, label_len, input_len i32")
    if labels.dim() not in (1, 2):
        raise CrnnError("ctc_align: labels must be 1-D (flat) or 2-D (dense rows)")
    lib = _lib.load()
    logits, labels = logits.contiguous(), labels.contiguous()
    label_len, input_len = label_len.contiguous(), input_len.contiguous()
    T, N, C = logits.shape
    if label_len.numel() != N or input_len.numel() != N or (labels.dim() == 2 and labels.shape[0] != N):
        raise CrnnError("ctc_align: labels (dense), label_len and input_len must hold one entry / row per utterance")
    dense = labels.dim() == 2
    if max_label_len is None:
        max_label_len = labels.shape[1] if dense else (int(label_len.max().item()) if N else 0)
    dev = logits.device
    start = torch.empty(labels.shape, dtype=torch.int32, device=dev)
    end = torch.empty(labels.shape, dtype=torch.int32, device=dev)
    peak = torch.empty(labels.shape, dtype=torch.float32, device=dev)
    lp = torch.empty(N, dtype=torch.float32, device=dev)
    # a labelling with no ids at all (every L = 0) still passes non-null pointers; dense rows of width 0 are the flat layout
    stride = labels.shape[1] if dense else 0
    if labels.numel() == 0:
        labels = torch.zeros(1, dtype=torch.int32, device=dev)
        bufs = [torch.empty(1, dtype=t.dtype, device=dev) for t in (start, end, peak)]
    else:
        bufs = [start, end, peak]
    nbytes = ctc_align_workspace_bytes(T, N, C, max_label_len)
    if isinstance(workspace, str):
        if workspace != "auto":
            raise CrnnError(f"ctc_align: workspace must be 'auto' or a cuda tensor, got {workspace!r}")
        workspace = _align_ws.get(dev)
        if workspace is None or workspace.numel() < nbytes:
            _align_ws.pop(dev, None)
            workspace = _align_ws[dev] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    if not (torch.is_tensor(workspace) and workspace.is_cuda and workspace.is_contiguous()):
        raise CrnnError("ctc_align: workspace must be a contiguous cuda tensor")
    check(lib.crnn_ctc_align(logits.data_ptr(), labels.data_ptr(), stride, label_len.data_ptr(), input_len.data_ptr(), T, N, C,
                             int(blank), int(max_label_len), bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), lp.data_ptr(),
                             workspace.data_ptr(), workspace.numel() * workspace.element_size(), _stream()))
    return start, end, peak, lp


def alignment_dict(labels, start, end, peak, path_logprob):
    """Host arrays of one alignment, dense [N, M] (entries past each length: label 0, span -1, peak 0), as Session.run returns
    them for "read_alignment" / "label_alignment": labels, start, end, x0 / x1 (the input columns [4*start, 4*end + 4) the span
    covers: frame t is conv5 output t, which reads pooled columns t and t+1), peak and path_logprob [N]."""
    start, end = np.asarray(start, np.int32), np.asarray(end, np.int32)
    return dict(labels=np.asarray(labels, np.int32), start=start, end=end,
                x0=np.where(start >= 0, 4 * start, -1).astype(np.int32), x1=np.where(end >= 0, 4 * end + 4, -1).astype(np.int32),
                peak=np.asarray(peak, np.float32), path_logprob=np.asarray(path_logprob, np.float32))


LEXICON_MAX_ENTRY = 63


class Lexicon(object):
    """A device-resident word list for lexicon-based reading (crnn_lexicon_candidates / crnn_ctc_lexicon_score): CSR `ids` i32
    (the entries' class ids concatenated) and `off` [K+1] i32 on `device`.  `entries` are id sequences over the charset's ids
    [1, nclasses-2] (0 is the CTC blank, nclasses-1 the decoders' blank), 1 .. 63 ids each; anything else raises ValueError.
    Exact duplicates are kept at their first occurrence only (`index_of` maps each kept entry back to its position in
    `entries`), so a tie between two slots is a tie between different words."""

    def __init__(self, entries, device="cuda", nclasses=64):
        kept, seen, index_of = [], set(), []
        for i, e in enumerate(entries):
            e = tuple(int(v) for v in e)
            if not e or len(e) > LEXICON_MAX_ENTRY:
                raise ValueError(f"Lexicon: entry {i} has {len(e)} ids; entries hold 1 .. {LEXICON_MAX_ENTRY}")
            bad = [v for v in e if not 1 <= v <= nclasses - 2]
            if bad:
                raise ValueError(f"Lexicon: entry {i} holds id {bad[0]} outside the charset's ids [1, {nclasses - 2}]")
            if e not in seen:
                seen.add(e)
                kept.append(e)
                index_of.append(i)
        if not kept:
            raise ValueError("Lexicon: no entries")
        self.entries = kept
        self.index_of = np.asarray(index_of, np.int64)
        lens = np.array([len(e) for e in kept], np.int32)
        off = np.zeros(len(kept) + 1, np.int32)
        np.cumsum(lens, out=off[1:])
        self.max_entry_len = int(lens.max())
        self.ids = torch.tensor(np.fromiter((v for e in kept for v in e), np.int32, int(off[-1])), device=device)
        self.off = torch.tensor(off, device=device)
        self.lens = lens

    def __len__(self):
        return len(self.entries)

    def padded(self, width=None):
        """[K, width] i32 host array of the entries, zero-padded (width: the longest entry by default)."""
        width = self.max_entry_len if width is None else int(width)
        out = np.zeros((len(self.entries), width), np.int32)
        for k, e in enumerate(self.entries):
            out[k, :len(e)] = e
        return out


def _cuda_i32(name, *tensors):
    if not all(torch.is_tensor(t) and t.is_cuda for t in tensors):
        raise CrnnError(f"{name} needs CUDA tensors (sm_90a); there is no CPU fallback")
    if any(t.dtype != torch.int32 for t in tensors):
        raise CrnnError(f"{name}: index tensors must be i32")


def lexicon_candidates(reads, read_len, lexicon, max_edit=3, max_candidates=64):
    """The lexicon entries nearest each read by edit distance (crnn_lexicon_candidates): reads [N, M] i32 cuda in the decoders'
    dense layout (dense_decoded), read_len [N] i32 cuda.  Returns device (cand, cand_dist) [N, max_candidates] i32 ordered by
    (distance, lexicon index), -1 past the count, and cand_total [N] i32 (the entries within max_edit; max_edit < 0: no
    threshold)."""
    _cuda_i32("lexicon_candidates", reads, read_len)
    if reads.dim() != 2 or read_len.numel() != reads.shape[0]:
        raise CrnnError("lexicon_candidates: reads must be [N, M] and read_len [N]")
    reads, read_len = reads.contiguous(), read_len.contiguous()
    N, M = reads.shape
    dev = reads.device
    cand = torch.empty((N, max_candidates), dtype=torch.int32, device=dev)
    dist = torch.empty((N, max_candidates), dtype=torch.int32, device=dev)
    total = torch.empty(N, dtype=torch.int32, device=dev)
    if N == 0:
        return cand, dist, total
    src = reads if reads.numel() else torch.zeros(1, dtype=torch.int32, device=dev)   # rows of width 0 still pass a pointer
    check(_lib.load().crnn_lexicon_candidates(src.data_ptr(), M, read_len.data_ptr(), N, lexicon.ids.data_ptr(), lexicon.off.data_ptr(),
                                              len(lexicon), lexicon.max_entry_len, int(max_edit), int(max_candidates), cand.data_ptr(),
                                              dist.data_ptr(), total.data_ptr(), _stream()))
    return cand, dist, total


def ctc_lexicon_score(logits, input_len, lexicon, cand, blank=0):
    """CTC scores of the candidates (crnn_ctc_lexicon_score): logits [T,N,64] f32 cuda, input_len [N] i32, cand [N, J] i32 as
    lexicon_candidates returns it.  Returns device score [N, J] f32 (ln p(entry | line); -inf for empty slots and infeasible
    entries, NaN for invalid ones), best [N] i32 (lexicon index of the highest finite score, lowest slot on ties, -1 if none) and
    best_score [N] f32."""
    _cuda_i32("ctc_lexicon_score", input_len, cand)
    if not (torch.is_tensor(logits) and logits.is_cuda and logits.dtype == torch.float32 and logits.dim() == 3):
        raise CrnnError("ctc_lexicon_score: logits must be a [T,N,64] f32 cuda tensor")
    logits, input_len, cand = logits.contiguous(), input_len.contiguous(), cand.contiguous()
    T, N, C = logits.shape
    if input_len.numel() != N or cand.dim() != 2 or cand.shape[0] != N:
        raise CrnnError("ctc_lexicon_score: input_len [N] and cand [N, J] must hold one entry / row per line")
    dev = logits.device
    J = cand.shape[1]
    score = torch.empty((N, J), dtype=torch.float32, device=dev)
    best = torch.empty(N, dtype=torch.int32, device=dev)
    best_score = torch.empty(N, dtype=torch.float32, device=dev)
    check(_lib.load().crnn_ctc_lexicon_score(logits.data_ptr(), input_len.data_ptr(), T, N, C, int(blank), lexicon.ids.data_ptr(),
                                             lexicon.off.data_ptr(), lexicon.max_entry_len, cand.data_ptr(), J, score.data_ptr(),
                                             best.data_ptr(), best_score.data_ptr(), _stream()))
    return score, best, best_score


def lexicon_decode(logits, input_len, reads, read_len, lexicon, max_edit=3, max_candidates=64):
    """Lexicon-based reading of a batch: the candidates of each read within max_edit, scored by CTC (blank 0, the blank warp-ctc
    trains), and the most probable one.  logits [T,N,64] f32, input_len [N], reads [N, M] and read_len [N] i32, all cuda.
    Returns host arrays: labels [N, max(M, longest entry)] i32 (the chosen entry's ids zero-padded; the read itself when no
    candidate has a finite score), index [N] (lexicon index, -1 when none), score [N] f32 (ln p of the chosen entry, -inf when
    none), distance [N] (edit distance of the chosen entry, -1 when none), candidates [N] (entries within max_edit)."""
    cand, dist, total = lexicon_candidates(reads, read_len, lexicon, max_edit, max_candidates)
    _, best, best_score = ctc_lexicon_score(logits, input_len, lexicon, cand, blank=0)
    cand, dist, total, best, best_score = (a.cpu().numpy() for a in (cand, dist, total, best, best_score))
    rd, rl = reads.cpu().numpy(), read_len.cpu().numpy()
    N = rd.shape[0]
    labels = np.zeros((N, max(rd.shape[1], lexicon.max_entry_len)), np.int32)
    distance = np.full(N, -1, np.int32)
    for n in range(N):
        k = int(best[n])
        if k >= 0:
            e = lexicon.entries[k]
            labels[n, :len(e)] = e
            distance[n] = dist[n][np.flatnonzero(cand[n] == k)[0]]
        else:
            L = min(max(int(rl[n]), 0), rd.shape[1])
            labels[n, :L] = rd[n, :L]
    return dict(labels=labels, index=best.astype(np.int32), score=best_score.astype(np.float32), distance=distance,
                candidates=total.astype(np.int32))


RESIZE_MAX_HEIGHT = 1024      # the tallest source line crnn_resize_lines_u8 takes


def resize_lines_u8(src, src_offset, src_h, src_w, out_w, W, max_h, out=None):
    """Native-size 8-bit gray lines -> the packed [N, W, 32] uint8 batch of forward_lines (crnn_resize_lines_u8): line i is
    src_h[i] x src_w[i] bytes, row-major, at src[src_offset[i]:], resized to 32 rows and out_w[i] columns with Pillow's 8-bit
    BILINEAR, byte for byte, and written width-major into slot i; columns out_w[i] .. W-1 are zero.  src uint8, src_offset [N]
    int64, src_h / src_w / out_w [N] int32, all cuda; max_h (host int) bounds every src_h[i], at most RESIZE_MAX_HEIGHT.  The
    per-line values are preconditions (include/crnn_ctc.h); out_w and W come from lib.lstm.test.line_size.  out: a contiguous
    [N, W, 32] uint8 cuda tensor, or None to allocate one.  No host fallback: CPU tensors raise CrnnError."""
    idx = (src_h, src_w, out_w)
    if not all(torch.is_tensor(t) and t.is_cuda for t in (src, src_offset) + idx):
        raise CrnnError("resize_lines_u8 needs CUDA tensors (sm_90a); there is no CPU fallback")
    if src.dtype != torch.uint8 or src_offset.dtype != torch.int64 or any(t.dtype != torch.int32 for t in idx):
        raise CrnnError("resize_lines_u8: src must be uint8, src_offset int64 and src_h, src_w, out_w int32")
    N = src_h.numel()
    if src_offset.numel() != N or src_w.numel() != N or out_w.numel() != N:
        raise CrnnError("resize_lines_u8: src_offset, src_h, src_w and out_w must hold one entry per line")
    src, src_offset, src_h, src_w, out_w = (t.contiguous() for t in (src, src_offset, src_h, src_w, out_w))
    if out is None:
        out = torch.empty((N, int(W), 32), dtype=torch.uint8, device=src.device)
    elif not (torch.is_tensor(out) and out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous()
              and tuple(out.shape) == (N, int(W), 32)):
        raise CrnnError(f"resize_lines_u8: out must be a contiguous [{N}, {int(W)}, 32] uint8 cuda tensor")
    check(_lib.load().crnn_resize_lines_u8(src.data_ptr(), src_offset.data_ptr(), src_h.data_ptr(), src_w.data_ptr(), out_w.data_ptr(),
                                           N, int(W), int(max_h), out.data_ptr(), _stream()))
    return out


PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
PNG_MAX_WIDTH = 1000000       # the widest PNG crnn_png_decode_gray_u8 reads (libpng's default limit)
PNG_STATUS = {0: "ok", 1: "bad header", 2: "bad chunk", 3: "bad CRC", 4: "bad zlib stream", 5: "bad DEFLATE data",
              6: "wrong amount of image data", 7: "bad filter type or palette index", 8: "a chunk the host reader acts on",
              9: "workspace too small"}


class ImageDecodeError(CrnnError):
    """Encoded files of an `images` feed the device decoders refused: ``entries`` their indices in the feed, ``status`` their codes
    (PNG_STATUS for a PNG entry, JPEG_STATUS for a JPEG one).  Raised as such when both kinds were refused in one feed."""

    def __init__(self, entries, status, message=None):
        self.entries, self.status = list(entries), list(status)
        super().__init__(message or "images: entries {} are files the device decoders refused (status {})".format(
            self.entries, self.status))


    @classmethod
    def mixed(cls, refused):
        """The error for refused files of both kinds: refused [(entry, code, kind)], kind "PNG" or "JPEG"; entries in feed order."""
        refused = sorted(refused)
        names = {"PNG": PNG_STATUS, "JPEG": JPEG_STATUS}
        entries = [e for e, _, _ in refused]
        return cls(entries, [c for _, c, _ in refused], "images: entries {} are files the device decoders refused ({})".format(
            entries, ", ".join("{} {}".format(k, names[k].get(c, str(c))) for _, c, k in refused)))


class PngDecodeError(ImageDecodeError):
    """Files of an `images` feed the device decoder refused, all of them PNG: ``entries`` their indices in the feed, ``status``
    their codes."""

    def __init__(self, entries, status):
        entries, status = list(entries), list(status)
        super().__init__(entries, status, "images: entries {} are PNG files the device decoder refused ({})".format(
            entries, ", ".join(PNG_STATUS.get(s, str(s)) for s in status)))


class JpegDecodeError(ImageDecodeError):
    """Files of an `images` feed the device decoder refused, all of them JPEG: ``entries`` their indices in the feed, ``status``
    their codes (JPEG_STATUS)."""

    def __init__(self, entries, status):
        entries, status = list(entries), list(status)
        super().__init__(entries, status, "images: entries {} are JPEG files the device decoder refused ({})".format(
            entries, ", ".join(JPEG_STATUS.get(s, str(s)) for s in status)))


def png_size(data):
    """(h, w) from a PNG file's signature and IHDR (bytes-like), or None when `data` does not start with them.  Only the fields
    are read: the rest of the header is the device decoder's to check."""
    b = bytes(data[:33])
    if len(b) < 33 or b[:8] != PNG_SIGNATURE or b[8:16] != b"\x00\x00\x00\x0dIHDR":
        return None
    return int.from_bytes(b[20:24], "big"), int.from_bytes(b[16:20], "big")


def png_plan(ihdr, file_len):
    """crnn_png_plan: ihdr [N, 13] uint8 (bytes 16 .. 28 of each file), file_len [N] int64 (host arrays) -> (ws_offset [N + 1]
    int64, workspace bytes).  File i's zlib stream and inflated scanlines lie in workspace[ws_offset[i]:ws_offset[i + 1]]."""
    ihdr = np.ascontiguousarray(ihdr, np.uint8)
    file_len = np.ascontiguousarray(file_len, np.int64)
    N = file_len.size
    if ihdr.shape != (N, 13):
        raise CrnnError(f"png_plan: ihdr must be [{N}, 13] uint8")
    off = np.zeros(N + 1, np.int64)
    nbytes = _lib.c_size_t()
    check(_lib.load().crnn_png_plan(ihdr.ctypes.data, file_len.ctypes.data, N, off.ctypes.data, ctypes.byref(nbytes)))
    return off, int(nbytes.value)


def decode_png_gray(files, file_offset, file_len, h, w, out_offset, ws_offset, rule, out=None, workspace=None, status=None):
    """PNG files -> 8-bit gray lines on the device (crnn_png_decode_gray_u8), byte for byte the host reader's: rule 0
    cv2.imread(path, 0), rule 1 Pillow's convert("L").  File i is files[file_offset[i]:][:file_len[i]]; its h[i] x w[i] image goes
    row-major to out[out_offset[i]:], the layout resize_lines_u8 reads.  files / out uint8, file_offset / file_len / out_offset
    [N] int64, h / w [N] int32, ws_offset [N + 1] int64 (png_plan's), all cuda.  out: None allocates sum(h * w) bytes;
    workspace: None allocates ws_offset's last entry (read back from the device when needed: pass it to stay asynchronous);
    status: a [N] int32 cuda tensor, or None.  Returns (out, status); a file with a non-zero status (PNG_STATUS) has an
    all-zero slot.  No host fallback: CPU tensors raise CrnnError."""
    return _decode_gray("decode_png_gray", "crnn_png_decode_gray_u8", files, file_offset, file_len, h, w, out_offset, ws_offset,
                        rule, out, workspace, status)


def _decode_gray(name, entry, files, file_offset, file_len, h, w, out_offset, ws_offset, rule, out, workspace, status):
    ints64, ints32 = (file_offset, file_len, out_offset, ws_offset), (h, w)
    if not all(torch.is_tensor(t) and t.is_cuda for t in (files,) + ints64 + ints32):
        raise CrnnError(f"{name} needs CUDA tensors (sm_90a); there is no CPU fallback")
    if files.dtype != torch.uint8 or any(t.dtype != torch.int64 for t in ints64) or any(t.dtype != torch.int32 for t in ints32):
        raise CrnnError(f"{name}: files must be uint8, file_offset, file_len, out_offset and ws_offset int64, h and w int32")
    N = h.numel()
    if any(t.numel() != N for t in (file_offset, file_len, out_offset, w)) or ws_offset.numel() != N + 1:
        raise CrnnError(f"{name}: one file_offset, file_len, out_offset, h and w per file and N + 1 ws_offset entries")
    files, file_offset, file_len, out_offset, ws_offset, h, w = (t.contiguous() for t in (files,) + ints64 + ints32)
    dev = files.device
    if out is None:
        out = torch.empty(max(int((h.long() * w.long()).sum().item()), 1), dtype=torch.uint8, device=dev)
    elif not (torch.is_tensor(out) and out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous()):
        raise CrnnError(f"{name}: out must be a contiguous uint8 cuda tensor")
    if workspace is None:
        workspace = torch.empty(max(int(ws_offset[-1].item()), 1), dtype=torch.uint8, device=dev)
    if status is None:
        status = torch.empty(N, dtype=torch.int32, device=dev)
    elif not (torch.is_tensor(status) and status.is_cuda and status.dtype == torch.int32 and status.numel() == N):
        raise CrnnError(f"{name}: status must be a [{N}] int32 cuda tensor")
    check(getattr(_lib.load(), entry)(files.data_ptr(), file_offset.data_ptr(), file_len.data_ptr(), N, h.data_ptr(), w.data_ptr(),
                                      out_offset.data_ptr(), int(rule), out.data_ptr(), status.data_ptr(), workspace.data_ptr(),
                                      ws_offset.data_ptr(), workspace.numel(), _stream()))
    return out, status


JPEG_STATUS = {0: "ok", 1: "bad header", 2: "unsupported JPEG process", 3: "bad marker segment", 4: "bad Huffman table",
               5: "bad entropy-coded data", 6: "bad restart marker", 7: "the host reader computes something else",
               8: "workspace too small"}
_JPEG_SOF = set(range(0xC0, 0xD0)) - {0xC4, 0xC8, 0xCC}


def jpeg_sof(data):
    """(marker, payload) of a JPEG file's first SOFn segment -- the marker code (0xC0 baseline, 0xC1 extended sequential, ...)
    and the segment's bytes after its length field -- found by walking the marker segments from SOI (only their headers are read,
    however long the segments before the frame); None when `data` is not such a prefix (a bad marker or segment length, or SOS /
    EOI before any SOF)."""
    b = memoryview(data).cast("B")
    n = len(b)
    if n < 2 or b[0] != 0xFF or b[1] != 0xD8:
        return None
    pos = 2
    while True:
        if pos >= n or b[pos] != 0xFF:
            return None
        while pos < n and b[pos] == 0xFF:
            pos += 1
        if pos + 3 > n:
            return None
        m = b[pos]
        if m == 0x00 or m == 0x01 or 0xD0 <= m <= 0xDA:        # no segment here, or the scan / EOI before a frame
            return None
        length = (b[pos + 1] << 8) | b[pos + 2]
        if length < 2 or pos + 1 + length > n:
            return None
        if m in _JPEG_SOF:
            payload = bytes(b[pos + 3:pos + 1 + length])
            return (m, payload) if len(payload) >= 6 else None
        pos += 1 + length


def jpeg_size(data):
    """(h, w) from a JPEG file's first SOFn segment (bytes-like), or None when `data` does not walk from SOI to one (jpeg_sof).
    Only the size is read: the rest of the file is the device decoder's to check."""
    sof = jpeg_sof(data)
    return None if sof is None else (int.from_bytes(sof[1][1:3], "big"), int.from_bytes(sof[1][3:5], "big"))


def jpeg_plan(sof, file_len, rule):
    """crnn_jpeg_plan: sof [N, 16] uint8 (each file's SOF payload after its length field, zero-filled to 16 bytes), file_len [N]
    int64 (host arrays), rule 0 / 1 -> (ws_offset [N + 1] int64, workspace bytes).  File i's record, restart segment table,
    coefficients and (rule 1, colour) planes lie in workspace[ws_offset[i]:ws_offset[i + 1]]."""
    sof = np.ascontiguousarray(sof, np.uint8)
    file_len = np.ascontiguousarray(file_len, np.int64)
    N = file_len.size
    if sof.shape != (N, 16):
        raise CrnnError(f"jpeg_plan: sof must be [{N}, 16] uint8")
    off = np.zeros(N + 1, np.int64)
    nbytes = _lib.c_size_t()
    check(_lib.load().crnn_jpeg_plan(sof.ctypes.data, file_len.ctypes.data, N, int(rule), off.ctypes.data, ctypes.byref(nbytes)))
    return off, int(nbytes.value)


def jpeg_sof_records(files):
    """[N, 16] uint8: each file's SOF payload zero-filled to 16 bytes, the `sof` of jpeg_plan (zeros where jpeg_sof finds none)."""
    rec = np.zeros((len(files), 16), np.uint8)
    for i, f in enumerate(files):
        sof = jpeg_sof(f)
        if sof is not None:
            p = sof[1][:16]
            rec[i, :len(p)] = np.frombuffer(p, np.uint8)
    return rec


def decode_jpeg_gray(files, file_offset, file_len, h, w, out_offset, ws_offset, rule, out=None, workspace=None, status=None):
    """JPEG files -> 8-bit gray lines on the device (crnn_jpeg_decode_gray_u8), byte for byte the host reader's: rule 0
    cv2.imread(path, 0), rule 1 Pillow's convert("L").  The arguments are decode_png_gray's; ws_offset is jpeg_plan's for the
    same rule and the workspace must be 16-byte aligned.  Returns (out, status); a file with a non-zero status (JPEG_STATUS) has
    an all-zero slot.  No host fallback: CPU tensors raise CrnnError."""
    return _decode_gray("decode_jpeg_gray", "crnn_jpeg_decode_gray_u8", files, file_offset, file_len, h, w, out_offset, ws_offset,
                        rule, out, workspace, status)


class GlyphAtlas(object):
    """A PIL font's glyphs on the device for crnn_render_lines_u8: ``glyphs`` [n, 8] i32 (advance, mask w, h, offset ox, oy, mask
    byte offset) and ``masks`` u8, from gen.glyph_atlas (which refuses a font whose cached glyph path does not reproduce
    ImageDraw.text).  ``charset``: cfg.CHARSET by default; charset index c is label id c + 1."""

    def __init__(self, font, charset=None, device="cuda"):
        from .lib.lstm.utils import gen
        glyphs, masks = gen.glyph_atlas(font, charset)
        self.nglyphs = glyphs.shape[0]
        self.max_adv = int(glyphs[:, 0].max())
        self.glyphs = torch.tensor(glyphs, device=device)
        self.masks = torch.tensor(masks, device=device)


def render_record_ints(max_len):
    """i32 entries of one line's layout record (include/crnn_ctc.h crnn_render_layout)."""
    return 8 + 4 * int(max_len)


def render_feed_ints(N, max_len):
    """i32 entries of crnn_render_layout's `feeds` for N lines of at most max_len characters."""
    return 4 + 2 * int(N) + int(N) * int(max_len)


def render_workspace_bytes(N, max_len, max_adv):
    """Bytes of device workspace crnn_render_lines_u8 needs for N lines of at most max_len glyphs of advance <= max_adv."""
    nbytes = _lib.c_size_t()
    check(_lib.load().crnn_render_workspace_size(int(N), int(max_len), int(max_adv), nbytes))
    return int(nbytes.value)


def _render_buf(t, shape, dtype, what):
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == dtype and t.is_contiguous() and tuple(t.shape) == tuple(shape)):
        raise CrnnError(f"{what} must be a contiguous {list(shape)} {dtype} cuda tensor")


def render_layout(seed, min_len, max_len, nw_lo, nw_hi, atlas, layout=None, feeds=None, N=None):
    """Layouts of one batch of the device line stream (crnn_render_layout) on the current stream: lines of min_len .. max_len
    characters of ``atlas``'s charset, seed ``seed`` (gen.batch_seed), bucket nw_lo < nw <= nw_hi (nw_hi 0: none).  Returns the
    device (layout [N, render_record_ints(max_len)], feeds [render_feed_ints(N, max_len)]) i32, written into the given tensors
    when they are passed (N from layout)."""
    if layout is None:
        layout = torch.empty((int(N), render_record_ints(max_len)), dtype=torch.int32, device=atlas.glyphs.device)
    N = layout.shape[0]
    if feeds is None:
        feeds = torch.empty(render_feed_ints(N, max_len), dtype=torch.int32, device=layout.device)
    _render_buf(layout, (N, render_record_ints(max_len)), torch.int32, "render_layout: layout")
    _render_buf(feeds, (render_feed_ints(N, max_len),), torch.int32, "render_layout: feeds")
    s = int(seed) & (2 ** 64 - 1)
    s = s - 2 ** 64 if s >= 2 ** 63 else s                  # the seed's 64 bits as the ABI's int64_t
    check(_lib.load().crnn_render_layout(s, N, int(min_len), int(max_len), int(nw_lo), int(nw_hi), atlas.glyphs.data_ptr(),
                                         atlas.nglyphs, layout.data_ptr(), feeds.data_ptr(), _stream()))
    return layout, feeds


def render_lines_u8(layout, max_len, atlas, W, workspace=None, out=None):
    """The [N, W, 32] uint8 batch of a device layout (crnn_render_lines_u8) on the current stream: glyphs of ``atlas``
    composited as Pillow's draw_bitmap blends them, then Pillow's BILINEAR resize, byte for byte.  W: the padded width (feeds[3]
    of render_layout).  workspace: u8 cuda tensor of render_workspace_bytes(N, max_len, atlas.max_adv) bytes, or None."""
    N = layout.shape[0]
    _render_buf(layout, (N, render_record_ints(max_len)), torch.int32, "render_lines_u8: layout")
    need = render_workspace_bytes(N, max_len, atlas.max_adv)
    if workspace is None:
        workspace = torch.empty(need, dtype=torch.uint8, device=layout.device)
    if out is None:
        out = torch.empty((N, int(W), 32), dtype=torch.uint8, device=layout.device)
    _render_buf(out, (N, int(W), 32), torch.uint8, "render_lines_u8: out")
    if not (torch.is_tensor(workspace) and workspace.is_cuda):
        raise CrnnError("render_lines_u8: workspace must be a cuda tensor")
    check(_lib.load().crnn_render_lines_u8(layout.data_ptr(), N, int(max_len), atlas.glyphs.data_ptr(), atlas.masks.data_ptr(),
                                           atlas.max_adv, int(W), workspace.data_ptr(), workspace.numel() * workspace.element_size(),
                                           out.data_ptr(), _stream()))
    return out


def render_layout_dict(layout, feeds):
    """A device layout and its feeds as host arrays laid out like gen.philox_layout's dict (chars, x, y, fill past each length
    zeroed; dx is not recorded)."""
    lay, f = layout.cpu().numpy().astype(np.int64), feeds.cpu().numpy()
    N, L = lay.shape[0], (lay.shape[1] - 8) // 4
    ln = lay[:, 0]
    live = np.arange(L)[None, :] < ln[:, None]
    d = {k: lay[:, c] for c, k in enumerate(("len", "bg", "x0", "canvas_w", "nw", "tsl", "label_off", "attempt"))}
    for j, k in enumerate(("chars", "x", "y", "fill")):
        d[k] = np.where(live, lay[:, 8 + j * L:8 + (j + 1) * L], 0)
    d.update(status=int(f[0]), max_nw=int(f[1]), W=int(f[3]), label_len=f[4:4 + N].copy(), time_steps=f[4 + N:4 + 2 * N].copy(),
             labels=f[4 + 2 * N:4 + 2 * N + int(f[2])].copy(), max_len=L)
    return d


def ctc_greedy(logits, input_len, tf_blank=TF_BLANK, strip=0):
    """Returns (out [N,T] i32 zero padded, out_len [N] i32) on device."""
    lib = _lib.load()
    T, N, C = logits.shape
    out = torch.empty((N, T), dtype=torch.int32, device=logits.device)
    out_len = torch.empty(N, dtype=torch.int32, device=logits.device)
    check(lib.crnn_ctc_greedy(logits.data_ptr(), input_len.data_ptr(), T, N, C, tf_blank, strip, out.data_ptr(),
                              out_len.data_ptr(), _stream()))
    return out, out_len


def _host_beam_inputs(logits, input_len):
    x = logits.detach().float().cpu().numpy() if torch.is_tensor(logits) else np.asarray(logits, dtype=np.float32)
    x = np.ascontiguousarray(x)
    il = input_len.detach().cpu().numpy() if torch.is_tensor(input_len) else np.asarray(input_len)
    return x, np.ascontiguousarray(il, dtype=np.int32)


def ctc_beam_search(logits, input_len, beam_width=100, merge_repeated=True, strip=0, num_threads=0):
    """The reference's decoder (network.py:656: ctc_beam_search_decoder, width 100, blank C-1, merge_repeated) on the HOST, as
    the TF op is.  logits: [T,N,C] f32 (cuda tensor -> copied back once, or numpy); returns (out [N,T] i32, out_len [N] i32,
    neg_log_prob [N] f32) as numpy arrays."""
    lib = _lib.load()
    x, il = _host_beam_inputs(logits, input_len)
    T, N, C = x.shape
    out = np.zeros((N, T), np.int32); out_len = np.zeros(N, np.int32); nlp = np.zeros(N, np.float32)
    check(lib.crnn_ctc_beam_search(x.ctypes.data, il.ctypes.data, T, N, C, int(beam_width), 1 if merge_repeated else 0, int(strip),
                                   out.ctypes.data, out_len.ctypes.data, nlp.ctypes.data, int(num_threads)))
    return out, out_len, nlp


def ctc_beam_search_topk(logits, input_len, beam_width=100, top_paths=1, merge_repeated=True, strip=0, num_threads=0):
    """ctc_beam_search_decoder's top_paths on the HOST: the `top_paths` best entries of ctc_beam_search's beam, by total (exact
    ties in insertion order; path 0 is ctc_beam_search's read).  1 <= top_paths <= beam_width.  Returns numpy (out [N,K,T] i32
    zero padded, out_len [N,K] i32, log_prob [N,K] f32 = TF's log_probability (<= 0), num_paths [N] i32); paths past
    num_paths have length 0 and log_prob -inf.  Equal labellings from different prefixes are all returned."""
    lib = _lib.load()
    x, il = _host_beam_inputs(logits, input_len)
    T, N, C = x.shape
    K = int(top_paths)
    out = np.zeros((N, max(K, 0), T), np.int32); out_len = np.zeros((N, max(K, 0)), np.int32)
    lp = np.zeros((N, max(K, 0)), np.float32); npaths = np.zeros(N, np.int32)
    check(lib.crnn_ctc_beam_search_topk(x.ctypes.data, il.ctypes.data, T, N, C, int(beam_width), K, 1 if merge_repeated else 0,
                                        int(strip), out.ctypes.data, out_len.ctypes.data, lp.ctypes.data, npaths.ctypes.data,
                                        int(num_threads)))
    return out, out_len, lp, npaths


_beam_ws = {}        # device -> ((T, N, C, beam_width), workspace tensor): the last shape's workspace, reused call to call


def beam_workspace_bytes(T, N, C, beam_width):
    """Bytes of device workspace crnn_ctc_beam_search_device needs for this shape (no CUDA call)."""
    nbytes = _lib.c_size_t()
    check(_lib.load().crnn_ctc_beam_workspace_size(int(T), int(N), int(C), int(beam_width), nbytes))
    return int(nbytes.value)


def _device_beam_inputs(name, logits, input_len, beam_width):
    """Checked contiguous (logits, input_len) and the device's cached workspace for their shape."""
    if not (torch.is_tensor(logits) and logits.is_cuda and torch.is_tensor(input_len) and input_len.is_cuda):
        raise CrnnError(f"{name} needs CUDA tensors; {name.replace('_device', '')} is the host decoder")
    if logits.dtype != torch.float32 or logits.dim() != 3 or input_len.dtype != torch.int32:
        raise CrnnError(f"{name}: logits must be [T,N,C] f32 and input_len i32")
    logits = logits.contiguous()
    input_len = input_len.contiguous()
    T, N, C = logits.shape
    if input_len.numel() != N:
        raise CrnnError(f"{name}: input_len must hold one entry per utterance")
    key = (T, N, C, int(beam_width))
    dev = logits.device
    cached = _beam_ws.get(dev)
    if cached is None or cached[0] != key:
        _beam_ws.pop(dev, None)
        nbytes = beam_workspace_bytes(T, N, C, beam_width)
        cached = _beam_ws[dev] = (key, torch.empty(nbytes, dtype=torch.uint8, device=dev))
    return logits, input_len, cached[1]


def ctc_beam_search_device(logits, input_len, beam_width=100, merge_repeated=True, strip=0):
    """The same decoder as ctc_beam_search (labellings identical to the host's), run on the GPU from device logits: one warp
    per utterance, asynchronous on the current stream, no host sync.  logits [T,N,C] f32 cuda (2 <= C <= 64), input_len [N]
    i32 cuda (clamped to [0, T]), 1 <= beam_width <= 128.  Returns device (out [N,T] i32 zero padded, out_len [N] i32,
    neg_log_prob [N] f32).  There is no host fallback: CPU tensors or an unsupported shape raise CrnnError."""
    lib = _lib.load()
    logits, input_len, ws = _device_beam_inputs("ctc_beam_search_device", logits, input_len, beam_width)
    T, N, C = logits.shape
    dev = logits.device
    out = torch.empty((N, T), dtype=torch.int32, device=dev)
    out_len = torch.empty(N, dtype=torch.int32, device=dev)
    nlp = torch.empty(N, dtype=torch.float32, device=dev)
    check(lib.crnn_ctc_beam_search_device(logits.data_ptr(), input_len.data_ptr(), T, N, C, int(beam_width), 1 if merge_repeated else 0,
                                          int(strip), out.data_ptr(), out_len.data_ptr(), nlp.data_ptr(), ws.data_ptr(), ws.numel(),
                                          _stream()))
    return out, out_len, nlp


def ctc_beam_search_topk_device(logits, input_len, beam_width=100, top_paths=1, merge_repeated=True, strip=0):
    """ctc_beam_search_topk on the GPU: ctc_beam_search_device's beam, inputs, workspace and stream rules, and
    ctc_beam_search_topk's outputs (identical labels, lengths and num_paths) as device tensors (out [N,K,T], out_len [N,K],
    log_prob [N,K], num_paths [N]).  Asynchronous, no host sync; no host fallback."""
    lib = _lib.load()
    logits, input_len, ws = _device_beam_inputs("ctc_beam_search_topk_device", logits, input_len, beam_width)
    T, N, C = logits.shape
    dev = logits.device
    K = int(top_paths)
    out = torch.empty((N, max(K, 0), T), dtype=torch.int32, device=dev)
    out_len = torch.empty((N, max(K, 0)), dtype=torch.int32, device=dev)
    lp = torch.empty((N, max(K, 0)), dtype=torch.float32, device=dev)
    npaths = torch.empty(N, dtype=torch.int32, device=dev)
    check(lib.crnn_ctc_beam_search_topk_device(logits.data_ptr(), input_len.data_ptr(), T, N, C, int(beam_width), K,
                                               1 if merge_repeated else 0, int(strip), out.data_ptr(), out_len.data_ptr(),
                                               lp.data_ptr(), npaths.data_ptr(), ws.data_ptr(), ws.numel(), _stream()))
    return out, out_len, lp, npaths


def dense_decoded(out, out_len):
    """sparse_tensor_to_dense(default 0) shape [N, max_len] (network.py:657); one D2H sync."""
    m = int(out_len.max().item()) if out_len.numel() else 0
    return out[:, :m].contiguous()


def dense_decoded_topk(out, out_len):
    """The K decodings of ctc_beam_search_topk(_device) (out [N,K,T], out_len [N,K]) as K [N, max_len] arrays, each what
    sparse_tensor_to_dense(decoded[k], default 0) gives: max_len is that path's longest read.  numpy or torch in, the same out
    (a torch input costs one D2H sync)."""
    K = out.shape[1]
    if torch.is_tensor(out_len):
        m = out_len.max(0).values.cpu().tolist() if out_len.numel() else [0] * K
    else:
        m = out_len.max(0).tolist() if out_len.size else [0] * K
    return [out[:, k, :int(m[k])].contiguous() if torch.is_tensor(out) else np.ascontiguousarray(out[:, k, :int(m[k])])
            for k in range(K)]


def test_gemm_tn_bf16(A, B, block_n, k_splits=0):
    """D[M,N] = A[K,M]^T @ B[K,N] through the MN-major wgmma path (tests only)."""
    lib = _lib.load()
    K, M = A.shape
    Nc = B.shape[1]
    D = torch.zeros((M, Nc), dtype=torch.float32, device=A.device)
    check(lib.crnn_test_gemm_tn_bf16(A.data_ptr(), B.data_ptr(), D.data_ptr(), M, Nc, K, block_n, k_splits, _stream()))
    return D


def test_gemm_bf16(A, B, block_n):
    lib = _lib.load()
    M, K = A.shape
    Nc = B.shape[0]
    D = torch.empty((M, Nc), dtype=torch.float32, device=A.device)
    check(lib.crnn_test_gemm_bf16(A.data_ptr(), B.data_ptr(), D.data_ptr(), M, Nc, K, block_n, _stream()))
    return D
