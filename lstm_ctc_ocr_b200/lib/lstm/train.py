"""Training solver with the reference's surface (lib/lstm/train.py): ``SolverWrapper(sess, network, imgdb, pre_train,
output_dir, logdir)``, ``snapshot``, ``restoreLabel``, ``train_model(sess, max_iters, restore)``, ``train_net(...)``.

Every iteration runs ``sess.run([loss, train_op], feed_dict)`` (train.py:129-130): forward, CTC loss + gradient, backward,
global-norm clip 10.0 and the optimizer ``cfg.TRAIN.SOLVER`` selects -- all on the GPU engine.  The selection is the reference's
(train.py:74-76): ``Adam`` -> AdamOptimizer(lr), ``RMS`` -> RMSPropOptimizer(lr) with TF's defaults (decay 0.9, momentum 0,
epsilon 1e-10), ANY other value -> MomentumOptimizer(lr, cfg.TRAIN.MOMENTUM).

Checkpoints are ``.npz`` files holding the TF variable names/layouts, the solver's slots, lr and the step, named
``<prefix>_ctc_iter_<k>.ckpt.npz`` with a TF-style ``checkpoint`` index file.  Slot keys per solver: ``adam_m/<var>`` and
``adam_v/<var>`` (Adam), ``momentum/<var>`` (Momentum), ``rms/<var>`` (the mean square) and ``rms_momentum/<var>`` (RMSProp)."""
import os
import re

import numpy as np

from ... import engine
from ...session import Session
from ..networks.network import Fetch
from .config import cfg
from .utils.gen import feed_dtype, get_batch
from .utils.timer import Timer
from .utils.training import accuracy_calculation


class Variable(object):
    """Scalar host variable (the reference keeps lr / global_step as tf.Variables, train.py:73,78)."""

    def __init__(self, value):
        self.value = value

    def eval(self):
        return self.value

    def assign(self, v):
        self.value = v
        return self


class TrainOp(Fetch):
    """What ``opt.apply_gradients(zip(clip_by_global_norm(tf.gradients(loss, tvars), 10.0), tvars), global_step)`` returns."""

    def __init__(self, net, lr, global_step, clip=10.0):
        super().__init__(net, "train_op")
        self.lr, self.global_step, self.clip = lr, global_step, clip

    def step_fn(self, eng, logits, grad, d_data, d_tsl):
        eng.backward(d_data, d_tsl, grad)             # data parallel: announces gradient buckets, reduced on a side stream meanwhile
        self.global_step.assign(self.global_step.eval() + 1)
        dp = getattr(eng, "_dp", None)
        if dp is not None:
            dp.step(self.lr.eval(), self.global_step.eval(), clip=self.clip)       # waits for the buckets; clip + update on the SUM / world
        else:
            eng.apply_gradients(self.lr.eval(), self.global_step.eval(), clip=self.clip)
        return None


def render_on_device(name):
    """cfg.RENDER ("host" or "device") -> True when train_model renders its default batches on the GPU."""
    if str(name) not in ("host", "device"):
        raise ValueError(f"RENDER must be 'host' or 'device', got {name!r}")
    return str(name) == "device"


def is_device_batch(imgs):
    """True for the pixels of a batch already on the GPU (a DeviceLineRenderer's uint8 cuda tensor)."""
    import torch
    return torch.is_tensor(imgs) and imgs.is_cuda


def solver_from_cfg(train_cfg):
    """cfg.TRAIN -> (engine solver name, momentum), chosen as the reference chooses its optimizer (train.py:74-76): SOLVER 'Adam'
    -> "Adam", 'RMS' -> "RMS" (TF defaults, no config key), every other value -> "Momentum" with TRAIN.MOMENTUM.  The momentum is
    returned for every solver; only Momentum reads it."""
    name = {"Adam": "Adam", "RMS": "RMS"}.get(train_cfg.SOLVER, "Momentum")
    return name, float(train_cfg.MOMENTUM)


class SolverWrapper(object):
    def __init__(self, sess, network, imgdb, pre_train, output_dir, logdir):
        self.net = network
        self.imgdb = imgdb
        self.pre_train = pre_train
        self.output_dir = output_dir
        self.logdir = logdir
        self.sess = sess
        print("done")

    # ---- checkpoints (train.py:23-37, 96-106) ---------------------------------------------------------------
    def snapshot(self, sess, iter):
        os.makedirs(self.output_dir, exist_ok=True)
        infix = ("_" + cfg.TRAIN.SNAPSHOT_INFIX) if cfg.TRAIN.SNAPSHOT_INFIX != "" else ""
        filename = cfg.TRAIN.SNAPSHOT_PREFIX + "_ctc" + infix + "_iter_{:d}".format(iter + 1) + ".ckpt"
        path = os.path.join(self.output_dir, filename)
        eng = sess.engine_for(self.net)
        blob = dict(eng.state_dict())
        if getattr(eng, "bn_moving", None) is not None:
            blob.update(eng.bn_moving_state())          # moving_mean / moving_variance of conv4_1, conv4_2 under TF's names
        if eng.adam_m is not None:
            blob.update(slot_arrays(eng))
        blob["global_step"] = np.array(getattr(self, "_global_step", Variable(0)).eval())
        blob["lr"] = np.array(getattr(self, "_lr", Variable(cfg.TRAIN.LEARNING_RATE)).eval())
        np.savez(path + ".npz", **blob)
        with open(os.path.join(self.output_dir, "checkpoint"), "w") as f:
            f.write('model_checkpoint_path: "{}"\n'.format(filename))
        print("Wrote snapshot to: {:s}".format(path))
        return path

    def _latest_checkpoint(self):
        idx = os.path.join(self.output_dir, "checkpoint")
        if not os.path.exists(idx):
            return None
        m = re.search(r'model_checkpoint_path: "(.*)"', open(idx).read())
        return os.path.join(self.output_dir, m.group(1)) if m else None

    def restore(self, sess, path):
        blob = np.load(path + ".npz")
        eng = sess.engine_for(self.net)
        eng.load_params({k: blob[k] for k in eng.table})
        if getattr(eng, "bn_moving", None) is not None:
            restore_bn_moving(eng, blob)
        loaded = getattr(sess, "params_loaded", None)     # Session: an fp8 evaluation engine recalibrates for the restored weights
        if loaded is not None:
            loaded(self.net)
        if eng.adam_m is not None:
            restore_slots(eng, blob)
        return blob

    def restoreLabel(self, label_vec, label_len):
        labels = []
        for l_len in label_len:
            labels.append(label_vec[:l_len])
            label_vec = label_vec[l_len:]
        return labels

    # ---- the loop (train.py:63-162) -----------------------------------------------------------------------------
    def _feed(self, batch, keep_prob):
        """feed_dict for one data-layer tuple (train.py:119-127); uint8 batches (cfg.FEED_DTYPE "uint8") go to data_u8."""
        imgs, flat_labels, label_len, time_steps = batch
        net = self.net
        if is_device_batch(imgs):                         # a DeviceLineRenderer batch: uint8 on the device, fed in place
            return {net.data_u8: imgs, net.labels: np.array(flat_labels), net.time_step_len: np.array(time_steps),
                    net.labels_len: np.array(label_len), net.keep_prob: keep_prob}
        # a PrefetchFeeder hands out an ndarray view of a page-locked ring slot: keep it (np.array would copy it to pageable memory)
        data = imgs if isinstance(imgs, np.ndarray) and imgs.ndim == 3 else np.array(imgs)
        return {(net.data_u8 if data.dtype == np.uint8 else net.data): data, net.labels: np.array(flat_labels), net.time_step_len: np.array(time_steps),
                net.labels_len: np.array(label_len), net.keep_prob: keep_prob}

    def _prepare(self, sess, restore, lr, global_step):
        """Variable initialisation, data-parallel broadcast and the optional resume (train.py:88-106)."""
        from ... import parallel, synthetic
        eng = sess.engine_for(self.net)
        if not getattr(eng, "_initialised", False):
            eng.load_params(synthetic.init_params(cfg.RNG_SEED))       # global_variables_initializer
            eng._initialised = True
        solver, momentum = solver_from_cfg(cfg.TRAIN)
        if eng.solver != solver:
            eng.set_solver(solver, momentum)                          # the slots start from TF's initial values
        else:
            eng.momentum = momentum                                   # same solver: its slots carry over (a second train_model)
        eng.set_training(True)
        if parallel.world_size() > 1 and getattr(eng, "_dp", None) is None:
            # parameter broadcast, global-batch BatchNorm over peer memory, overlapped gradient buckets (parallel.DataParallel)
            eng._dp = parallel.DataParallel(eng, sync_bn=bool(cfg.TRAIN.get("SYNC_BN", True)))
        if not restore:
            return 1
        path = self._latest_checkpoint()
        try:
            print("Restoring from {}...".format(path), end=" ")
            blob = self.restore(sess, path)
            first_iter = int(os.path.splitext(os.path.basename(path))[0].split("_")[-1])   # iteration from the file name
            global_step.assign(first_iter)
            lr.assign(float(blob["lr"]))
            print("done")
            return first_iter
        except Exception:
            raise Exception("Check your pretrained {:s}".format(str(path)))

    def _validate(self, sess, dense_decoded, val_gen, cache):
        """Accuracy on ONE cached validation batch (train.py:145-162)."""
        if "batch" not in cache:
            cache["batch"] = next(val_gen)
            cache["org"] = self.restoreLabel(cache["batch"][1], cache["batch"][2])
        res = sess.run(fetches=dense_decoded, feed_dict=self._feed(cache["batch"], 1.0))
        acc = accuracy_calculation(cache["org"], res, ignore_value=0)
        print("accuracy: {:.5f}".format(acc))
        return acc

    def train_model(self, sess, max_iters, restore=False, train_gen=None, val_gen=None):
        from ... import parallel
        dtype = feed_dtype(cfg.FEED_DTYPE)
        on_device = render_on_device(cfg.RENDER)
        if on_device:
            # batches rendered on the session's GPU: the host streams' seeds and rank handling, no producer processes
            dev = getattr(sess, "device", None)
            train_gen = train_gen or get_batch(num_workers=0, batch_size=cfg.TRAIN.BATCH_SIZE, on_device=True, device=dev)
            val_gen = val_gen or get_batch(num_workers=0, batch_size=cfg.VAL.BATCH_SIZE, on_device=True, device=dev)
        train_gen = train_gen or get_batch(num_workers=12, batch_size=cfg.TRAIN.BATCH_SIZE, vis=False, dtype=dtype)
        val_gen = val_gen or get_batch(num_workers=1, batch_size=cfg.VAL.BATCH_SIZE, vis=False, dtype=dtype)
        loss, dense_decoded = self.net.build_loss()
        lr, global_step = Variable(cfg.TRAIN.LEARNING_RATE), Variable(0)
        self._lr, self._global_step = lr, global_step
        train_op = TrainOp(self.net, lr, global_step, clip=10.0)
        first_iter = self._prepare(sess, restore, lr, global_step)
        if hasattr(sess, "attach_feeder"):
            sess.attach_feeder(train_gen)                  # PrefetchFeeder: the next batch's H2D copy overlaps the current step (no-op for plain generators)
        timer, history, val_cache = Timer(), [], {}
        loss_min = 0.015                                   # best-loss snapshot threshold (train.py:109)
        is_chief = parallel.rank() == 0
        for iter in range(first_iter, max_iters):
            timer.tic()
            if iter != 0 and iter % cfg.TRAIN.STEPSIZE == 0:
                lr.assign(lr.eval() * cfg.TRAIN.GAMMA)
            ctc_loss, _ = sess.run(fetches=[loss, train_op], feed_dict=self._feed(next(train_gen), 0.5))
            history.append(float(ctc_loss))
            step_seconds = timer.toc(average=False)
            if iter % cfg.TRAIN.DISPLAY == 0:
                print("iter: %d / %d, total loss: %.7f, lr: %.7f" % (iter, max_iters, ctc_loss, lr.eval()), end=" ")
                print("speed: {:.3f}s / iter".format(step_seconds))
            new_best = ctc_loss < loss_min
            if new_best or (iter + 1) % cfg.TRAIN.SNAPSHOT_ITERS == 0:
                if is_chief:
                    if new_best:
                        print("loss: ", ctc_loss, end=" ")
                        self.snapshot(sess, 1)             # the reference always names the best-loss snapshot iter_2
                    else:
                        self.snapshot(sess, iter)
                if new_best:
                    loss_min = ctc_loss
            if new_best or (iter + 1) % cfg.VAL.VAL_STEP == 0:
                self._validate(sess, dense_decoded, val_gen, val_cache)
        return history


def _to_dev(arr, eng):
    import torch
    return torch.as_tensor(np.asarray(arr, dtype=np.float32).reshape(-1), device=eng.device)


def slot_arrays(eng):
    """{"<slot prefix>/<TF variable>": array} of the engine's current solver slots (engine.SOLVER_SLOTS names the prefixes)."""
    out = {}
    for prefix, buf in eng.solver_slots().items():
        for k, (off, shp) in eng.table.items():
            n = int(np.prod(shp))
            out[prefix + "/" + k] = buf[off:off + n].view(*shp).cpu().numpy()
    return out


def restore_bn_moving(eng, blob):
    """Moving statistics from a checkpoint that holds them; an older one leaves TF's initial values (mean 0, variance 1), so it
    still resumes -- but an engine that evaluates with moving statistics refuses it: untrained statistics are a mistake."""
    files = set(getattr(blob, "files", blob))
    if all(k in files for k in engine.BN_MOVING_KEYS):
        eng.load_bn_moving({k: blob[k] for k in engine.BN_MOVING_KEYS})
        return
    if eng.bn_statistics == "moving":
        raise KeyError("cfg.TEST.BN_STATS is 'moving' but the checkpoint holds no moving statistics ({})".format(
            ", ".join(engine.BN_MOVING_KEYS)))
    eng.load_bn_moving(None)


def restore_slots(eng, blob):
    """Load the configured solver's slots from a checkpoint that holds them.  A params-only checkpoint leaves the slots freshly
    initialised as TF initialises them; one that holds only another solver's slots raises, as TF's Saver fails on a checkpoint
    without the graph's slot variables."""
    from ...engine import SOLVER_SLOTS
    slots = eng.solver_slots()
    files = set(blob.files)
    if all(p + "/" + k in files for p in slots for k in eng.table):
        for prefix, buf in slots.items():
            for k, (off, shp) in eng.table.items():
                buf[off:off + int(np.prod(shp))].copy_(_to_dev(blob[prefix + "/" + k], eng))
        return
    known = {p for pairs in SOLVER_SLOTS.values() for p, _ in pairs}
    held = sorted({f.split("/", 1)[0] for f in files if "/" in f} & known)
    if held:
        raise KeyError("checkpoint holds the slots {} but not all of those of the configured solver {} ({})".format(
            held, eng.solver, sorted(slots)))
    eng.reset_slots()


def train_net(network, imgdb, pre_train, output_dir, log_dir, max_iters=40000, restore=False):
    with Session() as sess:
        sw = SolverWrapper(sess, network, imgdb, pre_train, output_dir, logdir=log_dir)
        print("Solving...")
        sw.train_model(sess, max_iters, restore=restore)
        print("done solving")
