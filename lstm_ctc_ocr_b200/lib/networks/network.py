"""Network object with the reference's attribute surface (lib/networks/network.py:40-95,647-664).

The reference builds a TF1 graph through a chaining DSL; here the graph is fixed (it is the one
LSTM_train.setup/LSTM_test.setup build, LSTM_train.py:22-38) and runs as hand-written sm_90a
kernels in libcrnnctc.so.  What is preserved is the *surface* the solver touches: placeholders
``data/labels/time_step_len/labels_len/keep_prob``, the ``layers`` dict, ``feed``/``get_output``,
``build_loss() -> (loss, dense_decoded)``; handles are evaluated by ``Session.run``."""
from ..lstm.config import cfg


class Placeholder(object):
    """Stand-in for tf.placeholder: a named, typed slot filled through ``feed_dict``."""

    def __init__(self, name, dtype, shape):
        self.name, self.dtype, self.shape = name, dtype, shape

    def __repr__(self):
        return f"<Placeholder {self.name} {self.dtype} {self.shape}>"


class Fetch(object):
    """Stand-in for a TF tensor/op handle: something ``Session.run`` can evaluate."""

    def __init__(self, net, kind, name=None):
        self.net, self.kind, self.name = net, kind, name or kind

    def __repr__(self):
        return f"<Fetch {self.name}>"


DEFAULT_PADDING = "SAME"        # network.py:8

# The topology libcrnnctc.so implements, as the chain LSTM_train.setup / LSTM_test.setup build it (LSTM_train.py:22-38), in the
# vocabulary of the reference's layer DSL: (op, arguments after defaults).  The name 'pool2' is used twice there, the second
# max_pool overwriting the first in `layers` (network.py:33); kept as is.
TOPOLOGY = [
    ("conv_single", dict(k_h=3, k_w=3, c_o=64, s_h=1, s_w=1, name="conv1", c_i=1, bn=False, biased=True, relu=True, padding="SAME")),
    ("max_pool", dict(k_h=2, k_w=2, s_h=2, s_w=2, name="pool1", padding="VALID")),
    ("conv_single", dict(k_h=3, k_w=3, c_o=128, s_h=1, s_w=1, name="conv2", c_i=64, bn=False, biased=True, relu=True, padding="SAME")),
    ("max_pool", dict(k_h=2, k_w=2, s_h=2, s_w=2, name="pool2", padding="VALID")),
    ("conv_single", dict(k_h=3, k_w=3, c_o=256, s_h=1, s_w=1, name="conv3_1", c_i=128, bn=False, biased=True, relu=True, padding="SAME")),
    ("conv_single", dict(k_h=3, k_w=3, c_o=256, s_h=1, s_w=1, name="conv3_2", c_i=256, bn=False, biased=True, relu=True, padding="SAME")),
    ("max_pool", dict(k_h=1, k_w=2, s_h=1, s_w=2, name="pool2", padding="VALID")),
    ("conv_single", dict(k_h=3, k_w=3, c_o=512, s_h=1, s_w=1, name="conv4_1", c_i=256, bn=True, biased=True, relu=True, padding="SAME")),
    ("conv_single", dict(k_h=3, k_w=3, c_o=512, s_h=1, s_w=1, name="conv4_2", c_i=512, bn=True, biased=True, relu=True, padding="SAME")),
    ("max_pool", dict(k_h=1, k_w=2, s_h=1, s_w=2, name="pool3", padding="VALID")),
    ("conv_single", dict(k_h=2, k_w=2, c_o=512, s_h=1, s_w=1, name="conv5", c_i=512, bn=False, biased=True, relu=False, padding="VALID")),
    ("reshape_squeeze_layer", dict(d=512, name="reshaped_layer")),
    ("bi_lstm", dict(num_hids=512, num_layers=2, name="logits", img_shape=None)),
]
LAYER_NAMES = [kw["name"] for _, kw in TOPOLOGY]
# layers of the reference's DSL that exist (network.py:131-645) but are not on the CRNN+CTC path (SURVEY section 2: out of scope)
_OFF_PATH_LAYERS = ("lstm", "concat", "conv", "conv_zero", "conv_norm", "conv_final", "upconv", "relu", "avg_pool", "reshape_layer",
                    "spatial_reshape_layer", "lrn", "fc", "softmax", "spatial_softmax", "add", "batch_normalization", "negation",
                    "bn_scale_combo", "pva_negation_block", "pva_negation_block_v2", "pva_inception_res_stack",
                    "pva_inception_res_block", "scale", "dropout", "smooth_l1_dist")


class UnsupportedGraph(NotImplementedError):
    """The declared layer chain is not the one the sm_90a kernels implement (there is no generic graph executor behind this
    API and no fallback: the reference's LSTM_train / LSTM_test topology is the product)."""


def layer(op):
    """The reference's chaining decorator (network.py:19-38): default name, inputs from the previous call, result registered in
    `layers` and fed forward, `self` returned."""
    def layer_decorated(self, *args, **kwargs):
        name = kwargs.setdefault("name", self.get_unique_name(op.__name__))
        if len(self.inputs) == 0:
            raise RuntimeError("No input variables found for layer %s." % name)
        layer_input = self.inputs[0] if len(self.inputs) == 1 else list(self.inputs)
        layer_output = op(self, layer_input, *args, **kwargs)
        self.layers[name] = layer_output
        self.feed(layer_output)
        return self
    layer_decorated.__name__ = op.__name__
    layer_decorated.__doc__ = op.__doc__
    return layer_decorated


class Network(object):
    def __init__(self, inputs, trainable=True):
        self.inputs = []
        self.layers = dict(inputs)
        self.trainable = trainable
        self.setup()

    def setup(self):
        raise NotImplementedError("Must be subclassed.")

    def feed(self, *args):
        assert len(args) != 0
        self.inputs = []
        for layer in args:
            if isinstance(layer, str):
                try:
                    layer = self.layers[layer]
                except KeyError:
                    print(list(self.layers.keys()))
                    raise KeyError("Unknown layer name fed: %s" % layer)
            self.inputs.append(layer)
        return self

    @property
    def line_width(self):
        """Optional placeholder, not in the reference: each line's padded width W_i when several lines are packed into one batch.
        Feeding it evaluates every line as if it were run alone (per-line BatchNorm statistics and width boundaries,
        crnn_forward_lines).  Shared by every network built on this class."""
        ph = self.__dict__.get("_line_width")
        if ph is None:
            ph = self.__dict__["_line_width"] = Placeholder("line_width", "int32", [None])
        return ph

    @property
    def data_u8(self):
        """Optional placeholder, not in the reference: the batch as 8-bit pixels, uint8 [N, W, 32] in the layout of `data`.  The
        network's input is then data_u8 / 255 (an IEEE f32 division, the value `data` holds for the same pixel), and the bytes
        travel to the device as they are: a quarter of the host and PCIe traffic of `data`.  `data` keeps its meaning (a uint8
        array fed to it is widened to 0..255, as a TF float placeholder would cast it); feed one of the two.  Shared by every
        network built on this class."""
        ph = self.__dict__.get("_data_u8")
        if ph is None:
            ph = self.__dict__["_data_u8"] = Placeholder("data_u8", "uint8", [None, None, cfg.NUM_FEATURES])
        return ph

    @property
    def images(self):
        """Optional placeholder, not in the reference: a batch of text lines at their native size, a sequence of 2-D uint8 gray
        arrays (H_i x W_i, 1 <= H_i <= 1024).  Each line travels to the device as it is and is resized there to 32 rows with
        Pillow's BILINEAR, byte for byte (crnn_resize_lines_u8), then evaluated packed as with `line_width`: the batch, widths and
        time_step_len that prepare_line + pack_lines would build on the host.  Evaluation fetches only; feed it instead of data,
        data_u8, line_width and time_step_len.  Shared by every network built on this class."""
        ph = self.__dict__.get("_images")
        if ph is None:
            ph = self.__dict__["_images"] = Placeholder("images", "uint8", [None, None])
        return ph

    def get_output(self, layer):
        try:
            return self.layers[layer]
        except KeyError:
            print(list(self.layers.keys()))
            raise KeyError("Unknown layer name fed: %s" % layer)

    def get_unique_name(self, prefix):
        n = sum(t.startswith(prefix) for t in self.layers) + 1
        return "%s_%d" % (prefix, n)

    # ---- the layer DSL of the path (network.py:97-129,160-191,343-368): each call DECLARES a layer -- the arithmetic is the
    # fixed kernel pipeline of libcrnnctc.so -- and is checked against the topology those kernels implement, so a reference-style
    # `setup()` chain runs unchanged and anything else fails loudly instead of silently computing a different network.
    def validate_padding(self, padding):
        assert padding in ("SAME", "VALID")

    def _declare(self, op, input, **kw):
        d = self.__dict__.setdefault("_declared", [])
        pos = len(d)
        if pos >= len(TOPOLOGY):
            raise UnsupportedGraph(f"{op}({kw.get('name')}): the compiled network ends with bi_lstm('logits')")
        want_op, want = TOPOLOGY[pos]
        got = dict(kw)
        if op == "conv_single" and not got.get("c_i"):
            # `if not c_i: c_i = input.get_shape()[-1]` (network.py:164): the previous layer's channel count -- except on the
            # channel-less data placeholder, where the reference itself has to pass c_i=cfg.NCHANNELS (LSTM_train.py:24)
            got["c_i"] = want.get("c_i") if pos else cfg.NUM_FEATURES
        if op != want_op or got != want:
            diff = {k: (got.get(k), v) for k, v in want.items() if got.get(k) != v} if op == want_op else {}
            raise UnsupportedGraph(f"layer {pos} declared as {op}({kw}) but libcrnnctc.so implements {want_op}({want})"
                                   + (f"; differing (declared, compiled): {diff}" if diff else ""))
        src = input if isinstance(input, list) else [input]
        expect = ["time_step_len"] if op == "bi_lstm" else []
        prev = TOPOLOGY[pos - 1][1]["name"] if pos else "data"
        names = [getattr(x, "name", None) for x in src]
        if names[0] != prev or names[1:] != expect:
            raise UnsupportedGraph(f"{op}({kw.get('name')}) is fed from {names}; the compiled network feeds it from {[prev] + expect}")
        d.append((op, got))
        return Fetch(self, "logits") if op == "bi_lstm" else Fetch(self, "layer:" + kw["name"], kw["name"])

    @layer
    def conv_single(self, input, k_h, k_w, c_o, s_h, s_w, name, c_i=None, bn=False, biased=True, relu=True, padding=DEFAULT_PADDING,
                    trainable=True):
        """conv2d -> bias_add -> (batch-statistics batch_norm) -> relu (network.py:160-191)."""
        self.validate_padding(padding)
        return self._declare("conv_single", input, k_h=k_h, k_w=k_w, c_o=c_o, s_h=s_h, s_w=s_w, name=name, c_i=c_i, bn=bn, biased=biased,
                             relu=relu, padding=padding)

    @layer
    def max_pool(self, input, k_h, k_w, s_h, s_w, name, padding=DEFAULT_PADDING):
        """tf.nn.max_pool with ksize [1,k_h,k_w,1], strides [1,s_h,s_w,1] (network.py:343-350)."""
        self.validate_padding(padding)
        return self._declare("max_pool", input, k_h=k_h, k_w=k_w, s_h=s_h, s_w=s_w, name=name, padding=padding)

    @layer
    def reshape_squeeze_layer(self, input, d, name):
        """[N,H,W,C] -> [N,H*W,d] (network.py:361-368)."""
        return self._declare("reshape_squeeze_layer", input, d=int(d), name=name)

    @layer
    def bi_lstm(self, input, num_hids, num_layers, name, img_shape=None, trainable=True):
        """fw/bw LSTMCell(num_hids//2) under bidirectional_dynamic_rnn(sequence_length) + the num_hids -> NCLASSES projection,
        time-major logits (network.py:97-129); `num_layers` is unused by the reference too."""
        return self._declare("bi_lstm", input, num_hids=int(num_hids), num_layers=int(num_layers), name=name, img_shape=img_shape)

    def __getattr__(self, item):
        if item in _OFF_PATH_LAYERS:
            raise UnsupportedGraph(f"layer '{item}' of the reference's DSL is not on the CRNN+CTC path this library implements "
                                   "(conv_single, max_pool, reshape_squeeze_layer, bi_lstm)")
        raise AttributeError(item)

    def _declare_graph(self):
        """The chain LSTM_train.setup / LSTM_test.setup build (LSTM_train.py:22-38), issued through the DSL above."""
        self.feed("data")
        for op, kw in TOPOLOGY[:-1]:
            getattr(self, op)(**kw)
        op, kw = TOPOLOGY[-1]
        self.feed("reshaped_layer", "time_step_len")
        getattr(self, op)(**kw)

    def _check_declared(self):
        n = len(self.__dict__.get("_declared", []))
        if n != len(TOPOLOGY):
            raise UnsupportedGraph(f"the declared chain stops after {n} of {len(TOPOLOGY)} layers; the compiled network runs "
                                   "conv1 .. conv5, reshaped_layer and bi_lstm('logits')")

    def load(self, data_path, session, ignore_missing=False):
        """npy dict {scope: {var: array}} loader (network.py:50-63)."""
        import numpy as np
        data = np.load(data_path, allow_pickle=True, encoding="latin1").item()
        sd = {}
        for scope, sub in data.items():
            for var, arr in sub.items():
                sd[f"{scope}/{var}"] = arr
        session.assign(self, sd, ignore_missing=ignore_missing)

    def build_loss(self):
        """(loss, dense_decoded) handles; semantics of network.py:647-664 with the greedy decode of
        SURVEY §8(c) in place of the width-100 beam search."""
        if "labels" not in self.layers:
            raise KeyError("Unknown layer name fed: labels")
        self._check_declared()
        self._wd = float(cfg.TRAIN.WEIGHT_DECAY)
        return Fetch(self, "loss"), Fetch(self, "dense_decoded")
