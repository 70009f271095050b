"""Global run configuration with the reference's keys and defaults.

Mirrors lib/lstm/config.py of the reference: same key names, default values (config.py:12-72),
charset map (config.py:73-81), typed YAML merge (config.py:99-134) and ``--set`` overrides
(config.py:136-156).  Implemented on a small attribute dict (easydict is not a dependency)."""
import os
import os.path as osp
from ast import literal_eval
from time import localtime, strftime


class AttrDict(dict):
    """dict with attribute access (what the reference gets from easydict)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


_CHARSET = "0123456789abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ"

# key -> default, exactly the reference's values (lib/lstm/config.py:12-72); nested sections are AttrDicts
_DEFAULTS = {
    "GPU_ID": 1, "GPU_USAGE": 0.9,
    "OFFSET_TIME_STEP": -1, "POOL_SCALE": 4,                   # time_step = nw // POOL_SCALE + OFFSET_TIME_STEP
    "IMG_SHAPE": [32, 100], "IMG_HEIGHT": 32, "NCHANNELS": 1,
    "MAX_CHAR_LEN": 6, "MIN_LEN": 4, "MAX_LEN": 6,
    "BLANK_TOKEN": 0, "SPACE_INDEX": 0, "SPACE_TOKEN": "",
    "CHARSET": _CHARSET, "NCLASSES": len(_CHARSET) + 2,        # + CTC blank (0) + decoder blank (63)
    "FONT": "fonts/Ubuntu-M.ttf",
    # not in the reference: which decoder `dense_decoded` runs -- "greedy" (GPU kernel, the hot path) or "beam" (the reference's
    # ctc_beam_search_decoder semantics, network.py:656; decoded on the GPU, width BEAM_WIDTH <= 128)
    "DECODER": "greedy", "BEAM_WIDTH": 100,
    # not in the reference (it widens every line to f32 on the host): "uint8" builds training, validation and evaluation batches
    # as 8-bit pixels and feeds them through the networks' data_u8 placeholder -- a quarter of the host and PCIe bytes, the same
    # values on the device (x = u / 255 in f32); "float32" feeds data as the reference does
    "FEED_DTYPE": "float32",
    "NET_NAME": "lstm", "EXP_DIR": "default", "LOG_DIR": "default", "RNG_SEED": 3,
    "TRAIN": {
        "SOLVER": "Adam", "TXT": "annotation_train.txt",
        "LEARNING_RATE": 0.01, "MOMENTUM": 0.9, "GAMMA": 0.1, "STEPSIZE": 50000, "WEIGHT_DECAY": 0.0005,
        "DISPLAY": 10, "LOG_IMAGE_ITERS": 100, "NUM_EPOCHS": 2000,
        "NUM_HID": 512, "NUM_LAYERS": 2, "BATCH_SIZE": 64,
        "SNAPSHOT_ITERS": 5000, "SNAPSHOT_PREFIX": "lstm", "SNAPSHOT_INFIX": "",
        "SYNC_BN": True,        # not in the reference (single device): data-parallel runs use GLOBAL-batch BN statistics
    },
    "VAL": {"TXT": "annotation_val.txt", "VAL_STEP": 1000, "NUM_EPOCHS": 1000, "BATCH_SIZE": 128, "PRINT_NUM": 5},
    # not in the reference (one line per run): lines per packed evaluation batch of test_model, each line still evaluated as if
    # alone (DESIGN §5 has the measured rates behind the default)
    "TEST": {"BATCH_SIZE": 64,
             # not in the reference: "fp8" evaluates LSTM_test networks with e4m3 operands in conv3_1 .. conv5 (compute_dtype 4),
             # calibrated on a fixed rendered set when the weights are assigned
             "COMPUTE_DTYPE": "bf16",
             # not in the reference (it evaluates with is_training=True): "moving" normalises conv4_1 / conv4_2 of LSTM_test networks
             # with the moving mean / variance training tracks (TF's is_training=False); "batch" with the evaluated batch's statistics
             "BN_STATS": "batch",
             # not in the reference: True adds to each file's line of test_model the read's confidence exp(path_logprob) (the
             # probability of its best CTC alignment) and each character's peak posterior (Session.run's "read_alignment")
             "CONFIDENCE": False,
             # not in the reference (CRNN's lexicon-based transcription): a word-list file (one word per line) makes test_model read
             # each line as the most probable word (CTC score) among the LEXICON_CANDIDATES nearest words within edit distance
             # LEXICON_MAX_EDIT of the plain read (CRNN's delta = 3; < 0: no threshold); "" reads without a lexicon
             "LEXICON": "", "LEXICON_MAX_EDIT": 3, "LEXICON_CANDIDATES": 64},
}


def _defaults():
    c = AttrDict()
    for k, v in _DEFAULTS.items():
        c[k] = AttrDict(v) if isinstance(v, dict) else (list(v) if isinstance(v, list) else v)
    c.NUM_FEATURES = c.IMG_HEIGHT * c.NCHANNELS
    c.ROOT_DIR = osp.abspath(osp.join(osp.dirname(__file__), "..", "..", ".."))
    return c


cfg = _defaults()


def get_encode_decode_dict():
    """chars '0-9a-zA-Z' <-> ids 1..62; '' <-> 0 (config.py:73-81)."""
    enc = {ch: i for i, ch in enumerate(cfg.CHARSET, 1)}
    dec = {i: ch for ch, i in enc.items()}
    enc[cfg.SPACE_TOKEN] = cfg.SPACE_INDEX
    dec[cfg.SPACE_INDEX] = cfg.SPACE_TOKEN
    return enc, dec


def get_output_dir(imdb, weights_filename):
    d = osp.abspath(osp.join(cfg.ROOT_DIR, "output", cfg.EXP_DIR))
    if weights_filename is not None:
        d = osp.join(d, weights_filename)
    os.makedirs(d, exist_ok=True)
    return d


def get_log_dir(imdb):
    d = osp.abspath(osp.join(cfg.ROOT_DIR, "logs", cfg.LOG_DIR, imdb.name, strftime("%Y-%m-%d-%H-%M-%S", localtime())))
    os.makedirs(d, exist_ok=True)
    return d


def _merge(a, b, path=""):
    """Typed recursive merge with key-existence check (config.py:99-126)."""
    for k, v in a.items():
        if k not in b:
            raise KeyError(f"{path}{k} is not a valid config key")
        old = b[k]
        if isinstance(old, dict):
            if not isinstance(v, dict):
                raise ValueError(f"{path}{k}: expected a mapping")
            _merge(v, old, path + k + ".")
            continue
        if old is not None and type(old) is not type(v):
            if isinstance(old, float) and isinstance(v, int):
                v = float(v)
            else:
                raise ValueError(f"Type mismatch ({type(old)} vs. {type(v)}) for config key: {path}{k}")
        b[k] = v


def cfg_from_file(filename):
    import yaml
    with open(filename, "r") as f:
        _merge(yaml.safe_load(f) or {}, cfg)


def cfg_from_list(cfg_list):
    """``--set K V K V ...`` with literal_eval values (config.py:136-156)."""
    assert len(cfg_list) % 2 == 0
    for k, v in zip(cfg_list[0::2], cfg_list[1::2]):
        keys = k.split(".")
        d = cfg
        for sub in keys[:-1]:
            assert sub in d, f"{k} is not a valid config key"
            d = d[sub]
        assert keys[-1] in d, f"{k} is not a valid config key"
        try:
            value = literal_eval(v)
        except Exception:
            value = v
        assert type(value) is type(d[keys[-1]]), f"type {type(value)} does not match original type {type(d[keys[-1]])}"
        d[keys[-1]] = value
