"""fp64 restatements of the moving BatchNorm statistics of conv4_1 / conv4_2 (include/crnn_ctc.h, crnn_model_bind_bn_moving):
the per-step update, the fold into the conv weights and bias, and an fp64 forward that normalises with given statistics.

Every update and fold operation is one correctly rounded f64 operation, as the kernels compute them (bn_moving_update_kernel,
bn_fold_kernel, colscale_moving_kernel: explicit __d*_rn intrinsics, no fma contraction), so numpy / torch fp64 predict every
bit of the f32 and bf16 results.

Test infrastructure only (imported by tests/)."""
import numpy as np
import torch
import torch.nn.functional as F

DECAY = 0.999
EPS = float(np.float32(1e-3))          # cfg.bn_eps as the kernels read it (an f32)
LAYERS = ("conv4_1", "conv4_2")


def initial():
    """TF's initial moving statistics: [2 layers][mean, variance][512] f32, mean 0, variance 1."""
    m = np.zeros((2, 2, 512), np.float32)
    m[:, 1] = 1.0
    return m


def ema_update(moving, stats, count, decay=DECAY):
    """One training step: moving f32 [2][2][512], stats f64 [2][sum, sum of squares][512] over `count` positions ->
    the new f32 buffer.  moving -= (moving - batch value) * (1 - decay) in f64, rounded once."""
    st = np.asarray(stats, np.float64)
    mean = st[:, 0] / count
    var = np.maximum(st[:, 1] / count - mean * mean, 0.0)           # population variance
    f = 1.0 - np.float64(np.float32(decay))
    m = np.asarray(moving, np.float32).astype(np.float64)
    out = np.empty((2, 2, 512), np.float32)
    out[:, 0] = (m[:, 0] - (m[:, 0] - mean) * f).astype(np.float32)
    out[:, 1] = (m[:, 1] - (m[:, 1] - var) * f).astype(np.float32)
    return out


def bf16_rne(x):
    """Round fp64 values straight to bf16 (nearest even; normal range), returned as fp64: what cvt.rn.bf16.f64 does."""
    x = torch.as_tensor(x, dtype=torch.float64)
    m, e = torch.frexp(x)
    return torch.ldexp(torch.round(m * 256.0) / 256.0, e.to(torch.float64))


def fold(params, moving, eps=EPS):
    """{layer: dict(w=W' fp64 HWIO holding bf16 values, b=b' fp64 holding f32 values, s=s fp64 [512], w_exact=W*s fp64)}
    of the f32 parameters (TF names) and the f32 moving buffer."""
    out = {}
    mv = np.asarray(moving, np.float32).astype(np.float64)
    for l, k in enumerate(LAYERS):
        g = np.asarray(params[f"{k}/{k}/gamma"], np.float32).astype(np.float64)
        be = np.asarray(params[f"{k}/{k}/beta"], np.float32).astype(np.float64)
        b = np.asarray(params[f"{k}/biases"], np.float32).astype(np.float64)
        w = np.asarray(params[f"{k}/weights"], np.float32).astype(np.float64)
        s = g / np.sqrt(mv[l, 1] + np.float64(eps))
        ws = w * s
        out[k] = dict(w=bf16_rne(ws), w_exact=torch.as_tensor(ws), b=((b - mv[l, 0]) * s + be).astype(np.float32).astype(np.float64),
                      s=s)
    return out


def colscale_moving(colscale, s41, s42):
    """fp8: f32(colscale[2 + l] * s_l) of the [5][512] colscale table."""
    cs = np.asarray(colscale, np.float32).astype(np.float64)
    return np.stack([(cs[2] * s41).astype(np.float32), (cs[3] * s42).astype(np.float32)])


def forward(params, data, time_step_len, moving=None, folded=False, eps=EPS):
    """The oracle's fp64 forward (oracle.crnn_oracle.forward) with conv4_1 / conv4_2 normalised by the moving statistics
    `moving` [2][2][512]: unfolded, y = relu(gamma * (conv + b - mean) / sqrt(var + eps) + beta); folded=True, the exact fold
    relu(conv(x; W * s) + (b - mean) * s + beta) (no rounding).  moving=None: the oracle's batch statistics."""
    from oracle import crnn_oracle as O
    p = params
    dt = next(iter(p.values())).dtype
    x = torch.as_tensor(np.asarray(data)).to(dt)[:, None, :, :]
    mv = None if moving is None else torch.as_tensor(np.asarray(moving, np.float32)).to(dt)
    for name, kh, kw, ci, co, bn, relu, pad in O.CONV_SPECS:
        w, b = p[f"{name}/weights"], p[f"{name}/biases"]
        if bn and mv is not None:
            l = LAYERS.index(name)
            gamma, beta = p[f"{name}/{name}/gamma"], p[f"{name}/{name}/beta"]
            mean, var = mv[l, 0], mv[l, 1]
            wt = w.permute(3, 2, 0, 1)
            if folded:
                s = gamma / torch.sqrt(var + eps)
                y = F.conv2d(x, (w * s).permute(3, 2, 0, 1), (b - mean) * s + beta, padding=(kh // 2, kw // 2))
            else:
                y = F.conv2d(x, wt, b, padding=(kh // 2, kw // 2))
                y = (y - mean[None, :, None, None]) / torch.sqrt(var[None, :, None, None] + eps)
                y = y * gamma[None, :, None, None] + beta[None, :, None, None]
            x = torch.relu(y)
        else:
            x, _ = O.conv_single(x, w, b, (p[f"{name}/{name}/beta"], p[f"{name}/{name}/gamma"]) if bn else None, relu, pad)
        if name in O.POOL_AFTER:
            x = F.max_pool2d(x, O.POOL_AFTER[name], O.POOL_AFTER[name])
    N = x.shape[0]
    feat = x.permute(0, 2, 3, 1).reshape(N, -1, O.NUM_HID)
    fw = O.lstm_direction(feat, time_step_len, p[f"{O.LSTM_FW}/weights"], p[f"{O.LSTM_FW}/biases"], False)
    bw = O.lstm_direction(feat, time_step_len, p[f"{O.LSTM_BW}/weights"], p[f"{O.LSTM_BW}/biases"], True)
    logits = torch.cat([fw, bw], dim=2).reshape(-1, O.NUM_HID) @ p["logits/weights"] + p["logits/biases"]
    return logits.reshape(N, -1, O.NCLASSES).permute(1, 0, 2).contiguous()
