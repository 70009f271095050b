"""fp64 restatements of every stage of the bf16 forward and backward path, each on that stage's OWN inputs.

A stage function takes the operands the kernel reads (bf16 activations / gradients read back from the workspace, weights
rounded to bf16 as prepare_weights() rounds them, f32 biases) as fp64 tensors, on any one device, in the workspace layouts (NHWC, permuted
LSTM gate columns, reversed backward-direction rows, time-major logits) and returns the stage's output computed in fp64.
With the kernel's own inputs the only legitimate differences are the order of the f32 accumulation and the final rounding,
so a test can bound each element by about one bf16 ulp plus a small multiple of `acc`: the same operation applied to
|inputs| and |weights|, i.e. the scale the accumulation error is relative to.

Data and weight gradients are written as tiny fp64 torch functions differentiated by torch.autograd.grad with the GPU's own
upstream gradient as grad_outputs; `acc` is the same vector-Jacobian product on absolute values.  The BatchNorm backwards
are written out, so that a batch can be evaluated in image chunks: their batch sums (bn_sums, bn_bwd_sums) add over chunks.

`rnd` is the rounding the kernels apply INSIDE a stage (the bf16 h a recurrence step exchanges, the bf16 values the pool3
backward compares).  The GPU tests pass `bf16`; tests/test_stage_refs_cpu.py passes `ident` and chains the stages from the
oracle's fp64 activations, which must then reproduce the oracle's forward and gradients.

The f32-class paths (csrc/forward_x3.cu) use the same functions.  Their split-bf16 operands enter as (hi, lo) pairs
(`split`): wherever an activation and a weight are both pairs, the linear part of a stage is the split-operand product
ah*wh + al*wh + ah*wl that the kernels' virtual K = [hi | lo | hi] against [wh | wh | wl] computes, evaluated in fp64, so
the one dropped term al*wl is left out of the reference as well.  tf32 operands enter as plain values rounded by
`tf32_rna`.  `x3=True` selects the recurrence layout of that path: an input projection without bias in natural gate order
and natural frame order, the bias (+1 on f) added by the cell, the backward direction reading frame len-1-step.

Test infrastructure only (imported by tests/)."""
import numpy as np
import torch
import torch.nn.functional as F

HID = 256
UPC = 32            # hidden units per [i|j|f|o] column group of the permuted LSTM layout (lstm_perm in kernels.cu)


def bf16(x):
    """Round to bf16 the way the kernels do (f32 value, then round-to-nearest-even)."""
    return x.float().to(torch.bfloat16).double()


def f32(x):
    return x.float().double()


def ident(x):
    return x


# ---------------------------------------------------------------------------------------------------------- operands
def split(x):
    """(hi, lo) of the f32 value of x as forward_x3.cu's split2 stores it: hi = bf16 round-to-nearest-even of x, lo = bf16
    round-to-nearest-even of the f32 difference x - hi (exact in f32)."""
    x32 = x.float()
    hi = x32.to(torch.bfloat16)
    lo = (x32 - hi.float()).to(torch.bfloat16)
    return hi.double(), lo.double()


def split_value(x):
    """The value a split-stored x carries: hi + lo."""
    hi, lo = split(x)
    return hi + lo


def tf32_rna(x):
    """Round the f32 value of x to tf32 (10 explicit mantissa bits), nearest with ties away from zero
    (cvt.rna.tf32.f32): add half of the dropped 13-bit field to the magnitude bits, then clear the field."""
    u = x.float().contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (u & 0x80000000) | (((u & 0x7FFFFFFF) + 0x1000) & 0xFFFFE000)
    r = torch.where(r >= 2 ** 31, r - 2 ** 32, r)                 # back to the int32 bit pattern
    return r.to(torch.int32).view(torch.float32).double()


def is_pair(x):
    return isinstance(x, tuple)


def pair_value(x):
    return x[0] + x[1] if is_pair(x) else x


def pair_map(fn, x):
    """fn applied to a value or to both halves of a pair (slicing, reshaping, gathering)."""
    return (fn(x[0]), fn(x[1])) if is_pair(x) else fn(x)


def bilinear(fn, x, w):
    """fn(x, w) in fp64 for a bilinear fn (conv, matmul), and acc = fn(|x|, |w|).  If either operand is a (hi, lo) pair the
    result is the split-operand product fn(xh, wh) + fn(xl, wh) + fn(xh, wl) (a plain value counts as (value, 0))."""
    if not (is_pair(x) or is_pair(w)):
        return fn(x, w), fn(x.abs(), w.abs())
    xh, xl = x if is_pair(x) else (x, None)
    wh, wl = w if is_pair(w) else (w, None)
    y = fn(xh, wh if wl is None else wh + wl)           # xh*wh + xh*wl in one pass (wh + wl is exact in fp64)
    if xl is not None:
        y = y + fn(xl, wh)
    return y, fn(pair_value(x).abs() if xl is None else xh.abs() + xl.abs(),
                 pair_value(w).abs() if wl is None else wh.abs() + wl.abs())


def nchw(x):
    return x.permute(0, 3, 1, 2)


def nhwc(x):
    return x.permute(0, 2, 3, 1)


# ---------------------------------------------------------------------------------------------------------- layouts
def gate_perm(upc=UPC, device=None):
    """TF gate column j = g*256 + u  ->  its column in the permuted [1024] layout (kernels.cu: lstm_perm)."""
    j = torch.arange(4 * HID, device=device)
    g, u = j // HID, j % HID
    return (u // upc) * 4 * upc + g * upc + u % upc


def to_perm(z):
    """[..., 1024] TF gate order -> permuted column order."""
    out = torch.empty_like(z)
    out[..., gate_perm(device=z.device)] = z
    return out


def from_perm(z):
    """[..., 1024] permuted column order -> TF gate order."""
    return z[..., gate_perm(device=z.device)]


def clamp_lens(lens, T):
    return [min(max(int(v), 0), T) for v in lens]


def reverse_rows(x, lens, T):
    """tf.reverse_sequence over axis 1 of [N, H2, C]: row t < len goes to len-1-t, rows t >= len stay (an involution)."""
    L = torch.as_tensor(clamp_lens(lens, T), device=x.device)[:, None]
    t = torch.arange(x.shape[1], device=x.device)[None, :]
    src = torch.where(t < L, L - 1 - t, t)
    return torch.gather(x, 1, src[..., None].expand(x.shape))


def step_h(lstm_out, lens, T):
    """The h each recurrence step wrote, from lstm_out [N, H2, 512]: [2 dirs, N, T steps, 256], step s of the backward
    direction at frame len-1-s (rows of steps >= len meaningless)."""
    N = lstm_out.shape[0]
    L = torch.as_tensor(clamp_lens(lens, T), device=lstm_out.device)
    out = []
    for d in range(2):
        t = _step_frames(L[:, None], torch.arange(T, device=lstm_out.device)[None, :], d)
        out.append(torch.gather(lstm_out[..., d * HID:(d + 1) * HID], 1, t[..., None].expand(N, T, HID)))
    return torch.stack(out)


def unpack_gates(g, N):
    """Workspace `gates` [2*tiles, T, 4, 32, 128, 8] (common.cuh: lstm_gate_off) -> [2 dirs, N, T steps, 4 gates, 256]."""
    tiles = g.shape[0] // 2
    T = g.shape[1]
    return g.reshape(2, tiles, T, 4, 32, 128, 8).permute(0, 1, 5, 2, 3, 4, 6).reshape(2, tiles * 128, T, 4, HID)[:, :N]


def pack_gates(g, Npad):
    """Inverse of unpack_gates (rows past N zero)."""
    _, N, T, _, _ = g.shape
    full = g.new_zeros((2, Npad, T, 4, HID))
    full[:, :N] = g
    return full.reshape(2, Npad // 128, 128, T, 4, 32, 8).permute(0, 1, 3, 4, 5, 2, 6).reshape(2 * Npad // 128, T, 4, 32, 128, 8)


def unpack_csave(c, N):
    """Workspace `csave` [2*tiles, T, 64, 128, 4] (common.cuh: lstm_c_off) -> [2 dirs, N, T steps, 256]."""
    tiles = c.shape[0] // 2
    T = c.shape[1]
    return c.reshape(2, tiles, T, 64, 128, 4).permute(0, 1, 4, 2, 3, 5).reshape(2, tiles * 128, T, HID)[:, :N]


def pack_csave(c, Npad):
    _, N, T, _ = c.shape
    full = c.new_zeros((2, Npad, T, HID))
    full[:, :N] = c
    return full.reshape(2, Npad // 128, 128, T, 64, 4).permute(0, 1, 3, 4, 2, 5).reshape(2 * Npad // 128, T, 64, 128, 4)


# ---------------------------------------------------------------------------------------------------------- helpers
def _conv(x, w_hwio, b=None, padding=1):
    """NHWC x HWIO -> NHWC (fp64), SAME for 3x3 (padding 1), VALID for padding 0."""
    return nhwc(F.conv2d(nchw(x), w_hwio.permute(3, 2, 0, 1), b, padding=padding))


def _conv_acc(x, w, b, padding=1):
    """conv + bias and its accumulation scale; x and w may be split (hi, lo) pairs (see `bilinear`)."""
    y, acc = bilinear(lambda a, k: _conv(a, k, None, padding), x, w)
    if b is not None:
        y, acc = y + b, acc + b.abs()
    return y, acc


def pool22(x):
    """2x2 max pool of NHWC [N, H, W, C] -> (max, first arg-max dy*2+dx)."""
    N, H, W, C = x.shape
    v = x.reshape(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(N, H // 2, W // 2, C, 4)
    return v.max(dim=-1).values, first_argmax(v)


def pool12(x):
    """1x2 max pool over the W axis of NHWC [N, H, W, C] -> (max, first arg-max dx)."""
    N, H, W, C = x.shape
    v = x.reshape(N, H, W // 2, 2, C).permute(0, 1, 2, 4, 3)
    m, _ = v.max(dim=-1)
    return m, first_argmax(v)


def first_argmax(v):
    """Index of the FIRST maximum along the last axis."""
    m = v.max(dim=-1, keepdim=True).values
    k = v.shape[-1]
    idx = torch.arange(k, device=v.device).expand_as(v)
    return torch.where(v == m, idx, torch.full_like(idx, k)).min(dim=-1).values


def windows22(x):
    """The four values of each 2x2 window of NHWC x, window index dy*2+dx last: [N, H/2, W/2, C, 4]."""
    N, H, W, C = x.shape
    return x.reshape(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(N, H // 2, W // 2, C, 4)


def windows12(x):
    N, H, W, C = x.shape
    return x.reshape(N, H, W // 2, 2, C).permute(0, 1, 2, 4, 3)


def vjp(fn, inputs, dy):
    """fp64 autograd: gradients of fn(*inputs) w.r.t. every input, with dy as grad_outputs."""
    xs = [t.detach().clone().requires_grad_(True) for t in inputs]
    return [g.detach() if g is not None else None for g in torch.autograd.grad(fn(*xs), xs, dy, allow_unused=True)]


def vjp_acc(fn, inputs, dy):
    """(gradients, accumulation scale): the same vector-Jacobian product on |inputs| and |dy| (fn must be multilinear)."""
    return vjp(fn, inputs, dy), vjp(fn, [t.abs() for t in inputs], dy.abs())


# ---------------------------------------------------------------------------------------------------------- forward stages
def conv1_stage(data, w, b):
    """conv1 (3x3 SAME, Cin 1) + bias + ReLU + 2x2 pool.  data [N, W, 32] and w, b as f32 values (the kernel's split-bf16
    operands drop only the lo*lo term).  Returns out [N, W/2, 16, 64], acc, pre (conv + bias before ReLU), am."""
    x = data[..., None]
    pre, acc = _conv_acc(x, w, b)
    out, am = pool22(torch.relu(pre))
    return dict(out=out, acc=windows22(acc).max(-1).values, pre=pre, am=am)


def conv_relu_pool22_stage(x, w, b):
    """conv2: 3x3 SAME + bias + ReLU + 2x2 pool."""
    pre, acc = _conv_acc(x, w, b)
    out, am = pool22(torch.relu(pre))
    return dict(out=out, acc=windows22(acc).max(-1).values, pre=pre, am=am)


def conv_relu_stage(x, w, b):
    """conv3_1: 3x3 SAME + bias + ReLU."""
    pre, acc = _conv_acc(x, w, b)
    return dict(out=torch.relu(pre), acc=acc, pre=pre)


def conv_relu_pool12_stage(x, w, b):
    """conv3_2: 3x3 SAME + bias + ReLU + 1x2 pool over the image-height axis."""
    pre, acc = _conv_acc(x, w, b)
    out, am = pool12(torch.relu(pre))
    return dict(out=out, acc=windows12(acc).max(-1).values, pre=pre, am=am)


def conv_bias_stage(x, w, b):
    """conv4_x GEMM (EPI_STATS): 3x3 SAME + bias, the pre-BatchNorm activation."""
    out, acc = _conv_acc(x, w, b)
    return dict(out=out, acc=acc)


def bn_sums(x_pre):
    """The batch sums BatchNorm statistics come from, additive over image chunks: sum, sum of squares and sum of |x| per
    channel over every position of x_pre [N, H2, 4, C], and the count."""
    x = x_pre.reshape(-1, x_pre.shape[-1])
    return dict(sum=x.sum(0), sumsq=(x * x).sum(0), sum_acc=x.abs().sum(0), cnt=x.shape[0])


def bn_stats_stage(x_pre, gamma, beta, eps, sums=None, parts=None):
    """Batch statistics over every position of x_pre [N, H2, 4, C] (kernels.cu: bn_finalize_kernel): sums, mean, population
    variance, invstd, scale = gamma*invstd, shift = beta - mean*scale.  sums = (sum, sum of squares): finalize those (the
    workspace's own f64 sums) instead of x_pre's; the error scales still come from x_pre.  parts = bn_sums() added over
    the image chunks of a batch stands for x_pre's (x_pre is then not read)."""
    p = bn_sums(x_pre) if parts is None else parts
    cnt = p["cnt"]
    s1, s2 = (p["sum"], p["sumsq"]) if sums is None else sums
    mean = s1 / cnt
    var = (s2 / cnt - mean * mean).clamp_min(0)
    invstd = 1.0 / torch.sqrt(var + eps)
    scale = gamma * invstd
    # error scales of the coefficients derived from (slightly perturbed) sums: the mean cancels down from sum|x| / cnt, the
    # variance E[x^2] - mean^2 amplifies relative errors of the sums by E[x^2] / var, and the shift cancels beta against
    # mean * scale
    mean_acc = p["sum_acc"] / cnt
    cond = (s2 / cnt) / (var + eps)
    acc = dict(mean=mean_acc, invstd=invstd.abs() * cond, scale=scale.abs() * cond,
               shift=beta.abs() + scale.abs() * (mean_acc + mean.abs() * cond))
    return dict(sum=s1, sumsq=s2, sum_acc=p["sum_acc"], mean=mean, var=var, invstd=invstd, scale=scale,
                shift=beta - mean * scale, acc=acc)


def bn_apply_relu_stage(x_pre, scale, shift):
    """max(x*scale + shift, 0) with the workspace's f32 scale / shift."""
    y = x_pre * scale + shift
    return dict(out=torch.relu(y), acc=(x_pre * scale).abs() + shift.abs())


def bn_apply_relu_pool_stage(x_pre, scale, shift, rnd=bf16):
    """pool3: max over image-height pairs of rnd(max(x*scale + shift, 0)) (the pair is compared after the per-position
    rounding, kernels.cu: bn_apply_relu_pool12_kernel)."""
    y = torch.relu(x_pre * scale + shift)
    out, _ = pool12(rnd(y))
    acc = windows12((x_pre * scale).abs() + shift.abs()).max(-1).values
    return dict(out=out, acc=acc)


def conv5_stage(a4b, w, b):
    """conv5: 2x2 VALID over [N, H2, 2, 512] -> [N, T, 512] (frames t < T)."""
    y, acc = _conv_acc(a4b, w, b, padding=0)
    return dict(out=y[:, :, 0, :], acc=acc[:, :, 0, :])


def _forget_one(b):
    return torch.cat([torch.zeros(2 * HID), torch.ones(HID), torch.zeros(HID)]).to(b.device, b.dtype)


def xproj_stage(a5, wx_fw, wx_bw, b_fw, b_bw, lens, T, bias_rnd=f32, x3=False):
    """Input projection of both directions for all H2 rows of a5 [N, H2, 512]: z = a5 Wx + b (+1 on the forget gate, added
    in f32 by lstm_bias_prep: `bias_rnd`), gate columns permuted, backward-direction rows reversed by length (rows t >= len,
    the padding row t = T included, stay).  x3: z = a5 Wx only (the f32-class cell adds the bias), natural [i|j|f|o]
    columns and frame order in both directions; a5 and the weights may be split pairs."""
    outs, accs = [], []
    for d, (wx, b) in enumerate(((wx_fw, b_fw), (wx_bw, b_bw))):
        if x3:
            z, acc = bilinear(torch.matmul, a5, wx)
            outs.append(z)
            accs.append(acc)
            continue
        bias = bias_rnd(b + _forget_one(b))
        z = to_perm(a5 @ wx + bias)
        acc = to_perm(a5.abs() @ wx.abs() + bias.abs())
        if d == 1:
            z, acc = reverse_rows(z, lens, T), reverse_rows(acc, lens, T)
        outs.append(z)
        accs.append(acc)
    return dict(out=torch.cat(outs, -1), acc=torch.cat(accs, -1))


def _cell(z, c_prev):
    i, j, f, o = torch.sigmoid(z[..., :HID]), torch.tanh(z[..., HID:2 * HID]), torch.sigmoid(z[..., 2 * HID:3 * HID]), \
        torch.sigmoid(z[..., 3 * HID:])
    c = f * c_prev + i * j
    return torch.stack([i, j, f, o], -2), c, o * torch.tanh(c)


def _step_frames(L, s, d):
    """Frame each row reads at step s (of a [N] or [N, 1] step grid): s forward, len-1-s backward (s where s >= len)."""
    return torch.where(L > s, (L - 1 - s) if d else s + 0 * L, s + 0 * L)


def recurrence_stage(xproj, wh_fw, wh_bw, lens, T, rnd=bf16, biases=None):
    """Both LSTM directions over T steps from the projected inputs `xproj` (workspace layout) and W_h [256, 1024]; h is
    rounded by `rnd` (to a value) before it feeds the next step.  Returns lstm_out [N, H2, 512] (frames t >= len and the
    padding row zero), gates [2, N, T, 4, 256] and c [2, N, T, 256] per STEP (valid for steps < len).
    biases = (b_fw, b_bw) selects the x3 layout (xproj_stage(x3=True)): the step adds the bias and 1 on f itself and reads
    the xproj row of its own frame; W_h may then be a split pair."""
    N, H2, _ = xproj.shape
    L = torch.as_tensor(clamp_lens(lens, T), device=xproj.device)
    out = xproj.new_zeros((N, H2, 2 * HID))
    gates = xproj.new_zeros((2, N, T, 4, HID))
    cs = xproj.new_zeros((2, N, T, HID))
    ar = torch.arange(N, device=xproj.device)
    for d, wh in enumerate((wh_fw, wh_bw)):
        xd = xproj[..., d * 1024:(d + 1) * 1024]
        if biases is None:
            xd = from_perm(xd)
        h = xproj.new_zeros((N, HID))
        c = xproj.new_zeros((N, HID))
        for s in range(T):
            act = (s < L)[:, None]
            t = _step_frames(L, s, d)
            if biases is None:
                z = xd[:, s] + h @ wh
            else:
                z = xd[ar, t] + bilinear(torch.matmul, h, wh)[0] + biases[d] + _forget_one(biases[d])
            g, c_new, h_new = _cell(z, c)
            gates[d, :, s] = g
            cs[d, :, s] = c_new
            sel = (s < L)
            out[ar[sel], t[sel], d * HID:(d + 1) * HID] = h_new[sel]
            c = torch.where(act, c_new, c)
            h = torch.where(act, rnd(h_new), h)
    return dict(out=out, gates=gates, c=cs)


def recurrence_steps_isolated(xproj, wh_fw, wh_bw, lstm_out, c_steps, lens, T, biases=None):
    """Every recurrence step on its own inputs: z = xproj row + h_prev W_h with h_prev the step's predecessor read back from
    `lstm_out` (the bf16 h the kernel exchanged) and c_prev from the saved cell state `c_steps` [2, N, T, 256].  Returns
    gates / c [2, N, T, ...] and h [2, N, T, 256] per step (rows of steps >= len meaningless).
    biases = (b_fw, b_bw): the x3 layout (see recurrence_stage); lstm_out and W_h may be split pairs.  c_steps = None
    (the f32-class path saves no per-step cell state): c is carried in fp64 from step to step, teacher-forced by h only."""
    N = xproj.shape[0]
    L = torch.as_tensor(clamp_lens(lens, T), device=xproj.device)
    gates = xproj.new_zeros((2, N, T, 4, HID))
    cs = xproj.new_zeros((2, N, T, HID))
    hs = xproj.new_zeros((2, N, T, HID))
    s = torch.arange(T, device=xproj.device)
    for d, wh in enumerate((wh_fw, wh_bw)):
        # frame of step s, and of its predecessor s-1 (h_prev = 0 at s = 0)
        t_of = (L[:, None] - 1 - s[None, :]).clamp_min(0) if d else s[None, :].expand(N, T)
        if biases is None:
            xd = from_perm(xproj[:, :T, d * 1024:(d + 1) * 1024])                 # [N, T(step), 1024]
        else:
            xd = torch.gather(xproj[..., d * 1024:(d + 1) * 1024], 1, t_of[..., None].expand(N, T, 4 * HID))
            xd = xd + biases[d] + _forget_one(biases[d])
        def prev_h(out_d):
            """h of each step's predecessor from this direction's lstm_out columns [N, H2, 256] (zero at step 0)."""
            h = xproj.new_zeros((N, T, HID))
            if T > 1:
                h[:, 1:] = torch.gather(out_d, 1, t_of[:, :-1, None].expand(N, T - 1, HID))
            return h

        h_prev = pair_map(lambda v: prev_h(v[..., d * HID:(d + 1) * HID]), lstm_out)   # a pair stays a pair
        c_prev = xproj.new_zeros((N, T, HID))
        if T > 1 and c_steps is not None:
            c_prev[:, 1:] = c_steps[d, :, :-1]
        z = xd + bilinear(torch.matmul, h_prev, wh)[0]
        if c_steps is not None:
            g, c, h = _cell(z, c_prev)
        else:
            c = xproj.new_zeros((N, HID))
            g, cc, h = [], [], []
            for k in range(T):
                gk, c, hk = _cell(z[:, k], c)
                g.append(gk); cc.append(c); h.append(hk)
            g, c, h = torch.stack(g, 1), torch.stack(cc, 1), torch.stack(h, 1)
        gates[d], cs[d], hs[d] = g, c, h
    return dict(gates=gates, c=cs, h=hs)


def logits_stage(lstm_out, wl, bl, T):
    """512 -> 64 projection of frames t < T, time-major [T, N, 64] (frames past len see zero rows: the bias alone)."""
    y, acc = bilinear(torch.matmul, pair_map(lambda v: v[:, :T], lstm_out), wl)
    y, acc = y + bl, acc + bl.abs()
    return dict(out=y.permute(1, 0, 2), acc=acc.permute(1, 0, 2))


# ---------------------------------------------------------------------------------------------------------- backward stages
def dl_rows_stage(dlogits, H2):
    """dlogits [T, N, 64] (time-major) -> frame rows [N, H2, 64] (padding row t = T zero) and the logits bias gradient."""
    T, N, _ = dlogits.shape
    rows = dlogits.new_zeros((N, H2, 64))
    rows[:, :T] = dlogits.permute(1, 0, 2)
    return dict(dl_rows=rows, dbias=dlogits.sum((0, 1)), dbias_acc=dlogits.abs().sum((0, 1)))


def logits_bwd(lstm_out, dl_rows, wl):
    """From the frame rows of d logits: the 512 -> 64 weight gradient and d_lstm_out."""
    (dx, dw), (ax, aw) = vjp_acc(lambda x, w: x @ w, [lstm_out, wl], dl_rows)
    return dict(dw=dw, dw_acc=aw, d_lstm_out=dx, d_lstm_out_acc=ax)


def bptt_stage(d_out, gates, c_steps, wh_fw, wh_bw, lens, T, dz_in=None, rnd=bf16):
    """Backward recurrence of both directions.  gates [2, N, T, 4, 256] / c_steps [2, N, T, 256] are the saved per-step
    values, d_out [N, H2, 512] the gradient w.r.t. lstm_out.  dz of step s+1 enters step s through W_h^T: taken from
    `dz_in` (the workspace's dz_all: the bf16 values the kernel exchanged) when given, else rnd(own result).
    Returns dz_all [N, H2, 2048] in frame order with permuted gate columns (zero for frames >= len), and the cell gradient
    dc of every step [2, N, T, 256] (zero for steps >= len)."""
    N, H2, _ = d_out.shape
    L = torch.as_tensor(clamp_lens(lens, T), device=d_out.device)
    dz_all = d_out.new_zeros((N, H2, 2048))
    dcs = d_out.new_zeros((2, N, T, HID))
    ar = torch.arange(N, device=d_out.device)
    for d, wh in enumerate((wh_fw, wh_bw)):
        dz_next = d_out.new_zeros((N, 1024))
        dc_next = d_out.new_zeros((N, HID))
        f_next = d_out.new_zeros((N, HID))
        for s in range(T - 1, -1, -1):
            act = s < L
            t = torch.where(act, (L - 1 - s) if d else torch.full_like(L, s), torch.full_like(L, s))
            i, j, f, o = gates[d, :, s].unbind(-2)
            c = c_steps[d, :, s]
            c_prev = c_steps[d, :, s - 1] if s > 0 else torch.zeros_like(c)
            dh = d_out[ar, t, d * HID:(d + 1) * HID] + dz_next @ wh.t()
            tc = torch.tanh(c)
            dc = dc_next * f_next + dh * o * (1 - tc * tc)
            dz = torch.cat([dc * j * i * (1 - i), dc * i * (1 - j * j), dc * c_prev * f * (1 - f), dh * tc * o * (1 - o)], -1)
            m = act[:, None]                 # select, never multiply: saved gates of inactive steps are never written
            zero = dz.new_zeros(())
            dz = torch.where(m, dz, zero)
            dz_all[ar[act], t[act], d * 1024:(d + 1) * 1024] = to_perm(dz)[act]
            if dz_in is not None:
                dz_next = torch.where(m, from_perm(dz_in[ar, t, d * 1024:(d + 1) * 1024]), zero)
            else:
                dz_next = rnd(dz)
            dc_next, f_next = torch.where(m, dc, zero), torch.where(m, f, zero)
            dcs[d, :, s] = dc_next
    return dict(dz=dz_all, dc=dcs)


# tanh.approx.f32 (ptx.cuh: fast_tanh): the PTX ISA states a maximum relative error of 2^-10.987 for the .f32 type
D_TANH = 2.0 ** -10.987
# The f32 accumulation of one 128-deep partial product of the BPTT exchange: 8 wgmma k-steps, each losing at most one f32
# ulp of the partial sum (2^-23 of acc, test_gpu_stage_isolation_batch.py), so at most 2^-20 of acc.  A partial whose fp64
# value lies within 4x that (2^-18 of acc) of a bf16 rounding midpoint is allowed to round either way.
MMA_WINDOW = 2.0 ** -18
# relative error of a value recovered from its bf16 round-to-nearest-even q: |x - q| <= 2^-8 |x| <= 2^-8 / (1 - 2^-8) |q|
R_BF16 = 2.0 ** -8 / (1.0 - 2.0 ** -8)


def ulp_bf16(x):
    """One bf16 ulp of |x| (2^(floor(log2 |x|) - 7), |x| at least 2^-126), fp64 on x's device."""
    return torch.ldexp(torch.ones_like(x), torch.frexp(x.abs().clamp_min(2.0 ** -126)).exponent - 8)


def _shift_next(x):
    """x of step s+1 at step s along axis 1 (zero at the last step)."""
    out = torch.zeros_like(x)
    out[:, :-1] = x[:, 1:]
    return out


def bptt_steps_isolated(d_out, gates, c_steps, wh_fw, wh_bw, dz_all, lens, T, rnd=bf16):
    """Every BPTT step on its own operands, the GPU's dz_all [N, H2, 2048] among them: nothing carries from step to step,
    so a wrong step fails at that step.  Step s of direction d (frame s forward, len-1-s backward; active while s < len):
      exchange  dh = d_out[frame] + sum_r rnd(p_r): p_r = the GPU's dz of step s+1 (zero when s+1 >= len) restricted to the
                permuted gate columns r*128 .. r*128+127 (rank r of the cluster) times to_perm(W_h) over those columns,
                rounded to bf16 by the rank before the f32 sum (lstm_bwd.cuh);
      o         dz_o = dh tanh(c_s) o(1-o) on the saved gates / cell state;
      carry     dc_s = dc_{s+1} f_{s+1} + dh o (1 - tanh(c_s)^2), dc_{s+1} recovered from the GPU's stored dz of step s+1
                as dz_j / (i(1-j^2)) or dz_i / (j i(1-i)), whichever factor is larger (zero at s = len-1).  Where both
                factors are zero the reference's own dc_{s+1} is carried instead, with its allowance (`fallback`);
      i, j, f   dz_i = dc j i(1-i), dz_j = dc i(1-j^2), dz_f = dc c_{s-1} f(1-f) (c_{-1} = 0).
    gates [2, N, T, 4, 256], c_steps [2, N, T, 256]: the saved per-step values; d_out [N, H2, 512].  Returns per step
    [2, N, T, 4, 256] (TF gate order i, j, f, o): dz (the reference), gpu (the GPU's dz of that step), allow (what the
    kernel's roundings the reference does not restate can move: a partial within MMA_WINDOW of a bf16 rounding midpoint
    (one ulp of it), the bf16-stored dz the carry is recovered from (R_BF16), tanh.approx (D_TANH)), acc (the same
    expressions on absolute values, the scale of the f32 arithmetic); active [2, N, T]; dc / dc_hat [2, N, T, 256] (the
    reference's dc and the dc recovered from the GPU's dz of each step), recovered / fallback [2, N, T, 256] (where the
    carry INTO a step was recovered / carried), near_midpoint [2, N, T, 256] (partials with a one-ulp allowance).
    rnd = ident: the partials are not rounded (the fp64 chain of tests/test_stage_refs_cpu.py)."""
    N = d_out.shape[0]
    dev = d_out.device
    L = torch.as_tensor(clamp_lens(lens, T), device=dev)
    s = torch.arange(T, device=dev)
    act = s[None, :] < L[:, None]                                             # [N, T]
    has_next = _shift_next(act)
    keys = ("dz", "gpu", "allow", "acc", "dc", "dc_hat", "recovered", "fallback", "near_midpoint")
    out = {k: [] for k in keys}
    a3 = act[..., None]
    for d, wh in enumerate((wh_fw, wh_bw)):
        t_of = _step_frames(L[:, None], s[None, :], d)                       # [N, T]
        zp = torch.gather(dz_all[:, :, d * 1024:(d + 1) * 1024], 1, t_of[..., None].expand(N, T, 1024))
        zp = torch.where(a3, zp, zp.new_zeros(()))                           # the GPU's dz per step, permuted columns
        # ---- exchange: the 8 ranks' partial products of dz_{s+1}, each rounded to bf16, summed
        znr = _shift_next(zp).reshape(N, T, 8, 128)
        whp = to_perm(wh).reshape(HID, 8, 128)
        p = torch.einsum("ntrk,urk->ntru", znr, whp)                          # [N, T, 8 ranks, 256 units]
        window = MMA_WINDOW * torch.einsum("ntrk,urk->ntru", znr.abs(), whp.abs())
        del znr
        near = (bf16(p - window) != bf16(p + window)) if rnd is not ident else torch.zeros_like(p, dtype=torch.bool)
        allow_x = torch.where(near, ulp_bf16(p.abs() + window), p.new_zeros(())).sum(2)
        del window
        q = rnd(p)
        del p
        rec, rec_acc = q.sum(2), q.abs().sum(2)
        del q
        dh = torch.gather(d_out[..., d * HID:(d + 1) * HID], 1, t_of[..., None].expand(N, T, HID))
        zero = dh.new_zeros(())
        dht = torch.where(a3, dh + rec, zero)
        dht_acc = torch.where(a3, dh.abs() + rec_acc, zero)
        allow_x = torch.where(a3, allow_x, zero)
        i, j, f, o = (torch.where(a3, g, zero) for g in gates[d].unbind(-2))
        c = torch.where(a3, c_steps[d], zero)
        cp = torch.zeros_like(c)
        cp[:, 1:] = c[:, :-1]
        tc = torch.tanh(c)
        # ---- o column: nothing carried
        so = o * (1 - o)
        ref_o = dht * tc * so
        allow_o = allow_x * (tc * so).abs() + D_TANH * ref_o.abs()
        acc_o = dht_acc * (tc * so).abs()
        # ---- carry: dc of step s+1 recovered from the GPU's stored dz_j / dz_i of that step
        zs = from_perm(zp)
        fi, fj = j * i * (1 - i), i * (1 - j * j)
        use_j = fj.abs() >= fi.abs()
        fac = torch.where(use_j, fj, fi)
        ok = fac != 0
        dc_hat = torch.where(ok, torch.where(use_j, zs[..., HID:2 * HID], zs[..., :HID]) / torch.where(ok, fac, 1.0), zero)
        dch_n, f_n, ok_n = _shift_next(dc_hat), _shift_next(f), _shift_next(ok)
        hn = has_next[..., None]
        rec_ok, fb = hn & ok_n, hn & ~ok_n
        carry_r = torch.where(rec_ok, dch_n * f_n, zero)
        allow_cr = R_BF16 * carry_r.abs()
        acc_cr = carry_r.abs()
        sd = 1 - tc * tc
        d_own = dht * o * sd
        allow_own = allow_x * (o * sd).abs() + 2 * D_TANH * (1 + D_TANH) * (dht * o).abs() * tc * tc
        acc_own = dht_acc * o.abs() * (1 + tc * tc)
        dc, a_dc, acc_dc = carry_r + d_own, allow_cr + allow_own, acc_cr + acc_own
        if bool(fb.any()):
            # carried where nothing can be recovered: the reference's own dc_{s+1}, its allowance times f_{s+1}; a run of k
            # such steps settles after k + 1 passes
            for _ in range(T + 1):
                nxt = (torch.where(fb, _shift_next(dc) * f_n, carry_r) + d_own,
                       torch.where(fb, _shift_next(a_dc) * f_n.abs(), allow_cr) + allow_own,
                       torch.where(fb, _shift_next(acc_dc) * f_n.abs(), acc_cr) + acc_own)
                done = all(torch.equal(x, y) for x, y in zip(nxt, (dc, a_dc, acc_dc)))
                dc, a_dc, acc_dc = nxt
                if done:
                    break
        ref, allow, acc = [], [], []
        for fc in (fi, fj, cp * f * (1 - f)):
            ref.append(dc * fc)
            allow.append(a_dc * fc.abs())
            acc.append(acc_dc * fc.abs())
        ref.append(ref_o)
        allow.append(allow_o)
        acc.append(acc_o)
        out["dz"].append(torch.stack(ref, -2))
        out["allow"].append(torch.stack(allow, -2))
        out["acc"].append(torch.stack(acc, -2))
        out["gpu"].append(zs.reshape(N, T, 4, HID))
        out["dc"].append(torch.where(a3, dc, zero))
        out["dc_hat"].append(dc_hat)
        out["recovered"].append(rec_ok)
        out["fallback"].append(fb)
        out["near_midpoint"].append(near.sum(2) if rnd is not ident else torch.zeros_like(rec, dtype=torch.long))
    r = {k: torch.stack(v) for k, v in out.items()}
    r["active"] = act[None].expand(2, N, T)
    return r


def lstm_grads_stage(dz_all, a5, lstm_out, wx_fw, wx_bw, wh_fw, wh_bw):
    """Weight / bias gradients of both LSTM cells ([768, 1024] = [W_x; W_h], TF column order) and d_a5 = sum_dir dz W_x^T.
    h_prev of frame t is frame t-1 (forward) / t+1 (backward) of lstm_out, zero past the ends."""
    out = {}
    d_a5 = torch.zeros_like(a5)
    d_a5_acc = torch.zeros_like(a5)
    for d, (wx, wh) in enumerate(((wx_fw, wh_fw), (wx_bw, wh_bw))):
        dz = from_perm(dz_all[..., d * 1024:(d + 1) * 1024])
        ho = lstm_out[..., d * HID:(d + 1) * HID]
        hp = torch.zeros_like(ho)
        if d == 0:
            hp[:, 1:] = ho[:, :-1]
        else:
            hp[:, :-1] = ho[:, 1:]
        fn = lambda x, h, a, b, bias: x @ a + h @ b + bias
        (dx, _, dwx, dwh, db), (ax, _, awx, awh, ab) = vjp_acc(fn, [a5, hp, wx, wh, a5.new_zeros(1024)], dz)
        key = "fw" if d == 0 else "bw"
        out[key + "/weights"] = torch.cat([dwx, dwh], 0)
        out[key + "/weights_acc"] = torch.cat([awx, awh], 0)
        out[key + "/biases"] = db
        out[key + "/biases_acc"] = ab
        d_a5 = d_a5 + dx
        d_a5_acc = d_a5_acc + ax
    out["d_a5"] = d_a5
    out["d_a5_acc"] = d_a5_acc
    return out


def conv_bwd(dy, x, w, padding=1):
    """Data and weight gradients of a bias-free 3x3 SAME (padding 1) or 2x2 VALID (padding 0) conv, bias gradient = sum dy."""
    (dx, dw), (ax, aw) = vjp_acc(lambda a, b: _conv(a, b, None, padding), [x, w], dy)
    return dict(dx=dx, dx_acc=ax, dw=dw, dw_acc=aw, db=dy.sum((0, 1, 2)), db_acc=dy.abs().sum((0, 1, 2)))


def conv5_bwd(d_a5, a4b, w):
    """conv5 from d_a5 [N, H2, 512] (frames t < T): d_a4b, weight and bias gradients."""
    T = a4b.shape[1] - 1
    return conv_bwd(d_a5[:, :T, None, :], a4b, w, padding=0)


def bn_batch(x_pre, eps, parts=None):
    """fp64 batch mean and invstd of x_pre [N, H2, 4, C] (from bn_sums() over the whole batch when given as `parts`)."""
    p = bn_sums(x_pre) if parts is None else parts
    mean = p["sum"] / p["cnt"]
    var = (p["sumsq"] / p["cnt"] - mean * mean).clamp_min(0)
    return dict(mean=mean, invstd=1.0 / torch.sqrt(var + eps), cnt=p["cnt"])


def bn_bwd_sums(dy, dy_acc, x_pre, stats):
    """The batch reductions of a BatchNorm backward, additive over image chunks: d beta = sum dy, d gamma = sum dy*xhat
    and the same on the accumulation scale dy_acc of dy (at least |dy|)."""
    xhat = (x_pre - stats["mean"]) * stats["invstd"]
    red = (0, 1, 2)
    return dict(dbeta=dy.sum(red), dgamma=(dy * xhat).sum(red), dbeta_acc=dy_acc.sum(red),
                dgamma_acc=(dy_acc * xhat.abs()).sum(red))


def _bn_bwd(dy, dy_acc, x_pre, gamma, eps, stats, sums):
    """dx = gamma*invstd*(dy - mean(dy) - xhat*mean(dy*xhat)) with the batch statistics and sums of the whole batch (of
    dy's own images when not given), and its scale summed in absolute values.  The kernels evaluate it as A*dy + B + C*x
    with f32 coefficients (backward_kernels.cu: bn_bwd_coef_kernel), where B and C*x cancel down to the centred term; the
    2^-8 share of |B| + |C*x| lets a 2^-16 * acc bound cover their f32 rounding (2^-24)."""
    stats = bn_batch(x_pre, eps) if stats is None else stats
    sums = bn_bwd_sums(dy, dy_acc, x_pre, stats) if sums is None else sums
    mean, invstd, cnt = stats["mean"], stats["invstd"], stats["cnt"]
    xhat = (x_pre - mean) * invstd
    dx = gamma * invstd * (dy - sums["dbeta"] / cnt - xhat * (sums["dgamma"] / cnt))
    m1, m2 = sums["dbeta_acc"] / cnt, sums["dgamma_acc"] / cnt
    cx = (gamma * invstd * invstd).abs() * m2 * (x_pre.abs() + mean.abs())
    acc = (gamma * invstd).abs() * (dy_acc + m1 + xhat.abs() * m2) + 2.0 ** -8 * cx
    return dict(dx=dx, dx_acc=acc, **sums)


def bn_relu_pool_route(d_pooled, x_pre, bn, rnd=bf16):
    """The gradient at the BN4_2 output: the pooled gradient d_pooled [N, H2, 2, C] goes to the FIRST position of the pair
    whose rnd(max(x*scale+shift, 0)) is the larger (the forward rounded each position before taking the max), and only
    where that max is > 0; bn = the workspace's scale, shift."""
    yq = windows12(rnd(torch.relu(x_pre * bn[0] + bn[1])))
    first = yq[..., 0] >= yq[..., 1]
    pos = torch.maximum(yq[..., 0], yq[..., 1]) > 0
    mask = torch.stack([first & pos, ~first & pos], -1).to(x_pre.dtype)       # [N, H2, 2, C, 2]
    N, H2, W4, C = x_pre.shape
    return (d_pooled[..., None] * mask).permute(0, 1, 2, 4, 3).reshape(N, H2, W4, C)


def bn_relu_pool_bwd_stage(d_pooled, x_pre, bn, gamma, eps, rnd=bf16, stats=None, sums=None):
    """BN4_2 + ReLU + pool3 backward: x_pre [N, H2, 4, C] pre-BN, d_pooled [N, H2, 2, C], bn [4, C] = the workspace's
    scale, shift, mean, invstd.  The gradient is routed by bn_relu_pool_route; the BN itself is differentiated in fp64 with
    the statistics recomputed from x_pre.  Over image chunks of a batch, stats = bn_batch() of the whole batch and sums =
    bn_bwd_sums() added over its chunks (the dgamma / dbeta returned are then those of the whole batch)."""
    dyr = bn_relu_pool_route(d_pooled, x_pre, bn, rnd)
    return _bn_bwd(dyr, dyr.abs(), x_pre, gamma, eps, stats, sums)


def conv_relu_dgrad(dy, x_pre, bn, w, mask=None, rnd=bf16):
    """conv4_2's data gradient of dy = d_pre4b, stored as bf16 (`rnd`) and masked by conv4_1's ReLU: x*scale + shift > 0
    on the workspace's f32 scale / shift (what the forward applied) unless `mask` is given.  Returns it and its
    accumulation scale: the dgrad sum on absolute values plus one bf16 ulp of the stored gradient (its rounding may fall
    either way where the f32 and fp64 sums straddle a rounding boundary)."""
    if mask is None:
        mask = (f32(x_pre * bn[0] + bn[1]) > 0).to(x_pre.dtype)
    (g,), (g_abs,) = vjp_acc(lambda a: _conv(a, w), [torch.zeros_like(x_pre)], dy)
    g = rnd(g) * mask
    return g, g_abs * mask + 2.0 ** 9 * g.abs()


def conv_bn_relu_bwd_stage(dy, x_pre, bn, gamma, w, eps, mask=None, rnd=bf16, stats=None, sums=None):
    """conv4_2 data gradient + conv4_1's ReLU mask + BN4_1 backward as one stage (the workspace's d_pre4a is overwritten in
    place by the BN apply): x_pre [N, H2, 4, 512] pre-BN conv4_1, dy = d_pre4b, the gradient from conv_relu_dgrad; stats /
    sums as in bn_relu_pool_bwd_stage."""
    g, g_acc = conv_relu_dgrad(dy, x_pre, bn, w, mask, rnd)
    return _bn_bwd(g, g_acc, x_pre, gamma, eps, stats, sums)


def unpool_stage(d_pooled, pooled, am, win):
    """Un-pool + ReLU backward: the pooled gradient where pooled > 0, routed to window position am (dy*2+dx for the 2x2
    pool, dx for the 1x2 pool); zeros elsewhere.  Exact copies, no arithmetic."""
    g = torch.where(pooled > 0, d_pooled, torch.zeros_like(d_pooled))
    N, Hp, Wp, C = g.shape
    sel = torch.stack([(am == k).to(g.dtype) for k in range(win)], -1) * g[..., None]
    if win == 4:
        return sel.reshape(N, Hp, Wp, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(N, 2 * Hp, 2 * Wp, C)
    return sel.permute(0, 1, 2, 4, 3).reshape(N, Hp, 2 * Wp, C)


def masked_colsum(d_pooled, pooled):
    """Bias gradient of a conv followed by ReLU + max-pool: column sums of the pooled gradient where the pooled output > 0."""
    g = torch.where(pooled > 0, d_pooled, torch.zeros_like(d_pooled))
    return g.sum((0, 1, 2)), g.abs().sum((0, 1, 2))


def conv1_wgrad_stage(d_a1, a1, am1, data, w):
    """conv1 weight / bias gradient: d_a1 where a1 > 0, routed by am1 to its pre-pool position, against the f32 image."""
    g = unpool_stage(d_a1, a1, am1, 4)
    (dw,) = vjp(lambda b: _conv(data[..., None], b), [w], g)
    (aw,) = vjp(lambda b: _conv(data.abs()[..., None], b), [w.abs()], g.abs())
    return dict(dw=dw, dw_acc=aw, db=g.sum((0, 1, 2)), db_acc=g.abs().sum((0, 1, 2)))
