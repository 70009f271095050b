"""Drop-in for ``warpctc_tensorflow.ctc`` (the call at reference lib/networks/network.py:653-654).

    costs = ctc(activations, flat_labels, label_lengths, input_lengths, blank_label=0)

activations: [T, N, 64] f32 *unnormalised* logits (torch CUDA tensor, or numpy -> staged to the GPU);
returns costs [N] in the same container type.  With a torch tensor that requires grad the result is
differentiable: the kernel produces d cost/d logits in the same launch (as warp-ctc's op does) and the
backward is ``grad * dloss[None, :, None]`` -- the gradient the TF binding registers."""
import numpy as np
import torch

from . import engine


class _CTC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, activations, flat_labels, label_lengths, input_lengths, blank, max_label_len):
        costs, grad = engine.ctc_loss(activations.contiguous(), flat_labels, label_lengths, input_lengths, blank=blank,
                                      want_grad=True, max_label_len=max_label_len)
        ctx.save_for_backward(grad)
        return costs

    @staticmethod
    def backward(ctx, dcosts):
        (grad,) = ctx.saved_tensors
        return grad * dcosts[None, :, None], None, None, None, None, None


def _dev_i32(x, device):
    if torch.is_tensor(x):
        return x.to(device=device, dtype=torch.int32).contiguous()
    return torch.as_tensor(np.asarray(x, dtype=np.int32), device=device)


def ctc(activations, flat_labels, label_lengths, input_lengths, blank_label=0):
    as_numpy = not torch.is_tensor(activations)
    if not torch.cuda.is_available():
        raise engine.CrnnError("ctc: needs a CUDA device (sm_90a); there is no CPU fallback")
    if as_numpy:
        activations = torch.as_tensor(np.asarray(activations, dtype=np.float32), device="cuda")
    if not activations.is_cuda:
        raise engine.CrnnError("ctc: activations must live on the GPU (no CPU fallback)")
    dev = activations.device
    ll_host = label_lengths.cpu().numpy() if torch.is_tensor(label_lengths) else np.asarray(label_lengths)
    mll = int(ll_host.max()) if ll_host.size else 0
    # host-side checks the kernel cannot make (it is not told the length of flat_labels): warp-ctc reads sum(label_lengths) ids
    T, N, C = activations.shape
    n_lab = int(flat_labels.numel()) if torch.is_tensor(flat_labels) else int(np.asarray(flat_labels).size)
    if ll_host.shape != (N,) or (ll_host.size and int(ll_host.min()) < 0):
        raise ValueError("ctc: label_lengths must be [N], non-negative")
    if int(ll_host.sum()) != n_lab:
        raise ValueError(f"ctc: sum(label_lengths) = {int(ll_host.sum())} but flat_labels holds {n_lab} ids")
    if not torch.is_tensor(flat_labels) and n_lab:
        fl_host = np.asarray(flat_labels)
        if int(fl_host.min()) < 0 or int(fl_host.max()) >= C or bool((fl_host == int(blank_label)).any()):
            raise ValueError(f"ctc: label ids must lie in [0, {C}) and differ from the blank ({int(blank_label)})")
    fl, ll, il = _dev_i32(flat_labels, dev), _dev_i32(label_lengths, dev), _dev_i32(input_lengths, dev)
    if activations.requires_grad:
        costs = _CTC.apply(activations, fl, ll, il, int(blank_label), mll)
    else:
        costs, _ = engine.ctc_loss(activations.contiguous(), fl, ll, il, blank=int(blank_label), max_label_len=mll)
    return costs.cpu().numpy() if as_numpy else costs
