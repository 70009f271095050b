"""GPU diagnostic: per-stage error of the CUDA path against the oracle."""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lstm_ctc_ocr_b200 import engine  # noqa: E402
from oracle import crnn_oracle as O  # noqa: E402


def rel(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def main():
    dev = torch.device("cuda:0")
    print(torch.cuda.get_device_name(0))
    # ---- GEMM
    for bn, (M, Nc, K) in [(64, (300, 64, 512)), (128, (1000, 256, 576)), (256, (4096, 512, 2304))]:
        g = torch.Generator(device="cpu").manual_seed(bn)
        A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).to(dev)
        B = (torch.randn(Nc, K, generator=g) * 0.5).to(torch.bfloat16).to(dev)
        D = engine.test_gemm_bf16(A, B, bn)
        torch.cuda.synchronize()
        ref = A.float() @ B.float().t()
        print(f"gemm bn={bn} M={M} Nc={Nc} K={K} rel_err={rel(D.cpu(), ref.cpu()):.3e}", flush=True)
    # ---- CTC
    T, N = 24, 37
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((T, N, 64)) * 2).astype(np.float32)
    ll = rng.integers(1, 8, size=N).astype(np.int32); il = rng.integers(12, T + 1, size=N).astype(np.int32)
    ll[3] = 14; il[3] = 10      # infeasible
    lab = rng.integers(1, 63, size=int(ll.sum())).astype(np.int32)
    lab[1] = lab[0]
    costs_o, grad_o = O.ctc_loss_np(x, lab, ll, il)
    c, g = engine.ctc_loss(torch.tensor(x, device=dev), torch.tensor(lab, device=dev), torch.tensor(ll, device=dev),
                           torch.tensor(il, device=dev), want_grad=True)
    torch.cuda.synchronize()
    print("ctc costs rel", rel(c.cpu(), costs_o), "grad abs", float(np.abs(g.cpu().numpy() - grad_o).max()), flush=True)
    out, out_len = engine.ctc_greedy(torch.tensor(x, device=dev), torch.tensor(il, device=dev))
    dec_o = O.greedy_decode(x, il)
    dec = [out[i, :int(out_len[i])].cpu().tolist() for i in range(N)]
    print("greedy equal:", dec == dec_o, flush=True)
    # ---- forward, stage by stage
    for (N, W, widths) in [(4, 88, [88, 85, 60, 33]), (3, 100, None)]:
        pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
        data, lab, ll, tsl = O.synth_batch(N, W, seed=5, widths=widths)
        m = engine.CrnnModel()
        m.load_params(pn)
        t0 = time.time()
        logits = m.forward(torch.tensor(data, device=dev), torch.tensor(tsl, device=dev))
        torch.cuda.synchronize()
        print(f"forward N={N} W={W} ok in {time.time()-t0:.2f}s", flush=True)
        lo, acts = O.forward(O.to_torch(pn), data, tsl, return_all=True)
        T = W // 4 - 1
        for name in ["conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2"]:
            ref = acts[name].permute(0, 2, 3, 1).numpy()            # NCHW -> NHWC
            got = m.tap(name, N, W).cpu().numpy()
            print(f"  {name:8s} rel_err={rel(got, ref):.3e}  shape={got.shape}", flush=True)
        got = m.tap("conv5", N, W).cpu().numpy()[:, :T]
        print(f"  conv5    rel_err={rel(got, acts['reshaped_layer'].numpy()):.3e}")
        got = m.tap("lstm_out", N, W).cpu().numpy()[:, :T]
        print(f"  lstm_out rel_err={rel(got, acts['lstm_out'].numpy()):.3e}")
        print(f"  logits   rel_err={rel(logits.cpu().numpy(), lo.numpy()):.3e}  max|logit|={float(lo.abs().max()):.3f}", flush=True)
        costs, _ = engine.ctc_loss(logits, torch.tensor(lab, device=dev), torch.tensor(ll, device=dev), torch.tensor(tsl, device=dev))
        co, _ = O.ctc_loss_np(lo.numpy(), lab, ll, tsl)
        loss = m.total_loss(costs)
        lo_loss = co.mean() + float(O.l2_reg(O.to_torch(pn), 1e-5))
        print(f"  ctc costs rel={rel(costs.cpu(), co):.3e} loss={float(loss):.6f} oracle={lo_loss:.6f}", flush=True)
        del m


if __name__ == "__main__":
    main()
