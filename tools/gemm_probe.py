"""Micro-probe: plain wgmma GEMM throughput vs operand bytes per MMA cycle (is the conv mainloop L2-feed-bound?)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lstm_ctc_ocr_b200 import engine  # noqa: E402

dev = torch.device("cuda:0")
SKIP = os.environ.get('CRNN_PROBE_SKIP_TMA') == '1'
for (M, Nc, K, bn) in [(8192, 8192, 8192, 256), (8192, 8192, 8192, 128), (8192, 8192, 8192, 64), (262144, 512, 4608, 256), (262144, 512, 2304, 256),
                       (16384, 256, 8192, 256)]:
    A = torch.randn(M, K, device=dev).to(torch.bfloat16)
    B = torch.randn(Nc, K, device=dev).to(torch.bfloat16)
    for _ in range(2):
        D = engine.test_gemm_bf16(A, B, bn)
    torch.cuda.synchronize()
    if M <= 8192 and not SKIP:
        ref = A.float() @ B.float().t()
        print('   rel_err', float((D - ref).abs().max() / ref.abs().max()), flush=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        engine.test_gemm_bf16(A, B, bn)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    tiles = ((M + 127) // 128) * (Nc // bn)
    bytes_l2 = tiles * (K // 64) * (16384 + bn * 128)
    print(f"M={M} N={Nc} K={K} BLOCK_N={bn}: {ms:.3f} ms  {2.0*M*Nc*K/ms/1e9:.0f} TFLOP/s  smem-feed {bytes_l2/ms/1e9:.2f} TB/s (+ f32 D write {M*Nc*4/ms/1e9:.2f} TB/s)", flush=True)
    del A, B
