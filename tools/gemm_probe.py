"""Micro-probe: plain wgmma GEMM throughput vs operand bytes per MMA cycle (is the conv mainloop L2-feed-bound?).

Each BLOCK_N = 256 shape is also timed with a bf16 output (the register-side epilogue with TMA stores, EPI_BIAS_BF16 without
bias) and with the epilogue skipped (mainloop alone); the difference is the time the epilogue adds per tile."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lstm_ctc_ocr_b200 import engine  # noqa: E402

dev = torch.device("cuda:0")
SKIP = os.environ.get('CRNN_PROBE_SKIP_TMA') == '1'
SMS = torch.cuda.get_device_properties(dev).multi_processor_count


def run(A, B, bn, mode):
    os.environ['CRNN_PROBE_BF16_OUT'] = '1' if mode != 'f32' else '0'
    os.environ['CRNN_PROBE_SKIP_EPI'] = '1' if mode == 'no-epilogue' else '0'
    return engine.test_gemm_bf16(A, B, bn)


# (M, N, K, BLOCK_N): square GEMMs, then the conv4_2- and conv4_1-shaped GEMMs (262144 positions = batch 1024 x 64 x 4), the input projection
for (M, Nc, K, bn) in [(8192, 8192, 8192, 256), (8192, 8192, 8192, 128), (8192, 8192, 8192, 64), (262144, 512, 4608, 256), (262144, 512, 2304, 256),
                       (65536, 2048, 512, 256), (16384, 256, 8192, 256)]:
    A = torch.randn(M, K, device=dev).to(torch.bfloat16)
    B = torch.randn(Nc, K, device=dev).to(torch.bfloat16)
    modes = ['f32', 'bf16', 'no-epilogue'] if bn == 256 else ['f32']
    tiles = ((M + 127) // 128) * (Nc // bn)
    for mode in modes:
        for _ in range(2):
            D = run(A, B, bn, mode)
        torch.cuda.synchronize()
        if M <= 8192 and not SKIP and mode != 'no-epilogue':
            ref = A.float() @ B.float().t()
            out = D if mode == 'f32' else D.view(torch.bfloat16).reshape(-1)[:M * Nc].view(M, Nc).float()
            print('   rel_err', float((out - ref).abs().max() / ref.abs().max()), flush=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            run(A, B, bn, mode)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        bytes_l2 = tiles * (K // 64) * (16384 + bn * 128)
        us_tile = ms * 1e3 / ((tiles + SMS - 1) // SMS)
        print(f"M={M} N={Nc} K={K} BLOCK_N={bn} out={mode}: {ms:.3f} ms  {2.0*M*Nc*K/ms/1e9:.0f} TFLOP/s  {us_tile:.2f} us/tile-round  "
              f"smem-feed {bytes_l2/ms/1e9:.2f} TB/s", flush=True)
    del A, B
os.environ.pop('CRNN_PROBE_BF16_OUT', None)
os.environ.pop('CRNN_PROBE_SKIP_EPI', None)
