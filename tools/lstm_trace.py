"""Timeline of the persistent LSTM kernel (debug): CRNN_LSTM_TRACE=1 makes crnn_forward print clock64 stamps of CTAs 0 and 5
for steps 8..11 to stderr, one line per (CTA, warpgroup slot, step), in clocks since the CTA's earliest stamp.
lstm_mc_kernel: slot wg0 / wg1 = the MMA warpgroup of row half 0 / 1; events 5 xproj loads issued, 3 h_{s-1} landed
(the half's mbarrier), 4 MMAs done, 7 cell done, 8 h slice stored, 9 exchange issued, 10 output / saved-state stores issued.
Usage: python tools/lstm_trace.py [N] [W]"""
import os
import sys

os.environ["CRNN_LSTM_TRACE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from lstm_ctc_ocr_b200 import engine, synthetic  # noqa: E402

N = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
W = int(sys.argv[2]) if len(sys.argv) > 2 else 256
dev = torch.device("cuda:0")
m = engine.CrnnModel(device=dev)
m.load_params(synthetic.init_params(3))
data, lab, ll, tsl = synthetic.synth_batch(N, W, seed=3)
d, t = torch.tensor(data, device=dev), torch.tensor(tsl, device=dev)
for _ in range(2):
    m.forward(d, t)
torch.cuda.synchronize()
