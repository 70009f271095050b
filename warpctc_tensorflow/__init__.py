"""Import-name shim: the reference binds its CTC operator with ``import warpctc_tensorflow`` (lib/networks/network.py:6) and
calls ``warpctc_tensorflow.ctc(activations=..., flat_labels=..., label_lengths=..., input_lengths=...)`` (network.py:653-654).
With this repository's root on ``sys.path`` that import resolves here and the call runs the sm_90a CTC kernels of
libcrnnctc.so (``lstm_ctc_ocr_b200.warpctc.ctc``: same argument names and order, ``blank_label=0`` default, costs [N];
differentiable for torch tensors the way the TF binding's registered gradient is).  No CPU fallback."""
from lstm_ctc_ocr_b200.warpctc import ctc  # noqa: F401

__all__ = ["ctc"]
