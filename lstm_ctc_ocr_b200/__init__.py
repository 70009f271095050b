"""H100-native (sm_90a) CRNN+CTC hot path behind the model/solver API of ilovin/lstm_ctc_ocr."""
from ._lib import CrnnError, LIB_PATH  # noqa: F401
