"""Known-answer vectors published by the two third-party projects that hold the arithmetic of the reference's loss and
decode call sites (lib/networks/network.py:653-657): TensorFlow (`tf.nn.ctc_loss`, `ctc_greedy_decoder`,
`ctc_beam_search_decoder`) and baidu-research/warp-ctc (`compute_ctc_loss`).  Neither project is vendored under
the reference checkout nor installable here (SURVEY 8(c)), so these are the only externally held numbers the path can be pinned to.

Provenance [upstream-memory -- transcribed, not fetched: there is no network]:
  * CTC_LOSS: tensorflow/python/kernel_tests/ctc_loss_op_test.py::CTCLossTest.testBasic (two 5-frame, 6-class utterances,
    blank = class 5, inputs = log of the probability matrices below, expected loss = -log p(l|x), expected gradient w.r.t. the
    unnormalised inputs).  The same matrices, costs and gradients are warp-ctc's tests/test_cpu.cpp::options_test
    ("expected_grads // from tensorflow", `options.blank_label = 5`), i.e. BOTH dependencies of network.py:653-655 pin them.
  * GREEDY: tensorflow/python/kernel_tests/ctc_decoder_ops_test.py::CTCGreedyDecoderTest.testCTCGreedyDecoder (4 classes,
    blank = class 3, merge_repeated=True; frames past seq_len ignored).
  * BEAM: same file, testCTCDecoderBeamSearch (6 classes, blank = class 5, beam_width = 2, merge_repeated: the top path the
    test pins is [1, 0] although [0, 1, 0] carries more probability mass and wins at any beam width != 2 -- a vector that
    only an implementation with TF's candidate ordering and eviction rule reproduces).
  * LSTM_CELL: tensorflow/python/kernel_tests/rnn_cell_test.py::RNNCellTest.testBasicLSTMCell (two stacked 2-unit cells, every
    weight 0.5, zero biases, forget_bias 1.0, input [1, 1], every state entry 0.1; state_is_tuple=False packs [c, h] per layer).
    Uniform weights cannot tell gate ORDER apart; they pin the cell equations and the forget bias.

  * CONV / POOL / CLIP: tensorflow/python/kernel_tests/conv_ops_test.py::testConv2D1x1Filter and ::testConv2D2x2Filter (NHWC input
    [1,2,3,3] = 1..18, HWIO filters 1..9 / 1..36, stride 1, VALID -- the layout conventions of the checkpoint's conv kernels and
    conv5's 2x2 VALID case, network.py:160-182), pooling_ops_test.py::_testMaxPoolValidPadding ([1,3,3,3] = 1..27, 2x2 / stride 2
    VALID), clip_ops_test.py::testClipByGlobalNormClipped / NotClipped (lib/lstm/train.py:82).

Self-check of the transcription: `tests/test_oracle.py::test_third_party_known_answers_*` recomputes the two losses from the
matrices with an fp64 alpha recursion and gets 3.342113 and 5.422622 -- six matching digits on values nobody could guess --
and all 60 gradient entries to 1e-6; a mis-remembered digit anywhere in a matrix would break both."""
import numpy as np

# ---- ctc_loss_op_test.py::testBasic == warp-ctc options_test --------------------------------------------------------------
CTC_BLANK = 5
CTC_PROBS = [np.asarray(
    [[0.633766, 0.221185, 0.0917319, 0.0129757, 0.0142857, 0.0260553],
     [0.111121, 0.588392, 0.278779, 0.0055756, 0.00569609, 0.010436],
     [0.0357786, 0.633813, 0.321418, 0.00249248, 0.00272882, 0.0037688],
     [0.0663296, 0.643849, 0.280111, 0.00283995, 0.0035545, 0.00331533],
     [0.458235, 0.396634, 0.123377, 0.00648837, 0.00903441, 0.00623107]], dtype=np.float64), np.asarray(
    [[0.30176, 0.28562, 0.0831517, 0.0862751, 0.0816851, 0.161508],
     [0.24082, 0.397533, 0.0557226, 0.0546814, 0.0557528, 0.19549],
     [0.230246, 0.450868, 0.0389607, 0.038309, 0.0391602, 0.202456],
     [0.280884, 0.429522, 0.0326593, 0.0339046, 0.0326856, 0.190345],
     [0.423286, 0.315517, 0.0338439, 0.0393744, 0.0339315, 0.154046]], dtype=np.float64)]
CTC_TARGETS = [[0, 1, 2, 1, 0], [0, 1, 1, 0]]
CTC_LOSS = [3.34211, 5.42262]                      # = -loss_log_prob_{0,1}
CTC_GRAD = [np.asarray(
    [[-0.366234, 0.221185, 0.0917319, 0.0129757, 0.0142857, 0.0260553],
     [0.111121, -0.411608, 0.278779, 0.0055756, 0.00569609, 0.010436],
     [0.0357786, 0.633813, -0.678582, 0.00249248, 0.00272882, 0.0037688],
     [0.0663296, -0.356151, 0.280111, 0.00283995, 0.0035545, 0.00331533],
     [-0.541765, 0.396634, 0.123377, 0.00648837, 0.00903441, 0.00623107]], dtype=np.float64), np.asarray(
    [[-0.69824, 0.28562, 0.0831517, 0.0862751, 0.0816851, 0.161508],
     [0.24082, -0.602467, 0.0557226, 0.0546814, 0.0557528, 0.19549],
     [0.230246, 0.450868, 0.0389607, 0.038309, 0.0391602, -0.797544],
     [0.280884, -0.570478, 0.0326593, 0.0339046, 0.0326856, 0.190345],
     [-0.576714, 0.315517, 0.0338439, 0.0393744, 0.0339315, 0.154046]], dtype=np.float64)]


def ctc_case(num_classes=6, blank=CTC_BLANK, pad_logit=-60.0):
    """The two utterances as one warp-ctc style call: logits [T=5, N=2, num_classes] (log of the probabilities; classes the
    vectors do not have get `pad_logit`, i.e. probability < 1e-26), flat labels, lengths, and the expected costs / gradient in
    the same class numbering.  `blank` re-numbers the classes so that TF's blank (5) lands on `blank` and TF's labels
    0..4 fill the lowest remaining ids in order (blank=0: TF label k -> k+1, the warp-ctc convention of network.py:653)."""
    ids = [c for c in range(num_classes) if c != blank][:5]
    col = ids + [blank]                                             # TF class k -> col[k]
    T, N = 5, 2
    x = np.full((T, N, num_classes), pad_logit, np.float64)
    g = np.zeros((T, N, num_classes), np.float64)
    for n in range(N):
        x[:, n, col] = np.log(CTC_PROBS[n])
        g[:, n, col] = CTC_GRAD[n]
    flat = np.asarray([col[k] for tgt in CTC_TARGETS for k in tgt], np.int32)
    label_len = np.asarray([len(t) for t in CTC_TARGETS], np.int32)
    input_len = np.asarray([T, T], np.int32)
    return x, flat, label_len, input_len, np.asarray(CTC_LOSS), g


# ---- ctc_decoder_ops_test.py::testCTCGreedyDecoder --------------------------------------------------------------------------
GREEDY_BLANK = 3
GREEDY_INPUTS = [np.asarray(
    [[1.0, 0.0, 0.0, 0.0],
     [0.0, 0.0, 0.4, 0.6],
     [0.0, 0.0, 0.4, 0.6],
     [0.0, 0.9, 0.1, 0.0],
     [0.0, 0.0, 0.0, 0.0],      # t=4 (ignored: seq_len_0 = 4)
     [0.0, 0.0, 0.0, 0.0]]), np.asarray(
    [[0.1, 0.9, 0.0, 0.0],
     [0.0, 0.9, 0.1, 0.0],
     [0.0, 0.0, 0.1, 0.9],
     [0.0, 0.9, 0.1, 0.1],
     [0.9, 0.1, 0.0, 0.0],
     [0.0, 0.0, 0.0, 0.0]])]    # t=5 (ignored: seq_len_1 = 5)
GREEDY_SEQ_LEN = [4, 5]
GREEDY_DECODED = [[0, 1], [1, 1, 0]]               # merge_repeated=True


def greedy_case(num_classes=4, blank=GREEDY_BLANK, pad=-1.0):
    """[T=6, N=2, num_classes] scores with TF's blank moved to `blank` (labels keep their ids; needs blank >= 3)."""
    assert blank >= 3
    T, N = 6, 2
    x = np.full((T, N, num_classes), pad, np.float64)
    for n in range(N):
        x[:, n, :3] = GREEDY_INPUTS[n][:, :3]
        x[:, n, blank] = GREEDY_INPUTS[n][:, 3]
    return x, np.asarray(GREEDY_SEQ_LEN, np.int32), GREEDY_DECODED


# ---- ctc_decoder_ops_test.py::testCTCDecoderBeamSearch ---------------------------------------------------------------------
BEAM_BLANK = 5
BEAM_PROBS = np.asarray(
    [[0.30999, 0.309938, 0.0679938, 0.0673362, 0.0708352, 0.173908],
     [0.215136, 0.439699, 0.0370931, 0.0393967, 0.0381581, 0.230517],
     [0.199959, 0.489485, 0.0233221, 0.0251417, 0.0233289, 0.238763],
     [0.279611, 0.452966, 0.0204795, 0.0209126, 0.0194803, 0.20655],
     [0.51286, 0.288951, 0.0243026, 0.0220788, 0.0219297, 0.129878],
     [0.155251, 0.164444, 0.173517, 0.176138, 0.169979, 0.160671]])      # "random entry added in at time=5" (past seq_len)
BEAM_SEQ_LEN = 5
BEAM_WIDTH = 2
BEAM_TOP_PATHS = [[1, 0], [0, 1, 0]]               # decode_truth: beam 0, beam 1


def beam_case():
    """[T=8, N=1, 6]: log(p) + 2.0 ("add arbitrary offset - this is fine"), padded with two all-zero frames to max_time 8."""
    x = np.zeros((8, 1, 6), np.float64)
    x[:6, 0] = np.log(BEAM_PROBS) + 2.0
    return x, np.asarray([BEAM_SEQ_LEN], np.int32)


# ---- rnn_cell_test.py::testBasicLSTMCell ----------------------------------------------------------------------------------
LSTM_X = np.asarray([[1.0, 1.0]])
LSTM_STATE0 = 0.1                                   # every entry of [c1, h1, c2, h2]
LSTM_WEIGHT = 0.5                                   # constant_initializer(0.5) for both [4, 8] matrices; biases 0
LSTM_OUT = np.asarray([[0.24024698, 0.24024698]])
LSTM_STATE = np.asarray([[0.68967271, 0.68967271, 0.44848421, 0.44848421, 0.39897051, 0.39897051, 0.24024698, 0.24024698]])


# ---- conv_ops_test.py::testConv2D1x1Filter / testConv2D2x2Filter, pooling_ops_test.py::_testMaxPoolValidPadding --------------
CONV_INPUT_NHWC = np.arange(1, 19, dtype=np.float64).reshape(1, 2, 3, 3)
CONV_1X1_FILTER_HWIO = np.arange(1, 10, dtype=np.float64).reshape(1, 1, 3, 3)
CONV_1X1_EXPECTED = [30.0, 36.0, 42.0, 66.0, 81.0, 96.0, 102.0, 126.0, 150.0, 138.0, 171.0, 204.0, 174.0, 216.0, 258.0, 210.0, 261.0, 312.0]
CONV_2X2_FILTER_HWIO = np.arange(1, 37, dtype=np.float64).reshape(2, 2, 3, 3)
CONV_2X2_EXPECTED = [2271.0, 2367.0, 2463.0, 2901.0, 3033.0, 3165.0]         # VALID, stride 1 -> [1,1,2,3]
POOL_INPUT_NHWC = np.arange(1, 28, dtype=np.float64).reshape(1, 3, 3, 3)
POOL_2X2_S2_VALID_EXPECTED = [13.0, 14.0, 15.0]

# ---- clip_ops_test.py::testClipByGlobalNormClipped / testClipByGlobalNormNotClipped ----------------------------------------------
CLIP_X0 = np.asarray([[-2.0, 0.0, 0.0], [4.0, 0.0, 0.0]])
CLIP_X1 = np.asarray([1.0, -2.0])
CLIP_GLOBAL_NORM = 5.0
CLIP_AT_4 = (np.asarray([[-1.6, 0.0, 0.0], [3.2, 0.0, 0.0]]), np.asarray([0.8, -1.6]))       # clip_norm 4.0
CLIP_AT_6 = (CLIP_X0, CLIP_X1)                                                               # clip_norm 6.0: unchanged
