// Backward pass + optimizer orchestration: what tf.gradients / clip_by_global_norm / {Adam, RMSProp, Momentum}Optimizer
// .apply_gradients do in the reference's train_op (lib/lstm/train.py:73-83), as hand-written sm_90a kernels.
//   data gradients   : K-major wgmma GEMMs (csrc/gemm.cuh) with transformed weights
//   weight gradients : MN-major "TN" wgmma GEMMs with split-K f32 reduction (csrc/gemm_tn.cuh)
//   BPTT             : persistent cluster kernel (csrc/lstm_bwd.cuh)
//   BN / pool / ReLU / bias / conv1 / clip + solver update : HBM-bound kernels (csrc/backward_kernels.cu)
#include <cmath>
#include <cstring>

#include "backward_kernels.cuh"
#include "conv1_wgrad_tc.cuh"
#include "conv_swap.cuh"
#include "gemm_launch.h"
#include "kernels.cuh"
#include "lstm_bwd.cuh"
#include "model_internal.h"

extern "C" int crnn_model_set_training(crnn_model* m, int flag) {
  if (!m) return crnn_fail(CRNN_INVALID_VALUE, "set_training: null model");
  if (flag && m->cfg.compute_dtype >= 2) return crnn_fail(CRNN_UNSUPPORTED, "set_training: the f32-class and fp8 paths (compute_dtype 2, 3, 4) are forward only");
  if (flag && !m->wblock_bwd) {
    const size_t nB[9] = {512 * 4608, 256 * 4608, 256 * 2304, 128 * 2304, 64 * 1152, 1024 * 1024, 512 * 64, 512 * 2048, 512 * 1024};
    size_t tot = 1024;
    for (size_t v : nB) tot += align_up(v * 2);
    CUDA_TRY(cudaMalloc(&m->wblock_bwd, tot));
    uint8_t* p = reinterpret_cast<uint8_t*>(m->wblock_bwd);
    __nv_bfloat16** dst[9] = {&m->Bd_c42, &m->Bd_c41, &m->Bd_c32, &m->Bd_c31, &m->Bd_c2, &m->Bd_c5, &m->Bld, &m->Bxb, &m->Bhb};
    for (int i = 0; i < 9; ++i) { *dst[i] = reinterpret_cast<__nv_bfloat16*>(p); p += align_up(nB[i] * 2); }
    m->grad_sumsq = reinterpret_cast<double*>(p);
    CRNN_TRY(make_tmap_2d(&m->tD_c42, m->Bd_c42, 512, 4608, 4608, 256));
    CRNN_TRY(make_tmap_2d(&m->tD_c41, m->Bd_c41, 256, 4608, 4608, 256));
    CRNN_TRY(make_tmap_2d(&m->tD_c32, m->Bd_c32, 256, 2304, 2304, 256));
    CRNN_TRY(make_tmap_2d(&m->tD_c31, m->Bd_c31, 128, 2304, 2304, 128));
    CRNN_TRY(make_tmap_2d(&m->tDs_c2, m->Bd_c2, 64, 1152, 1152, 128));
    CRNN_TRY(make_tmap_2d(&m->tD_c5, m->Bd_c5, 1024, 1024, 1024, 256));
    CRNN_TRY(make_tmap_2d(&m->tD_l, m->Bld, 512, 64, 64, 256));
    CRNN_TRY(make_tmap_2d(&m->tD_x, m->Bxb, 512, 2048, 2048, 256));
    CRNN_TRY(make_tmap_2d(&m->tD_h256, m->Bhb, 512, 1024, 1024, 256));
    m->dirty_bwd = true;
  }
  m->training = flag != 0;
  return CRNN_OK;
}

static int prepare_weights_bwd(crnn_model* m, cudaStream_t st) {
  CRNN_TRY(launch_dgrad_weight(m->P("conv4_2/weights"), m->Bd_c42, 512, 512, st));
  CRNN_TRY(launch_dgrad_weight(m->P("conv4_1/weights"), m->Bd_c41, 256, 512, st));
  CRNN_TRY(launch_dgrad_weight(m->P("conv3_2/weights"), m->Bd_c32, 256, 256, st));
  CRNN_TRY(launch_dgrad_weight(m->P("conv3_1/weights"), m->Bd_c31, 128, 256, st));
  CRNN_TRY(launch_dgrad_weight(m->P("conv2/weights"), m->Bd_c2, 64, 128, st));
  CRNN_TRY(launch_conv5_dgrad_weight(m->P("conv5/weights"), m->Bd_c5, st));
  CRNN_TRY(launch_cast_bf16(m->P("logits/weights"), m->Bld, 512 * 64, st));
  CRNN_TRY(launch_lstm_bwd_weight(m->P("logits/bidirectional_rnn/fw/lstm_cell/weights"), m->P("logits/bidirectional_rnn/bw/lstm_cell/weights"),
                                  m->Bxb, m->Bhb, st));
  m->dirty_bwd = false;
  return CRNN_OK;
}

static gemm_tn::Params tn_plain(int M, int Ncols, long long rows, float* out, long long ldo) {
  gemm_tn::Params p;
  memset(&p, 0, sizeof(p));
  p.num_taps = 1;
  p.num_m_tiles = (M + 127) / 128;
  p.M = M; p.N = Ncols;
  p.k_blocks_total = (int)((rows + 63) / 64);
  p.out = out; p.ldo = ldo;
  return p;
}
static gemm_tn::Params tn_conv(int N, int H, int Wd, int Cin, int Cout, float* out, int merged) {
  gemm_tn::Params p;
  memset(&p, 0, sizeof(p));
  p.num_taps = 9;
  p.num_m_tiles = (Cin + 127) / 128;
  p.M = Cin; p.N = Cout;
  p.bh = 32 / Wd; p.Wd = Wd; p.H = H; p.Nimg = N; p.Cin = Cin;
  p.sb_per_img = (H + p.bh - 1) / p.bh;
  p.merged = merged;
  p.kb_per_img = p.sb_per_img / 2;
  p.k_blocks_total = merged ? N * p.kb_per_img : (N * p.sb_per_img + 1) / 2;
  p.out = out; p.ldo = Cout; p.tap_stride = (long long)Cin * Cout;
  return p;
}

// `u8` (crnn_backward_u8): `data` holds uint8 pixels, read only by conv1's weight gradient
static int backward_impl(crnn_model* m, const void* data, bool u8, const int* time_step_len, const float* dlogits, int N, int W,
                         void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  if (!m || !data || !time_step_len || !dlogits || !workspace) return crnn_fail(CRNN_INVALID_VALUE, "backward: null pointer");
  // conv1's weight gradient loads f32 pixels as float4, the dlogits rows are read as float4
  if (!u8) CRNN_TRY(check_aligned(data, 16, "backward", "data"));
  CRNN_TRY(check_aligned(dlogits, 16, "backward", "dlogits"));
  if (!m->params || !m->grads) return crnn_fail(CRNN_NOT_BOUND, "backward: bind params and grads first");
  if (!m->training) return crnn_fail(CRNN_INVALID_VALUE, "backward: call crnn_model_set_training(m, 1) before the forward pass");
  Plan& pl = m->plan;
  if (pl.N != N || pl.W != W || pl.ws != workspace || !pl.train)
    return crnn_fail(CRNN_INVALID_VALUE, "backward: no training-mode forward ran on this workspace for (N=%d, W=%d)", N, W);
  size_t need = 0;
  CRNN_TRY(crnn_model_workspace_size(m, N, W, 1, &need));
  if (workspace_bytes < need) return crnn_fail(CRNN_WORKSPACE_TOO_SMALL, "backward: workspace %zu < %zu", workspace_bytes, need);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (m->dirty_bwd) CRNN_TRY(prepare_weights_bwd(m, st));
  const int H1 = pl.H1, H2 = pl.H2, T = pl.T, sms = m->num_sms - m->bwd_sm_reserve;
  const long long R = (long long)N * H2;
  auto G = [&](const std::string& n) { return m->grads + m->find(n)->offset; };
  auto notify = [&](const char* first, const char* next) {     // gradients of tensors [first, next) of the table are final
    if (!m->grad_cb) return;
    const long long o = m->find(first)->offset;
    const long long e = next ? m->find(next)->offset : m->total;
    m->grad_cb(m->grad_user, o, e - o, stream);
  };
  cudaEvent_t* ev = nullptr;
  if (m->prof_on && m->prof_used_bwd < m->prof_slots) ev = &m->prof_events_bwd[(size_t)(m->prof_used_bwd++) * (kNumBwdStages + 1)];
  int evi = 0;
#define BMARK() do { if (ev) CUDA_TRY(cudaEventRecord(ev[evi++], st)); } while (0)
  BMARK();
  CUDA_TRY(cudaMemsetAsync(m->grads, 0, (size_t)m->total * sizeof(float), st));
  // moving statistics: one update per training step, from the sums this step's forward normalised with (pl.stats, over the global
  // batch when data parallel: both exchanges leave the global sums there)
  if (m->bn_moving) {
    CRNN_TRY(launch_bn_moving_update(pl.stats, (double)N * H2 * 4 * m->dp_world, m->bn_moving, m->bn_decay, st));
    m->bn_fold_dirty = true;
  }

  // ------------------------------------------------------------------ 512 -> 64 projection (network.py:118-128)
  CRNN_TRY(launch_dlogits_rows(dlogits, pl.dl_rows, G("logits/biases"), T, N, H2, st));
  {
    gemm_tn::Params p = tn_plain(512, 64, R, G("logits/weights"), 64);
    p.num_n_tiles = 1;
    CRNN_TRY((launch_gemm_tn<64, gemm_tn::TN_PLAIN, 6>(pl.tT_lstm_all, pl.tT_dl, p, sms, st)));
  }
  {
    gemm::Params p;
    memset(&p, 0, sizeof(p));
    p.M = (int)R; p.num_m_tiles = (p.M + 127) / 128; p.num_n_tiles = 2; p.num_k_blocks = 1; p.kb_per_shift = 1;
    p.Nc = 512; p.out = pl.d_lstm_out; p.ldo = 512;
    CRNN_TRY((launch_gemm<256, gemm::A_PLAIN, gemm::EPI_BIAS_BF16, 4>(pl.tG_dl, m->tD_l, p, sms, st, &pl.tO_dlo)));
  }
  BMARK();
  // ------------------------------------------------------------------ BPTT through both directions
  // dz rows of the padding frames (t = T) are never written by the recurrence, yet dW_x, dW_h, the LSTM bias sums and the conv5
  // data gradient read them as K rows: zero them in every backward, whatever the workspace held before the forward
  CUDA_TRY(cudaMemset2DAsync(pl.dz_all + (size_t)T * 2048, (size_t)H2 * 2048 * 2, 0, 2048 * 2, N, st));
  {
    lstm_bwd::Params lp;
    lp.gates = pl.gates; lp.csave = pl.csave; lp.d_out = pl.d_lstm_out; lp.dz_all = pl.dz_all;
    lp.seq_len = time_step_len; lp.Nimg = N; lp.Npad = pl.Npad; lp.H = H2; lp.T = T; lp.tiles_per_dir = pl.Npad / 128;
    static bool attr = false;
    if (!attr) {
      CUDA_TRY(cudaFuncSetAttribute(lstm_bwd::lstm_bwd_ks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lstm_bwd::ks::SMEM_BYTES));
      attr = true;
    }
    CRNN_TRY(launch_cluster(lstm_bwd::lstm_bwd_ks_kernel, lstm_bwd::CS, lstm_bwd::CS * 2 * lp.tiles_per_dir, lstm_bwd::ks::NUM_THREADS,
                            lstm_bwd::ks::SMEM_BYTES, st, m->tD_h256, lp, pl.bptt_x));
  }
  BMARK();
  {
    const std::string fw = "logits/bidirectional_rnn/fw/lstm_cell", bw = "logits/bidirectional_rnn/bw/lstm_cell";
    const long long dW = m->find(bw + "/weights")->offset - m->find(fw + "/weights")->offset;
    const long long db = m->find(bw + "/biases")->offset - m->find(fw + "/biases")->offset;
    CRNN_TRY(launch_colsum_bf16(pl.dz_all, R, 2048, G(fw + "/biases"), true, db, st));
    {  // dW_x (rows 0..511 of both [768,1024] matrices) = a5^T dz
      gemm_tn::Params p = tn_plain(512, 2048, R, G(fw + "/weights"), 1024);
      p.num_n_tiles = 8; p.lstm_cols = 1; p.dir_stride = dW;
      CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_PLAIN, 4>(pl.tT_a5, pl.tT_dz, p, sms, st)));
    }
    {  // dW_h forward direction: previous step = frame t-1
      gemm_tn::Params p = tn_plain(256, 1024, R, G(fw + "/weights"), 1024);
      p.num_n_tiles = 4; p.lstm_cols = 1; p.out_row_offset = 512; p.a_row_shift = -1;
      CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_PLAIN, 4>(pl.tT_lstm_fw, pl.tT_dz_fw, p, sms, st)));
    }
    {  // dW_h backward direction: previous step = frame t+1
      gemm_tn::Params p = tn_plain(256, 1024, R, G(bw + "/weights"), 1024);
      p.num_n_tiles = 4; p.lstm_cols = 1; p.out_row_offset = 512; p.a_row_shift = +1;
      CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_PLAIN, 4>(pl.tT_lstm_bw, pl.tT_dz_bw, p, sms, st)));
    }
    // LSTM (both directions) and the 512 -> 64 projection are the tail of the flat buffer: their gradients are final here
    if (m->grad_cb) {
      const long long o = m->find(fw + "/weights")->offset;
      m->grad_cb(m->grad_user, o, m->total - o, stream);
    }
    {  // dx = dz W_x^T  ->  gradient w.r.t. the conv5 feature rows
      gemm::Params p;
      memset(&p, 0, sizeof(p));
      p.M = (int)R; p.num_m_tiles = (p.M + 127) / 128; p.num_n_tiles = 2; p.num_k_blocks = 32; p.kb_per_shift = 32;
      p.Nc = 512; p.out = pl.d_a5; p.ldo = 512;
      CRNN_TRY((launch_gemm<256, gemm::A_PLAIN, gemm::EPI_BIAS_BF16, 4>(pl.tG_dz, m->tD_x, p, sms, st, &pl.tG_da5)));
    }
  }
  BMARK();
  // ------------------------------------------------------------------ conv5 (2x2 VALID)
  CRNN_TRY(launch_colsum_bf16(pl.d_a5, R, 512, G("conv5/biases"), false, 0, st));
  for (int r = 0; r < 2; ++r) {
    gemm_tn::Params p = tn_plain(1024, 512, R, G("conv5/weights") + (size_t)r * 1024 * 512, 512);
    p.num_n_tiles = 2; p.a_row_shift = r;
    CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_PLAIN, 4>(pl.tT_a4b, pl.tT_da5, p, sms, st)));
  }
  notify("conv5/weights", "logits/bidirectional_rnn/fw/lstm_cell/weights");
  {
    gemm::Params p;
    memset(&p, 0, sizeof(p));
    p.M = (int)R; p.num_m_tiles = (p.M + 127) / 128; p.num_n_tiles = 4; p.num_k_blocks = 16; p.kb_per_shift = 8; p.row_shift_mul = -1;
    p.Nc = 1024; p.out = pl.d_a4b; p.ldo = 1024;
    CRNN_TRY((launch_gemm<256, gemm::A_PLAIN, gemm::EPI_BIAS_BF16, 4>(pl.tG_da5, m->tD_c5, p, sms, st, &pl.tO_da4b)));
  }
  BMARK();
  // ------------------------------------------------------------------ conv4_2: pool3 + ReLU + batch-stat BN backward
  CUDA_TRY(cudaMemsetAsync(pl.bn_bwd_sums, 0, 2 * 2 * 512 * sizeof(double), st));
  const size_t P4 = (size_t)N * H2 * 4;
  const double P4g = (double)P4 * m->dp_world;         // positions of the batch the BN statistics were taken over
  // data parallel: [sum dy, sum dy*xhat] over the GLOBAL batch (exchanged over peer memory / the callback), local sums kept for dgamma/dbeta
  double* sums42 = pl.bn_bwd_sums + 1024;
  double* sums41 = pl.bn_bwd_sums;
  double* gsum42 = m->dp_world > 1 ? pl.bn_bwd_sums + 3072 : sums42;
  double* gsum41 = m->dp_world > 1 ? pl.bn_bwd_sums + 2048 : sums41;
  CRNN_TRY(launch_bn_bwd_reduce(pl.d_a4b, pl.a4b_pre, pl.bn + 2048, sums42, P4 / 2, 512, st));
  if (m->dp_world > 1) CRNN_TRY(dp_allreduce_1024(m, sums42, gsum42, st));
  CRNN_TRY(launch_bn_bwd_apply(true, pl.d_a4b, pl.a4b_pre, pl.d_pre4b, pl.bn + 2048, m->P("conv4_2/conv4_2/gamma"), gsum42, sums42, P4g,
                               P4 / 2, 512, pl.bn_bwd_coef, G("conv4_2/conv4_2/gamma"), G("conv4_2/conv4_2/beta"), st));
  // conv4_2/biases: a bias in front of a batch-statistics BatchNorm has an analytically ZERO gradient (the BN backward projects
  // the column sums of d(pre-BN) out); it stays at the zero the buffer was cleared to instead of summing 134 MB of rounding noise
  BMARK();
  {
    gemm_tn::Params p = tn_conv(N, H2, 4, 512, 512, G("conv4_2/weights"), pl.wm4);
    p.num_n_tiles = 2;
    CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_CONV, 4>(pl.tW_a4a, pl.tW_p4b, p, sms, st)));
  }
  notify("conv4_2/weights", "conv5/weights");
  BMARK();
  {
    // pass 1 of conv4_1's BatchNorm/ReLU backward (the two per-channel sums) rides in this epilogue: no separate read of the
    // 268 MB gradient + 268 MB pre-BN activation
    gemm::Params p = conv_params(N, H2, 4, 512, 512, 256, nullptr, pl.d_pre4a, pl.mg4);
    p.mask = pl.a4a_pre; p.bnp = pl.bn; p.stats = sums41;
    CRNN_TRY((launch_gemm<256, gemm::A_CONV3, gemm::EPI_CONV_STORE_BNRED, 4>(pl.tG_p4b, m->tD_c42, p, sms, st)));
  }
  BMARK();
  // ------------------------------------------------------------------ conv4_1: ReLU + BN backward
  if (m->dp_world > 1) CRNN_TRY(dp_allreduce_1024(m, sums41, gsum41, st));
  CRNN_TRY(launch_bn_bwd_apply(false, pl.d_pre4a, pl.a4a_pre, pl.d_pre4a, pl.bn, m->P("conv4_1/conv4_1/gamma"), gsum41, sums41, P4g, P4, 512,
                               pl.bn_bwd_coef, G("conv4_1/conv4_1/gamma"), G("conv4_1/conv4_1/beta"), st));
  // conv4_1/biases: analytically zero as well (see conv4_2)
  BMARK();
  {
    gemm_tn::Params p = tn_conv(N, H2, 4, 256, 512, G("conv4_1/weights"), pl.wm4);
    p.num_n_tiles = 2;
    CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_CONV, 4>(pl.tW_a3p, pl.tW_p4a, p, sms, st)));
  }
  notify("conv4_1/weights", "conv4_2/weights");
  BMARK();
  {
    gemm::Params p = conv_params(N, H2, 4, 512, 256, 256, nullptr, pl.d_a3p, pl.mg4);
    CRNN_TRY((launch_gemm<256, gemm::A_CONV3, gemm::EPI_CONV_STORE, 4>(pl.tG_p4a, m->tD_c41, p, sms, st, &pl.tO_da3p)));
  }
  BMARK();
  // ------------------------------------------------------------------ conv3_2: 1x2 pool + ReLU backward
  CRNN_TRY(launch_unpool_relu_bwd(2, pl.d_a3p, pl.a3p, pl.am3, pl.d_pre32, (size_t)N * H2 * 4, H2, 4, 256, st));
  // bias gradient = column sums of the POOLED gradient where the pooled output is positive (each value is routed to one position)
  CRNN_TRY(launch_colsum_masked_bf16(pl.d_a3p, pl.a3p, (long long)N * H2 * 4, 256, G("conv3_2/biases"), st));
  BMARK();
  {
    gemm_tn::Params p = tn_conv(N, H2, 8, 256, 256, G("conv3_2/weights"), pl.wm3);
    p.num_n_tiles = 1;
    CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_CONV, 4>(pl.tW_a3, pl.tW_p32, p, sms, st)));
  }
  notify("conv3_2/weights", "conv4_1/weights");
  BMARK();
  {
    // conv3_1's ReLU backward rides in this epilogue (zero where a3 == 0): saves one read + one write of the 268 MB gradient
    gemm::Params p = conv_params(N, H2, 8, 256, 256, 256, nullptr, pl.d_pre31, pl.mg3);
    p.mask = pl.a3;
    CRNN_TRY((launch_gemm<256, gemm::A_CONV3, gemm::EPI_CONV_STORE_MASK, 4>(pl.tG_p32, m->tD_c32, p, sms, st)));
  }
  BMARK();
  // ------------------------------------------------------------------ conv3_1: bias gradient (its ReLU backward is fused above)
  CRNN_TRY(launch_colsum_bf16(pl.d_pre31, (long long)N * H2 * 8, 256, G("conv3_1/biases"), false, 0, st));
  BMARK();
  {
    gemm_tn::Params p = tn_conv(N, H2, 8, 128, 256, G("conv3_1/weights"), pl.wm3);
    p.num_n_tiles = 1;
    CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_CONV, 4>(pl.tW_a2, pl.tW_p31, p, sms, st)));
  }
  notify("conv3_1/weights", "conv3_2/weights");
  BMARK();
  {
    // conv3_1's data gradient has 128 output channels: position-major it is an N = 128 tile (half the MMA rate); swapped, the 128
    // channels fill the M side and N is 256 positions (32 H rows x 8)
    convsw::DgradParams p;
    p.Nimg = N; p.H = H2; p.tiles_per_img = (H2 + 31) / 32; p.out = pl.d_a2;
    CRNN_TRY((launch_conv_dgrad_swap<8, 4, 128>(pl.tG_p31s, m->tD_c31, p, sms, st)));
  }
  BMARK();
  // ------------------------------------------------------------------ conv2: 2x2 pool + ReLU backward
  CRNN_TRY(launch_unpool_relu_bwd(4, pl.d_a2, pl.a2, pl.am2, pl.d_pre2, (size_t)N * H2 * 8, H2, 8, 128, st));
  CRNN_TRY(launch_colsum_masked_bf16(pl.d_a2, pl.a2, (long long)N * H2 * 8, 128, G("conv2/biases"), st));
  BMARK();
  {
    // operands swapped: A = d(pre-activation) [positions x 128 co] on the M side, B = a1 with FOUR tap-shifted 64-channel boxes
    // per 256-column N tile (columns = (tap, ci)); 3 N tiles cover the 9 taps.  N = 256 runs the MMA at full rate where the
    // Cout = 128 N tile of the straight formulation halves it.
    gemm_tn::Params p = tn_conv(N, H1, 16, 64, 128, G("conv2/weights"), pl.wm2);
    p.tap_pack_n = 1; p.num_taps = 1; p.num_m_tiles = 1; p.num_n_tiles = 3; p.M = 128; p.N = 9 * 64; p.ldo = 128; p.tap_stride = 0;
    CRNN_TRY((launch_gemm_tn<256, gemm_tn::TN_CONV, 4>(pl.tW_p2, pl.tW_a1, p, sms, st)));
  }
  BMARK();
  {
    convsw::DgradParams p;
    p.Nimg = N; p.H = H1; p.tiles_per_img = (H1 + 15) / 16; p.out = pl.d_a1;
    CRNN_TRY((launch_conv_dgrad_swap<16, 2, 64>(pl.tG_p2s, m->tDs_c2, p, sms, st)));
  }
  BMARK();
  // ------------------------------------------------------------------ conv1 (Cin = 1): pool1 + ReLU backward folded in; tensor-core
  // kernel with thread-built operands (conv1_wgrad_tc.cuh)
  CRNN_TRY(launch_conv1_wgrad_tc(pl.d_a1, pl.a1, pl.am1, data, u8, G("conv1/weights"), G("conv1/biases"), N, W, sms, st));
  notify("conv1/weights", "conv3_1/weights");
  BMARK();
#undef BMARK
  return CRNN_OK;
}

extern "C" int crnn_backward(crnn_model* m, const float* data, const int* time_step_len, const float* dlogits, int N, int W,
                             void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  return backward_impl(m, data, false, time_step_len, dlogits, N, W, workspace, workspace_bytes, stream);
}
extern "C" int crnn_backward_u8(crnn_model* m, const uint8_t* data, const int* time_step_len, const float* dlogits, int N, int W,
                                void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  // the uint8 kernel loads each row's pixels as 4-byte words
  CRNN_TRY(check_aligned(data, 4, "backward_u8", "uint8 data"));
  return backward_impl(m, data, true, time_step_len, dlogits, N, W, workspace, workspace_bytes, stream);
}

// The half of every solver step that does not depend on the solver: grads <- grads + wd*wd_mul*w on the L2-regularised tensors
// (conv kernels + logits matrix) and the global sum of squares into m->grad_sumsq, which the update kernels turn into the clip
// scale.
static int finish_gradients(crnn_model* m, float wd_mul, cudaStream_t st) {
  WdSegs segs;
  segs.n = 0;
  for (auto& c : kConvs) {
    const TensorInfo* t = m->find(std::string(c.name) + "/weights");
    segs.off[segs.n] = t->offset; segs.cnt[segs.n] = t->count; segs.n++;
  }
  const TensorInfo* t = m->find("logits/weights");
  segs.off[segs.n] = t->offset; segs.cnt[segs.n] = t->count; segs.n++;
  return launch_grad_finish(m->grads, m->params, segs, m->cfg.weight_decay * wd_mul, m->total, m->grad_sumsq, st);
}

// grads <- grads + wd*wd_mul*w on the regularised tensors; g <- g*grad_mul; clip by global norm; TF Adam.
// Data-parallel use: all-reduce(SUM) the flat gradient buffer first, then call with grad_mul = 1/world, wd_mul = world.
extern "C" int crnn_clip_adam_step(crnn_model* m, float lr, float clip, int step, float grad_mul, float wd_mul,
                                   crnn_stream_t stream) {
  if (!m || step < 1) return crnn_fail(CRNN_INVALID_VALUE, "clip_adam_step: bad args");
  if (!m->params || !m->grads || !m->adam_m || !m->adam_v) return crnn_fail(CRNN_NOT_BOUND, "clip_adam_step: bind params, grads and Adam slots");
  if (!m->grad_sumsq) return crnn_fail(CRNN_INVALID_VALUE, "clip_adam_step: call crnn_model_set_training(m, 1) first");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CRNN_TRY(finish_gradients(m, wd_mul, st));
  const double b1 = 0.9, b2 = 0.999;
  const float lr_t = (float)(lr * std::sqrt(1.0 - std::pow(b2, step)) / (1.0 - std::pow(b1, step)));
  CRNN_TRY(launch_clip_adam(m->params, m->grads, m->adam_m, m->adam_v, m->grad_sumsq, grad_mul, clip, lr_t, (float)b1, (float)b2, 1e-8f,
                            m->total, st));
  m->dirty = true;
  m->dirty_bwd = true;
  return CRNN_OK;
}

// Same gradient finish and clip, then TF MomentumOptimizer; accum lives in the buffer bound as adam_m.
extern "C" int crnn_clip_momentum_step(crnn_model* m, float lr, float momentum, float clip, float grad_mul, float wd_mul,
                                       crnn_stream_t stream) {
  if (!m || !(momentum >= 0.f)) return crnn_fail(CRNN_INVALID_VALUE, "clip_momentum_step: bad args (momentum must be >= 0)");
  if (!m->params || !m->grads || !m->adam_m) return crnn_fail(CRNN_NOT_BOUND, "clip_momentum_step: bind params, grads and adam_m (accum)");
  if (!m->grad_sumsq) return crnn_fail(CRNN_INVALID_VALUE, "clip_momentum_step: call crnn_model_set_training(m, 1) first");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CRNN_TRY(finish_gradients(m, wd_mul, st));
  CRNN_TRY(launch_clip_momentum(m->params, m->grads, m->adam_m, m->grad_sumsq, grad_mul, clip, lr, momentum, m->total, st));
  m->dirty = true;
  m->dirty_bwd = true;
  return CRNN_OK;
}

// Same gradient finish and clip, then TF RMSPropOptimizer (not centred); mom lives in adam_m, ms in adam_v.
extern "C" int crnn_clip_rmsprop_step(crnn_model* m, float lr, float decay, float momentum, float epsilon, float clip, float grad_mul,
                                      float wd_mul, crnn_stream_t stream) {
  if (!m || !(decay >= 0.f && decay <= 1.f) || !(momentum >= 0.f) || !(epsilon >= 0.f))
    return crnn_fail(CRNN_INVALID_VALUE, "clip_rmsprop_step: bad args (decay in [0, 1], momentum >= 0, epsilon >= 0)");
  if (!m->params || !m->grads || !m->adam_m || !m->adam_v)
    return crnn_fail(CRNN_NOT_BOUND, "clip_rmsprop_step: bind params, grads, adam_m (mom) and adam_v (ms)");
  if (!m->grad_sumsq) return crnn_fail(CRNN_INVALID_VALUE, "clip_rmsprop_step: call crnn_model_set_training(m, 1) first");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CRNN_TRY(finish_gradients(m, wd_mul, st));
  CRNN_TRY(launch_clip_rmsprop(m->params, m->grads, m->adam_m, m->adam_v, m->grad_sumsq, grad_mul, clip, lr, decay, momentum, epsilon,
                               m->total, st));
  m->dirty = true;
  m->dirty_bwd = true;
  return CRNN_OK;
}

// global gradient norm of the last solver step (before clipping, after averaging); host-synchronising helper
extern "C" int crnn_last_grad_norm(crnn_model* m, float grad_mul, float* out, crnn_stream_t stream) {
  if (!m || !out || !m->grad_sumsq) return crnn_fail(CRNN_INVALID_VALUE, "last_grad_norm: bad args");
  double v = 0;
  CUDA_TRY(cudaMemcpyAsync(&v, m->grad_sumsq, sizeof(double), cudaMemcpyDeviceToHost, reinterpret_cast<cudaStream_t>(stream)));
  CUDA_TRY(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(stream)));
  *out = (float)(std::sqrt(v) * grad_mul);
  return CRNN_OK;
}

// MN-major GEMM unit-test entry: D[M,N] (zeroed by the caller) += A[K,M]^T B[K,N]
extern "C" int crnn_test_gemm_tn_bf16(const void* A, const void* B, float* D, int M, int Ncols, int K, int block_n,
                                      int k_splits, crnn_stream_t stream) {
  if (!A || !B || !D || M <= 0 || Ncols <= 0 || K <= 0 || (M % 8) || (Ncols % 8)) return crnn_fail(CRNN_INVALID_VALUE, "test_gemm_tn: bad args");
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  CUtensorMap ta, tb;
  CRNN_TRY(make_tmap_2d_box(&ta, A, K, M, M, 64, 64));
  CRNN_TRY(make_tmap_2d_box(&tb, B, K, Ncols, Ncols, 64, 64));
  gemm_tn::Params p = tn_plain(M, Ncols, K, D, Ncols);
  p.num_n_tiles = (Ncols + block_n - 1) / block_n;
  p.k_splits = k_splits;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (block_n == 64) return launch_gemm_tn<64, gemm_tn::TN_PLAIN, 6>(ta, tb, p, sms, st);
  if (block_n == 128) return launch_gemm_tn<128, gemm_tn::TN_PLAIN, 6>(ta, tb, p, sms, st);
  if (block_n == 256) return launch_gemm_tn<256, gemm_tn::TN_PLAIN, 4>(ta, tb, p, sms, st);
  return crnn_fail(CRNN_INVALID_VALUE, "test_gemm_tn: block_n must be 64/128/256");
}

extern "C" int crnn_profile_bwd_num_stages(void) { return kNumBwdStages; }
extern "C" const char* crnn_profile_bwd_stage_name(int i) { return (i >= 0 && i < kNumBwdStages) ? kBwdStageNames[i] : ""; }
extern "C" int crnn_profile_bwd_read(crnn_model* m, float* ms_out, int* backwards) {
  if (!m || !ms_out || !backwards) return crnn_fail(CRNN_INVALID_VALUE, "profile_bwd_read: null");
  *backwards = m->prof_used_bwd;
  for (int f = 0; f < m->prof_used_bwd; ++f) {
    cudaEvent_t* ev = &m->prof_events_bwd[(size_t)f * (kNumBwdStages + 1)];
    CUDA_TRY(cudaEventSynchronize(ev[kNumBwdStages]));
    for (int s = 0; s < kNumBwdStages; ++s) CUDA_TRY(cudaEventElapsedTime(ms_out + (size_t)f * kNumBwdStages + s, ev[s], ev[s + 1]));
  }
  return CRNN_OK;
}
