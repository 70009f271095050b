// Internal declarations shared by model.cu (forward) and backward.cu (gradients / optimizer).
#pragma once
#include <string>
#include <vector>

#include <cuda.h>

#include "common.cuh"
#include "gemm.cuh"

int make_tmap_2d(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride, uint32_t box_rows);
int make_tmap_nhwc(CUtensorMap* m, const void* base, int N, int H, int Wd, int C, int bh);
// f32 tensors read as tf32 operands: 32-element (128 B) boxes along the contiguous dimension
int make_tmap_2d_f32(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride, uint32_t box_rows);
int make_tmap_nhwc_f32(CUtensorMap* m, const void* base, int N, int H, int Wd, int C, int bh);
// e4m3 tensors (UINT8 elements): 128-element (128 B) boxes along the contiguous dimension
int make_tmap_2d_u8(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride, uint32_t box_rows);
int make_tmap_nhwc_u8(CUtensorMap* m, const void* base, int N, int H, int Wd, int C, int bh);
size_t align_up(size_t v, size_t a = 1024);
int make_tmap_2d_box(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride, uint32_t box_cols,
                     uint32_t box_rows);

struct TensorInfo {
  std::string name;
  int ndim;
  int64_t shape[4];
  int64_t offset;
  int64_t count;
};

struct ConvSpec { const char* name; int kh, kw, ci, co; bool bn; };
static const ConvSpec kConvs[7] = {   // lib/networks/LSTM_train.py:24-34
    {"conv1", 3, 3, 1, 64, false},    {"conv2", 3, 3, 64, 128, false},  {"conv3_1", 3, 3, 128, 256, false},
    {"conv3_2", 3, 3, 256, 256, false}, {"conv4_1", 3, 3, 256, 512, true}, {"conv4_2", 3, 3, 512, 512, true},
    {"conv5", 2, 2, 512, 512, false}};

static const char* kStageNames[] = {"conv1_pool1", "conv2_pool2", "conv3_1", "conv3_2_pool", "conv4_1_gemm", "bn4_1_apply",
                                    "conv4_2_gemm", "bn4_2_apply_pool3", "conv5", "lstm_xproj", "lstm_recurrence", "logits"};
static const int kNumStages = 12;
static const char* kBwdStageNames[] = {"zero+logits_bwd", "lstm_bptt", "lstm_wgrad+dx", "conv5_bwd", "bn4_2_bwd", "conv4_2_wgrad",
                                       "conv4_2_dgrad", "bn4_1_bwd", "conv4_1_wgrad", "conv4_1_dgrad", "conv3_2_bwd_elem", "conv3_2_wgrad",
                                       "conv3_2_dgrad", "conv3_1_bwd_elem", "conv3_1_wgrad", "conv3_1_dgrad", "conv2_bwd_elem", "conv2_wgrad",
                                       "conv2_dgrad", "conv1_wgrad"};
static const int kNumBwdStages = 20;

static const int kMaxChunks = 16;

struct Plan {
  int N = 0, W = 0, H1 = 0, H2 = 0, T = 0, Npad = 0;
  void* ws = nullptr;
  __nv_bfloat16 *a1, *a2, *a3, *a3p, *a4a_pre, *a4a, *a4b_pre, *a4b, *a5, *xproj, *lstm_out, *h_state;
  double* stats;        // [2 layers][2][512]
  float* bn;            // [2 layers][4][512]: scale, shift, mean, invstd
  // packed evaluation (crnn_forward_lines), past the inference layout; line_w == nullptr after any other forward, stats_l / bn_l ==
  // nullptr also under moving statistics
  int* line_w = nullptr;      // [N] clamped line widths
  bool moving = false;        // the last forward normalised conv4_x with the moving statistics (no a4x_pre, bn or stats written)
  double* stats_l = nullptr;  // [2 layers][N][2][512]
  float* bn_l = nullptr;      // [2 layers][N][4][512]
  CUtensorMap tA_c2s;   // conv2 input through 128-position boxes regardless of H (swapped-operand kernel, conv_swap.cuh)
  CUtensorMap tA_c31, tA_c32, tA_c41, tA_c42, tA_c5, tA_x, tA_l;
  // output maps of the register-side GEMM epilogues (gemm::frag_epi) where no input map above has the producing layer's tile
  // geometry: conv3_1 stores through tA_c32 and conv5 through tA_x; conv1_tc_kernel stores its pooled tiles through tO_c1
  CUtensorMap tO_c1, tO_c2s, tO_c32, tO_c41, tO_c42, tO_x;
  // conv A maps use 128-position boxes (`mg*` = 1) when a tile's 4 sub-boxes are contiguous rows of one image;
  // the weight-gradient GEMMs read the same tensors through 64- or 32-position boxes (tW_*)
  int mg2 = 0, mg3 = 0, mg4 = 0, wm2 = 0, wm3 = 0, wm4 = 0;
  CUtensorMap tW_a1, tW_a2, tW_a3, tW_a3p, tW_a4a, tW_p4b, tW_p4a, tW_p32, tW_p31, tW_p2;
  // compute_dtype 4: UINT8 views of the e4m3 activations, which live in the first half of the bf16 buffers a2, a3, a3p, a4a, a4b
  // (forward_fp8.cu): A operands of conv3_1 .. conv5, conv3_1 stores through q_c32, conv2 / conv3_2 through qO_c2s / qO_c32
  CUtensorMap q_c31, q_c32, q_c41, q_c42, q_c5, qO_c2s, qO_c32;
  // moving statistics: conv4_2's pooled output a4b as a conv output (Wd = 2), bf16 and e4m3
  CUtensorMap tO_m42, qO_m42;
  // ---- training only -------------------------------------------------------------------------------------------
  bool train = false;
  uint8_t *am1, *am2, *am3;                       // arg-max window indices of pool1 / pool2 / the 1x2 pool after conv3_2
  __nv_bfloat16* gates;                           // [2][N][T][4][256] post-activation gates
  float* csave;                                   // [2][N][T][256]
  __nv_bfloat16 *dl_rows, *d_lstm_out, *dz_all, *d_a5, *d_a4b, *d_pre4b, *d_pre4a, *d_a3p, *d_pre32, *d_pre31, *d_a2,
      *d_pre2, *d_a1;
  uint8_t* bptt_x;                                // lstm_bwd_ks_kernel exchange buffer [2][units][8 dst][8 src][8 KB]
  double* bn_bwd_sums;                            // [2 layers][2][512]
  float* bn_bwd_coef;                             // [3][512] scratch
  // K-major A maps of gradient buffers (data-gradient GEMMs)
  CUtensorMap tG_dl, tG_dz, tG_da5, tG_p4b, tG_p4a, tG_p32;
  CUtensorMap tG_p2s, tG_p31s;                    // d_pre2 / d_pre31 through 128-position boxes regardless of H (conv_dgrad_swap_kernel)
  CUtensorMap tO_dlo, tO_da4b, tO_da3p;           // data-gradient GEMM outputs (the others store through tG_da5 / tG_p4a)
  // MN-major (TN) maps: 2-D [rows, C] with 64x64 boxes, and the NHWC maps above reused for TN_CONV
  CUtensorMap tT_lstm_fw, tT_lstm_bw, tT_lstm_all, tT_dl, tT_a5, tT_dz, tT_dz_fw, tT_dz_bw, tT_a4b, tT_da5;
};

struct crnn_model {
  crnn_config cfg;
  int num_sms = 132;
  std::vector<TensorInfo> tensors;
  int64_t total = 0;
  float *params = nullptr, *grads = nullptr, *adam_m = nullptr, *adam_v = nullptr;
  bool dirty = true;
  // bf16 K-major operand copies of the weights (B matrices [Cout][K])
  __nv_bfloat16 *Bc2 = nullptr, *Bc31, *Bc32, *Bc41, *Bc42, *Bc5, *Bx, *Bh, *Bl;
  float* xbias = nullptr;    // [2048] permuted LSTM bias with forget_bias folded in
  double* sumsq = nullptr;
  void* wblock = nullptr;
  CUtensorMap tB_c2, tB_c31, tB_c32, tB_c41, tB_c42, tB_c5, tB_x, tB_l, tB_h128;
  // training: bf16 operands of the data-gradient GEMMs (allocated by crnn_model_set_training)
  bool training = false;
  bool dirty_bwd = true;
  void* wblock_bwd = nullptr;
  __nv_bfloat16 *Bd_c42 = nullptr, *Bd_c41, *Bd_c32, *Bd_c31, *Bd_c2, *Bd_c5, *Bld, *Bxb, *Bhb;
  CUtensorMap tD_c42, tD_c41, tD_c32, tD_c31, tD_c5, tD_l, tD_x;
  CUtensorMap tDs_c2;        // conv2 dgrad weights through a 128-row box (rows 64..127 out of bounds -> zero fill): conv2_dgrad_swap_kernel
  CUtensorMap tD_h256;       // W_h^T operand of the BPTT (Bhb), box = 256 unit rows
  double* grad_sumsq = nullptr;
  // ---- moving BatchNorm statistics of conv4_1 / conv4_2 (crnn_model_bind_bn_moving / crnn_model_set_bn_statistics)
  float* bn_moving = nullptr;            // caller-owned [2 layers][mean, variance][512] f32; updated by every crnn_backward
  float bn_decay = 0.999f;
  bool bn_use_moving = false;            // evaluation forwards normalise conv4_x with bn_moving (training forwards never do)
  bool bn_fold_dirty = true;             // params, bn_moving or the mode changed since the folded operands were derived
  void* wblock_bnm = nullptr;            // folded operands, allocated by the first crnn_model_bind_bn_moving
  __nv_bfloat16 *Bm41 = nullptr, *Bm42 = nullptr;   // bf16(W * s) [Cout][K]
  float* bm_bias = nullptr;              // [2][512] (b - mean) * s + beta
  double* bm_scale = nullptr;            // [2][512] s = gamma / sqrt(var + eps)
  CUtensorMap tB_m41, tB_m42;
  Plan plan;
  void* x3 = nullptr;        // state of the f32-class path (compute_dtype 2, forward_x3.cu)
  void* fp8 = nullptr;       // e4m3 weights and scales of compute_dtype 4 (forward_fp8.cu)
  // ---- data parallelism (SURVEY 8(e)): BatchNorm statistics over the GLOBAL batch + per-bucket "gradient ready" notifications
  int dp_rank = 0, dp_world = 1;
  crnn_allreduce_fn xchg_cb = nullptr;   // fallback exchange of the [2][512] f64 BN sums (e.g. NCCL through the host language)
  void* xchg_user = nullptr;
  void** d_peers = nullptr;              // device array [world] of peer inbox pointers (own inbox at [rank]); nullptr = no peer memory
  int* d_peer_err = nullptr;
  unsigned long long peer_epoch = 0;
  int bwd_sm_reserve = 0;                // SMs left free by the persistent backward kernels (for overlapped collectives)
  crnn_grad_ready_fn grad_cb = nullptr;
  void* grad_user = nullptr;
  std::vector<cudaEvent_t> chunk_events;   // crnn_forward_host: one per H2D chunk + one "staging free" event
  // per-stage CUDA-event profiling (crnn_profile_*): events are recorded on the caller's stream between stages
  std::vector<cudaEvent_t> prof_events;   // [slots][kNumStages + 1]
  int prof_slots = 0, prof_used = 0;
  bool prof_on = false;
  std::vector<cudaEvent_t> prof_events_bwd;   // [slots][kNumBwdStages + 1]
  int prof_used_bwd = 0;

  const TensorInfo* find(const std::string& n) const {
    for (auto& t : tensors) if (t.name == n) return &t;
    return nullptr;
  }
  float* P(const std::string& n) const { return params + find(n)->offset; }
};

// f32-class ("3xbf16") forward path, forward_x3.cu
size_t x3_workspace_size(int N, int W);
int x3_forward(crnn_model* m, const void* data, bool u8, const int* time_step_len, int N, int W, float* logits_out, void* workspace,
               size_t workspace_bytes, cudaStream_t st);
int x3_debug_tap(crnn_model* m, const char* name, float* dst, size_t dst_elems, void* workspace, cudaStream_t st);
int x3_debug_tap_raw(crnn_model* m, const char* name, void* dst, size_t dst_bytes, void* workspace, cudaStream_t st);
void x3_destroy(crnn_model* m);
void x3_params_changed(crnn_model* m);

// fp8 inference path (compute_dtype 4), forward_fp8.cu; the orchestration is model.cu's forward
namespace convsw { struct Params; }
int fp8_create(crnn_model* m);        // e4m3 weights, scales and scratch of a compute_dtype 4 model, allocated once at create
void fp8_destroy(crnn_model* m);
void fp8_params_changed(crnn_model* m);
bool fp8_calibrated(const crnn_model* m);
int fp8_prepare(crnn_model* m, cudaStream_t st);
int fp8_plan_maps(Plan& pl);
int fp8_conv2(crnn_model* m, convsw::Params p, bool lines, int sms, cudaStream_t st);
// moving = true (layers 2, 3): conv4_x with the folded BatchNorm, e4m3 a4a (EPI_RELU) / pooled a4b (EPI_RELU_POOL12) out
int fp8_conv_gemm(crnn_model* m, int layer, gemm::Params p, bool lines, int sms, cudaStream_t st, bool moving = false);
int fp8_fold_moving(crnn_model* m, bool refolded, cudaStream_t st);   // colscale of conv4_x times the moving-statistics scale
int fp8_bn_apply(crnn_model* m, int layer, const float* bn, bool lines, cudaStream_t st);
int fp8_conv5(crnn_model* m, gemm::Params p, int sms, cudaStream_t st);
int fp8_finish_calibration(crnn_model* m, cudaStream_t st);
int fp8_get_scales(crnn_model* m, float* host);
int fp8_set_scales(crnn_model* m, const float* host);
int fp8_dequant_tap(crnn_model* m, int idx, const void* src, float* dst, size_t n, cudaStream_t st);
int fp8_debug_tap_raw(crnn_model* m, const std::string& name, void* dst, size_t dst_bytes, cudaStream_t st, int* status);

// SyncBN exchange (peer.cu): sums of `in` [1024] f64 over all ranks -> `out` (may alias `in`); optionally fused with the BN finalize
int dp_allreduce_1024(crnn_model* m, const double* in, double* out, cudaStream_t st);
int dp_allreduce_bn_finalize(crnn_model* m, double* stats, double count_global, const float* gamma, const float* beta, float eps,
                             float* bn /*scale, shift, mean, invstd: [4][512]*/, cudaStream_t st);

size_t layout_plan(Plan& pl, int N, int W, uint8_t* base, bool train, bool lines = false, bool moving = false);
int prepare_weights(crnn_model* m, cudaStream_t st);
int ensure_plan(crnn_model* m, int N, int W, void* ws, cudaStream_t st);
int bn_fold_moving(crnn_model* m, bool* refolded, cudaStream_t st);

static inline gemm::Params conv_params(int N, int H, int Wd, int Cin, int Cout, int block_n, const float* bias, void* out,
                                       int merged = 0) {
  gemm::Params p;
  memset(&p, 0, sizeof(p));
  p.bh = 32 / Wd;
  p.Wd = Wd; p.H = H; p.Nimg = N;
  p.sb_per_img = (H + p.bh - 1) / p.bh;
  p.num_m_tiles = (N * p.sb_per_img + 3) / 4;
  p.num_n_tiles = Cout / block_n;
  p.cin_blocks = Cin / 64;
  p.num_k_blocks = 9 * p.cin_blocks;
  p.Nc = Cout;
  p.bias = bias;
  p.out = out;
  p.merged = merged;
  return p;
}


