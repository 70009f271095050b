// Host side of libcrnnctc.so: model handle, parameter table (TF variable names/layouts), workspace plan,
// TMA tensor maps, forward orchestration.  Graph restated from lib/networks/LSTM_train.py:22-38.
#include <cstdarg>
#include <cstring>
#include <string>
#include <vector>

#include <cstdlib>
#include <condition_variable>
#include <mutex>
#include <thread>

#include "gemm_launch.h"
#include "lstm.cuh"
#include "conv_swap.cuh"
#include "conv1_tc.cuh"
#include "kernels.cuh"
#include "model_internal.h"

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[1024] = "";
int crnn_fail(int status, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return status;
}
extern "C" const char* crnn_last_error(void) { return g_err; }
extern "C" int crnn_version(void) { return 104; }
extern "C" const char* crnn_status_string(int s) {
  switch (s) {
    case CRNN_OK: return "CRNN_OK";
    case CRNN_INVALID_VALUE: return "CRNN_INVALID_VALUE";
    case CRNN_CUDA_ERROR: return "CRNN_CUDA_ERROR";
    case CRNN_NOT_BOUND: return "CRNN_NOT_BOUND";
    case CRNN_UNSUPPORTED: return "CRNN_UNSUPPORTED";
    case CRNN_WORKSPACE_TOO_SMALL: return "CRNN_WORKSPACE_TOO_SMALL";
  }
  return "CRNN_UNKNOWN";
}

extern "C" int crnn_host_is_pinned(const void* host_ptr) {
  if (!host_ptr) return 0;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, host_ptr) != cudaSuccess) { cudaGetLastError(); return 0; }
  return a.type == cudaMemoryTypeHost ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ TMA maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// 2-D bf16 map over [rows, cols] with arbitrary row stride (elements); box = [64 cols, box_rows], 128B swizzle.
int make_tmap_2d(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride,
                        uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled(2d) failed: %d", (int)r);
  return CRNN_OK;
}
int make_tmap_2d_box(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride, uint32_t box_cols,
                     uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled(2d box) failed: %d", (int)r);
  return CRNN_OK;
}
// 4-D bf16 map over NHWC [N, H, Wd, C]; box = [64 ch, Wd, bh, 1]; OOB (halo) elements read as zero.
int make_tmap_nhwc(CUtensorMap* m, const void* base, int N, int H, int Wd, int C, int bh) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Wd, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)Wd * C * 2, (cuuint64_t)H * Wd * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)Wd, (cuuint32_t)bh, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled(4d) failed: %d", (int)r);
  return CRNN_OK;
}
int make_tmap_2d_f32(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride * 4};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled(2d f32) failed: %d", (int)r);
  return CRNN_OK;
}
int make_tmap_nhwc_f32(CUtensorMap* m, const void* base, int N, int H, int Wd, int C, int bh) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Wd, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)Wd * C * 4, (cuuint64_t)H * Wd * C * 4};
  cuuint32_t box[4] = {32, (cuuint32_t)Wd, (cuuint32_t)bh, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled(4d f32) failed: %d", (int)r);
  return CRNN_OK;
}
int make_tmap_2d_u8(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride};
  cuuint32_t box[2] = {128, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled(2d u8) failed: %d", (int)r);
  return CRNN_OK;
}
int make_tmap_nhwc_u8(CUtensorMap* m, const void* base, int N, int H, int Wd, int C, int bh) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Wd, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C, (cuuint64_t)Wd * C, (cuuint64_t)H * Wd * C};
  cuuint32_t box[4] = {128, (cuuint32_t)Wd, (cuuint32_t)bh, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return crnn_fail(CRNN_CUDA_ERROR, "cuTensorMapEncodeTiled(4d u8) failed: %d", (int)r);
  return CRNN_OK;
}

static void add_tensor(crnn_model* m, const std::string& name, std::initializer_list<int64_t> shp) {
  TensorInfo t;
  t.name = name;
  t.ndim = (int)shp.size();
  t.count = 1;
  int i = 0;
  for (int k = 0; k < 4; ++k) t.shape[k] = 1;
  for (auto s : shp) { t.shape[i++] = s; t.count *= s; }
  t.offset = m->total;
  m->total += t.count;
  m->tensors.push_back(t);
}

extern "C" int crnn_model_create(const crnn_config* cfg, crnn_model** out) {
  if (!cfg || !out) return crnn_fail(CRNN_INVALID_VALUE, "model_create: null");
  if (cfg->img_height != 32 || cfg->nclasses != 64 || cfg->num_hid != 512)
    return crnn_fail(CRNN_UNSUPPORTED, "model_create: only IMG_HEIGHT=32, NCLASSES=64, NUM_HID=512 (the reference's net)");
  if (cfg->compute_dtype < 1 || cfg->compute_dtype > 4)
    return crnn_fail(CRNN_UNSUPPORTED, "model_create: compute_dtype must be 1 (bf16 operands), 2 (f32-class split-bf16 operands), 3 (tf32 "
                                       "operands) or 4 (e4m3 operands in conv3_1 .. conv5, inference only)");
  crnn_model* m = new crnn_model();
  m->cfg = *cfg;
  for (auto& c : kConvs) {
    add_tensor(m, std::string(c.name) + "/weights", {c.kh, c.kw, c.ci, c.co});
    add_tensor(m, std::string(c.name) + "/biases", {c.co});
    if (c.bn) {
      add_tensor(m, std::string(c.name) + "/" + c.name + "/beta", {c.co});
      add_tensor(m, std::string(c.name) + "/" + c.name + "/gamma", {c.co});
    }
  }
  for (const char* d : {"fw", "bw"}) {
    std::string s = std::string("logits/bidirectional_rnn/") + d + "/lstm_cell";
    add_tensor(m, s + "/weights", {768, 1024});
    add_tensor(m, s + "/biases", {1024});
  }
  add_tensor(m, "logits/weights", {512, 64});
  add_tensor(m, "logits/biases", {64});

  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    delete m;
    return crnn_fail(CRNN_CUDA_ERROR, "model_create: no CUDA device (this library has no CPU fallback)");
  }
  if (prop.major != 9) {
    delete m;
    return crnn_fail(CRNN_UNSUPPORTED, "model_create: needs sm_90 (found sm_%d%d)", prop.major, prop.minor);
  }
  m->num_sms = prop.multiProcessorCount;

  // one allocation for all derived operand copies
  const size_t nB[9] = {128 * 576, 256 * 1152, 256 * 2304, 512 * 2304, 512 * 4608, 512 * 2048, 2048 * 512, 2048 * 256, 64 * 512};
  size_t tot = 0;
  for (size_t v : nB) tot += (v * 2 + 1023) / 1024 * 1024;
  tot += 2048 * 4 + 1024;
  if (cudaMalloc(&m->wblock, tot) != cudaSuccess) { delete m; return crnn_fail(CRNN_CUDA_ERROR, "model_create: cudaMalloc"); }
  uint8_t* p = reinterpret_cast<uint8_t*>(m->wblock);
  __nv_bfloat16** dst[9] = {&m->Bc2, &m->Bc31, &m->Bc32, &m->Bc41, &m->Bc42, &m->Bc5, &m->Bx, &m->Bh, &m->Bl};
  for (int i = 0; i < 9; ++i) { *dst[i] = reinterpret_cast<__nv_bfloat16*>(p); p += (nB[i] * 2 + 1023) / 1024 * 1024; }
  m->xbias = reinterpret_cast<float*>(p); p += 2048 * 4;
  m->sumsq = reinterpret_cast<double*>(p);
  int st = CRNN_OK;
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_c2, m->Bc2, 128, 576, 576, 128);
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_c31, m->Bc31, 256, 1152, 1152, 256);
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_c32, m->Bc32, 256, 2304, 2304, 256);
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_c41, m->Bc41, 512, 2304, 2304, 256);
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_c42, m->Bc42, 512, 4608, 4608, 256);
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_c5, m->Bc5, 512, 2048, 2048, 256);
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_x, m->Bx, 2048, 512, 512, 256);
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_h128, m->Bh, 2048, 256, 256, 128);
  if (st == CRNN_OK) st = make_tmap_2d(&m->tB_l, m->Bl, 64, 512, 512, 64);
  if (st == CRNN_OK && cfg->compute_dtype == 4) st = fp8_create(m);
  if (st != CRNN_OK) { cudaFree(m->wblock); delete m; return st; }
  *out = m;
  return CRNN_OK;
}

extern "C" int crnn_model_destroy(crnn_model* m) {
  if (!m) return CRNN_OK;
  x3_destroy(m);
  fp8_destroy(m);
  if (m->wblock) cudaFree(m->wblock);
  if (m->wblock_bwd) cudaFree(m->wblock_bwd);
  if (m->wblock_bnm) cudaFree(m->wblock_bnm);
  if (m->d_peers) cudaFree(m->d_peers);
  for (auto e : m->prof_events) cudaEventDestroy(e);
  for (auto e : m->prof_events_bwd) cudaEventDestroy(e);
  for (auto e : m->chunk_events) cudaEventDestroy(e);
  delete m;
  return CRNN_OK;
}
extern "C" int crnn_num_tensors(const crnn_model* m) { return m ? (int)m->tensors.size() : 0; }
extern "C" int64_t crnn_param_count(const crnn_model* m) { return m ? m->total : 0; }
extern "C" int crnn_param_info(const crnn_model* m, int index, const char** tf_name, int64_t* offset, int64_t shape[4],
                               int* ndim) {
  if (!m || index < 0 || index >= (int)m->tensors.size()) return crnn_fail(CRNN_INVALID_VALUE, "param_info: bad index");
  const TensorInfo& t = m->tensors[index];
  if (tf_name) *tf_name = t.name.c_str();
  if (offset) *offset = t.offset;
  if (shape) for (int k = 0; k < 4; ++k) shape[k] = t.shape[k];
  if (ndim) *ndim = t.ndim;
  return CRNN_OK;
}
extern "C" int crnn_model_bind(crnn_model* m, float* params, float* grads, float* adam_m, float* adam_v) {
  if (!m || !params) return crnn_fail(CRNN_INVALID_VALUE, "model_bind: null params");
  // bias rows, the L2 sums and every solver step read and write the four buffers as float4
  CRNN_TRY(check_aligned(params, 16, "model_bind", "params"));
  CRNN_TRY(check_aligned(grads, 16, "model_bind", "grads"));
  CRNN_TRY(check_aligned(adam_m, 16, "model_bind", "adam_m"));
  CRNN_TRY(check_aligned(adam_v, 16, "model_bind", "adam_v"));
  m->params = params; m->grads = grads; m->adam_m = adam_m; m->adam_v = adam_v;
  m->dirty = true;
  m->dirty_bwd = true;
  m->bn_fold_dirty = true;
  x3_params_changed(m);
  fp8_params_changed(m);
  return CRNN_OK;
}
extern "C" int crnn_model_params_changed(crnn_model* m) {
  if (!m) return crnn_fail(CRNN_INVALID_VALUE, "null model");
  m->dirty = true;
  m->dirty_bwd = true;
  m->bn_fold_dirty = true;
  x3_params_changed(m);
  fp8_params_changed(m);
  return CRNN_OK;
}

// ---- moving BatchNorm statistics of conv4_1 / conv4_2
extern "C" int crnn_model_bind_bn_moving(crnn_model* m, float* moving, float decay) {
  if (!m) return crnn_fail(CRNN_INVALID_VALUE, "bind_bn_moving: null model");
  if (!(decay >= 0.f && decay <= 1.f)) return crnn_fail(CRNN_INVALID_VALUE, "bind_bn_moving: decay %g outside [0, 1]", (double)decay);
  CRNN_TRY(check_aligned(moving, 4, "bind_bn_moving", "moving"));
  if (m->cfg.compute_dtype == 2 || m->cfg.compute_dtype == 3)
    return crnn_fail(CRNN_UNSUPPORTED, "bind_bn_moving: moving statistics run on the bf16 and fp8 paths (compute_dtype 1, 4)");
  if (moving && !m->wblock_bnm) {
    const size_t b41 = align_up((size_t)512 * 2304 * 2), b42 = align_up((size_t)512 * 4608 * 2);
    CUDA_TRY(cudaMalloc(&m->wblock_bnm, b41 + b42 + align_up(2 * 512 * 4) + 2 * 512 * 8));
    uint8_t* p = reinterpret_cast<uint8_t*>(m->wblock_bnm);
    m->Bm41 = reinterpret_cast<__nv_bfloat16*>(p); p += b41;
    m->Bm42 = reinterpret_cast<__nv_bfloat16*>(p); p += b42;
    m->bm_bias = reinterpret_cast<float*>(p); p += align_up(2 * 512 * 4);
    m->bm_scale = reinterpret_cast<double*>(p);
    CRNN_TRY(make_tmap_2d(&m->tB_m41, m->Bm41, 512, 2304, 2304, 256));
    CRNN_TRY(make_tmap_2d(&m->tB_m42, m->Bm42, 512, 4608, 4608, 256));
  }
  m->bn_moving = moving;
  m->bn_decay = decay;
  m->bn_fold_dirty = true;
  fp8_params_changed(m);      // fp8 scales calibrated on the old statistics are stale
  return CRNN_OK;
}

extern "C" int crnn_model_set_bn_statistics(crnn_model* m, int moving) {
  if (!m) return crnn_fail(CRNN_INVALID_VALUE, "set_bn_statistics: null model");
  if (moving != 0 && moving != 1) return crnn_fail(CRNN_INVALID_VALUE, "set_bn_statistics: 0 (batch) or 1 (moving), got %d", moving);
  if (m->cfg.compute_dtype == 2 || m->cfg.compute_dtype == 3)
    return crnn_fail(CRNN_UNSUPPORTED, "set_bn_statistics: moving statistics run on the bf16 and fp8 paths (compute_dtype 1, 4)");
  if (moving && m->training)
    return crnn_fail(CRNN_INVALID_VALUE, "set_bn_statistics: a model in training mode normalises with batch statistics");
  if (m->bn_use_moving != (moving != 0)) {
    m->bn_use_moving = moving != 0;
    m->bn_fold_dirty = true;
    fp8_params_changed(m);    // the fp8 scales of a4a / a4b belong to one mode
  }
  return CRNN_OK;
}

// the folded conv4_x operands for the bound moving statistics, re-derived when params, the buffer or the mode changed
int bn_fold_moving(crnn_model* m, bool* refolded, cudaStream_t st) {
  *refolded = false;
  if (!m->bn_fold_dirty) return CRNN_OK;
  const struct { const char* n; int K; __nv_bfloat16* d; } L[2] = {{"conv4_1", 2304, m->Bm41}, {"conv4_2", 4608, m->Bm42}};
  for (int l = 0; l < 2; ++l) {
    const std::string nm(L[l].n);
    CRNN_TRY(launch_bn_fold(m->P(nm + "/weights"), L[l].K, 512, m->P(nm + "/biases"), m->P(nm + "/" + nm + "/gamma"),
                            m->P(nm + "/" + nm + "/beta"), m->bn_moving + l * 1024, m->cfg.bn_eps, L[l].d, m->bm_bias + l * 512,
                            m->bm_scale + l * 512, st));
  }
  m->bn_fold_dirty = false;
  *refolded = true;
  return CRNN_OK;
}

// f32 TF-layout parameters -> bf16 K-major GEMM operands (B[co][(kh,kw,ci)] == transpose of HWIO flattened)
int prepare_weights(crnn_model* m, cudaStream_t st) {
  struct { const char* n; __nv_bfloat16* d; int R, C; } cv[6] = {
      {"conv2/weights", m->Bc2, 576, 128},    {"conv3_1/weights", m->Bc31, 1152, 256}, {"conv3_2/weights", m->Bc32, 2304, 256},
      {"conv4_1/weights", m->Bc41, 2304, 512}, {"conv4_2/weights", m->Bc42, 4608, 512}, {"conv5/weights", m->Bc5, 2048, 512}};
  for (auto& c : cv) CRNN_TRY(launch_transpose_cast(m->P(c.n), c.R, c.C, c.C, c.d, c.R, false, st));
  const char* dirs[2] = {"logits/bidirectional_rnn/fw/lstm_cell", "logits/bidirectional_rnn/bw/lstm_cell"};
  for (int d = 0; d < 2; ++d) {
    const float* w = m->P(std::string(dirs[d]) + "/weights");                 // [768,1024], rows [x(512); h(256)]
    CRNN_TRY(launch_transpose_cast(w, 512, 1024, 1024, m->Bx + (size_t)d * 1024 * 512, 512, true, st));
    CRNN_TRY(launch_transpose_cast(w + 512 * 1024, 256, 1024, 1024, m->Bh + (size_t)d * 1024 * 256, 256, true, st));
  }
  CRNN_TRY(launch_lstm_bias_prep(m->P(std::string(dirs[0]) + "/biases"), m->P(std::string(dirs[1]) + "/biases"), m->xbias, st));
  CRNN_TRY(launch_transpose_cast(m->P("logits/weights"), 512, 64, 64, m->Bl, 512, false, st));
  // L2 term depends only on the parameters: computed here, consumed by crnn_total_loss
  SumsqSegs segs;
  segs.n = 0;
  for (auto& c : kConvs) {
    const TensorInfo* t = m->find(std::string(c.name) + "/weights");
    segs.off[segs.n] = t->offset; segs.cnt[segs.n] = t->count; segs.n++;
  }
  const TensorInfo* t = m->find("logits/weights");
  segs.off[segs.n] = t->offset; segs.cnt[segs.n] = t->count; segs.n++;
  CRNN_TRY(launch_sumsq(m->params, segs, m->sumsq, st));
  m->dirty = false;
  return CRNN_OK;
}

// ------------------------------------------------------------------------------------------------ workspace
size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// `lines` (crnn_forward_lines, inference only): the packed-line region past the inference layout -- line widths [N] i32, then, unless
// conv4_x normalise with the `moving` statistics, per-line statistics [2][N][2][512] f64 and coefficients [2][N][4][512] f32
size_t layout_plan(Plan& pl, int N, int W, uint8_t* base, bool train, bool lines, bool moving) {
  pl.N = N; pl.W = W; pl.H1 = W / 2; pl.H2 = W / 4; pl.T = W / 4 - 1;
  pl.Npad = (N + 127) / 128 * 128;
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* p = base ? base + off : nullptr; off += align_up(bytes); return p; };
  const size_t n = N, h1 = pl.H1, h2 = pl.H2;
  pl.a1 = (__nv_bfloat16*)take(n * h1 * 16 * 64 * 2);
  pl.a2 = (__nv_bfloat16*)take(n * h2 * 8 * 128 * 2);
  pl.a3 = (__nv_bfloat16*)take(n * h2 * 8 * 256 * 2);
  pl.a3p = (__nv_bfloat16*)take(n * h2 * 4 * 256 * 2);
  pl.a4a_pre = (__nv_bfloat16*)take(n * h2 * 4 * 512 * 2);
  pl.a4a = (__nv_bfloat16*)take(n * h2 * 4 * 512 * 2);
  pl.a4b_pre = (__nv_bfloat16*)take(n * h2 * 4 * 512 * 2);
  pl.a4b = (__nv_bfloat16*)take(n * h2 * 2 * 512 * 2);
  pl.a5 = (__nv_bfloat16*)take(n * h2 * 512 * 2);
  pl.xproj = (__nv_bfloat16*)take(n * h2 * 2048 * 2);
  pl.lstm_out = (__nv_bfloat16*)take(n * h2 * 512 * 2);
  pl.h_state = (__nv_bfloat16*)take((size_t)2 * 2 * pl.Npad * 256 * 2);
  pl.stats = (double*)take(2 * 2 * 512 * 8);
  pl.bn = (float*)take(2 * 4 * 512 * 4);
  pl.line_w = lines ? (int*)take(n * 4) : nullptr;
  pl.stats_l = lines && !moving ? (double*)take(2 * n * 2 * 512 * 8) : nullptr;
  pl.bn_l = lines && !moving ? (float*)take(2 * n * 4 * 512 * 4) : nullptr;
  pl.train = train;
  if (train) {
    const size_t T = pl.T;
    pl.am1 = (uint8_t*)take(n * h1 * 16 * 64);
    pl.am2 = (uint8_t*)take(n * h2 * 8 * 128);
    pl.am3 = (uint8_t*)take(n * h2 * 4 * 256);
    pl.gates = (__nv_bfloat16*)take((size_t)2 * pl.Npad * T * 1024 * 2);     // per 128-row batch tile (common.cuh: lstm_gate_off)
    pl.csave = (float*)take((size_t)2 * pl.Npad * T * 256 * 4);
    pl.dl_rows = (__nv_bfloat16*)take(n * h2 * 64 * 2);
    pl.d_lstm_out = (__nv_bfloat16*)take(n * h2 * 512 * 2);
    pl.dz_all = (__nv_bfloat16*)take(n * h2 * 2048 * 2);
    pl.bptt_x = (uint8_t*)take((size_t)2 * (2 * pl.Npad / 128) * 64 * 8192);
    pl.d_a5 = (__nv_bfloat16*)take(n * h2 * 512 * 2);
    pl.d_a4b = (__nv_bfloat16*)take(n * h2 * 2 * 512 * 2);
    pl.d_pre4b = (__nv_bfloat16*)take(n * h2 * 4 * 512 * 2);
    pl.d_pre4a = (__nv_bfloat16*)take(n * h2 * 4 * 512 * 2);
    pl.d_a3p = (__nv_bfloat16*)take(n * h2 * 4 * 256 * 2);
    pl.d_pre32 = (__nv_bfloat16*)take(n * h2 * 8 * 256 * 2);
    pl.d_pre31 = (__nv_bfloat16*)take(n * h2 * 8 * 256 * 2);
    pl.d_a2 = (__nv_bfloat16*)take(n * h2 * 8 * 128 * 2);
    pl.d_pre2 = (__nv_bfloat16*)take(n * h1 * 16 * 128 * 2);
    pl.d_a1 = (__nv_bfloat16*)take(n * h1 * 16 * 64 * 2);
    pl.bn_bwd_sums = (double*)take(4 * 2 * 512 * 8);      // [local | global-batch] x [2 layers][2][512]
    pl.bn_bwd_coef = (float*)take(3 * 512 * 4);
  }
  return off;
}

extern "C" int crnn_model_workspace_size(const crnn_model* m, int N, int W, int train, size_t* bytes) {
  if (!m || !bytes) return crnn_fail(CRNN_INVALID_VALUE, "workspace_size: null");
  if (N <= 0 || W < 8 || (W % 4) != 0) return crnn_fail(CRNN_INVALID_VALUE, "workspace_size: need N>0, W>=8, W%%4==0 (gen.py:58)");
  if (m->cfg.compute_dtype == 4 && train) return crnn_fail(CRNN_UNSUPPORTED, "workspace_size: the fp8 path (compute_dtype 4) is inference only");
  if (m->cfg.compute_dtype == 2 || m->cfg.compute_dtype == 3) {
    if (train) return crnn_fail(CRNN_UNSUPPORTED, "workspace_size: the f32-class paths (compute_dtype 2, 3) are forward + CTC only");
    *bytes = x3_workspace_size(N, W);
    return CRNN_OK;
  }
  Plan pl;
  *bytes = layout_plan(pl, N, W, nullptr, train != 0);
  return CRNN_OK;
}

static int build_plan(crnn_model* m, int N, int W, void* ws, cudaStream_t st) {
  Plan& pl = m->plan;
  layout_plan(pl, N, W, reinterpret_cast<uint8_t*>(ws), m->training);
  pl.ws = ws;
  pl.mg2 = (pl.H1 % 8) == 0; pl.mg3 = (pl.H2 % 16) == 0; pl.mg4 = (pl.H2 % 32) == 0;
  pl.wm2 = (pl.H1 % 4) == 0; pl.wm3 = (pl.H2 % 8) == 0; pl.wm4 = (pl.H2 % 16) == 0;
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c2s, pl.a1, N, pl.H1, 16, 64, 8));
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c31, pl.a2, N, pl.H2, 8, 128, pl.mg3 ? 16 : 4));
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c32, pl.a3, N, pl.H2, 8, 256, pl.mg3 ? 16 : 4));
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c41, pl.a3p, N, pl.H2, 4, 256, pl.mg4 ? 32 : 8));
  CRNN_TRY(make_tmap_nhwc(&pl.tA_c42, pl.a4a, N, pl.H2, 4, 512, pl.mg4 ? 32 : 8));
  // conv5 (2x2 VALID over [N,H2,2,512]): output (n,t) = rows n*H2+t and n*H2+t+1 of the [N*H2, 1024] view
  CRNN_TRY(make_tmap_2d(&pl.tA_c5, pl.a4b, (uint64_t)N * pl.H2, 1024, 1024, 128));
  CRNN_TRY(make_tmap_2d(&pl.tA_x, pl.a5, (uint64_t)N * pl.H2, 512, 512, 128));
  CRNN_TRY(make_tmap_2d(&pl.tA_l, pl.lstm_out, (uint64_t)N * pl.H2, 512, 512, 128));
  CRNN_TRY(make_tmap_nhwc(&pl.tO_c1, pl.a1, N, pl.H1, 16, 64, 4));               // conv1_tc_kernel's pooled warpgroup tile: 4 pooled rows
  CRNN_TRY(make_tmap_nhwc(&pl.tO_c2s, pl.a2, N, pl.H2, 8, 128, 8));             // conv2_swap_kernel's pooled tile: 8 pooled rows
  CRNN_TRY(make_tmap_nhwc(&pl.tO_c32, pl.a3p, N, pl.H2, 4, 256, pl.mg3 ? 16 : 4));     // conv3_2's pooled tile: 64 positions
  CRNN_TRY(make_tmap_nhwc(&pl.tO_c41, pl.a4a_pre, N, pl.H2, 4, 512, pl.mg4 ? 32 : 8));
  CRNN_TRY(make_tmap_nhwc(&pl.tO_c42, pl.a4b_pre, N, pl.H2, 4, 512, pl.mg4 ? 32 : 8));
  CRNN_TRY(make_tmap_nhwc(&pl.tO_m42, pl.a4b, N, pl.H2, 2, 512, pl.mg4 ? 32 : 8));     // moving statistics: conv4_2's pooled tile
  CRNN_TRY(make_tmap_2d(&pl.tO_x, pl.xproj, (uint64_t)N * pl.H2, 2048, 2048, 128));
  if (m->cfg.compute_dtype == 4) CRNN_TRY(fp8_plan_maps(pl));
  if (pl.train) {
    const uint64_t R = (uint64_t)N * pl.H2;
    // K-major A operands (box = [64 K-elements, 128 rows])
    CRNN_TRY(make_tmap_2d(&pl.tG_dl, pl.dl_rows, R, 64, 64, 128));
    CRNN_TRY(make_tmap_2d(&pl.tG_dz, pl.dz_all, R, 2048, 2048, 128));
    CRNN_TRY(make_tmap_2d(&pl.tG_da5, pl.d_a5, R, 512, 512, 128));
    CRNN_TRY(make_tmap_nhwc(&pl.tG_p4b, pl.d_pre4b, N, pl.H2, 4, 512, pl.mg4 ? 32 : 8));
    CRNN_TRY(make_tmap_nhwc(&pl.tG_p4a, pl.d_pre4a, N, pl.H2, 4, 512, pl.mg4 ? 32 : 8));
    CRNN_TRY(make_tmap_nhwc(&pl.tG_p32, pl.d_pre32, N, pl.H2, 8, 256, pl.mg3 ? 16 : 4));
    CRNN_TRY(make_tmap_nhwc(&pl.tG_p2s, pl.d_pre2, N, pl.H1, 16, 128, 8));
    CRNN_TRY(make_tmap_nhwc(&pl.tG_p31s, pl.d_pre31, N, pl.H2, 8, 256, 16));
    CRNN_TRY(make_tmap_2d(&pl.tO_dlo, pl.d_lstm_out, R, 512, 512, 128));
    CRNN_TRY(make_tmap_2d(&pl.tO_da4b, pl.d_a4b, R, 1024, 1024, 128));
    CRNN_TRY(make_tmap_nhwc(&pl.tO_da3p, pl.d_a3p, N, pl.H2, 4, 256, pl.mg4 ? 32 : 8));
    // weight-gradient (TN_CONV) views: 64-position boxes when two sub-boxes are contiguous rows of one image, else 32
    CRNN_TRY(make_tmap_nhwc(&pl.tW_a1, pl.a1, N, pl.H1, 16, 64, pl.wm2 ? 4 : 2));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_p2, pl.d_pre2, N, pl.H1, 16, 128, pl.wm2 ? 4 : 2));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_a2, pl.a2, N, pl.H2, 8, 128, pl.wm3 ? 8 : 4));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_p31, pl.d_pre31, N, pl.H2, 8, 256, pl.wm3 ? 8 : 4));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_a3, pl.a3, N, pl.H2, 8, 256, pl.wm3 ? 8 : 4));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_p32, pl.d_pre32, N, pl.H2, 8, 256, pl.wm3 ? 8 : 4));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_a3p, pl.a3p, N, pl.H2, 4, 256, pl.wm4 ? 16 : 8));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_p4a, pl.d_pre4a, N, pl.H2, 4, 512, pl.wm4 ? 16 : 8));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_a4a, pl.a4a, N, pl.H2, 4, 512, pl.wm4 ? 16 : 8));
    CRNN_TRY(make_tmap_nhwc(&pl.tW_p4b, pl.d_pre4b, N, pl.H2, 4, 512, pl.wm4 ? 16 : 8));
    // MN-major (TN) operands: box = [64 channels, 64 rows]
    CRNN_TRY(make_tmap_2d_box(&pl.tT_lstm_all, pl.lstm_out, R, 512, 512, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_lstm_fw, pl.lstm_out, R, 256, 512, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_lstm_bw, pl.lstm_out + 256, R, 256, 512, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_dl, pl.dl_rows, R, 64, 64, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_a5, pl.a5, R, 512, 512, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_dz, pl.dz_all, R, 2048, 2048, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_dz_fw, pl.dz_all, R, 1024, 2048, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_dz_bw, pl.dz_all + 1024, R, 1024, 2048, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_a4b, pl.a4b, R, 1024, 1024, 64, 64));
    CRNN_TRY(make_tmap_2d_box(&pl.tT_da5, pl.d_a5, R, 512, 512, 64, 64));
  }
  return CRNN_OK;
}

int ensure_plan(crnn_model* m, int N, int W, void* ws, cudaStream_t st) {
  Plan& pl = m->plan;
  if (pl.N != N || pl.W != W || pl.ws != ws || pl.train != m->training) return build_plan(m, N, W, ws, st);
  return CRNN_OK;
}

// ---- host-side copy pool (crnn_forward_pageable): a pageable numpy batch has to be moved into page-locked staging before it can
// be DMA'd; one host thread alone takes longer for the 33.6 MB of a batch than the whole GPU step.  A few persistent workers split every
// copy; the caller copies one share itself and waits for the rest.
namespace {
class CopyPool {
 public:
  static CopyPool& get() { static CopyPool* p = new CopyPool(); return *p; }   // leaked on purpose: workers may outlive static destructors
  void copy(void* dst, const void* src, size_t bytes, int threads) {
    if (threads > kMax + 1) threads = kMax + 1;
    if (threads < 2 || bytes < (1u << 20)) { memcpy(dst, src, bytes); return; }
    std::unique_lock<std::mutex> call_lock(call_mu_);                // one copy at a time
    ensure(threads - 1);
    const size_t share = ((bytes / threads) + 4095) & ~size_t(4095);
    {
      std::lock_guard<std::mutex> lk(mu_);
      dst_ = static_cast<uint8_t*>(dst); src_ = static_cast<const uint8_t*>(src); bytes_ = bytes; share_ = share;
      active_ = threads - 1; pending_ = threads - 1; ++gen_;
    }
    cv_.notify_all();
    const size_t own = (size_t)(threads - 1) * share;               // the caller takes the last share
    if (own < bytes) memcpy(static_cast<uint8_t*>(dst) + own, static_cast<const uint8_t*>(src) + own, bytes - own);
    std::unique_lock<std::mutex> lk(mu_);
    done_.wait(lk, [&] { return pending_ == 0; });
  }

 private:
  static constexpr int kMax = 15;
  void ensure(int n) {
    while ((int)workers_.size() < n) {
      const int id = (int)workers_.size();
      workers_.emplace_back([this, id] { run(id); });
      workers_.back().detach();
    }
  }
  void run(int id) {
    uint64_t seen = 0;
    for (;;) {
      uint8_t* d; const uint8_t* s; size_t n, share;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        if (id >= active_) continue;
        d = dst_; s = src_; n = bytes_; share = share_;
      }
      const size_t b = (size_t)id * share;
      if (b < n) memcpy(d + b, s + b, (b + share <= n) ? share : n - b);
      {
        std::lock_guard<std::mutex> lk(mu_);
        if (--pending_ == 0) done_.notify_one();
      }
    }
  }
  std::mutex mu_, call_mu_;
  std::condition_variable cv_, done_;
  std::vector<std::thread> workers_;
  uint8_t* dst_ = nullptr; const uint8_t* src_ = nullptr;
  size_t bytes_ = 0, share_ = 0;
  int active_ = 0, pending_ = 0;
  uint64_t gen_ = 0;
};
}  // namespace

// The events of the host-fed forwards' copy handshake, created on first use: [c] = image range c copied (recorded on the copy
// stream), [kMaxChunks] = the work queued on the compute stream before the copies (it may still read the staging tensor).
static int ensure_chunk_events(crnn_model* m) {
  if (m->chunk_events.empty()) {
    m->chunk_events.resize(kMaxChunks + 1);
    for (auto& e : m->chunk_events) CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  return CRNN_OK;
}

// One forward call: where its batch lies and how it is computed.
//   host == nullptr (crnn_forward, crnn_forward_lines, calibration): `data` is the batch on the device.
//   host != nullptr, pageable == nullptr (crnn_forward_host): the batch is in page-locked host memory; it is copied to `data` on
//     `copy_st` in `chunks` image ranges, each range's front end starting once its copy has landed.
//   pageable != nullptr (crnn_forward_pageable): the batch is in ordinary host memory; the copy pool (`host_threads`) moves each range
//     into the page-locked staging `host` first.
//   line_width != nullptr (crnn_forward_lines): every image is a line evaluated as if alone.
//   u8 (the crnn_*_u8 twins): the batch holds uint8 pixels, one byte per element instead of four.
// The precision is the model's (bf16 or, compute_dtype 4, e4m3); `calib` (crnn_model_calibrate_fp8) runs the bf16 front end up to
// conv4_2's BatchNorm, then reduces the fp8 scales.
struct FwdCall {
  const void* data = nullptr;
  const void* host = nullptr;
  const void* pageable = nullptr;
  int host_threads = 1, chunks = 1;
  bool u8 = false;
  cudaStream_t copy_st = nullptr;
  const int* line_width = nullptr;
  bool calib = false;
  // bytes of n images of width W, and image n of one of the batch pointers
  size_t bytes(size_t n, int W) const { return n * W * 32 * (u8 ? 1 : sizeof(float)); }
  uint8_t* at(const void* base, size_t n, int W) const {
    return const_cast<uint8_t*>(static_cast<const uint8_t*>(base)) + bytes(n, W);
  }
};

// The batch in image ranges of `nc`: `compute(n0, n1)` queues range [n0, n1)'s work on `st`.  A host-fed batch reaches the device on
// `copy_st`: the copies wait for the work queued earlier on `st` (it may still read the staging tensor), and `st` waits for range c's
// copy before range c's work.  From page-locked memory every range's DMA is queued before the first range's work; from pageable memory
// the host copy of range c + 1 overlaps the GPU work on range c.  So the host buffers may be reused once the work queued on `copy_st`
// has completed, and a graph captured on `st` takes the copies in.
template <class F>
static int for_each_range(crnn_model* m, const FwdCall& a, int N, int W, int nc, cudaStream_t st, F&& compute) {
  const bool fed = a.host != nullptr;
  auto copy = [&](int c) -> int {
    const int n0 = c * nc, n = (n0 + nc < N) ? nc : N - n0;
    if (a.pageable != nullptr) CopyPool::get().copy(a.at(a.host, n0, W), a.at(a.pageable, n0, W), a.bytes(n, W), a.host_threads);
    CUDA_TRY(cudaMemcpyAsync(a.at(a.data, n0, W), a.at(a.host, n0, W), a.bytes(n, W), cudaMemcpyHostToDevice, a.copy_st));
    CUDA_TRY(cudaEventRecord(m->chunk_events[c], a.copy_st));
    return CRNN_OK;
  };
  if (fed) {
    CRNN_TRY(ensure_chunk_events(m));
    CUDA_TRY(cudaEventRecord(m->chunk_events[kMaxChunks], st));
    CUDA_TRY(cudaStreamWaitEvent(a.copy_st, m->chunk_events[kMaxChunks], 0));
  }
  for (int c = 0; fed && a.pageable == nullptr && c * nc < N; ++c) CRNN_TRY(copy(c));
  for (int c = 0; c * nc < N; ++c) {
    if (fed && a.pageable != nullptr) CRNN_TRY(copy(c));
    if (fed) CUDA_TRY(cudaStreamWaitEvent(st, m->chunk_events[c], 0));
    const int n0 = c * nc;
    CRNN_TRY(compute(n0, (n0 + nc < N) ? n0 + nc : N));
  }
  return CRNN_OK;
}

// The BiLSTM recurrence: ONE persistent launch, a cluster of 8 CTAs per (direction, 128-sample tile) -- csrc/lstm.cuh.
// CRNN_LSTM_TRACE=1 records a debug timeline and prints it to stderr after every launch (tools/lstm_trace.py reads it).
static int launch_lstm_forward(crnn_model* m, const int* time_step_len, cudaStream_t st) {
  constexpr int CS = 8;
  const Plan& pl = m->plan;
  lstm::Params lp;
  lp.xproj = pl.xproj; lp.h_state = pl.h_state; lp.lstm_out = pl.lstm_out; lp.seq_len = time_step_len;
  lp.Nimg = pl.N; lp.Npad = pl.Npad; lp.H = pl.H2; lp.T = pl.T; lp.tiles_per_dir = pl.Npad / 128;
  lp.gates = pl.train ? pl.gates : nullptr; lp.csave = pl.train ? pl.csave : nullptr;
  static long long* d_trace = nullptr;
  const bool want_trace = getenv("CRNN_LSTM_TRACE") != nullptr;
  if (want_trace && d_trace == nullptr) CUDA_TRY(cudaMalloc(&d_trace, 2 * 2 * 4 * 16 * sizeof(long long)));
  if (want_trace) CUDA_TRY(cudaMemsetAsync(d_trace, 0, 2 * 2 * 4 * 16 * sizeof(long long), st));
  lp.trace = want_trace ? d_trace : nullptr;
  auto kern = lstm::lstm_mc_kernel<CS>;
  static bool attr = false;
  if (!attr) {
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lstm::CfgMc<CS>::SMEM_BYTES));
    attr = true;
  }
  CRNN_TRY(launch_cluster(kern, CS, CS * 2 * lp.tiles_per_dir, lstm::MC_THREADS, lstm::CfgMc<CS>::SMEM_BYTES, st, m->tB_h128, lp));
  if (want_trace) {
    long long h[2 * 2 * 4 * 16];            // [CTA 0 / 5][warpgroup slot][step 8..11][event]
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaMemcpy(h, d_trace, sizeof(h), cudaMemcpyDeviceToHost));
    for (int c = 0; c < 2; ++c) {
      long long t0 = 0;                       // earliest stamp of the CTA: both warpgroups on one time axis
      for (int i = c * 128; i < (c + 1) * 128; ++i)
        if (h[i] && (!t0 || h[i] < t0)) t0 = h[i];
      for (int wg = 0; wg < 2; ++wg)
        for (int s = 0; s < 4; ++s) {
          const long long* r = h + ((c * 2 + wg) * 4 + s) * 16;
          bool any = false;
          for (int e = 0; e < 16; ++e) any = any || r[e];
          if (!any) continue;
          fprintf(stderr, "lstm_trace cta%d wg%d step%d:", c ? 5 : 0, wg, 8 + s);
          for (int e = 0; e < 12; ++e) fprintf(stderr, " %lld", r[e] ? r[e] - t0 : -1);
          fprintf(stderr, "\n");
        }
    }
  }
  return CRNN_OK;
}

// The forward pass of every entry point (FwdCall).  A chunked front end (crnn_forward_host / _pageable) runs the batch-independent
// conv1 .. conv3_2 + pools per image range, so the copy (33.6 MB at batch 1024 x 32x256) hides behind that compute instead of
// preceding it; from conv4_1 on (batch-statistics BatchNorm) the batch is processed whole.  Packed lines: the conv epilogues zero each
// activation past the line's width and conv4_x use per-line batch statistics.  compute_dtype 4 runs conv3_1 .. conv5 on e4m3 operands
// (forward_fp8.cu); it and the f32-class paths (forward_x3.cu) copy a host-fed batch whole, then compute.
static int forward(crnn_model* m, FwdCall a, const int* time_step_len, int N, int W, float* logits_out, void* workspace,
                   size_t workspace_bytes, crnn_stream_t stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool calib = a.calib, fp8 = m && m->cfg.compute_dtype == 4 && !calib;
  if (!m || !a.data || !time_step_len || (!logits_out && !calib) || !workspace) return crnn_fail(CRNN_INVALID_VALUE, "forward: null pointer");
  // conv1 loads f32 pixels as float4 and the logits epilogues store float4 (the uint8 twins check their 4-byte rule first)
  if (!a.u8) CRNN_TRY(check_aligned(a.data, 16, "forward", a.host ? "data_staging" : "data"));
  CRNN_TRY(check_aligned(logits_out, 16, "forward", "logits_out"));
  if (!m->params) return crnn_fail(CRNN_NOT_BOUND, "forward: call crnn_model_bind first");
  const bool moving = m->bn_use_moving && !m->training;     // training forwards always normalise with batch statistics
  if (moving && !m->bn_moving)
    return crnn_fail(CRNN_NOT_BOUND, "forward: moving BatchNorm statistics selected but no buffer bound (crnn_model_bind_bn_moving)");
  if (N <= 0 || W < 8 || (W % 4) != 0) return crnn_fail(CRNN_INVALID_VALUE, "forward: need N>0, W>=8, W%%4==0");
  size_t need = 0;
  CRNN_TRY(crnn_model_workspace_size(m, N, W, m->training ? 1 : 0, &need));
  if (workspace_bytes < need) return crnn_fail(CRNN_WORKSPACE_TOO_SMALL, "forward: workspace %zu < %zu", workspace_bytes, need);
  if ((reinterpret_cast<uintptr_t>(workspace) & 1023) != 0) return crnn_fail(CRNN_INVALID_VALUE, "forward: workspace must be 1024-byte aligned");
  if (fp8 || calib) {
    if (fp8 && !fp8_calibrated(m))
      return crnn_fail(CRNN_INVALID_VALUE, "forward: the fp8 model (compute_dtype 4) has no activation scales: calibration is missing "
                                           "(crnn_model_calibrate_fp8 or crnn_model_set_fp8_scales after the last parameter change)");
    if (m->dp_world > 1) return crnn_fail(CRNN_UNSUPPORTED, "forward: the fp8 path runs on one device (no data parallelism)");
  }
  const bool x3 = m->cfg.compute_dtype == 2 || m->cfg.compute_dtype == 3;
  if (fp8 || calib || x3) {
    // copy-then-compute: the whole batch as one range, no work in it
    CRNN_TRY(for_each_range(m, a, N, W, N, st, [](int, int) -> int { return CRNN_OK; }));
    a.host = a.pageable = nullptr;
    a.chunks = 1;
  }
  if (x3) return x3_forward(m, a.data, a.u8, time_step_len, N, W, logits_out, workspace, workspace_bytes, st);
  if (m->dirty) CRNN_TRY(prepare_weights(m, st));
  if (fp8) CRNN_TRY(fp8_prepare(m, st));
  if (moving) {
    bool refolded = false;
    CRNN_TRY(bn_fold_moving(m, &refolded, st));
    if (fp8) CRNN_TRY(fp8_fold_moving(m, refolded, st));
  }
  Plan& pl = m->plan;
  CRNN_TRY(ensure_plan(m, N, W, workspace, st));
  const bool lines = a.line_width != nullptr;
  layout_plan(pl, N, W, reinterpret_cast<uint8_t*>(workspace), pl.train, lines, moving);    // this call's packed-line region, or none
  pl.moving = moving;
  const int H1 = pl.H1, H2 = pl.H2, sms = m->num_sms;
  if (lines) CRNN_TRY(launch_clamp_line_width(a.line_width, pl.line_w, N, W, st));
  cudaEvent_t* ev = nullptr;
  if (!calib && m->prof_on && m->prof_used < m->prof_slots) ev = &m->prof_events[(size_t)(m->prof_used++) * (kNumStages + 1)];
  int evi = 0;
#define STAGE_MARK() do { if (ev) CUDA_TRY(cudaEventRecord(ev[evi++], st)); } while (0)
  STAGE_MARK();

  // ---- front end, per image range [n0, n1): conv1+pool1, conv2+pool2, conv3_1, conv3_2+pool (all batch-independent)
  const int sb3 = (H2 + 3) / 4;                      // 32-position sub-boxes per image of the conv3 layers (Wd = 8 -> 4 H rows)
  const int sb2 = (H1 + 1) / 2;                      // the same at conv2's input resolution (Wd = 16 -> 2 H rows)
  int chunks = a.chunks < 1 ? 1 : a.chunks > kMaxChunks ? kMaxChunks : a.chunks;
  int nc = (N + chunks - 1) / chunks;
  // a range must start on a tile-PAIR boundary of every layer (128-position tiles = 4 sub-boxes, pairs = 8)
  if (chunks > 1 && ((nc * sb3) % 8 != 0 || (nc * sb2) % 8 != 0)) { chunks = 1; nc = N; }
  CRNN_TRY(for_each_range(m, a, N, W, nc, st, [&](int n0, int n1) -> int {
    const int cn = n1 - n0;
    const bool mark = (n1 == N) && chunks == 1;      // per-stage events only make sense for an unchunked front end
    // conv1 + pool1 (tensor cores, split-bf16 operands: conv1_tc.cuh)
    {
      const size_t o1 = (size_t)n0 * H1 * 16 * 64;
      CRNN_TRY(launch_conv1_tc(pl.tO_c1, a.at(a.data, n0, W), a.u8, m->P("conv1/weights"), m->P("conv1/biases"), n0,
                               pl.train ? pl.am1 + o1 : nullptr, cn, W, sms, st, pl.line_w));
    }
    if (mark) STAGE_MARK();
    // conv2 + ReLU + pool2
    {
      convsw::Params p;
      p.Nimg = cn; p.img0 = n0; p.H = H1; p.tiles_per_img = (H1 + 15) / 16; p.bias = m->P("conv2/biases"); p.out = pl.a2;
      p.argmax = pl.train ? pl.am2 : nullptr;
      p.line_w = pl.line_w;
      if (fp8) CRNN_TRY(fp8_conv2(m, p, lines, sms, st));
      else if (pl.train) CRNN_TRY(launch_conv2_swap<true>(pl.tA_c2s, m->tB_c2, pl.tO_c2s, p, sms, st));
      else CRNN_TRY(launch_conv2_swap_lines(lines, pl.tA_c2s, m->tB_c2, pl.tO_c2s, p, sms, st));
    }
    if (mark) STAGE_MARK();
    // conv3_1 + ReLU
    {
      gemm::Params p = conv_params(N, H2, 8, 128, 256, 256, m->P("conv3_1/biases"), pl.a3, pl.mg3);
      if (chunks > 1) { p.m_tile0 = n0 * sb3 / 4; p.num_m_tiles = cn * sb3 / 4; }
      p.line_w = pl.line_w;
      if (fp8) CRNN_TRY(fp8_conv_gemm(m, 0, p, lines, sms, st));
      else CRNN_TRY((launch_gemm_lines<256, gemm::A_CONV3, gemm::EPI_RELU, 4>(lines, pl.tA_c31, m->tB_c31, p, sms, st, &pl.tA_c32)));
    }
    if (mark) STAGE_MARK();
    // conv3_2 + ReLU + height pool
    {
      gemm::Params p = conv_params(N, H2, 8, 256, 256, 256, m->P("conv3_2/biases"), pl.a3p, pl.mg3);
      if (chunks > 1) { p.m_tile0 = n0 * sb3 / 4; p.num_m_tiles = cn * sb3 / 4; }
      if (pl.train) {
        p.argmax = pl.am3;
        CRNN_TRY((launch_gemm<256, gemm::A_CONV3, gemm::EPI_RELU_POOL12_T, 4>(pl.tA_c32, m->tB_c32, p, sms, st)));
      } else {
        p.line_w = pl.line_w;
        if (fp8) CRNN_TRY(fp8_conv_gemm(m, 1, p, lines, sms, st));
        else CRNN_TRY((launch_gemm_lines<256, gemm::A_CONV3, gemm::EPI_RELU_POOL12, 4>(lines, pl.tA_c32, m->tB_c32, p, sms, st, &pl.tO_c32)));
      }
    }
    if (mark) STAGE_MARK();
    return CRNN_OK;
  }));
  if (chunks > 1) for (int i = 0; i < 4; ++i) STAGE_MARK();     // keep the event layout (front-end stages read as ~0)

  // ---- conv4_1 + BN + ReLU, conv4_2 + BN + ReLU + pool3, each a GEMM, a BatchNorm finalize and an apply.  The statistics are the
  // batch's (over the GLOBAL batch when it is sharded over ranks: the exchange is fused into the finalize kernel) or each line's own.
  // With the moving statistics the BatchNorm is folded into the weights and bias: conv4_1 + BN + ReLU is conv3_1's EPI_RELU GEMM,
  // conv4_2 + BN + ReLU + pool3 conv3_2's EPI_RELU_POOL12 GEMM, and the finalize and apply do not run (their events read ~0).
  const struct { const char* name; int cin; const CUtensorMap *tA, *tB, *tO, *tB_m, *tO_m; __nv_bfloat16 *pre, *out; } L[2] = {
      {"conv4_1", 256, &pl.tA_c41, &m->tB_c41, &pl.tO_c41, &m->tB_m41, &pl.tA_c42, pl.a4a_pre, pl.a4a},
      {"conv4_2", 512, &pl.tA_c42, &m->tB_c42, &pl.tO_c42, &m->tB_m42, &pl.tO_m42, pl.a4b_pre, pl.a4b}};
  double* const stats = lines ? pl.stats_l : pl.stats;              // [2 layers][N or 1][2][512]
  float* const bn_all = lines ? pl.bn_l : pl.bn;                    // [2 layers][N or 1][4][512]
  const size_t per_layer = lines ? (size_t)N * 512 : 512;
  if (!moving) CUDA_TRY(cudaMemsetAsync(stats, 0, 2 * per_layer * 2 * sizeof(double), st));
  for (int l = 0; l < 2; ++l) {
    const std::string nm(L[l].name);
    gemm::Params p = conv_params(N, H2, 4, L[l].cin, 512, 256, moving ? m->bm_bias + l * 512 : m->P(nm + "/biases"),
                                 moving ? L[l].out : L[l].pre, pl.mg4);
    p.line_w = pl.line_w;
    if (!moving) p.stats = stats + l * per_layer * 2;
    if (fp8) CRNN_TRY(fp8_conv_gemm(m, 2 + l, p, lines, sms, st, moving));
    else if (moving && l == 0) CRNN_TRY((launch_gemm_lines<256, gemm::A_CONV3, gemm::EPI_RELU, 4>(lines, *L[0].tA, *L[0].tB_m, p, sms, st, L[0].tO_m)));
    else if (moving) CRNN_TRY((launch_gemm_lines<256, gemm::A_CONV3, gemm::EPI_RELU_POOL12, 4>(lines, *L[1].tA, *L[1].tB_m, p, sms, st, L[1].tO_m)));
    else CRNN_TRY((launch_gemm_lines<256, gemm::A_CONV3, gemm::EPI_STATS, 4>(lines, *L[l].tA, *L[l].tB, p, sms, st, L[l].tO)));
    STAGE_MARK();
    if (!moving) {
      float* bn = bn_all + l * per_layer * 4;
      const float *gamma = m->P(nm + "/" + nm + "/gamma"), *beta = m->P(nm + "/" + nm + "/beta");
      const double bn_count = (double)N * H2 * 4;
      if (lines) CRNN_TRY(launch_bn_finalize_lines(p.stats, pl.line_w, gamma, beta, m->cfg.bn_eps, bn, N, 512, st));
      else if (m->dp_world > 1) CRNN_TRY(dp_allreduce_bn_finalize(m, p.stats, bn_count * m->dp_world, gamma, beta, m->cfg.bn_eps, bn, st));
      else CRNN_TRY(launch_bn_finalize(p.stats, bn_count, gamma, beta, m->cfg.bn_eps, bn, bn + 512, bn + 1024, bn + 1536, 512, st));
      if (fp8) CRNN_TRY(fp8_bn_apply(m, l, bn, lines, st));
      else if (lines && l == 0) CRNN_TRY(launch_bn_apply_relu_lines(pl.a4a_pre, pl.a4a, bn, pl.line_w, N, H2, 4, 512, st));
      else if (lines) CRNN_TRY(launch_bn_apply_relu_pool12_lines(pl.a4b_pre, pl.a4b, bn, pl.line_w, N, H2, 2, 512, st));
      else if (l == 0) CRNN_TRY(launch_bn_apply_relu(pl.a4a_pre, pl.a4a, bn, bn + 512, (size_t)N * H2 * 4, 512, st));
      else CRNN_TRY(launch_bn_apply_relu_pool12(pl.a4b_pre, pl.a4b, bn, bn + 512, (size_t)N * H2 * 2, 512, st));
    }
    STAGE_MARK();
  }
  if (calib) return fp8_finish_calibration(m, st);
  // conv5 (2x2 VALID, no activation): plain GEMM, K-blocks 0..15 from row m, 16..31 from row m+1
  {
    gemm::Params p;
    memset(&p, 0, sizeof(p));
    p.M = N * H2;
    p.num_m_tiles = (p.M + 127) / 128; p.num_n_tiles = 2; p.num_k_blocks = 32; p.kb_per_shift = 16; p.row_shift_mul = 1;
    p.Nc = 512; p.bias = m->P("conv5/biases"); p.out = pl.a5; p.ldo = 512;
    if (fp8) CRNN_TRY(fp8_conv5(m, p, sms, st));
    else CRNN_TRY((launch_gemm<256, gemm::A_PLAIN, gemm::EPI_BIAS_BF16, 4>(pl.tA_c5, m->tB_c5, p, sms, st, &pl.tA_x)));
  }
  STAGE_MARK();
  // LSTM input projection for all frames and both directions: [N*H2, 512] x [512, 2048]
  {
    gemm::Params p;
    memset(&p, 0, sizeof(p));
    p.M = N * H2;
    p.num_m_tiles = (p.M + 127) / 128; p.num_n_tiles = 8; p.num_k_blocks = 8; p.kb_per_shift = 8;
    p.Nc = 2048; p.bias = m->xbias; p.out = pl.xproj; p.ldo = 2048;
    p.H = H2; p.T = pl.T; p.seq_len = time_step_len;
    CRNN_TRY((launch_gemm<256, gemm::A_PLAIN, gemm::EPI_XPROJ, 4>(pl.tA_x, m->tB_x, p, sms, st, &pl.tO_x)));
  }
  STAGE_MARK();
  // rows t = T (= H2-1) of lstm_out are never produced by a time step, yet the logits GEMM and the backward's dW_h GEMMs read
  // them (dW_h as h_{-1} / h_{T} of the neighbouring image): zero them in every forward, whatever the workspace held before
  CUDA_TRY(cudaMemset2DAsync(pl.lstm_out + (size_t)pl.T * 512, (size_t)H2 * 512 * 2, 0, 512 * 2, N, st));
  CRNN_TRY(launch_lstm_forward(m, time_step_len, st));
  STAGE_MARK();
  // 512 -> 64 projection, written time-major [T, N, 64] (network.py:126-128)
  {
    gemm::Params p;
    memset(&p, 0, sizeof(p));
    p.M = N * H2;
    p.num_m_tiles = (p.M + 127) / 128; p.num_n_tiles = 1; p.num_k_blocks = 8; p.kb_per_shift = 8;
    p.Nc = 64; p.bias = m->P("logits/biases"); p.out = logits_out; p.H = H2; p.T = pl.T; p.Nimg = N;
    CRNN_TRY((launch_gemm<64, gemm::A_PLAIN, gemm::EPI_LOGITS, 8>(pl.tA_l, m->tB_l, p, sms, st)));
  }
  STAGE_MARK();
#undef STAGE_MARK
  return CRNN_OK;
}

// the uint8 kernels load each row's pixels as 4-byte words
static int check_u8_aligned(const void* p, const char* fn) { return check_aligned(p, 4, fn, "uint8 data"); }

// a device-fed batch of floats or (u8) uint8 pixels
static FwdCall device_batch(const void* data, bool u8) {
  FwdCall a;
  a.data = data; a.u8 = u8;
  return a;
}
// a batch in page-locked (pageable == nullptr) or ordinary host memory, copied to `data` on `copy_stream`
static FwdCall host_batch(const void* host, const void* pageable, const void* data, bool u8, int chunks, int host_threads,
                          crnn_stream_t copy_stream) {
  FwdCall a = device_batch(data, u8);
  a.host = host; a.pageable = pageable; a.chunks = chunks; a.host_threads = host_threads < 1 ? 1 : host_threads;
  a.copy_st = reinterpret_cast<cudaStream_t>(copy_stream);
  return a;
}

extern "C" int crnn_forward(crnn_model* m, const float* data, const int* time_step_len, int N, int W, float* logits_out,
                            void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  return forward(m, device_batch(data, false), time_step_len, N, W, logits_out, workspace, workspace_bytes, stream);
}
extern "C" int crnn_forward_u8(crnn_model* m, const uint8_t* data, const int* time_step_len, int N, int W, float* logits_out,
                               void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  CRNN_TRY(check_u8_aligned(data, "forward_u8"));
  return forward(m, device_batch(data, true), time_step_len, N, W, logits_out, workspace, workspace_bytes, stream);
}

extern "C" int crnn_forward_host(crnn_model* m, const float* host_data, float* data_staging, const int* time_step_len, int N, int W,
                                 float* logits_out, void* workspace, size_t workspace_bytes, int chunks, crnn_stream_t stream,
                                 crnn_stream_t copy_stream) {
  if (!host_data || !data_staging) return crnn_fail(CRNN_INVALID_VALUE, "forward_host: null pointer");
  return forward(m, host_batch(host_data, nullptr, data_staging, false, chunks, 1, copy_stream), time_step_len, N, W, logits_out, workspace,
                 workspace_bytes, stream);
}
extern "C" int crnn_forward_host_u8(crnn_model* m, const uint8_t* host_data, uint8_t* data_staging, const int* time_step_len, int N,
                                    int W, float* logits_out, void* workspace, size_t workspace_bytes, int chunks, crnn_stream_t stream,
                                    crnn_stream_t copy_stream) {
  CRNN_TRY(check_u8_aligned(data_staging, "forward_host_u8"));
  if (!host_data || !data_staging) return crnn_fail(CRNN_INVALID_VALUE, "forward_host: null pointer");
  return forward(m, host_batch(host_data, nullptr, data_staging, true, chunks, 1, copy_stream), time_step_len, N, W, logits_out, workspace,
                 workspace_bytes, stream);
}

extern "C" int crnn_forward_pageable(crnn_model* m, const float* pageable_data, float* pinned_staging, float* data_staging,
                                     const int* time_step_len, int N, int W, float* logits_out, void* workspace, size_t workspace_bytes,
                                     int chunks, int host_threads, crnn_stream_t stream, crnn_stream_t copy_stream) {
  if (!pageable_data || !pinned_staging || !data_staging) return crnn_fail(CRNN_INVALID_VALUE, "forward_pageable: null pointer");
  return forward(m, host_batch(pinned_staging, pageable_data, data_staging, false, chunks, host_threads, copy_stream), time_step_len, N, W,
                 logits_out, workspace, workspace_bytes, stream);
}
extern "C" int crnn_forward_pageable_u8(crnn_model* m, const uint8_t* pageable_data, uint8_t* pinned_staging, uint8_t* data_staging,
                                        const int* time_step_len, int N, int W, float* logits_out, void* workspace, size_t workspace_bytes,
                                        int chunks, int host_threads, crnn_stream_t stream, crnn_stream_t copy_stream) {
  CRNN_TRY(check_u8_aligned(data_staging, "forward_pageable_u8"));
  if (!pageable_data || !pinned_staging || !data_staging) return crnn_fail(CRNN_INVALID_VALUE, "forward_pageable: null pointer");
  return forward(m, host_batch(pinned_staging, pageable_data, data_staging, true, chunks, host_threads, copy_stream), time_step_len, N, W,
                 logits_out, workspace, workspace_bytes, stream);
}

extern "C" int crnn_host_copy(void* dst, const void* src, size_t bytes, int threads) {
  if ((!dst || !src) && bytes) return crnn_fail(CRNN_INVALID_VALUE, "host_copy: null pointer");
  CopyPool::get().copy(dst, src, bytes, threads < 1 ? 1 : threads);
  return CRNN_OK;
}

// ---- fp8 (compute_dtype 4) scales
static int check_calibrate(const crnn_model* m) {
  if (!m) return crnn_fail(CRNN_INVALID_VALUE, "calibrate_fp8: null model");
  if (m->cfg.compute_dtype != 4) return crnn_fail(CRNN_UNSUPPORTED, "calibrate_fp8: the model is not an fp8 model (compute_dtype 4)");
  return CRNN_OK;
}
extern "C" int crnn_model_calibrate_fp8(crnn_model* m, const float* data, const int* time_step_len, int N, int W, void* workspace,
                                        size_t workspace_bytes, crnn_stream_t stream) {
  CRNN_TRY(check_calibrate(m));
  FwdCall a = device_batch(data, false);
  a.calib = true;
  return forward(m, a, time_step_len, N, W, nullptr, workspace, workspace_bytes, stream);
}
extern "C" int crnn_model_calibrate_fp8_u8(crnn_model* m, const uint8_t* data, const int* time_step_len, int N, int W, void* workspace,
                                           size_t workspace_bytes, crnn_stream_t stream) {
  CRNN_TRY(check_u8_aligned(data, "calibrate_fp8_u8"));
  CRNN_TRY(check_calibrate(m));
  FwdCall a = device_batch(data, true);
  a.calib = true;
  return forward(m, a, time_step_len, N, W, nullptr, workspace, workspace_bytes, stream);
}
extern "C" int crnn_model_get_fp8_scales(crnn_model* m, float* scales_host) {
  if (!m || !scales_host) return crnn_fail(CRNN_INVALID_VALUE, "get_fp8_scales: null");
  if (m->cfg.compute_dtype != 4) return crnn_fail(CRNN_UNSUPPORTED, "get_fp8_scales: the model is not an fp8 model (compute_dtype 4)");
  return fp8_get_scales(m, scales_host);
}
extern "C" int crnn_model_set_fp8_scales(crnn_model* m, const float* scales_host) {
  if (!m || !scales_host) return crnn_fail(CRNN_INVALID_VALUE, "set_fp8_scales: null");
  if (m->cfg.compute_dtype != 4) return crnn_fail(CRNN_UNSUPPORTED, "set_fp8_scales: the model is not an fp8 model (compute_dtype 4)");
  return fp8_set_scales(m, scales_host);
}

// packed evaluation: the inference plan with its packed-line region (layout_plan)
extern "C" int crnn_lines_workspace_size(const crnn_model* m, int N, int W, size_t* bytes) {
  if (!m || !bytes) return crnn_fail(CRNN_INVALID_VALUE, "lines_workspace_size: null");
  if (N <= 0 || W < 8 || (W % 4) != 0) return crnn_fail(CRNN_INVALID_VALUE, "lines_workspace_size: need N>0, W>=8, W%%4==0");
  if (m->cfg.compute_dtype == 2 || m->cfg.compute_dtype == 3)
    return crnn_fail(CRNN_UNSUPPORTED, "lines_workspace_size: packed evaluation runs on the bf16 and fp8 paths (compute_dtype 1, 4)");
  Plan pl;
  *bytes = layout_plan(pl, N, W, nullptr, false, true, m->bn_use_moving);
  return CRNN_OK;
}

// the checks of a packed batch, before the forward's own
static int check_lines(crnn_model* m, const void* data, const int* line_width, const int* time_step_len, int N, int W, const float* logits_out,
                       const void* workspace, size_t workspace_bytes) {
  if (!m || !data || !line_width || !time_step_len || !logits_out || !workspace) return crnn_fail(CRNN_INVALID_VALUE, "forward_lines: null pointer");
  if (m->cfg.compute_dtype == 2 || m->cfg.compute_dtype == 3)
    return crnn_fail(CRNN_UNSUPPORTED, "forward_lines: packed evaluation runs on the bf16 and fp8 paths (compute_dtype 1, 4)");
  if (m->training)
    return crnn_fail(CRNN_INVALID_VALUE, "forward_lines: evaluation only; the model is in training mode (training uses whole-batch statistics)");
  size_t need = 0;
  CRNN_TRY(crnn_lines_workspace_size(m, N, W, &need));
  if (workspace_bytes < need) return crnn_fail(CRNN_WORKSPACE_TOO_SMALL, "forward_lines: workspace %zu < %zu", workspace_bytes, need);
  return CRNN_OK;
}
extern "C" int crnn_forward_lines(crnn_model* m, const float* data, const int* line_width, const int* time_step_len, int N, int W,
                                  float* logits_out, void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  CRNN_TRY(check_lines(m, data, line_width, time_step_len, N, W, logits_out, workspace, workspace_bytes));
  FwdCall a = device_batch(data, false);
  a.line_width = line_width;
  return forward(m, a, time_step_len, N, W, logits_out, workspace, workspace_bytes, stream);
}
extern "C" int crnn_forward_lines_u8(crnn_model* m, const uint8_t* data, const int* line_width, const int* time_step_len, int N, int W,
                                     float* logits_out, void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  CRNN_TRY(check_u8_aligned(data, "forward_lines_u8"));
  CRNN_TRY(check_lines(m, data, line_width, time_step_len, N, W, logits_out, workspace, workspace_bytes));
  FwdCall a = device_batch(data, true);
  a.line_width = line_width;
  return forward(m, a, time_step_len, N, W, logits_out, workspace, workspace_bytes, stream);
}

// ------------------------------------------------------------------------------------------------ profiling
extern "C" int crnn_profile_begin(crnn_model* m, int max_forwards) {
  if (!m || max_forwards < 0) return crnn_fail(CRNN_INVALID_VALUE, "profile_begin: bad args");
  const size_t need = (size_t)max_forwards * (kNumStages + 1);
  while (m->prof_events.size() < need) {
    cudaEvent_t e;
    CUDA_TRY(cudaEventCreate(&e));
    m->prof_events.push_back(e);
  }
  const size_t need_b = (size_t)max_forwards * (kNumBwdStages + 1);
  while (m->prof_events_bwd.size() < need_b) {
    cudaEvent_t e;
    CUDA_TRY(cudaEventCreate(&e));
    m->prof_events_bwd.push_back(e);
  }
  m->prof_slots = max_forwards; m->prof_used = 0; m->prof_used_bwd = 0; m->prof_on = max_forwards > 0;
  return CRNN_OK;
}
extern "C" int crnn_profile_num_stages(void) { return kNumStages; }
extern "C" const char* crnn_profile_stage_name(int i) { return (i >= 0 && i < kNumStages) ? kStageNames[i] : ""; }
// Host-synchronising: waits for the recorded events. ms_out [forwards][kNumStages]
extern "C" int crnn_profile_read(crnn_model* m, float* ms_out, int* forwards) {
  if (!m || !ms_out || !forwards) return crnn_fail(CRNN_INVALID_VALUE, "profile_read: null");
  m->prof_on = false;
  *forwards = m->prof_used;
  for (int f = 0; f < m->prof_used; ++f) {
    cudaEvent_t* ev = &m->prof_events[(size_t)f * (kNumStages + 1)];
    CUDA_TRY(cudaEventSynchronize(ev[kNumStages]));
    for (int s = 0; s < kNumStages; ++s) CUDA_TRY(cudaEventElapsedTime(ms_out + (size_t)f * kNumStages + s, ev[s], ev[s + 1]));
  }
  return CRNN_OK;
}

extern "C" int crnn_total_loss(crnn_model* m, const float* costs, int N, float* loss_out, crnn_stream_t stream) {
  if (!m || !costs || !loss_out || N <= 0) return crnn_fail(CRNN_INVALID_VALUE, "total_loss: bad args");
  if (!m->params) return crnn_fail(CRNN_NOT_BOUND, "total_loss: call crnn_model_bind first");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (m->dirty) CRNN_TRY(prepare_weights(m, st));
  return launch_total_loss(costs, N, m->sumsq, m->cfg.weight_decay, loss_out, st);
}

extern "C" int crnn_debug_tap(crnn_model* m, const char* name, float* dst, size_t dst_elems, void* workspace,
                              crnn_stream_t stream) {
  if (!m || !name || !dst) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: null");
  if (m->cfg.compute_dtype == 2 || m->cfg.compute_dtype == 3)
    return x3_debug_tap(m, name, dst, dst_elems, workspace, reinterpret_cast<cudaStream_t>(stream));
  Plan& pl = m->plan;
  if (pl.ws == nullptr || pl.ws != workspace) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: no forward ran on this workspace");
  const size_t n = pl.N, h1 = pl.H1, h2 = pl.H2;
  const __nv_bfloat16* src = nullptr;
  size_t cnt = 0;
  std::string s(name);
  if (s == "conv1") { src = pl.a1; cnt = n * h1 * 16 * 64; }
  else if (s == "conv2") { src = pl.a2; cnt = n * h2 * 8 * 128; }
  else if (s == "conv3_1") { src = pl.a3; cnt = n * h2 * 8 * 256; }
  else if (s == "conv3_2") { src = pl.a3p; cnt = n * h2 * 4 * 256; }
  else if (s == "conv4_1") { src = pl.a4a; cnt = n * h2 * 4 * 512; }
  else if (s == "conv4_2") { src = pl.a4b; cnt = n * h2 * 2 * 512; }
  else if (s == "conv5") { src = pl.a5; cnt = n * h2 * 512; }
  else if (s == "lstm_out") { src = pl.lstm_out; cnt = n * h2 * 512; }
  else if (s == "xproj") { src = pl.xproj; cnt = n * h2 * 2048; }
  else if (s == "a4a_pre" || s == "a4b_pre") {
    if (pl.moving) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: %s: the last forward used moving statistics (no pre-BN output)", name);
    src = s == "a4a_pre" ? pl.a4a_pre : pl.a4b_pre;
    cnt = n * h2 * 4 * 512;
  }
  else {
    // saved state and backward buffers: only a training-mode plan holds them
    const struct { const char* name; const __nv_bfloat16* p; size_t cnt; } train_taps[] = {
        {"gates", pl.gates, (size_t)2 * pl.Npad * pl.T * 1024}, {"dl_rows", pl.dl_rows, n * h2 * 64},
        {"d_lstm_out", pl.d_lstm_out, n * h2 * 512},           {"dz_all", pl.dz_all, n * h2 * 2048},
        {"d_a5", pl.d_a5, n * h2 * 512},                       {"d_a4b", pl.d_a4b, n * h2 * 2 * 512},
        {"d_pre4b", pl.d_pre4b, n * h2 * 4 * 512},             {"d_pre4a", pl.d_pre4a, n * h2 * 4 * 512},
        {"d_a3p", pl.d_a3p, n * h2 * 4 * 256},                 {"d_pre32", pl.d_pre32, n * h2 * 8 * 256},
        {"d_pre31", pl.d_pre31, n * h2 * 8 * 256},             {"d_a2", pl.d_a2, n * h2 * 8 * 128},
        {"d_pre2", pl.d_pre2, n * h1 * 16 * 128},              {"d_a1", pl.d_a1, n * h1 * 16 * 64}};
    for (auto& t : train_taps)
      if (s == t.name) {
        if (!pl.train) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: %s exists only in a training-mode plan", name);
        src = t.p; cnt = t.cnt;
      }
    if (src == nullptr) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: unknown tap %s", name);
  }
  if (dst_elems < cnt) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap: dst too small (%zu < %zu)", dst_elems, cnt);
  if (m->cfg.compute_dtype == 4) {
    // the five e4m3 operands, dequantised with their scale (a calibration leaves the bf16 values in the same buffers, but a tap
    // reads the last forward, which an fp8 model runs in e4m3)
    const __nv_bfloat16* q[5] = {pl.a2, pl.a3, pl.a3p, pl.a4a, pl.a4b};
    for (int i = 0; i < 5; ++i)
      if (src == q[i]) return fp8_dequant_tap(m, i, src, dst, cnt, reinterpret_cast<cudaStream_t>(stream));
  }
  return launch_bf16_to_f32(src, dst, cnt, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int crnn_debug_tap_raw(crnn_model* m, const char* name, void* dst, size_t dst_bytes, void* workspace,
                                  crnn_stream_t stream) {
  if (!m || !name || !dst) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: null");
  if (m->cfg.compute_dtype == 2 || m->cfg.compute_dtype == 3)
    return x3_debug_tap_raw(m, name, dst, dst_bytes, workspace, reinterpret_cast<cudaStream_t>(stream));
  std::string s(name);
  if (m->cfg.compute_dtype == 4) {
    int status = CRNN_OK;
    if (fp8_debug_tap_raw(m, s, dst, dst_bytes, reinterpret_cast<cudaStream_t>(stream), &status)) return status;
  }
  // the folded operands of the moving statistics (model state, not workspace): bf16 [Cout][K] and f32 [2][512]
  if (s == "moving_w_conv4_1" || s == "moving_w_conv4_2" || s == "moving_bias") {
    if (!m->wblock_bnm || m->bn_fold_dirty)
      return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: %s: no forward with the current moving statistics ran yet", name);
    const void* src = s == "moving_bias" ? (const void*)m->bm_bias : s == "moving_w_conv4_1" ? (const void*)m->Bm41 : (const void*)m->Bm42;
    const size_t bytes = s == "moving_bias" ? 2 * 512 * sizeof(float) : (size_t)512 * (s == "moving_w_conv4_1" ? 2304 : 4608) * 2;
    if (dst_bytes < bytes) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: dst too small (%zu < %zu bytes)", dst_bytes, bytes);
    CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, reinterpret_cast<cudaStream_t>(stream)));
    return CRNN_OK;
  }
  Plan& pl = m->plan;
  if (pl.ws == nullptr || pl.ws != workspace) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: no forward ran on this workspace");
  if (pl.moving && (s == "bn" || s == "stats"))
    return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: %s: the last forward used moving statistics (no batch statistics)", name);
  const size_t n = pl.N, h1 = pl.H1, h2 = pl.H2;
  const void* src = nullptr;
  size_t bytes = 0;
  bool train_only = false;
  const bool q8 = m->cfg.compute_dtype == 4;
  if (q8 && s == "conv2") { src = pl.a2; bytes = n * h2 * 8 * 128; }                 // e4m3 operands, byte for byte
  else if (q8 && s == "conv3_1") { src = pl.a3; bytes = n * h2 * 8 * 256; }
  else if (q8 && s == "conv3_2") { src = pl.a3p; bytes = n * h2 * 4 * 256; }
  else if (q8 && s == "conv4_1") { src = pl.a4a; bytes = n * h2 * 4 * 512; }
  else if (q8 && s == "conv4_2") { src = pl.a4b; bytes = n * h2 * 2 * 512; }
  else if (s == "bn" && pl.line_w) { src = pl.bn_l; bytes = 2 * n * 4 * 512 * sizeof(float); }
  else if (s == "stats" && pl.line_w) { src = pl.stats_l; bytes = 2 * n * 2 * 512 * sizeof(double); }
  else if (s == "bn") { src = pl.bn; bytes = 2 * 4 * 512 * sizeof(float); }
  else if (s == "stats") { src = pl.stats; bytes = 2 * 2 * 512 * sizeof(double); }
  else if (s == "am1") { src = pl.am1; bytes = n * h1 * 16 * 64; train_only = true; }
  else if (s == "am2") { src = pl.am2; bytes = n * h2 * 8 * 128; train_only = true; }
  else if (s == "am3") { src = pl.am3; bytes = n * h2 * 4 * 256; train_only = true; }
  else if (s == "csave") { src = pl.csave; bytes = (size_t)2 * pl.Npad * pl.T * 256 * sizeof(float); train_only = true; }
  else return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: unknown tap %s", name);
  if (train_only && !pl.train) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: %s exists only in a training-mode plan", name);
  if (dst_bytes < bytes) return crnn_fail(CRNN_INVALID_VALUE, "debug_tap_raw: dst too small (%zu < %zu bytes)", dst_bytes, bytes);
  CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, reinterpret_cast<cudaStream_t>(stream)));
  return CRNN_OK;
}

extern "C" int crnn_test_gemm_bf16(const void* A, const void* B, float* D, int M, int Nc, int K, int block_n,
                                   crnn_stream_t stream) {
  if (!A || !B || !D || M <= 0 || Nc <= 0 || K <= 0 || (K % 64) != 0 || (Nc % block_n) != 0)
    return crnn_fail(CRNN_INVALID_VALUE, "test_gemm: bad args");
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  CUtensorMap ta, tb;
  CRNN_TRY(make_tmap_2d(&ta, A, M, K, K, 128));
  CRNN_TRY(make_tmap_2d(&tb, B, Nc, K, K, block_n));
  gemm::Params p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.Nc = Nc;
  p.num_m_tiles = (M + 127) / 128; p.num_n_tiles = Nc / block_n; p.num_k_blocks = K / 64; p.kb_per_shift = p.num_k_blocks;
  p.out = D;
  if (const char* e = getenv("CRNN_PROBE_SKIP_TMA")) p.debug_skip_tma = (e[0] == '1');
  if (const char* e = getenv("CRNN_PROBE_SKIP_EPI")) p.debug_skip_epilogue = (e[0] == '1');
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // probe: CRNN_PROBE_BF16_OUT=1 writes D as bf16 [M, Nc] (EPI_BIAS_BF16 without bias, the register-side epilogue with TMA stores)
  if (const char* e = getenv("CRNN_PROBE_BF16_OUT"); e && e[0] == '1' && block_n == 256) {
    CUtensorMap to;
    CRNN_TRY(make_tmap_2d(&to, D, M, Nc, Nc, 128));
    p.ldo = Nc;
    return launch_gemm<256, gemm::A_PLAIN, gemm::EPI_BIAS_BF16, 4>(ta, tb, p, sms, st, &to);
  }
  if (block_n == 64) return launch_gemm<64, gemm::A_PLAIN, gemm::EPI_F32, 8>(ta, tb, p, sms, st);
  if (block_n == 128) return launch_gemm<128, gemm::A_PLAIN, gemm::EPI_F32, 6>(ta, tb, p, sms, st);
  if (block_n == 256) return launch_gemm<256, gemm::A_PLAIN, gemm::EPI_F32, 4>(ta, tb, p, sms, st);
  return crnn_fail(CRNN_INVALID_VALUE, "test_gemm: block_n must be 64/128/256");
}
