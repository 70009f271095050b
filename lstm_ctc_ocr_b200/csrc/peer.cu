// Data-parallel exchange of the BatchNorm batch statistics over NVLink peer memory, fused into the BN finalize kernel
// (SURVEY 8(e): "optional SyncBN: allreduce of [sum x, sum x^2] per BN layer in forward and the matching two vectors in backward").
//
// The reference is single-device: tf.contrib.layers.batch_norm(is_training=True) at lib/networks/network.py:177-178 normalises
// with the statistics of the WHOLE batch.  With the batch sharded over `world` GPUs the same function needs the 2 x 512 f64
// sums of every rank.  They are 8 KB: far below the size where a ring/tree collective pays, and they sit on the forward critical
// path twice per step.  So there is no collective launch at all here: the kernel that finalises the statistics
//   1. stores this rank's 1024 doubles into slot [parity][rank] of EVERY rank's inbox (P2P stores over NVLink/NVSwitch; the
//      inboxes are cudaMalloc'ed buffers shared through CUDA IPC),
//   2. fences at system scope and publishes a monotonically increasing epoch in flag[rank] of every inbox (st.release.sys),
//   3. waits until the `world` flags of its OWN inbox reached the epoch (ld.acquire.sys, bounded spin),
//   4. sums the `world` slots in rank order -- the same order on every rank, so all replicas compute bit-identical statistics --
//      and (forward) turns them straight into the BN scale / shift / mean / inv-std vectors.
// Two inbox slots alternate by epoch parity: a rank can only be two exchanges ahead of a peer after that peer has finished
// reading the older slot (its own flag for the exchange in between is published after that read, in stream order).
#include "model_internal.h"

namespace {

constexpr int MAX_WORLD = 16;
constexpr long long SPIN_LIMIT = 60000000000ll;      // ~30 s of SM clocks: a missing peer becomes an error flag, not a hang

struct Inbox {
  unsigned long long flag[MAX_WORLD];
  unsigned long long pad[MAX_WORLD];
  double data[2][MAX_WORLD][1024];
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ double ld_volatile_f64(const double* p) {
  double v;
  asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

// FINALIZE = false: out[i] = sum over ranks of in[i]                                   (backward sums)
// FINALIZE = true : additionally BN scale/shift/mean/invstd from the global [sum, sumsq] (forward), network.py:177-178
template <bool FINALIZE>
__global__ void __launch_bounds__(1024) peer_allreduce_kernel(const double* in, double* out, Inbox* const* peers,
                                                             int rank, int world, unsigned long long epoch, int* err, double count,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                             float* __restrict__ bn) {
  __shared__ double sh[1024];
  const int i = threadIdx.x;
  const double v = in[i];
  const int par = (int)(epoch & 1ull);
  for (int p = 0; p < world; ++p) peers[p]->data[par][rank][i] = v;
  __threadfence_system();
  __syncthreads();
  Inbox* me = peers[rank];
  if (i < world) {
    st_release_sys(&peers[i]->flag[rank], epoch);
    const long long t0 = clock64();
    while (ld_acquire_sys(&me->flag[i]) < epoch) {
      if (clock64() - t0 > SPIN_LIMIT) { *err = 1; break; }
    }
  }
  __syncthreads();
  double s = 0.0;
  for (int p = 0; p < world; ++p) s += ld_volatile_f64(&me->data[par][p][i]);
  out[i] = s;
  if (FINALIZE) {
    sh[i] = s;
    __syncthreads();
    if (i < 512) {
      const double mean = sh[i] / count;
      double var = sh[512 + i] / count - mean * mean;            // population variance
      if (var < 0) var = 0;
      const double invstd = 1.0 / sqrt(var + (double)eps);
      bn[i] = (float)(gamma[i] * invstd);
      bn[512 + i] = (float)(beta[i] - mean * gamma[i] * invstd);
      bn[1024 + i] = (float)mean;
      bn[1536 + i] = (float)invstd;
    }
  }
}

__global__ void bn_finalize_512_kernel(const double* __restrict__ stats, double count, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, float eps, float* __restrict__ bn) {
  const int i = threadIdx.x;
  const double mean = stats[i] / count;
  double var = stats[512 + i] / count - mean * mean;
  if (var < 0) var = 0;
  const double invstd = 1.0 / sqrt(var + (double)eps);
  bn[i] = (float)(gamma[i] * invstd);
  bn[512 + i] = (float)(beta[i] - mean * gamma[i] * invstd);
  bn[1024 + i] = (float)mean;
  bn[1536 + i] = (float)invstd;
}

}  // namespace

extern "C" size_t crnn_peer_inbox_bytes(void) { return sizeof(Inbox); }

extern "C" int crnn_peer_inbox_create(void** dev_ptr, unsigned char handle[64]) {
  if (!dev_ptr || !handle) return crnn_fail(CRNN_INVALID_VALUE, "peer_inbox_create: null");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
  void* p = nullptr;
  CUDA_TRY(cudaMalloc(&p, sizeof(Inbox)));
  CUDA_TRY(cudaMemset(p, 0, sizeof(Inbox)));
  CUDA_TRY(cudaDeviceSynchronize());     // the memset is ordered on the legacy stream only: done before any stream's exchange
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); return crnn_fail(CRNN_CUDA_ERROR, "cudaIpcGetMemHandle: %s", cudaGetErrorString(e)); }
  memcpy(handle, &h, 64);
  *dev_ptr = p;
  return CRNN_OK;
}
extern "C" int crnn_peer_inbox_open(const unsigned char handle[64], void** dev_ptr) {
  if (!dev_ptr || !handle) return crnn_fail(CRNN_INVALID_VALUE, "peer_inbox_open: null");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  CUDA_TRY(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return CRNN_OK;
}
extern "C" int crnn_peer_inbox_close(void* dev_ptr) {
  if (dev_ptr) CUDA_TRY(cudaIpcCloseMemHandle(dev_ptr));
  return CRNN_OK;
}
extern "C" int crnn_peer_inbox_destroy(void* dev_ptr) {
  if (dev_ptr) CUDA_TRY(cudaFree(dev_ptr));
  return CRNN_OK;
}

extern "C" int crnn_model_set_data_parallel(crnn_model* m, int rank, int world, crnn_allreduce_fn allreduce, void* user) {
  if (!m || world < 1 || rank < 0 || rank >= world || world > MAX_WORLD) return crnn_fail(CRNN_INVALID_VALUE, "set_data_parallel: bad rank/world");
  m->dp_rank = rank; m->dp_world = world; m->xchg_cb = allreduce; m->xchg_user = user;
  return CRNN_OK;
}

extern "C" int crnn_model_set_grad_ready_callback(crnn_model* m, crnn_grad_ready_fn fn, void* user) {
  if (!m) return crnn_fail(CRNN_INVALID_VALUE, "set_grad_ready_callback: null model");
  m->grad_cb = fn; m->grad_user = user;
  return CRNN_OK;
}

extern "C" int crnn_model_set_backward_sm_reserve(crnn_model* m, int sms) {
  if (!m || sms < 0 || sms > m->num_sms / 2) return crnn_fail(CRNN_INVALID_VALUE, "set_backward_sm_reserve: bad value");
  m->bwd_sm_reserve = sms;
  return CRNN_OK;
}

extern "C" int crnn_model_set_peers(crnn_model* m, int rank, int world, void* const* inbox_ptrs_host) {
  if (!m || world < 1 || rank < 0 || rank >= world || world > MAX_WORLD) return crnn_fail(CRNN_INVALID_VALUE, "set_peers: bad rank/world");
  if (m->d_peers) { cudaFree(m->d_peers); m->d_peers = nullptr; }
  if (!inbox_ptrs_host) return CRNN_OK;                          // peers cleared: exchanges fall back to the callback
  for (int i = 0; i < world; ++i)
    if (!inbox_ptrs_host[i]) return crnn_fail(CRNN_INVALID_VALUE, "set_peers: inbox pointer %d is null", i);
  CUDA_TRY(cudaMalloc(&m->d_peers, sizeof(void*) * MAX_WORLD + sizeof(int)));
  CUDA_TRY(cudaMemset(m->d_peers, 0, sizeof(void*) * MAX_WORLD + sizeof(int)));
  CUDA_TRY(cudaMemcpy(m->d_peers, inbox_ptrs_host, sizeof(void*) * world, cudaMemcpyHostToDevice));
  // a copy from pageable memory may return before its DMA lands, and the next exchange may run on a non-blocking stream
  CUDA_TRY(cudaDeviceSynchronize());
  m->d_peer_err = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(m->d_peers) + sizeof(void*) * MAX_WORLD);
  m->dp_rank = rank; m->dp_world = world;
  m->peer_epoch = 0;
  return CRNN_OK;
}

extern "C" int crnn_peer_error(crnn_model* m, int* err_host) {
  if (!m || !err_host) return crnn_fail(CRNN_INVALID_VALUE, "peer_error: null");
  *err_host = 0;
  if (m->d_peer_err) CUDA_TRY(cudaMemcpy(err_host, m->d_peer_err, sizeof(int), cudaMemcpyDeviceToHost));
  return CRNN_OK;
}

int dp_allreduce_1024(crnn_model* m, const double* in, double* out, cudaStream_t st) {
  if (m->dp_world <= 1) {
    if (in != out) CUDA_TRY(cudaMemcpyAsync(out, in, 1024 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    return CRNN_OK;
  }
  if (m->d_peers) {
    ++m->peer_epoch;
    peer_allreduce_kernel<false><<<1, 1024, 0, st>>>(in, out, reinterpret_cast<Inbox* const*>(m->d_peers), m->dp_rank, m->dp_world,
                                                     m->peer_epoch, m->d_peer_err, 0.0, nullptr, nullptr, 0.f, nullptr);
    CUDA_TRY(cudaGetLastError());
    return CRNN_OK;
  }
  if (!m->xchg_cb) return crnn_fail(CRNN_INVALID_VALUE, "data parallel: neither peer inboxes nor an all-reduce callback are set");
  if (in != out) CUDA_TRY(cudaMemcpyAsync(out, in, 1024 * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (m->xchg_cb(m->xchg_user, out, 1024, 1, reinterpret_cast<crnn_stream_t>(st)) != 0)
    return crnn_fail(CRNN_CUDA_ERROR, "data parallel: the all-reduce callback failed");
  return CRNN_OK;
}

int dp_allreduce_bn_finalize(crnn_model* m, double* stats, double count_global, const float* gamma, const float* beta, float eps,
                             float* bn, cudaStream_t st) {
  if (m->dp_world > 1 && m->d_peers) {
    ++m->peer_epoch;
    peer_allreduce_kernel<true><<<1, 1024, 0, st>>>(stats, stats, reinterpret_cast<Inbox* const*>(m->d_peers), m->dp_rank, m->dp_world,
                                                    m->peer_epoch, m->d_peer_err, count_global, gamma, beta, eps, bn);
    CUDA_TRY(cudaGetLastError());
    return CRNN_OK;
  }
  CRNN_TRY(dp_allreduce_1024(m, stats, stats, st));
  bn_finalize_512_kernel<<<1, 512, 0, st>>>(stats, count_global, gamma, beta, eps, bn);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
