// Launch helpers for the wgmma GEMM kernels (shared by model.cu and backward.cu).
#pragma once
#include "gemm.cuh"
#include "gemm_tn.cuh"

// `out` is the tensor map the register-side epilogues (gemm::frag_epi) store through: NHWC box [64, Wd, bh (x4 merged), 1] for
// conv outputs, [64, 128] over [M, ldo] for plain ones.  The other epilogues take no map.
template <int BN, int AM, int EPI, int ST, int KIND = 0, bool LINES = false>
static int launch_gemm(const CUtensorMap& a, const CUtensorMap& b, const gemm::Params& p, int num_sms, cudaStream_t st,
                       const CUtensorMap* out = nullptr) {
  if (gemm::frag_epi(BN, EPI) && out == nullptr) return crnn_fail(CRNN_INVALID_VALUE, "launch_gemm: epilogue %d needs an output tensor map", EPI);
  auto kern = gemm::gemm_kernel<BN, AM, EPI, ST, KIND, LINES>;
  constexpr int smem = gemm::Smem<BN, ST, gemm::slice_cols(BN, EPI)>::BYTES;
  static bool attr = false;
  if (!attr) {
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < num_sms ? tiles : num_sms;
  kern<<<grid, gemm::NUM_THREADS, smem, st>>>(a, b, out ? *out : a, p);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

// launch_gemm with LINES picked at run time: `lines` = a packed evaluation batch (crnn_forward_lines)
template <int BN, int AM, int EPI, int ST, int KIND = 0>
static int launch_gemm_lines(bool lines, const CUtensorMap& a, const CUtensorMap& b, const gemm::Params& p, int num_sms, cudaStream_t st,
                             const CUtensorMap* out = nullptr) {
  if (lines) return launch_gemm<BN, AM, EPI, ST, KIND, true>(a, b, p, num_sms, st, out);
  return launch_gemm<BN, AM, EPI, ST, KIND, false>(a, b, p, num_sms, st, out);
}

// Launch of a kernel in clusters of `cluster` CTAs along x (the LSTM recurrence and its BPTT)
template <class... KArgs, class... Args>
static int launch_cluster(void (*kern)(KArgs...), int cluster, int grid, int threads, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, args...));
  return CRNN_OK;
}

// Split-K factor of a weight-gradient GEMM.  Work items (output tile x K chunk) all cost the same and the persistent CTAs take them
// round-robin, so the launch lasts  ceil(items / workers) rounds x (K blocks per chunk + epilogue).  A fixed "about 3 items per
// worker" can leave a mostly idle last round.  Pick the factor that minimises the modelled time (ties: fewer chunks = fewer f32
// reduction atomics).
static inline int pick_k_splits(int tiles, int k_blocks_total, int workers) {
  const int kEpi = 6;                            // epilogue + pipeline refill of one item, in K-block units
  int best = 1;
  long long best_cost = -1;
  const int kmax = k_blocks_total < 4 * workers ? k_blocks_total : 4 * workers;
  for (int k = 1; k <= kmax; ++k) {
    const long long rounds = ((long long)tiles * k + workers - 1) / workers;
    const long long cost = rounds * ((k_blocks_total + k - 1) / k + kEpi);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = k; }
  }
  return best;
}

template <int BN, int AM, int ST>
static int launch_gemm_tn(const CUtensorMap& a, const CUtensorMap& b, gemm_tn::Params p, int num_sms, cudaStream_t st) {
  auto kern = gemm_tn::gemm_tn_kernel<BN, AM, ST>;
  constexpr int smem = gemm_tn::Smem<BN, ST>::BYTES;
  static bool attr = false;
  if (!attr) {
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  const int tiles = p.num_taps * p.num_m_tiles * p.num_n_tiles;
  if (p.k_splits <= 0) p.k_splits = pick_k_splits(tiles, p.k_blocks_total, num_sms);
  const int items = tiles * p.k_splits;
  const int grid = items < num_sms ? items : num_sms;
  kern<<<grid, gemm_tn::NUM_THREADS, smem, st>>>(a, b, p);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}
