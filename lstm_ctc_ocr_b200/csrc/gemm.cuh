// Persistent warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   D[128 x BLOCK_N tile, f32] = A[rows x K] (bf16, K-major, TMA) * B[Nc x K]^T (bf16, K-major, TMA)
//
// Roles (384 threads): warpgroup 0 = TMA producer (warp 0, one lane per box; the warpgroup gives its registers to the MMA
// warpgroups), warpgroups 1 and 2 = MMA (rows 0..63 / 64..127 of the tile, accumulators in registers) and epilogue.
// Pipeline: STAGES-deep smem ring (full/empty mbarriers, TMA <-> MMA; the producer runs ahead into the next tile while
// the epilogue of this one drains).  The finished accumulators are staged in shared memory (ptx::acc_store_slice) so that
// every epilogue thread owns one accumulator ROW: 8 warps, accumulator quadrant q = warp % 4 (32 rows), two warps per
// quadrant each draining half of the staged columns.  At BLOCK_N = 256 the tile goes through one 128 x 64 f32 buffer (32 KB)
// a 64-column slice at a time, not as a whole (128 KB): that leaves room for a 4-stage ring, where the full tile would leave 2.
// Narrower tiles and EPI_CONV_STORE_BNRED stage the whole tile (slice_cols).  The MMA warpgroups run with 240
// registers (the producer keeps 24): the first slices drain while the later slices' accumulators are still in registers.
// The bf16-output epilogues at BLOCK_N = 256 (frag_epi) do not stage f32 at all: they finish the values in the fragment registers,
// write bf16 into the staging region (the whole 64 KB tile, 3 stages) in the layout of the output tensor map and leave through asynchronous TMA stores
// (frag_epilogue), so the next tile's MMAs start while the stores drain.
//
// A-operand modes
//   A_PLAIN  rows are consecutive rows of a 2-D [rows, K] tensor map; conv5 (2x2 VALID over [N,H,2,512]) reads
//            row m for the first half of K and row m+1 for the second half (kb_per_shift).
//   A_CONV3  implicit GEMM for a 3x3 SAME convolution over an NHWC activation [N, H, Wd, C]: a tile is
//            4 sub-boxes of 32 output positions (bh = 32/Wd rows of H x full Wd); K-block kb = tap (r,s) x
//            64-channel block; the producer issues one 4-D TMA box per sub-box at coordinates shifted by
//            (r-1, s-1) -- out-of-bounds elements are zero-filled by TMA, which *is* the SAME padding.
//
// Epilogues: see enum Epi.  In run_epilogue every epilogue thread owns one accumulator row; frag_epilogue works on the fragments.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace gemm {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;                      // bf16 elements per K-block = one 128 B swizzle row
constexpr int UMMA_K = 16;
constexpr int A_STAGE_BYTES = BLOCK_M * 128;     // 16 KB
constexpr int NUM_THREADS = 384;                 // warpgroup 0 producer, warpgroups 1..2 MMA + epilogue
constexpr int MAX_SMEM = 232448;                 // opt-in shared memory per block (227 KB)

enum AMode { A_PLAIN = 0, A_CONV3 = 1 };
enum Epi {
  EPI_F32 = 0,          // D f32 row-major [M, Nc] (tests)
  EPI_BIAS_BF16 = 1,    // + bias -> bf16 row-major [M, ldo]            (conv5, LSTM input projection)
  EPI_RELU = 2,         // conv: + bias, ReLU -> bf16 NHWC              (conv3_1)
  EPI_RELU_POOL12 = 4,  // conv: + bias, ReLU, max over Wd pairs        (conv3_2 + pool), needs Wd=8
  EPI_STATS = 5,        // conv: + bias -> bf16 pre-BN, per-channel sum / sum^2 (f64 atomics) (conv4_x)
  EPI_LOGITS = 7,       // + bias -> f32 time-major [T, N, 64]
  EPI_XPROJ = 8,        // + bias -> bf16 [N*H, 2048]; columns >= 1024 (backward direction) stored reversed-by-length
  EPI_CONV_STORE = 9,   // conv: plain bf16 NHWC store (data-gradient convolutions)
  EPI_RELU_POOL12_T = 11,  // training variant of EPI_RELU_POOL12: also emits the arg-max window index (uint8)
  EPI_CONV_STORE_MASK = 13,  // EPI_CONV_STORE with the ReLU backward of the PRODUCING layer folded in: zero where p.mask (its bf16 output, same NHWC layout) is 0
  EPI_CONV_STORE_BNRED = 14, // EPI_CONV_STORE + pass 1 of the BatchNorm/ReLU backward of the PRODUCING layer: per-channel f64 sums of the
                             // ReLU-masked gradient and of gradient * xhat (p.mask = its pre-BN bf16 output, p.bnp = scale|shift|mean|invstd)
  EPI_CONV_F32 = 12     // conv: raw f32 accumulators, NHWC store (f32-class path, forward_x3.cu: bias/BN/ReLU/pool + hi/lo split follow)
};

struct Params {
  int num_m_tiles, num_n_tiles, num_k_blocks;
  int m_tile0;           // first M tile of this launch (batch-chunked launches of the conv front end); tiles m_tile0 .. m_tile0+num_m_tiles-1
  int kb_per_shift;      // A_PLAIN: K-block kb reads A columns (kb % kb_per_shift)*64 of row (m + kb / kb_per_shift);
                         // == num_k_blocks for an ordinary GEMM; conv5 (2x2 VALID) uses 16 -> rows t and t+1
  int merged;            // conv: the tile's 4 sub-boxes are contiguous H rows of one image -> one 128-position TMA box
  int debug_skip_tma;    // probe only: producer arrives without loading (measures the MMA/epilogue ceiling)
  int debug_skip_epilogue;  // probe only: tiles end after the mainloop, nothing is stored (measures the mainloop alone)
  int row_shift_mul;     // +1 (conv5 forward: rows m, m+1) or -1 (conv5 data gradient: rows m, m-1)
  // split-bf16 ("3xbf16", f32-class) operands: the activation tensor stores [hi | lo] halves and the K loop visits
  // [hi | lo | hi] against weights [wh | wh | wl]; a virtual K-block index >= the fold wraps back onto the hi half.  0 = off.
  int cin_phys;          // A_CONV3: physical 64-channel blocks per tap (= 2*Cin/64 when cin_blocks = 3*Cin/64)
  int kb_phys;           // A_PLAIN: physical K-blocks per row shift (kb_per_shift counts the virtual ones)
  int M;                 // valid rows (plain modes)
  int Nc;                // total output columns
  // conv geometry (A_CONV3 and conv epilogues)
  int cin_blocks;        // Cin / 64
  int sb_per_img;        // ceil(H / bh)
  int bh, Wd, H, Nimg;
  // epilogue
  const float* bias;     // [Nc]
  void* out;             // primary output
  int ldo;               // row stride of `out` in elements (plain modes)
  double* stats;         // [2][Nc] (EPI_STATS)
  const __nv_bfloat16* mask;   // EPI_CONV_STORE_MASK: post-ReLU activation of the layer whose pre-activation gradient is being written
  const float* bnp;      // EPI_CONV_STORE_BNRED: [4][Nc] scale, shift, mean, invstd of the producing layer's BatchNorm
  uint8_t* argmax;       // EPI_RELU_POOL12_T: window index of the max, same shape as `out`
  // EPI_XPROJ (backward-direction rows reversed by length), EPI_LOGITS (time-major rows)
  const int* seq_len;    // [Nimg]
  int T;
  // LINES instantiations (packed evaluation, crnn_forward_lines): [Nimg] clamped line widths in input columns; conv rows at
  // h >= line_w[n] / 4 (every LINES layer runs at H = W/4) are stored as zero, and EPI_STATS sums go to slot n of `stats` [Nimg][2][Nc]
  const int* line_w;
  // KIND 2 (e4m3 operands, forward_fp8.cu): y = acc * colscale[col] + bias[col] (colscale = activation scale x weight scale);
  // EPI_RELU / EPI_RELU_POOL12 store e4m3(y / *oscale), the next GEMM's operand scale (a power of two)
  const float* colscale;
  const float* oscale;
};

__device__ __forceinline__ float warp_colsum32(const float (&v)[32], int lane) {
  // Sum over the 32 lanes of a warp for each of 32 per-lane registers; lane l returns column l's total.
  float r16[16], r8[8], r4[4], r2[2];
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    float send = (lane & 16) ? v[i] : v[i + 16];
    float keep = (lane & 16) ? v[i + 16] : v[i];
    r16[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float send = (lane & 8) ? r16[i] : r16[i + 8];
    float keep = (lane & 8) ? r16[i + 8] : r16[i];
    r8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float send = (lane & 4) ? r8[i] : r8[i + 4];
    float keep = (lane & 4) ? r8[i + 4] : r8[i];
    r4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float send = (lane & 2) ? r4[i] : r4[i + 2];
    float keep = (lane & 2) ? r4[i + 2] : r4[i];
    r2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  float send = (lane & 1) ? r2[0] : r2[1];
  float keep = (lane & 1) ? r2[1] : r2[0];
  return keep + __shfl_xor_sync(0xffffffffu, send, 1);
}

// Accumulator columns staged in shared memory at a time (see the header).  While a slice drains, the accumulators of the
// later slices stay live in registers (96 at BLOCK_N = 256).  EPI_CONV_STORE_BNRED's epilogue does not fit in the registers
// left beside them (it spills), so it stages the whole tile; it only serves the training backward pass.
// BLOCK_N = 128 measured slower in 64-column slices (6 stages) than whole (5 stages), so it stays whole.  The register-side
// bf16 epilogues (frag_epi) stage the whole bf16 tile in the bytes of 128 f32 columns: with 3 stages that measured faster than
// two 32 KB halves through one buffer with 4 stages (the halves wait on each other's stores).  EPI_RELU_POOL12's pooled tile
// needs only 32 KB.
constexpr int slice_cols(int block_n, int epi) {
  return (block_n < 256 || epi == EPI_CONV_STORE_BNRED) ? block_n
       : (epi == EPI_RELU || epi == EPI_STATS || epi == EPI_BIAS_BF16 || epi == EPI_XPROJ || epi == EPI_CONV_STORE) ? 128 : 64;
}

// STAGES is the requested ring depth; S the depth that fits next to the staged accumulator slice of SLICE_N columns
template <int BLOCK_N, int STAGES, int SLICE_N>
struct Smem {
  static constexpr int B_STAGE_BYTES = BLOCK_N * 128;
  static constexpr int ACC_BYTES = BLOCK_M * SLICE_N * 4;
  static constexpr int FIT = (MAX_SMEM - ACC_BYTES - 256 - 1024) / (A_STAGE_BYTES + B_STAGE_BYTES);
  static constexpr int S = STAGES < FIT ? STAGES : FIT;
  static constexpr int ACC_OFFSET = S * (A_STAGE_BYTES + B_STAGE_BYTES);
  static constexpr int BAR_OFFSET = ACC_OFFSET + ACC_BYTES;
  static constexpr int BYTES = BAR_OFFSET + 256 + 1024;   // barriers + alignment slack
};
static_assert(Smem<256, 4, 64>::S == 4, "a 64-column staging slice leaves room for a 4-stage ring at BLOCK_N = 256");

// Epilogues that run on the accumulator fragments and leave through TMA stores (frag_epilogue); the staging region then holds the
// bf16 tile (slice_cols = 128 "f32 columns" = 64 KB, 3 stages) or the pooled tile (32 KB, 4 stages) instead of an f32 slice.
constexpr bool frag_epi(int block_n, int epi) {
  return block_n == 256 && (epi == EPI_RELU || epi == EPI_RELU_POOL12 || epi == EPI_STATS || epi == EPI_BIAS_BF16 ||
                            epi == EPI_XPROJ || epi == EPI_CONV_STORE);
}

// bf16x2 word of staged row `row`, tile-half column c (even) 0..127: [64-column box][row][128 B], 16-B chunks XOR-swizzled by
// (row & 7) -- the SWIZZLE_128B layout the output tensor maps read, and conflict-free for fragment-order 32-bit writes
__device__ __forceinline__ uint32_t* stg_word(uint8_t* buf, int box_bytes, int row, int c) {
  return reinterpret_cast<uint32_t*>(buf + (c >> 6) * box_bytes + row * 128 + ((((c >> 3) & 7) ^ (row & 7)) << 4) + ((c & 7) << 1));
}
// e4m3 word (4 columns, c % 4 == 0) of staged row `row`, tile-half column c 0..127: one [row][128 B] box per half, same swizzle
__device__ __forceinline__ uint32_t* stg_word8(uint8_t* buf, int row, int c) {
  return reinterpret_cast<uint32_t*>(buf + row * 128 + ((((c >> 4) & 7) ^ (row & 7)) << 4) + (c & 15));
}

// EPI_STATS column sums of 32 staged rows rg*32 .. rg*32+31 at 32-bit word cw (two bf16 channels) of a 128-B box row:
// {sum lo, sum hi, sum lo^2, sum hi^2}.  The rows are added in the order of warp_colsum32 over 32 lanes (rows 16 apart first,
// then 8, 4, 2, 1), so the f32 partial sums are those of the row-per-thread epilogue, bit for bit.  Evaluated depth first:
// few partial sums are live next to the accumulators of the tile's second half.
template <int W>
__device__ __forceinline__ float4 rowsum_tree(const uint8_t* box, int rg, int cw, int i) {
  if constexpr (W == 32) {
    const int r = rg * 32 + i;
    const uint32_t v = *reinterpret_cast<const uint32_t*>(box + r * 128 + (((cw >> 2) ^ (r & 7)) << 4) + ((cw & 3) << 2));
    const float x = ptx::bf16_lo(v), y = ptx::bf16_hi(v);
    return make_float4(x, y, __fmul_rn(x, x), __fmul_rn(y, y));     // no contraction of the squares into the additions
  } else {
    const float4 a = rowsum_tree<W * 2>(box, rg, cw, i), b = rowsum_tree<W * 2>(box, rg, cw, i + W);
    return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}

// conv tiles: accumulator row r of tile m_blk is a real output position (h < H, image < Nimg); LINES: and h lies inside its line
template <bool LINES>
__device__ __forceinline__ bool conv_row_valid(const Params& p, int m_blk, int r) {
  const int g = m_blk * 4 + (r >> 5);
  const int n_img = g / p.sb_per_img;
  const int h = (g - n_img * p.sb_per_img) * p.bh + (r & 31) / p.Wd;
  if (LINES) return n_img < p.Nimg && h < (__ldg(p.line_w + n_img) >> 2);
  return n_img < p.Nimg && h < p.H;
}

// Register-side epilogue of one finished tile (frag_epi).  The MMA thread applies bias / ReLU / pooling to its own fragment
// registers with the same per-element operations as run_epilogue, writes bf16x2 words into the swizzled staging buffer, and one
// thread (`issuer`) sends the buffer to global memory with asynchronous TMA stores; the warpgroups then go on to the next
// tile's mainloop while the stores drain.  The whole bf16 tile is staged (64 KB: a 3-stage ring, see slice_cols), written and
// stored in two 128-column halves; before the first half of a tile is written, the issuer waits until the previous tile's stores
// have read the buffer.  The pooled tile (64 rows, 32 KB) keeps the 4-stage ring.
//   conv outputs: 4-D NHWC map, box [64 ch, Wd, bh (x4 when merged), 1]; TMA drops rows with h >= H or image >= Nimg.
//   plain outputs: 2-D [M, ldo] map, box [64, 128]; rows >= M are dropped.
//   EPI_STATS: per-channel sum / sum of squares of the bf16-rounded outputs, read back from the staging buffer (invalid rows
//   are staged as zero): thread = (column pair, 32-row group), 2048 f64 atomics per tile.
//   EPI_XPROJ, columns >= 1024: rows reversed by sequence length.  When H divides 128 a tile holds whole sequences, so the
//   reversal is a permutation of staging rows; otherwise the thread stores its words to the reversed rows directly.
//   LINES (conv epilogues): rows past their line are staged as zero like invalid rows, and a 32-row statistics group -- one
//   sub-box, which never spans two images -- adds into its own image's sums.
//   KIND 2 (e4m3 operands): every value is acc * colscale + bias first; EPI_RELU / EPI_RELU_POOL12 (Q8) then store e4m3 of
//   y / oscale: the pool max is taken in f32 (rounding is monotonic), lane l ^ 1 holds the neighbouring column pair, so one
//   shuffle turns two 2-byte pairs into one 4-column word, and a half tile is one [rows][128 B] box.
template <int EPI, bool LINES = false, int KIND = 0>
__device__ __forceinline__ void frag_epilogue(const Params& p, const float (&d)[128], uint8_t* stg, const CUtensorMap* tmO,
                                              const int m_blk, const int n_blk, const int wgi, const bool issuer) {
  constexpr bool POOL = (EPI == EPI_RELU_POOL12);
  constexpr bool CONV = (EPI == EPI_RELU || POOL || EPI == EPI_STATS || EPI == EPI_CONV_STORE);
  constexpr bool RELU = (EPI == EPI_RELU || POOL);
  constexpr bool Q8 = (KIND == 2) && RELU;              // e4m3 output
  constexpr int BOX_BYTES = (POOL ? 64 : 128) * 128;     // one [rows][64 columns] bf16 box = one [rows][128 columns] e4m3 box
  constexpr int NBX = Q8 ? 1 : 2;                        // boxes per 128-column half
  const int t = threadIdx.x & 127, l = t & 31;
  const int r0 = wgi * 64 + 16 * (t >> 5) + (l >> 2);   // fragment rows r0 and r0 + 8
  const int col0 = n_blk * 256;
  bool ok0 = true, ok1 = true;
  if (EPI == EPI_STATS || LINES) { ok0 = conv_row_valid<LINES>(p, m_blk, r0); ok1 = conv_row_valid<LINES>(p, m_blk, r0 + 8); }
  int s0 = r0, s1 = r0 + 8;                              // staging rows (EPI_XPROJ: destination rows)
  bool direct = false;
  if (EPI == EPI_XPROJ && col0 >= 1024) {
    int dr[2] = {r0, r0 + 8};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int grow = m_blk * 128 + dr[i];
      if (grow < p.M) {
        const int n = grow / p.H, tt = grow - n * p.H;
        const int len = min(max(__ldg(p.seq_len + n), 0), p.T);
        if (tt < len) dr[i] = n * p.H + (len - 1 - tt) - m_blk * 128;
      }
    }
    s0 = dr[0]; s1 = dr[1];
    direct = (128 % p.H) != 0;
  }
  float inv_os = 1.f;
  if constexpr (Q8) inv_os = 1.f / __ldg(p.oscale);     // a power of two: multiplying by it is the exact division
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    uint8_t* buf = stg + hf * NBX * BOX_BYTES;
    if (hf == 0) {
      if (issuer) ptx::bulk_wait_read_all();            // the previous stores have read the buffer
      ptx::bar_sync(1, 256);
    }
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const int j = hf * 16 + jj;
      const int c = 8 * jj + 2 * (l & 3);                // column within the half
      float2 b = make_float2(0.f, 0.f);
      if (EPI != EPI_CONV_STORE && p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + hf * 128 + c));
      uint32_t v0, v1;
      if constexpr (KIND == 2) {
        const float2 cs = __ldg(reinterpret_cast<const float2*>(p.colscale + col0 + hf * 128 + c));
        float y0 = __fmaf_rn(d[4 * j], cs.x, b.x), y1 = __fmaf_rn(d[4 * j + 1], cs.y, b.y);
        float y2 = __fmaf_rn(d[4 * j + 2], cs.x, b.x), y3 = __fmaf_rn(d[4 * j + 3], cs.y, b.y);
        if constexpr (Q8) {
          y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); y2 = fmaxf(y2, 0.f); y3 = fmaxf(y3, 0.f);
          if (POOL) {                                    // rows r and r ^ 1 (w pair) sit in lanes l and l ^ 4
            y0 = fmaxf(y0, __shfl_xor_sync(0xffffffffu, y0, 4));
            y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, 4));
            y2 = fmaxf(y2, __shfl_xor_sync(0xffffffffu, y2, 4));
            y3 = fmaxf(y3, __shfl_xor_sync(0xffffffffu, y3, 4));
          }
          const uint32_t q0 = ptx::pack_e4m3x2(y0 * inv_os, y1 * inv_os), q8 = ptx::pack_e4m3x2(y2 * inv_os, y3 * inv_os);
          // even lanes keep row r0 (columns c .. c+3), odd lanes row r0 + 8 (columns c-2 .. c+1)
          const bool even = (l & 1) == 0;
          const uint32_t r = __shfl_xor_sync(0xffffffffu, even ? q8 : q0, 1);
          const uint32_t word = even ? (q0 | (r << 16)) : (r | (q8 << 16));
          const int row = even ? r0 : r0 + 8;
          const bool ok = even ? ok0 : ok1;
          // pooled: lanes l and l ^ 4 hold the same pooled rows; the lanes with (l & 4) == 0 store them
          if (!POOL || (l & 4) == 0) *stg_word8(buf, POOL ? row >> 1 : row, even ? c : c - 2) = ok ? word : 0u;
          continue;
        }
        v0 = ptx::pack_bf16x2(y0, y1);
        v1 = ptx::pack_bf16x2(y2, y3);
        if (EPI == EPI_BIAS_BF16 || EPI == EPI_STATS) {
          *stg_word(buf, BOX_BYTES, s0, c) = ok0 ? v0 : 0u;
          *stg_word(buf, BOX_BYTES, s1, c) = ok1 ? v1 : 0u;
          continue;
        }
      }
      if (EPI == EPI_CONV_STORE) {
        v0 = ptx::pack_bf16x2(d[4 * j], d[4 * j + 1]);
        v1 = ptx::pack_bf16x2(d[4 * j + 2], d[4 * j + 3]);
      } else if (RELU) {
        v0 = ptx::pack_bf16x2(fmaxf(d[4 * j] + b.x, 0.f), fmaxf(d[4 * j + 1] + b.y, 0.f));
        v1 = ptx::pack_bf16x2(fmaxf(d[4 * j + 2] + b.x, 0.f), fmaxf(d[4 * j + 3] + b.y, 0.f));
      } else {
        v0 = ptx::pack_bf16x2(d[4 * j] + b.x, d[4 * j + 1] + b.y);
        v1 = ptx::pack_bf16x2(d[4 * j + 2] + b.x, d[4 * j + 3] + b.y);
      }
      if (POOL) {
        // rows r and r ^ 1 (w pair) sit in lanes l and l ^ 4; rounding to bf16 is monotonic, so max after packing == packing after max
        v0 = ptx::hmax2_bf16(v0, __shfl_xor_sync(0xffffffffu, v0, 4));
        v1 = ptx::hmax2_bf16(v1, __shfl_xor_sync(0xffffffffu, v1, 4));
        // both lanes of the pair now hold both pooled rows: lane l stores the first, lane l ^ 4 the second (conflict-free); the
        // rows of a w pair share h, so either lane's validity is the pooled row's
        if ((l & 4) == 0) *stg_word(buf, BOX_BYTES, r0 >> 1, c) = ok0 ? v0 : 0u;
        else *stg_word(buf, BOX_BYTES, (r0 + 8) >> 1, c) = ok1 ? v1 : 0u;
      } else if (EPI == EPI_XPROJ && direct) {
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out) + col0 + hf * 128 + c;
        if (m_blk * 128 + r0 < p.M) *reinterpret_cast<uint32_t*>(out + (size_t)(m_blk * 128 + s0) * p.ldo) = v0;
        if (m_blk * 128 + r0 + 8 < p.M) *reinterpret_cast<uint32_t*>(out + (size_t)(m_blk * 128 + s1) * p.ldo) = v1;
      } else {
        *stg_word(buf, BOX_BYTES, s0, c) = ok0 ? v0 : 0u;
        *stg_word(buf, BOX_BYTES, s1, c) = ok1 ? v1 : 0u;
      }
    }
    if (EPI == EPI_XPROJ && direct) continue;
    ptx::fence_proxy_async_smem();                       // generic-proxy writes -> visible to the TMA (async proxy) reads
    ptx::bar_sync(1, 256);
    if (issuer) {
#pragma unroll
      for (int bx = 0; bx < NBX; ++bx) {
        const int c = col0 + hf * 128 + bx * 64;
        uint8_t* src = buf + bx * BOX_BYTES;
        if (CONV) {
          const int nb = p.merged ? 1 : 4;
          for (int sb = 0; sb < nb; ++sb) {
            const int g = m_blk * 4 + sb;
            const int n = g / p.sb_per_img;
            ptx::tma_store_4d(tmO, src + sb * (BOX_BYTES / 4), c, 0, (g - n * p.sb_per_img) * p.bh, n);
          }
        } else {
          ptx::tma_store_2d(tmO, src, c, m_blk * 128);
        }
      }
      ptx::bulk_commit();
    }
    if (EPI == EPI_STATS) {
      // thread = (column pair cp, rows rg*32 .. rg*32+31); a warp reads whole 128-B rows: conflict-free
      const int tt = threadIdx.x - 128;
      const int cp = tt & 63, rg = tt >> 6, cw = cp & 31;
      const uint8_t* bb = buf + (cp >> 5) * BOX_BYTES;
      const float4 s = rowsum_tree<1>(bb, rg, cw, 0);
      const int c = col0 + hf * 128 + 2 * cp;
      double* st = p.stats;
      if (LINES) {
        const int n = (m_blk * 4 + rg) / p.sb_per_img;
        if (n >= p.Nimg) continue;                         // padding sub-box past the last image: all rows zero
        st += (size_t)n * 2 * p.Nc;
      }
      atomicAdd(st + c, (double)s.x);
      atomicAdd(st + c + 1, (double)s.y);
      atomicAdd(st + p.Nc + c, (double)s.z);
      atomicAdd(st + p.Nc + c + 1, (double)s.w);
    }
  }
}

// Epilogue of tile columns [c_lo, c_hi): thread (q, lane) owns accumulator row q*32+lane of the 128-row tile.  `acc` holds
// the NC staged columns c_acc .. c_acc+NC-1 of the tile.
template <int BLOCK_N, int NC, int EPI>
__device__ __forceinline__ void run_epilogue(const Params& p, float* acc, const int m_blk, const int n_blk, const int q,
                                             const int lane, const int c_lo, const int c_hi, const int c_acc) {
  const int row = q * 32 + lane;
  const int col0 = n_blk * BLOCK_N;

  // ---- conv row geometry (one sub-box of 32 positions per warp)
  int n_img = 0, h = 0, w = 0;
  bool valid = true;
  if (EPI == EPI_RELU || EPI == EPI_RELU_POOL12 || EPI == EPI_STATS || EPI == EPI_RELU_POOL12_T || EPI == EPI_CONV_F32 ||
      EPI == EPI_CONV_STORE_MASK || EPI == EPI_CONV_STORE_BNRED) {
    const int g = m_blk * 4 + q;
    n_img = g / p.sb_per_img;
    const int hb = g - n_img * p.sb_per_img;
    const int hl = lane / p.Wd;
    w = lane - hl * p.Wd;
    h = hb * p.bh + hl;
    valid = (n_img < p.Nimg) && (h < p.H);
  }

  if (EPI == EPI_F32) {
    const int grow = m_blk * BLOCK_M + row;
    float* out = reinterpret_cast<float*>(p.out) + (size_t)grow * p.Nc + col0;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
      if (grow < p.M) {
#pragma unroll
        for (int i = 0; i < 32; i += 4)
          *reinterpret_cast<uint4*>(out + c0 + i) = make_uint4(v[i], v[i + 1], v[i + 2], v[i + 3]);
      }
    }
  } else if (EPI == EPI_BIAS_BF16 || EPI == EPI_XPROJ) {
    const int grow = m_blk * BLOCK_M + row;
    int drow = grow;
    if (EPI == EPI_XPROJ && col0 >= 1024 && grow < p.M) {
      // tf.reverse_sequence(len) on the backward direction's input, done once at write time
      const int n = grow / p.H, t = grow - n * p.H;
      const int len = min(max(__ldg(p.seq_len + n), 0), p.T);
      if (t < len) drow = n * p.H + (len - 1 - t);
    }
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)drow * p.ldo + col0;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
      uint32_t pk[16];
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        const float4 b = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + col0 + c0 + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
        pk[i / 2] = ptx::pack_bf16x2(__uint_as_float(v[i]) + b.x, __uint_as_float(v[i + 1]) + b.y);
        pk[i / 2 + 1] = ptx::pack_bf16x2(__uint_as_float(v[i + 2]) + b.z, __uint_as_float(v[i + 3]) + b.w);
      }
      if (grow < p.M) {
#pragma unroll
        for (int i = 0; i < 16; i += 8)
          ptx::st_global_v8(out + c0 + 2 * i, pk[i], pk[i + 1], pk[i + 2], pk[i + 3], pk[i + 4], pk[i + 5], pk[i + 6], pk[i + 7]);
      }
    }
  } else if (EPI == EPI_LOGITS) {
    const int grow = m_blk * BLOCK_M + row;
    const int n = grow / p.H, t = grow - n * p.H;
    const bool ok = (grow < p.M) && (t < p.T);
    float* out = reinterpret_cast<float*>(p.out) + ((size_t)t * p.Nimg + n) * p.Nc + col0;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
      if (ok) {
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + c0 + i));
          *reinterpret_cast<float4*>(out + c0 + i) =
              make_float4(__uint_as_float(v[i]) + b.x, __uint_as_float(v[i + 1]) + b.y,
                          __uint_as_float(v[i + 2]) + b.z, __uint_as_float(v[i + 3]) + b.w);
        }
      }
    }
  } else if (EPI == EPI_RELU || EPI == EPI_RELU_POOL12) {
    __nv_bfloat16* outb = reinterpret_cast<__nv_bfloat16*>(p.out);
    size_t off;
    if (EPI == EPI_RELU) off = (((size_t)n_img * p.H + h) * p.Wd + w) * p.Nc;
    else off = (((size_t)n_img * p.H + h) * (p.Wd >> 1) + (w >> 1)) * p.Nc;
    __nv_bfloat16* out = outb + off + col0;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
      uint32_t pk[16];
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + c0 + i));
        pk[i / 2] = ptx::pack_bf16x2(fmaxf(__uint_as_float(v[i]) + b.x, 0.f), fmaxf(__uint_as_float(v[i + 1]) + b.y, 0.f));
        pk[i / 2 + 1] = ptx::pack_bf16x2(fmaxf(__uint_as_float(v[i + 2]) + b.z, 0.f), fmaxf(__uint_as_float(v[i + 3]) + b.w, 0.f));
      }
      if (EPI == EPI_RELU) {
        if (valid) {
#pragma unroll
          for (int i = 0; i < 16; i += 8)
            ptx::st_global_v8(out + c0 + 2 * i, pk[i], pk[i + 1], pk[i + 2], pk[i + 3], pk[i + 4], pk[i + 5], pk[i + 6], pk[i + 7]);
        }
      } else {
        // lane = hl*8 + w: partner lane^1 (w pair); rounding to bf16 is monotonic, so max after packing == packing after max
#pragma unroll
        for (int i = 0; i < 16; ++i) pk[i] = ptx::hmax2_bf16(pk[i], __shfl_xor_sync(0xffffffffu, pk[i], 1));
        const int sub = lane & 1;
        uint4 o0, o1;
        o0.x = sub ? pk[8] : pk[0];  o0.y = sub ? pk[9] : pk[1];  o0.z = sub ? pk[10] : pk[2]; o0.w = sub ? pk[11] : pk[3];
        o1.x = sub ? pk[12] : pk[4]; o1.y = sub ? pk[13] : pk[5]; o1.z = sub ? pk[14] : pk[6]; o1.w = sub ? pk[15] : pk[7];
        if (valid) {
          *reinterpret_cast<uint4*>(out + c0 + 16 * sub) = o0;
          *reinterpret_cast<uint4*>(out + c0 + 16 * sub + 8) = o1;
        }
      }
    }
  } else if (EPI == EPI_CONV_STORE_MASK) {
    const size_t off = (((size_t)n_img * p.H + h) * p.Wd + w) * p.Nc + col0;
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out) + off;
    const __nv_bfloat16* msk = p.mask + off;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint4 mk[4];
      if (valid) {
#pragma unroll
        for (int i = 0; i < 4; ++i) mk[i] = __ldg(reinterpret_cast<const uint4*>(msk + c0) + i);     // issued before the accumulator reads
      }
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
      if (valid) {
        const uint32_t* mw = reinterpret_cast<const uint32_t*>(mk);
        uint32_t pk[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          // the activation is post-ReLU (>= 0): "> 0" is "bf16 bits, sign aside, non-zero"; rounding then masking == masking then rounding
          const uint32_t keep = ((mw[i] & 0x7FFFu) ? 0xFFFFu : 0u) | ((mw[i] & 0x7FFF0000u) ? 0xFFFF0000u : 0u);
          pk[i] = ptx::pack_bf16x2(__uint_as_float(v[2 * i]), __uint_as_float(v[2 * i + 1])) & keep;
        }
#pragma unroll
        for (int i = 0; i < 16; i += 8)
          ptx::st_global_v8(out + c0 + 2 * i, pk[i], pk[i + 1], pk[i + 2], pk[i + 3], pk[i + 4], pk[i + 5], pk[i + 6], pk[i + 7]);
      }
    }
  } else if (EPI == EPI_CONV_STORE_BNRED) {
    // same sums as bn_bwd_reduce_kernel<false> (backward_kernels.cu), taken on the bf16-rounded gradient the apply pass will read
    const size_t off = (((size_t)n_img * p.H + h) * p.Wd + w) * p.Nc + col0;
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out) + off;
    const __nv_bfloat16* xp = p.mask + off;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint4 xq[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) xq[i] = valid ? __ldg(reinterpret_cast<const uint4*>(xp + c0) + i) : make_uint4(0u, 0u, 0u, 0u);
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
      const uint32_t* xw = reinterpret_cast<const uint32_t*>(xq);
      uint32_t pk[16];
      float f[32], f2[32];
      const float* bc = p.bnp + col0 + c0;
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        const float4 sc = __ldg(reinterpret_cast<const float4*>(bc + i));
        const float4 sh = __ldg(reinterpret_cast<const float4*>(bc + p.Nc + i));
        const float4 mu = __ldg(reinterpret_cast<const float4*>(bc + 2 * p.Nc + i));
        const float4 is = __ldg(reinterpret_cast<const float4*>(bc + 3 * p.Nc + i));
        pk[i / 2] = ptx::pack_bf16x2(__uint_as_float(v[i]), __uint_as_float(v[i + 1]));
        pk[i / 2 + 1] = ptx::pack_bf16x2(__uint_as_float(v[i + 2]), __uint_as_float(v[i + 3]));
        const float x0 = ptx::bf16_lo(xw[i / 2]), x1 = ptx::bf16_hi(xw[i / 2]), x2 = ptx::bf16_lo(xw[i / 2 + 1]), x3 = ptx::bf16_hi(xw[i / 2 + 1]);
        const float d0 = (valid && fmaf(x0, sc.x, sh.x) > 0.f) ? ptx::bf16_lo(pk[i / 2]) : 0.f;
        const float d1 = (valid && fmaf(x1, sc.y, sh.y) > 0.f) ? ptx::bf16_hi(pk[i / 2]) : 0.f;
        const float d2 = (valid && fmaf(x2, sc.z, sh.z) > 0.f) ? ptx::bf16_lo(pk[i / 2 + 1]) : 0.f;
        const float d3 = (valid && fmaf(x3, sc.w, sh.w) > 0.f) ? ptx::bf16_hi(pk[i / 2 + 1]) : 0.f;
        f[i] = d0; f[i + 1] = d1; f[i + 2] = d2; f[i + 3] = d3;
        f2[i] = d0 * (x0 - mu.x) * is.x; f2[i + 1] = d1 * (x1 - mu.y) * is.y; f2[i + 2] = d2 * (x2 - mu.z) * is.z; f2[i + 3] = d3 * (x3 - mu.w) * is.w;
      }
      if (valid) {
#pragma unroll
        for (int i = 0; i < 16; i += 8)
          ptx::st_global_v8(out + c0 + 2 * i, pk[i], pk[i + 1], pk[i + 2], pk[i + 3], pk[i + 4], pk[i + 5], pk[i + 6], pk[i + 7]);
      }
      const float s1 = warp_colsum32(f, lane);
      const float s2 = warp_colsum32(f2, lane);
      atomicAdd(p.stats + col0 + c0 + lane, (double)s1);
      atomicAdd(p.stats + p.Nc + col0 + c0 + lane, (double)s2);
    }
  } else if (EPI == EPI_CONV_F32) {
    float* out = reinterpret_cast<float*>(p.out) + (((size_t)n_img * p.H + h) * p.Wd + w) * p.Nc + col0;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
      if (valid) {
#pragma unroll
        for (int i = 0; i < 32; i += 4)
          *reinterpret_cast<uint4*>(out + c0 + i) = make_uint4(v[i], v[i + 1], v[i + 2], v[i + 3]);
      }
    }
  } else if (EPI == EPI_RELU_POOL12_T) {
    // Training variant: max over the pooling window carried as an integer key
    //   key = (bf16 bits of relu(x) << 2) | (1 - window_index)
    // post-ReLU bf16 bit patterns are monotone as unsigned integers, so max(key) picks the largest value and, among
    // equal values, the FIRST window position (the tie-break of TF/torch max-pool gradients).
    const size_t off = (((size_t)n_img * p.H + h) * (p.Wd >> 1) + (w >> 1)) * p.Nc;
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out) + off + col0;
    uint8_t* amx = p.argmax + off + col0;
    const uint32_t kidx = (uint32_t)(lane & 1);
    const uint32_t kinv = 1u - kidx;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + c0 + i));
        const uint32_t p0 = ptx::pack_bf16x2(fmaxf(__uint_as_float(v[i]) + b.x, 0.f), fmaxf(__uint_as_float(v[i + 1]) + b.y, 0.f));
        const uint32_t p1 = ptx::pack_bf16x2(fmaxf(__uint_as_float(v[i + 2]) + b.z, 0.f), fmaxf(__uint_as_float(v[i + 3]) + b.w, 0.f));
        v[i] = ((p0 & 0xFFFFu) << 2) | kinv;
        v[i + 1] = ((p0 >> 16) << 2) | kinv;
        v[i + 2] = ((p1 & 0xFFFFu) << 2) | kinv;
        v[i + 3] = ((p1 >> 16) << 2) | kinv;
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = max(v[i], __shfl_xor_sync(0xffffffffu, v[i], 1));
      // each lane of the window stores its 16 of the 32 columns
      constexpr int NS = 2, PER = 32 / NS;
      const int sub = lane & 1;
      uint32_t sel[PER];
#pragma unroll
      for (int i = 0; i < PER; ++i) {
        uint32_t x = v[i];
#pragma unroll
        for (int j = 1; j < NS; ++j) x = (sub == j) ? v[j * PER + i] : x;
        sel[i] = x;
      }
      if (valid) {
#pragma unroll
        for (int i = 0; i < PER; i += 8) {
          uint4 o;
          o.x = ((sel[i] >> 2) & 0xFFFFu) | ((sel[i + 1] >> 2) << 16);
          o.y = ((sel[i + 2] >> 2) & 0xFFFFu) | ((sel[i + 3] >> 2) << 16);
          o.z = ((sel[i + 4] >> 2) & 0xFFFFu) | ((sel[i + 5] >> 2) << 16);
          o.w = ((sel[i + 6] >> 2) & 0xFFFFu) | ((sel[i + 7] >> 2) << 16);
          *reinterpret_cast<uint4*>(out + c0 + sub * PER + i) = o;
          const uint32_t km = 1u;
          uint2 a;
          a.x = (km - (sel[i] & km)) | ((km - (sel[i + 1] & km)) << 8) | ((km - (sel[i + 2] & km)) << 16) | ((km - (sel[i + 3] & km)) << 24);
          a.y = (km - (sel[i + 4] & km)) | ((km - (sel[i + 5] & km)) << 8) | ((km - (sel[i + 6] & km)) << 16) | ((km - (sel[i + 7] & km)) << 24);
          *reinterpret_cast<uint2*>(amx + c0 + sub * PER + i) = a;
        }
      }
    }
  } else if (EPI == EPI_STATS) {
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out) + (((size_t)n_img * p.H + h) * p.Wd + w) * p.Nc + col0;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 32) {
      uint32_t v[32];
      ptx::acc_ld<NC, 32>(acc, row, c0 - c_acc, v);
      float f[32], f2[32];
      uint32_t pk[16];
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + c0 + i));
        f[i] = __uint_as_float(v[i]) + b.x;
        f[i + 1] = __uint_as_float(v[i + 1]) + b.y;
        f[i + 2] = __uint_as_float(v[i + 2]) + b.z;
        f[i + 3] = __uint_as_float(v[i + 3]) + b.w;
        pk[i / 2] = ptx::pack_bf16x2(f[i], f[i + 1]);
        pk[i / 2 + 1] = ptx::pack_bf16x2(f[i + 2], f[i + 3]);
      }
      if (valid) {
#pragma unroll
        for (int i = 0; i < 16; i += 8)
          ptx::st_global_v8(out + c0 + 2 * i, pk[i], pk[i + 1], pk[i + 2], pk[i + 3], pk[i + 4], pk[i + 5], pk[i + 6], pk[i + 7]);
      }
      // statistics of the values the next layer will actually read (bf16-rounded), masked to valid rows
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float a = valid ? ptx::bf16_lo(pk[i]) : 0.f, b = valid ? ptx::bf16_hi(pk[i]) : 0.f;
        f[2 * i] = a; f[2 * i + 1] = b;
        f2[2 * i] = a * a; f2[2 * i + 1] = b * b;
      }
      const float s1 = warp_colsum32(f, lane);
      const float s2 = warp_colsum32(f2, lane);
      atomicAdd(p.stats + col0 + c0 + lane, (double)s1);
      atomicAdd(p.stats + p.Nc + col0 + c0 + lane, (double)s2);
    }
  }
}

// KIND 0: bf16 operands, 64 elements per 128 B K-block.  KIND 1: f32 words read as tf32, 32 elements per K-block
// (forward_x3.cu, compute_dtype 3); tensor maps are FLOAT32 with 32-element boxes, everything else is shared.
// KIND 2: e4m3 operands, 128 elements per K-block (forward_fp8.cu, compute_dtype 4); UINT8 tensor maps with 128-element
// boxes, four k32 MMAs per K-block, register-side epilogues only (see frag_epilogue).
// LINES: packed evaluation lines (Params::line_w), frag_epi conv epilogues only
template <int BLOCK_N, int AMODE, int EPI, int STAGES, int KIND = 0, bool LINES = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
            const Params p) {
  static_assert(BLOCK_N == 64 || BLOCK_N == 128 || BLOCK_N == 256, "BLOCK_N");
  constexpr bool FRAG = frag_epi(BLOCK_N, EPI);          // tmO (output map) is read only by these
  static_assert(!LINES || (FRAG && AMODE == A_CONV3 && (KIND == 0 || KIND == 2)), "line masks exist in the register-side conv epilogues only");
  static_assert(KIND != 2 || (BLOCK_N == 256 && (EPI == EPI_RELU || EPI == EPI_RELU_POOL12 || EPI == EPI_STATS || EPI == EPI_BIAS_BF16)),
                "e4m3 GEMMs: conv3_1, conv3_2, conv4_x and conv5");
  constexpr int SLICE_N = slice_cols(BLOCK_N, EPI);
  using SM = Smem<BLOCK_N, STAGES, SLICE_N>;
  constexpr int S = SM::S;
  constexpr int B_STAGE_BYTES = BLOCK_N * 128;
  constexpr int KELEMS = KIND == 2 ? 128 : KIND ? 32 : BLOCK_K;        // operand elements per 128 B K-block

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + S * A_STAGE_BYTES;
  float* acc_tile = reinterpret_cast<float*>(smem + SM::ACC_OFFSET);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + S;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;

  if (warp_idx == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    if (FRAG) ptx::prefetch_tmap(&tmO);
    for (int s = 0; s < S; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);              // one arrive per MMA warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    // ===================== TMA producer =====================
    // One lane per TMA box: a single thread issuing 5 boxes per K-block serialises the conv mainloop on the issue latency.
    // Lanes 0..nA-1 load the A sub-boxes, lane nA loads B; lane 0 also arms the transaction count.  conv: when the tile's 4
    // sub-boxes are contiguous rows of one image (p.merged), a single 128-position box replaces them.
    ptx::setmaxnreg_dec<24>();
    const int nA = (AMODE == A_CONV3 && !p.merged) ? 4 : 1;
    if (warp_idx == 0 && lane <= nA) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = p.m_tile0 + tile / p.num_n_tiles, n_blk = tile % p.num_n_tiles;
        const int b_row = n_blk * BLOCK_N;
        // per-tile coordinates of this lane's A box (conv): image n, first H row h0
        int cn = 0, ch0 = 0;
        if (AMODE == A_CONV3 && lane < nA) {
          const int g = m_blk * 4 + lane;
          cn = g / p.sb_per_img;
          ch0 = (g - cn * p.sb_per_img) * p.bh;
        }
        int tap = 0, cb = 0;                    // conv K-block decomposition, advanced incrementally
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          if (p.debug_skip_tma) {
            if (lane == 0) ptx::mbar_arrive(&full_bar[stage]);
          } else {
            if (lane == 0) ptx::mbar_arrive_expect_tx(&full_bar[stage], A_STAGE_BYTES + B_STAGE_BYTES);
            if (lane < nA) {
              uint8_t* a_dst = smem_a + stage * A_STAGE_BYTES;
              if (AMODE == A_PLAIN) {
                const int rs = kb / p.kb_per_shift;
                int kc = kb - rs * p.kb_per_shift;
                if (p.kb_phys > 0 && kc >= p.kb_phys) kc -= p.kb_phys;
                ptx::tma_load_2d(&tmA, &full_bar[stage], a_dst, kc * KELEMS, m_blk * BLOCK_M + rs * p.row_shift_mul);
              } else {
                const int r = tap / 3, sx = tap - 3 * r;
                const int cbp = (p.cin_phys > 0 && cb >= p.cin_phys) ? cb - p.cin_phys : cb;
                ptx::tma_load_4d(&tmA, &full_bar[stage], a_dst + lane * 4096, cbp * KELEMS, sx - 1, ch0 + r - 1, cn);
              }
            } else {
              ptx::tma_load_2d(&tmB, &full_bar[stage], smem_b + stage * B_STAGE_BYTES, kb * KELEMS, b_row);
            }
          }
          if (++cb == p.cin_blocks) { cb = 0; ++tap; }
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA warpgroups (rows wgi*64 ..) + epilogue =====================
    ptx::setmaxnreg_inc<240>();
    const int wgi = (warp_idx >> 2) - 1;
    const int q = warp_idx & 3;                      // accumulator row quadrant drained by this warp
    const int chalf = (warp_idx - 4) >> 2;           // warps 4..7 take the first half of each staged slice, warps 8..11 the second
    const bool arriver = (warp_idx & 3) == 0 && lane == 0;
    const bool issuer = FRAG && threadIdx.x == 128;  // issues and waits on the epilogue's TMA stores
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = p.m_tile0 + tile / p.num_n_tiles, n_blk = tile % p.num_n_tiles;
      float d[BLOCK_N / 2];
      int prev = -1;
      for (int kb = 0; kb < p.num_k_blocks; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint64_t a_desc = ptx::make_desc_k_sw128(ptx::smem_u32(smem_a + stage * A_STAGE_BYTES + wgi * 64 * 128));
        const uint64_t b_desc = ptx::make_desc_k_sw128(ptx::smem_u32(smem_b + stage * B_STAGE_BYTES));
        wg::fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
          // advance 16 bf16 (8 tf32, 32 e4m3) = 32 B along K inside the 128 B swizzle row: +2 in the (addr >> 4) field
          if constexpr (KIND == 2) wg::mma_e4m3<BLOCK_N>(d, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
          else if (KIND) wg::mma_tf32<BLOCK_N>(d, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
          else wg::mma_bf16<BLOCK_N>(d, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
        }
        wg::commit();
        wg::wait<1>();                               // the previous K-block's MMAs have retired: free its smem slot
        if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
      wg::wait<0>();
      wg::fence_operand(d);
      if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
      if (p.debug_skip_epilogue) continue;
      if constexpr (FRAG) {
        frag_epilogue<EPI, LINES, KIND>(p, d, reinterpret_cast<uint8_t*>(acc_tile), &tmO, m_blk, n_blk, wgi, issuer);
      } else {
#pragma unroll
        for (int s = 0; s < BLOCK_N / SLICE_N; ++s) {
          ptx::bar_sync(1, 256);                     // the previous slice's (tile's) epilogue reads are done
          ptx::acc_store_slice<BLOCK_N, SLICE_N>(acc_tile, d, wgi * 64, s);
          ptx::bar_sync(1, 256);
          const int c_lo = s * SLICE_N + chalf * (SLICE_N / 2);
          run_epilogue<BLOCK_N, SLICE_N, EPI>(p, acc_tile, m_blk, n_blk, q, lane, c_lo, c_lo + SLICE_N / 2, s * SLICE_N);
        }
      }
    }
    if (FRAG && issuer) ptx::bulk_wait_all();        // the CTA's shared memory must outlive its last stores
  }
}

}  // namespace gemm
