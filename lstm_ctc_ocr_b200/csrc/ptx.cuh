// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma descriptors, clusters.
// No CUTLASS/CuTe dependency; bit layouts of the descriptors are documented next to each builder.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ------------------------------------------------------------------ bulk copies without a tensor map (1-D, 16-B granules)
__device__ __forceinline__ void bulk_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(reinterpret_cast<uint64_t>(src_gmem)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_store_1d(void* dst_gmem, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(reinterpret_cast<uint64_t>(dst_gmem)),
               "r"(smem_u32(src_smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every committed bulk group of this thread has completed (writes included): before a CTA that issued stores exits
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// 1-D bulk copy global -> the SAME smem offset of every CTA in `cta_mask`; each destination's mbarrier (same offset) gets the bytes
__device__ __forceinline__ void bulk_load_1d_mc(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar, uint16_t cta_mask) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(dst_smem)), "l"(reinterpret_cast<uint64_t>(src_gmem)), "r"(bytes), "r"(smem_u32(bar)), "h"(cta_mask)
               : "memory");
}
// ------------------------------------------------------------------ TMA loads (tile mode, OOB -> 0)
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const void* tmap, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const void* tmap, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}

// 128-bit vector reduction into global memory (PTX ISA 8.1, sm_90+): one L2 atomic transaction for 4 consecutive floats
__device__ __forceinline__ void red_add_v4_f32(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// smem tile -> global through a tensor map (bulk async group; complete with bulk_commit / bulk_wait_read_all)
__device__ __forceinline__ void tma_store_4d(const void* tmap, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}

// ------------------------------------------------------------------ wgmma operand descriptors (sm_90)
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [62,64) layout type: 0 = no swizzle (8-row x 16-B core matrices), 1 = SWIZZLE_128B
// K-major, no swizzle: `lbo` = byte distance between the two core matrices of one K=16 step, `sbo` = between 8-row groups.
__device__ __forceinline__ uint64_t make_desc_k_nosw(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo >> 4) << 16;
  d |= static_cast<uint64_t>(sbo >> 4) << 32;
  return d;
}
// K-major, 128-byte swizzle (rows of 128 B as written by TMA, 8-row atoms of 1024 B): SBO = 1024 B between 8-row groups.
// One K step (16 bf16 / 8 tf32 = 32 B) inside the swizzle row is +2 in the address field.
__device__ __forceinline__ uint64_t make_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// round-to-nearest f32 -> tf32 (the tensor core would otherwise truncate)
__device__ __forceinline__ float round_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}

// register budget of a warpgroup (all four warps execute it): producers give registers up, MMA warpgroups take them
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------ accumulator tile staged in shared memory
// The MMA warpgroups hold the accumulators in the wgmma fragment layout; the epilogues own one accumulator ROW per thread.
// The tile goes through shared memory as [rows][NC] f32 whose 16-B chunks are XOR-swizzled by (row & 7): fragment stores are
// at most 2-way conflicted and row-per-thread 16-B reads of a quarter-warp hit 8 different chunks (conflict-free).
template <int NC>
__device__ __forceinline__ float* acc_chunk(float* tile, int row, int c4) {
  return tile + row * NC + ((c4 ^ (row & 7)) << 2);
}
// fragment of one m64 x N wgmma (this thread's warpgroup) -> rows row0 .. row0+63, columns col0 .. col0+N-1
template <int N, int NC>
__device__ __forceinline__ void acc_store(float* tile, const float (&d)[N / 2], int row0, int col0 = 0) {
  const int t = threadIdx.x & 127, l = t & 31;
  const int r = row0 + 16 * (t >> 5) + (l >> 2);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int c = col0 + 8 * j + 2 * (l & 3);
    *reinterpret_cast<float2*>(acc_chunk<NC>(tile, r, c >> 2) + (c & 3)) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(acc_chunk<NC>(tile, r + 8, c >> 2) + (c & 3)) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// column slice s of the same fragment: columns s*NC .. s*NC+NC-1 (registers 4j .. 4j+3 of column groups j = s*NC/8 ..) ->
// rows row0 .. row0+63, columns 0 .. NC-1 of an NC-wide tile.  Call it with a constant s (an unrolled slice loop), so that the
// register indices stay compile-time constants.
template <int N, int NC>
__device__ __forceinline__ void acc_store_slice(float* tile, const float (&d)[N / 2], int row0, int s) {
  const int t = threadIdx.x & 127, l = t & 31;
  const int r = row0 + 16 * (t >> 5) + (l >> 2);
#pragma unroll
  for (int jj = 0; jj < NC / 8; ++jj) {
    const int j = s * (NC / 8) + jj;
    const int c = 8 * jj + 2 * (l & 3);
    *reinterpret_cast<float2*>(acc_chunk<NC>(tile, r, c >> 2) + (c & 3)) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(acc_chunk<NC>(tile, r + 8, c >> 2) + (c & 3)) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// row-per-thread read of NV consecutive columns c0 .. c0+NV-1 (c0 % 4 == 0) of `row`, as raw f32 bits
template <int NC, int NV>
__device__ __forceinline__ void acc_ld(float* tile, int row, int c0, uint32_t (&v)[NV]) {
#pragma unroll
  for (int i = 0; i < NV / 4; ++i) {
    const float4 x = *reinterpret_cast<const float4*>(acc_chunk<NC>(tile, row, (c0 >> 2) + i));
    v[4 * i] = __float_as_uint(x.x); v[4 * i + 1] = __float_as_uint(x.y);
    v[4 * i + 2] = __float_as_uint(x.z); v[4 * i + 3] = __float_as_uint(x.w);
  }
}


// ------------------------------------------------------------------ cluster helpers
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `local_smem_addr` in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t mapa(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
// wait with acquire at CLUSTER scope: pairs with mbar_arrive_cluster (release.cluster) of a peer CTA whose global writes are read next
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// TMA load multicast: the box lands at the same smem offset, and completes on the mbarrier at the same offset, in every CTA
// of `cta_mask` (one L2 read feeds the whole cluster)
__device__ __forceinline__ void tma_load_2d_mc(const void* tmap, uint64_t* bar, void* dst, int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
// ------------------------------------------------------------------ misc math / packing
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ uint32_t hmax2_bf16(uint32_t a, uint32_t b) {
  __nv_bfloat162 x = *reinterpret_cast<__nv_bfloat162*>(&a);
  __nv_bfloat162 y = *reinterpret_cast<__nv_bfloat162*>(&b);
  __nv_bfloat162 r = __hmax2(x, y);
  return *reinterpret_cast<uint32_t*>(&r);
}
// two f32 -> two e4m3 (round to nearest even, saturating to +-448; NaN stays NaN): `lo` in bits 0..7, `hi` in bits 8..15
__device__ __forceinline__ uint32_t pack_e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// four f32 -> one 32-bit word of e4m3, a in the lowest byte
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  return pack_e4m3x2(a, b) | (pack_e4m3x2(c, d) << 16);
}
__device__ __forceinline__ float e4m3_to_f32(uint32_t byte) {
  uint32_t h;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"((uint16_t)byte));
  return __half2float(__ushort_as_half((unsigned short)(h & 0xFFFFu)));
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }

// ------------------------------------------------------------------ 32-B global store as two 16-B stores (32-B aligned address)
__device__ __forceinline__ void st_global_v8(void* ptr, uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e, uint32_t f,
                                             uint32_t g, uint32_t h) {
  uint4* p = reinterpret_cast<uint4*>(ptr);
  p[0] = make_uint4(a, b, c, d);
  p[1] = make_uint4(e, f, g, h);
}

// ------------------------------------------------------------------ f32 pairs packed in 64 bits (two IEEE fma.rn)
__device__ __forceinline__ uint64_t pack_f32x2(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack_f32x2(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t ffma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  unpack_f32x2(a, a0, a1); unpack_f32x2(b, b0, b1); unpack_f32x2(c, c0, c1);
  return pack_f32x2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// One MUFU op each (the LSTM cell epilogue is MUFU-bound: 5 transcendentals per hidden unit per step).
// tanh.approx.f32: max relative error ~2^-11, far below the bf16 rounding of h that follows.
__device__ __forceinline__ float fast_tanh(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_sigmoid(float x) { return fmaf(0.5f, fast_tanh(0.5f * x), 0.5f); }

}  // namespace ptx
