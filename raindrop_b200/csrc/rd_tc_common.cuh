// Shared device-side PTX wrappers (mbarrier, TMA, wgmma, mma.sync) and host-side tensor-map helpers of
// the tensor-core kernels (rd_obprop_tc.cu, rd_tc_gemm.cu, rd_attn_tc.cu).  sm_90a.
#pragma once
#include <cuda.h>
#include <stdint.h>

#include <mutex>

#include "rd_common.cuh"

namespace rd {
namespace tc {

constexpr int SMEM_LIMIT = 232448;   // 227 KB of dynamic shared memory per CTA

__device__ __forceinline__ float rn_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}

// ---- PTX wrappers -------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(bar), "r"(parity) : "memory");
}
// non-blocking: has the phase of this parity completed?
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  return done != 0;
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// ---- split of an fp32 operand for the error-compensated ("3xTF32") products ----------------------------------------
// hi = the top 19 bits (exactly representable in TF32), lo = x - hi (exact).  hi*hi + hi*lo + lo*hi reproduces the fp32
// product to ~2^-22 relative, independent of how the tensor core converts a raw fp32 bit pattern.
__device__ __forceinline__ uint32_t tf32_hi(float x) { return __float_as_uint(x) & 0xFFFFE000u; }
__device__ __forceinline__ uint32_t tf32_lo(float x) { return __float_as_uint(x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u)); }

// ---- warp-level tensor-core MMA: D[16x8] += A[16x8] . B[8x8], TF32 operands, fp32 accumulate -------------------------
// fragments (g = lane / 4, t = lane % 4):  a0 (g, t)  a1 (g+8, t)  a2 (g, t+4)  a3 (g+8, t+4)
//                                          b0 (k=t, n=g)  b1 (k=t+4, n=g)
//                                          d0 (g, 2t)  d1 (g, 2t+1)  d2 (g+8, 2t)  d3 (g+8, 2t+1)
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// error-compensated: small terms first, then hi.hi
__device__ __forceinline__ void mma_tf32x3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint32_t bh0,
                                           uint32_t bh1, uint32_t bl0, uint32_t bl1) {
  mma_tf32(d, al, bh0, bh1);
  mma_tf32(d, ah, bl0, bl1);
  mma_tf32(d, ah, bh0, bh1);
}

// ---- warpgroup MMA (wgmma) synchronisation; the TF32 MMA itself, wgmma_tf32<N>, is in rd_wgmma_tf32.cuh -------------
// A fragment of warp w of the warpgroup: rows 16w .. 16w+15, same (g, t) layout as mma_tf32 above.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// shared-memory matrix descriptor of a K-major tile written by TMA with CU_TENSOR_MAP_SWIZZLE_128B: rows of 128 bytes
// (32 fp32 of K), 8-row groups 1024 bytes apart (SBO), layout type 1 = 128-byte swizzle.  Moving along K inside the
// 128-byte row is a plain advance of the start address (32 bytes per 8-wide k-step).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// byte offset of element (row, col) (col < 32) inside such a tile
__device__ __forceinline__ uint32_t sw128_offset(int row, int col) {
  return (uint32_t)(row * 128 + ((((col >> 2) ^ row) & 7) << 4) + (col & 3) * 4);
}

// ---- host side -----------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// cuTensorMapEncodeTiled costs a few microseconds of host time; a training step re-encodes the same
// ~90 maps every step (same buffers, same shapes), so keep them in a small direct-mapped cache.
struct TmapKey {
  const void* addr; int rank; int swizzle; cuuint64_t dims[5]; cuuint64_t strides[4]; cuuint32_t box[5];
  bool operator==(const TmapKey& o) const {
    if (addr != o.addr || rank != o.rank || swizzle != o.swizzle) return false;
    for (int i = 0; i < 5; ++i) if (dims[i] != o.dims[i] || box[i] != o.box[i]) return false;
    for (int i = 0; i < 4; ++i) if (strides[i] != o.strides[i]) return false;
    return true;
  }
};
struct TmapSlot { bool valid = false; TmapKey key; CUtensorMap map; };

inline int encode(CUtensorMap* m, const void* addr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                  const cuuint32_t* box, CUtensorMapSwizzle sw, const char* what) {
  constexpr int NSLOT = 512;
  static thread_local TmapSlot cache[NSLOT];
  TmapKey k{};
  k.addr = addr; k.rank = rank; k.swizzle = (int)sw;
  for (int i = 0; i < rank; ++i) { k.dims[i] = dims[i]; k.box[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) k.strides[i] = strides_bytes[i];
  uint64_t h = reinterpret_cast<uintptr_t>(addr) * 0x9E3779B97F4A7C15ull;
  h ^= (dims[0] * 0xC2B2AE3D27D4EB4Full) ^ ((uint64_t)box[rank - 1] << 17) ^ (rank > 1 ? dims[1] * 0x165667B19E3779F9ull : 0);
  TmapSlot& slot = cache[(h >> 40) % NSLOT];
  if (slot.valid && slot.key == k) { *m = slot.map; return 0; }
  EncodeTiledFn fn = get_encode();
  if (!fn) { set_error("cuTensorMapEncodeTiled not available from the driver"); return -3; }
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(addr), dims, strides_bytes,
                  box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(%s) failed: CUresult %d", what, (int)r); return -3; }
  slot.valid = true; slot.key = k; slot.map = *m;
  return 0;
}

// cudaFuncSetAttribute(max dynamic shared memory) once per (kernel, device): a process that touches a second
// GPU has to opt in there as well (the attribute is per device).
inline int ensure_max_smem(const void* fn, int bytes) {
  struct Slot { const void* fn; int dev; };
  static Slot done[256];
  static int n = 0;
  static std::mutex mu;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  for (int i = 0; i < n; ++i) if (done[i].fn == fn && done[i].dev == dev) return 0;
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(smem): %s", cudaGetErrorString(e)); return -1; }
  if (n < 256) { done[n].fn = fn; done[n].dev = dev; ++n; }
  return 0;
}

inline int num_sms() {
  static int n[16] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  const int slot = (dev >= 0 && dev < 16) ? dev : 0;
  if (n[slot] == 0) {
    cudaDeviceGetAttribute(&n[slot], cudaDevAttrMultiProcessorCount, dev);
    if (n[slot] <= 0) n[slot] = 132;
  }
  return n[slot];
}

}  // namespace tc
}  // namespace rd
