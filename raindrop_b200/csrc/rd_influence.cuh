// Code shared by the influence kernels (rd_influence.cu: psg_dot_kernel, rd_projection.cu: grad_proj_kernel): the
// TF32 remainder image of a block of rows and the shared-memory ring their TMA producers fill.  sm_90a.
#pragma once
#include "rd_tc_common.cuh"

namespace rd {

// lo[i] = G[i] - (top 19 bits of G[i]) for i < n (n % 4 == 0, both 16-byte aligned): the exact remainder that, with the
// raw rows read as TF32 by the tensor cores, makes an error-compensated B operand (psg_lo_kernel, rd_influence.cu)
int grad_lo_image(const float* G, long long n, float* lo, cudaStream_t st);

namespace tc {

// The ring: one TMA thread fills STAGES stages, consumer warps drain them in the same order.  Barriers, 8 bytes each from
// `bar`: full[s] (one arrival, the producer's expect_tx, completed by the TMA bytes), then empty[s] (one arrival per
// consumer warp).

// a stage and the parity of its current use
template <int STAGES>
struct RingPos {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
  }
};

template <int STAGES>
struct TmaRing {
  uint32_t bar;
  __device__ __forceinline__ uint32_t full(int s) const { return bar + 8u * s; }
  __device__ __forceinline__ uint32_t empty(int s) const { return bar + 8u * (STAGES + s); }
  // one thread, before the CTA's first __syncthreads()
  __device__ __forceinline__ void init(uint32_t consumer_warps) const {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), consumer_warps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // producer: waits until stage p.stage is free and arms it for `bytes` of TMA; the loads then signal full(stage)
  __device__ __forceinline__ int produce(RingPos<STAGES>& p, uint32_t bytes) const {
    mbar_wait(empty(p.stage), p.phase ^ 1u);
    mbar_expect_tx(full(p.stage), bytes);
    const int s = p.stage;
    p.advance();
    return s;
  }
  // consumer: waits until stage p.stage has landed
  __device__ __forceinline__ int consume(RingPos<STAGES>& p) const {
    mbar_wait(full(p.stage), p.phase);
    const int s = p.stage;
    p.advance();
    return s;
  }
  // consumer warp: hands the oldest stage it still holds back to the producer
  __device__ __forceinline__ void release(RingPos<STAGES>& p, int lane) const {
    __syncwarp();
    if (lane == 0) mbar_arrive(empty(p.stage));
    p.advance();
  }
};

}  // namespace tc
}  // namespace rd
