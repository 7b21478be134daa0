// Observation-propagation layer forward on the Hopper tensor cores (sm_90a).
//
//   out[r, :] = relu(x[r, :] . W^T + b) * s[r % N]            x: [B*N, C] fp32, W: [C, C] fp32
//
// which is what `Observation_progation` computes on the live path (code/Ob_propagation.py:187-228:
// the message relu(lin_value(x_i)) depends on the target only, so segment-softmax + scatter-add
// collapse to the per-node factor s, see rd_node_scale).  Roofline: 8*C bytes and 2*C^2 flops per
// row -> C/4 flop/B (60 at P19): HBM-bound, so the design goal is to stream x exactly once.  The GEMM
// itself is the shared wgmma kernel (rd_tc_gemm.cu: persistent CTAs, TMA ring, register accumulators,
// fused epilogue); this file picks the tiling and the mode.  For the second layer the epilogue stores
// straight into the [T, B, D] encoder input (code/models_rd.py:338-341): no separate permute pass.
// fp32 bits are fed to the tensor core unchanged in the single-pass mode, so callers hand in
// TF32-representable operands (round_tf32 / round_out of the producing layer).
#include <cuda.h>
#include <stdlib.h>

#include "rd_obprop_tc.cuh"
#include "rd_tc_common.cuh"
#include "rd_tc_gemm.cuh"

namespace rd {
using namespace tc;

bool obprop_tc_supported(int C) {
  static int env = -1;
  if (env < 0) { const char* e = getenv("RD_OBPROP_TC"); env = (e && e[0] == '0') ? 0 : 1; }
  return env == 1 && C % 4 == 0 && C >= 16;
}

bool obprop_tc_exact(int64_t rows, int C, int mode) {
  static int env = -1;
  if (env < 0) { const char* e = getenv("RD_OBPROP_EXACT"); env = e ? (e[0] == '0' ? 1 : 2) : 0; }
  if (mode == 0) mode = env;
  if (mode == 1) return false;
  if (mode == 2) return true;
  return 2.0 * (double)rows * C * C <= 2.0e9;
}

__global__ void round_tf32_kernel(const float* __restrict__ x, long long n, float* __restrict__ y) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x[i]));
    y[i] = __uint_as_float(r);
  }
}

int round_tf32(const float* x, int64_t n, float* y, cudaStream_t st) {
  if (n <= 0) return 0;
  round_tf32_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(x, n, y);
  RD_CHECK_LAUNCH("round_tf32_kernel");
  return 0;
}

int obprop_tc_fwd(const ObpropTcArgs& a, cudaStream_t st) {
  if (a.perm && a.pdob != 4) { set_error("obprop_tc_fwd: permuted store needs d_ob == 4"); return -2; }
  if (a.perm && a.gate) { set_error("obprop_tc_fwd: gate is only built for the plain layout"); return -2; }
  if (a.rows > 0x7fffffffLL) { set_error("obprop_tc_fwd: too many rows"); return -2; }
  const bool exact = a.W_lo != nullptr;
  if (exact && a.round_out) { set_error("obprop_tc_fwd: the error-compensated mode does not round its output"); return -2; }
  TcNtArgs n;
  n.A = a.x; n.lda = a.C; n.B = a.W; n.B_lo = a.W_lo; n.M = a.rows; n.N = a.C; n.K = a.C; n.C = a.out;
  tc_nt_plan(a.rows, a.C, exact, &n.BN, &n.n_tiles);
  n.bias = a.bias; n.relu = a.relu; n.scale = a.scale; n.scale_mod = a.scale_mod;
  n.gate = a.gate; n.gate_ld = a.C; n.round_out = a.round_out;
  n.perm = a.perm; n.pB = a.pB; n.pN = a.pN; n.pD = a.pD;
  return tc_nt(n, st);
}

}  // namespace rd
