// Tensor-core GEMMs (rd_tc_gemm.cu): the shared wgmma NT kernel, the encoder's error-compensated GEMM and the grouped
// weight gradients.
#pragma once
#include "rd_common.cuh"

namespace rd {

// C[M, N] = epi(A[M, K] . B[N, K]^T) on the wgmma tensor cores; B_lo != null selects the error-compensated mode
// (3xTF32: A is split in registers, B_lo = B - trunc19(B) is precomputed), else single-pass TF32 on operands the caller
// keeps TF32-representable.  epi = +bias[col] -> relu -> *scale[row % scale_mod] -> *(gate > 0 ? gate_scale : 0) ->
// dropout (+ keep bits) -> +resid -> RN to TF32 (round_out); perm != 0 stores row b*pN + n, col t*4 + k into
// C[(t*pB + b)*pD + n*4 + k].  BN and n_tiles (BN * n_tiles >= N) are the caller's tiling of N, normally from
// tc_nt_plan; BN must be one of the widths the kernel is instantiated for in the chosen mode.
struct TcNtArgs {
  const float* A = nullptr; long long lda = 0;
  const float* B = nullptr; const float* B_lo = nullptr;
  long long M = 0; int N = 0, K = 0, BN = 0, n_tiles = 0;
  float* C = nullptr;
  const float* bias = nullptr; int relu = 0;
  const float* scale = nullptr; int scale_mod = 1;
  const float* gate = nullptr; long long gate_ld = 0; float gate_scale = 1.f;
  float drop_p = 0.f; const uint64_t* rng = nullptr; uint32_t drop_site = 0; DropRep rep;
  uint32_t* drop_mask = nullptr; int drop_mask_ld = 0;
  const float* resid = nullptr; long long resid_ld = 0;
  int round_out = 0;
  int perm = 0, pB = 0, pN = 0, pD = 0;
};
int tc_nt(const TcNtArgs& a, cudaStream_t st);
// Tiling of N for an M x N tc_nt problem (exact: error-compensated mode): the instantiated width and n-tile count that
// minimise the busiest SM's work over the device's SMs.  Deterministic for a given (M, N, mode, SM count);
// the environment variable RD_TC_NT_BN=<width> forces a width (debugging, and tests that compare plans).
void tc_nt_plan(long long M, int N, bool exact, int* BN, int* n_tiles);

// C[M,N] = epi( A[M,K] . B[N,K]^T ) with fp32-level accuracy on the TF32 tensor cores ("3xTF32"):
//   A = A_hi + A_lo, B = B_hi + B_lo (hi = top 19 bits, what the MMA reads; lo = exact remainder)
//   A.B^T ~= A_hi.B_hi^T + A_lo.B_hi^T + A_hi.B_lo^T          (dropped term ~2^-22 relative)
// A (activations) is split on the fly in registers; B (a weight) comes with its precomputed
// remainder B_lo (split_weights below).  epi = +bias[j] -> relu -> *gate -> dropout -> +resid.
struct TcGemmArgs {
  const float* A = nullptr; long long lda = 0;
  const float* B = nullptr; const float* B_lo = nullptr;   // [N, K] row-major, ld = K
  long long M = 0; int N = 0, K = 0;
  float* C = nullptr;                                        // [M, N] row-major, ld = N
  const float* bias = nullptr; int relu = 0;
  const float* gate = nullptr; long long gate_ld = 0; float gate_scale = 1.f;
  float drop_p = 0.f; const uint64_t* rng = nullptr; uint32_t drop_site = 0;
  DropRep rep;                                               // replicate rows: dropout drawn through rep_remap
  uint32_t* drop_mask = nullptr; int drop_mask_ld = 0;      // optional: keep bits of the dropout decisions, word [row*ld + col/32]
  const float* resid = nullptr; long long resid_ld = 0;
};
bool tc_gemm_supported(const TcGemmArgs& a);
void tc_gemm_set_debug(unsigned long long* buf);     // %globaltimer phase stamps [CTA][8] (debug)
int tc_gemm(const TcGemmArgs& a, cudaStream_t st);

// Weight gradient on the tensor cores: dW[Nout, Kin] = sum_r dY[r, Nout]^T X[r, Kin], db[Nout] = sum_r dY[r, :]
// (the bias gradient rides along as one extra "ones" column of X).  The row range is split across CTAs; partial tiles
// go to `partial` (tc_wgrad_partial_floats(...) floats) and are summed in a fixed order (deterministic).
bool tc_wgrad_supported(int Nout, int Kin, long long ldy, long long ldx, const void* dY, const void* X);
long long tc_wgrad_partial_floats(int Nout, int Kin, long long rows);
int tc_wgrad(const float* dY, long long ldy, const float* X, long long ldx, long long rows, int Nout, int Kin,
             float* dW, float* db, float* partial, cudaStream_t st);
// Grouped form: ONE tensor-core launch + ONE reduction launch for up to WG_MAX independent problems
// (each with its own `partial` buffer of tc_wgrad_partial_floats(...) floats, 16-byte aligned).
constexpr int WG_MAX = 12;
struct WgradItem { const float* dY; long long ldy; const float* X; long long ldx; long long rows; int Nout, Kin;
                   float* dW; float* db; float* partial; };
// Column sums riding along in the group's reduction launch: out[c] = sum_{s < nsplit} partial[s*stride + c], c < ncols
constexpr int CS_MAX = 36;
struct ColsumItem { const float* partial; long long stride; int nsplit, ncols; float* out; };
// The plan of one group: the tile width (0 when n = 0: no tensor-core launch), the rows target of its row splits and,
// per problem in the caller's order, the split count and the rows per split (a multiple of 32; the last split may be
// shorter).  Nld = N + 1 rounded up to 4 is the row stride of a problem's partial slabs.
struct WSplit { int nsplit, rows_per_split, Nld; };
struct WgradPlan { int BN, rows_target; WSplit sp[WG_MAX]; };
// plan (optional): the plan the call ran, written back
int tc_wgrad_group(const WgradItem* items, int n, const ColsumItem* cs, int ncs, cudaStream_t st,
                   WgradPlan* plan = nullptr);
void tc_wgrad_set_debug(unsigned long long* buf);    // per-CTA phase cycles [CTA][16] of tc_wgrad_kernel (debug)

// One launch for all weights of a step: lo = W - trunc19(W); t = W^T; t_lo = W^T - trunc19(W^T).
// optional extras for the single-pass-TF32 layers: rn = RN_tf32(W), rn_t = RN_tf32(W)^T
struct WeightSplit { const float* w; int rows, cols; float* lo; float* t; float* t_lo; float* rn = nullptr; float* rn_t = nullptr; };
// Optional step prologue done by thread 0 of the same launch: capture {seed, counter + step_offset} of the dropout stream
// into rng_captured (advance != 0: counter += 1 afterwards) and zero one ticket word.
struct StepPrologue { uint64_t* rng_state = nullptr; uint64_t* rng_captured = nullptr; int advance = 0; unsigned* zero_counter = nullptr;
                      uint64_t step_offset = 0; };
int split_weights(const WeightSplit* items, int n, cudaStream_t st, const StepPrologue* pro = nullptr);   // n <= 16

}  // namespace rd
