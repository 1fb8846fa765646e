// Interface of the float32-accurate tensor-core product (bjx_gemm.cu) used by the large-D dense path (bjx_dense.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bjx {

// Operand planes: a float32 row x[0..K) is stored as two binary16 rows (x1 | x2), each KP = K rounded up to 8 long,
// of 2^s x with x1 = fp16(2^s x), x2 = fp16(2^s x - x1).
__host__ __device__ __forceinline__ int plane_stride(int K) { return (K + 7) & ~7; }

// The power of two 2^s that lifts amax into [2^e, 2^(e+1)).  Zero / non-finite maxima leave the row unscaled (their
// NaN / inf propagate like the reference's).
__host__ __device__ __forceinline__ float pow2_lift_to(float amax, int e) {
  if (!(amax > 0.f) || amax > 3.0e38f) return 1.f;
  union { float f; uint32_t u; } b;
  b.f = amax;
  int s = e - ((int)((b.u >> 23) & 0xffu) - 127);
  s = s < -126 ? -126 : (s > 126 ? 126 : s);
  b.u = (uint32_t)(s + 127) << 23;
  return b.f;
}
// Exact splits (the row maximum is known): lift to [2^13, 2^14), two binades below binary16's largest finite value.
__host__ __device__ __forceinline__ float pow2_lift(float amax) { return pow2_lift_to(amax, 13); }
// Splits in the GEMM epilogue, where only the PREVIOUS production's row maximum is known: aim at [2^6, 2^7), the middle
// of the window [2^-3, 2^15.5) in which the split is exact to 2^-22 of the row maximum (below 2^-3 the second term's
// subnormal spacing 2^-24 shows; above 2^15.5 binary16 overflows).
__host__ __device__ __forceinline__ float plane_lift(float stale_max) { return pow2_lift_to(stale_max, 6); }
constexpr float kPlaneWindowLo = 0.125f;      // 2^-3
constexpr float kPlaneWindowHi = 46340.0f;    // 2^15.5

struct GemmEpilogue {
  float alpha;                 // row factor: (alpha_dev ? alpha_dev[r] * alpha : alpha) * x_unscale[r] * mat_unscale[0]
  const float* alpha_dev;      // [M] per-chain step sizes, or null
  const float* x_unscale;      // [M] 2^-s_r of the activation planes
  const float* mat_unscale;    // [1] 2^-s_A of the constant matrix
  float beta;                  // lincomb: y = alpha_r acc + beta Cin
  int has_cin;
  int double_kick;             // y = alpha_r acc + (alpha_r acc + Cin)
  int planes;                  // also emit the operand planes of y
  float* out_unscale;          // [M] 2^-s of the emitted planes
  const float* stale_max;      // [M] row maxima of the previous production of this variable (chooses the lift)
  float* next_max;             // [M] this production's row maxima (atomic max; zero on entry)
  float* zero_max;             // [M] cleared for the production after this one
};

struct GemmCall {
  const uint16_t* x_planes;    // [M, 2, KP]
  const uint16_t* a_planes;    // [N, 2, KP]
  float* Y;                    // [M, N]
  const float* Cin;            // [M, N] (may alias Y)
  uint16_t* planes_out;        // [M, 2, KP_out]
  int M, N, K, KP, KP_out;
  GemmEpilogue epi;
};

// returns 0 on success, a small positive code naming the failing stage otherwise
int gemm_f16x3(const GemmCall& g, cudaStream_t stream);

}  // namespace bjx
