// Large-D dense path (D > 128): HMC with a dense inverse mass matrix and/or a dense Gaussian target
// (BASELINE config 2: 1024-D correlated Gaussian, dense mass matrix).  The two linear maps of every
// leapfrog -- v = M^-1 p (blackjax/mcmc/integrators.py:242 -> metrics.py:263-270 -> util.py:57-61) and
// grad = -P q (the target's autodiff) -- are [C,D] x [D,D] GEMMs on the tensor cores (bjx_gemm.cu); the
// elementwise glue (half kicks, energies, accept/select) are the streaming row kernels below.
#include <vector>

#include "bjx_handle.h"
#include "bjx_internal.h"
#include <cuda_fp16.h>

#include "bjx_gemm.h"
#include "bjx_prng.cuh"

using namespace bjx;

namespace bjx {

constexpr int kRowWarps = 8;

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float max4(float m, float4 v) {
  return fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
}

// ---- float32 -> 2 x binary16 operand split (see bjx_gemm.cu / bjx_gemm.h) -----------------------------------
__device__ __forceinline__ void split2(float x, uint16_t& h1, uint16_t& h2) {
  const __half a = __float2half_rn(x);
  const __half b = __float2half_rn(x - __half2float(a));
  h1 = __half_as_ushort(a);
  h2 = __half_as_ushort(b);
}
__device__ __forceinline__ uint2 pack4(const uint16_t (&v)[4]) {
  return make_uint2((uint32_t)v[0] | ((uint32_t)v[1] << 16), (uint32_t)v[2] | ((uint32_t)v[3] << 16));
}
// the (x1 | x2) planes of four consecutive elements of a row (plane stride KP), lifted by sc
__device__ __forceinline__ void store_planes(uint16_t* row, int KP, int k, float4 v, float sc) {
  uint16_t p1[4], p2[4];
  split2(v.x * sc, p1[0], p2[0]);
  split2(v.y * sc, p1[1], p2[1]);
  split2(v.z * sc, p1[2], p2[2]);
  split2(v.w * sc, p1[3], p2[3]);
  *reinterpret_cast<uint2*>(row + k) = pack4(p1);
  *reinterpret_cast<uint2*>(row + (size_t)KP + k) = pack4(p2);
}

// Activation rows, one warp per row: X [R, K] float32 -> planes [R, 2, KP] binary16 of 2^s_r x with the exact lift
// (row maximum into [2^13, 2^14)), unscale[r] = 2^-s_r; optionally the row maximum itself (for the fused epilogue's
// next lift) and a cleared accumulator for the production after that.
__global__ void k_rows_split2(int R, int K, const float* __restrict__ x, uint16_t* __restrict__ xs, float* __restrict__ unscale,
                              float* __restrict__ rowmax, float* __restrict__ rowmax_zero) {
  const int lane = threadIdx.x & 31, r = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (r >= R) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)r * K);
  float amax = 0.f;
  for (int i = lane; i < K / 4; i += 32) amax = max4(amax, xr[i]);
  amax = wmax(amax);
  const float sc = pow2_lift(amax);
  const int KP = plane_stride(K);
  uint16_t* row = xs + (size_t)r * 2 * KP;
  for (int i = lane; i < K / 4; i += 32) store_planes(row, KP, 4 * i, xr[i], sc);  // second read: L1/L2
  if (lane == 0) {
    unscale[r] = 1.0f / sc;
    if (rowmax) rowmax[r] = amax;
    if (rowmax_zero) rowmax_zero[r] = 0.f;
  }
}

// Rows whose fused-epilogue planes were written with a lift that left the exact window (bjx_gemm.h) are re-split
// here from the float32 row with the exact lift.  One thread checks one row (two floats); flagged rows -- none in a
// stable trajectory -- are redone by the whole warp.
__global__ void k_planes_fixup(int R, int K, const float* __restrict__ y, uint16_t* __restrict__ ys,
                               const float* __restrict__ stale_max, const float* __restrict__ new_max,
                               float* __restrict__ unscale) {
  const int lane = threadIdx.x & 31;
  const int r0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32;
  const int r = r0 + lane;
  asm volatile("griddepcontrol.wait;" ::: "memory");  // launched programmatically dependent on the product before it
  bool bad = false;
  if (r < R) {
    const float mx = new_max[r];
    const float t = mx * plane_lift(stale_max[r]);
    bad = (mx > 0.f) && (mx <= 3.0e38f) && !(t >= kPlaneWindowLo && t < kPlaneWindowHi);
  }
  unsigned todo = __ballot_sync(0xffffffffu, bad);
  const int KP = plane_stride(K);
  while (todo) {
    const int rr = r0 + (__ffs(todo) - 1);
    todo &= todo - 1;
    const float sc = pow2_lift(new_max[rr]);
    const float4* xr = reinterpret_cast<const float4*>(y + (size_t)rr * K);
    uint16_t* row = ys + (size_t)rr * 2 * KP;
    for (int i = lane; i < K / 4; i += 32) store_planes(row, KP, 4 * i, xr[i], sc);
    if (lane == 0) unscale[rr] = 1.0f / sc;
  }
}

// max |x| of a constant matrix into *out (float bits; non-negative floats order like ints); *out zeroed beforehand
__global__ void k_absmax(long long n4, const float* __restrict__ x, float* out) {
  float m = 0.f;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n4; t += (long long)gridDim.x * blockDim.x)
    m = max4(m, reinterpret_cast<const float4*>(x)[t]);
  m = wmax(m);
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));
}
// Constant matrices: A [R, K] float32 -> planes [R, 2, KP] binary16 (a1 | a2) of 2^s_A a; *unscale = 2^-s_A
__global__ void k_matrix_split2(long long R, int K, const float* __restrict__ x, uint16_t* __restrict__ xs,
                                const float* __restrict__ amax, float* __restrict__ unscale) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const float sc = pow2_lift(amax[0]);
  if (t == 0) unscale[0] = 1.0f / sc;
  if (t >= R * K / 4) return;
  const long long e = t * 4;
  const long long r = e / K;
  const int k = (int)(e % K);
  const int KP = plane_stride(K);
  store_planes(xs + r * 2 * KP, KP, k, reinterpret_cast<const float4*>(x)[t], sc);
}

// Opening pass of a trajectory on the fused path, one warp per row: the first half kick p += (eps_c/2) g
// (integrators.py:235-239), the exact planes of the new p for the first q-update product, and the row maxima of p
// and q that seed the fused epilogues' lifts (slot 0 = maximum, slot 1 = cleared accumulator).
__global__ void k_rows_open(int C, int D, float* __restrict__ p, const float* __restrict__ g, const float* __restrict__ q,
                            float eps, const float* __restrict__ eps_dev, uint16_t* __restrict__ p_planes,
                            float* __restrict__ p_unscale, float* __restrict__ pmax0, float* __restrict__ pmax1,
                            float* __restrict__ qmax0, float* __restrict__ qmax1) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (c >= C) return;
  const size_t ro = (size_t)c * D;
  const float eh = (eps_dev ? eps_dev[c] : eps) * 0.5f;
  float pm = 0.f, qm = 0.f;
  for (int i = lane; i < D / 4; i += 32) {
    float4 pv = __ldcs(reinterpret_cast<const float4*>(p + ro) + i);
    const float4 gv = __ldcs(reinterpret_cast<const float4*>(g + ro) + i);
    pv.x = fmaf(eh, gv.x, pv.x); pv.y = fmaf(eh, gv.y, pv.y); pv.z = fmaf(eh, gv.z, pv.z); pv.w = fmaf(eh, gv.w, pv.w);
    reinterpret_cast<float4*>(p + ro)[i] = pv;  // re-read below: keep it cached
    pm = max4(pm, pv);
    if (q) qm = max4(qm, __ldcs(reinterpret_cast<const float4*>(q + ro) + i));
  }
  pm = wmax(pm);
  qm = wmax(qm);
  const float sc = pow2_lift(pm);
  const int KP = plane_stride(D);
  uint16_t* row = p_planes + (size_t)c * 2 * KP;
  for (int i = lane; i < D / 4; i += 32) store_planes(row, KP, 4 * i, reinterpret_cast<const float4*>(p + ro)[i], sc);
  if (lane == 0) {
    p_unscale[c] = 1.0f / sc;
    pmax0[c] = pm;
    pmax1[c] = 0.f;
    if (q) { qmax0[c] = qm; qmax1[c] = 0.f; }
  }
}

// z[c, i] = normal(key_c, (D,))[i] with key_c = split(rng_key_c, n)[sub] when sub >= 0 (hmc.py:299,302 -> util.py:89-91:
// sub = 0; elliptical_slice.py:205: sub = 1), the chain's key itself when sub < 0
__global__ void k_dense_normal(int C, int D, const uint32_t* __restrict__ keys, float* __restrict__ z, int sub,
                               int key_shared, uint32_t chain_offset) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n4 = (long long)C * D / 4;
  if (t >= n4) return;
  const long long e = t * 4;
  const int c = (int)(e / D);
  const uint32_t i = (uint32_t)(e % D);
  Key km = key_shared ? fold_in(Key{keys[0], keys[1]}, chain_offset + (uint32_t)c) : Key{keys[2 * c], keys[2 * c + 1]};
  if (sub >= 0) km = fold_in(km, (uint32_t)sub);
  float4 o;
  o.x = normal_at(km, i);
  o.y = normal_at(km, i + 1);
  o.z = normal_at(km, i + 2);
  o.w = normal_at(km, i + 3);
  reinterpret_cast<float4*>(z)[t] = o;
}

// y[c,:] = a[:] * x[c,:]  (diagonal metric with a dense target)
__global__ void k_rows_scale(int C, int D, const float* __restrict__ a, long long a_stride, const float* __restrict__ x,
                             float* __restrict__ y) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n4 = (long long)C * D / 4;
  if (t >= n4) return;
  const long long e = t * 4;
  const int c = (int)(e / D);
  const int i = (int)(e % D);
  const float4 av = *reinterpret_cast<const float4*>(a + (size_t)c * a_stride + i);
  const float4 xv = __ldcs(reinterpret_cast<const float4*>(x) + t);
  __stcs(reinterpret_cast<float4*>(y) + t, make_float4(av.x * xv.x, av.y * xv.y, av.z * xv.z, av.w * xv.w));
}

// x[c,:] += (eps_c * coef) * y[c,:]     (integrators.py:199-203,235-239)
__global__ void k_rows_axpy(int C, int D, float* __restrict__ x, const float* __restrict__ y, float eps,
                            const float* __restrict__ eps_dev, float coef) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n4 = (long long)C * D / 4;
  if (t >= n4) return;
  const int c = (int)(t * 4 / D);
  const float a = (eps_dev ? eps_dev[c] : eps) * coef;
  float4 xv = __ldcs(reinterpret_cast<const float4*>(x) + t);
  const float4 yv = __ldcs(reinterpret_cast<const float4*>(y) + t);
  xv.x = fmaf(a, yv.x, xv.x); xv.y = fmaf(a, yv.y, xv.y); xv.z = fmaf(a, yv.z, xv.z); xv.w = fmaf(a, yv.w, xv.w);
  __stcs(reinterpret_cast<float4*>(x) + t, xv);
}

// e[c] = -logp[c] + 0.5 * sum_i v[c,i] p[c,i]      (trajectory.py:745-748, metrics.py:263-270)
__global__ void k_rows_energy(int C, int D, const float* __restrict__ v, const float* __restrict__ p,
                              const float* __restrict__ logp, float* __restrict__ e, float p_sign) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (c >= C) return;
  const float4* vr = reinterpret_cast<const float4*>(v + (size_t)c * D);
  const float4* pr = reinterpret_cast<const float4*>(p + (size_t)c * D);
  float acc = 0.f;
  for (int i = lane; i < D / 4; i += 32) {
    const float4 a = __ldcs(vr + i), b = __ldcs(pr + i);
    acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
  }
  acc = wsum(acc);
  if (lane == 0) e[c] = -logp[c] + 0.5f * acc * p_sign;
}

// Gradient + second half kick for one leapfrog, streaming the row:
//   TARGET 2 (dense Gaussian): g = -P q was written by the GEMM epilogue (alpha = -1); logp = 1/2 q.g + offset
//   TARGET 0 (diag Gaussian) : g = -(q - mean) / s^2;      logp = -1/2 sum (q-mean)^2/s^2 + offset
//   then (if p != null) p += (eps_c * 0.5) * g                                  (integrators.py:134-141)
//   and, when another leapfrog follows (kicks == 2), that step's first half kick p += (eps_c * 0.5) * g
//   (integrators.py:235-239) -- same gradient, two separately rounded FMAs, one pass over the row.
template <int TARGET>
__global__ void k_rows_grad_kick(int C, int D, const float* __restrict__ q, const float* __restrict__ aux,
                                 const float* __restrict__ inv_var, const float* __restrict__ mean, float offset,
                                 float* __restrict__ p, float eps, const float* __restrict__ eps_dev,
                                 float* __restrict__ g_out, float* __restrict__ logp_out, int kicks,
                                 uint16_t* __restrict__ p_split /* [C,2,KP] binary16 planes of the new p, or null */,
                                 float* __restrict__ p_unscale) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (c >= C) return;
  const size_t ro = (size_t)c * D;
  const float eps_c = eps_dev ? eps_dev[c] : eps;
  const float eh = eps_c * 0.5f;
  float acc = 0.f, amax = 0.f;
  for (int i = lane; i < D / 4; i += 32) {
    const float4 qv = __ldcs(reinterpret_cast<const float4*>(q + ro) + i);
    float4 gv;
    if (TARGET == 2) {
      gv = __ldcs(reinterpret_cast<const float4*>(aux + ro) + i);  // aux == g_out: already the gradient
      acc = fmaf(qv.x, gv.x, acc); acc = fmaf(qv.y, gv.y, acc); acc = fmaf(qv.z, gv.z, acc); acc = fmaf(qv.w, gv.w, acc);
    } else {
      const float4 w = __ldg(reinterpret_cast<const float4*>(inv_var) + i);
      float4 d = qv;
      if (mean) {
        const float4 m = __ldg(reinterpret_cast<const float4*>(mean) + i);
        d = make_float4(qv.x - m.x, qv.y - m.y, qv.z - m.z, qv.w - m.w);
      }
      gv = make_float4(d.x * -w.x, d.y * -w.y, d.z * -w.z, d.w * -w.w);
      acc = fmaf(d.x, gv.x, acc); acc = fmaf(d.y, gv.y, acc); acc = fmaf(d.z, gv.z, acc); acc = fmaf(d.w, gv.w, acc);
    }
    if (TARGET != 2) __stcs(reinterpret_cast<float4*>(g_out + ro) + i, gv);
    if (p) {
      float4 pv = __ldcs(reinterpret_cast<const float4*>(p + ro) + i);
      pv.x = fmaf(eh, gv.x, pv.x); pv.y = fmaf(eh, gv.y, pv.y); pv.z = fmaf(eh, gv.z, pv.z); pv.w = fmaf(eh, gv.w, pv.w);
      if (kicks == 2) {
        pv.x = fmaf(eh, gv.x, pv.x); pv.y = fmaf(eh, gv.y, pv.y); pv.z = fmaf(eh, gv.z, pv.z); pv.w = fmaf(eh, gv.w, pv.w);
      }
      if (p_split) {
        reinterpret_cast<float4*>(p + ro)[i] = pv;  // re-read below: keep it cached
        amax = max4(amax, pv);
      } else {
        __stcs(reinterpret_cast<float4*>(p + ro) + i, pv);
      }
    }
  }
  if (p_split) {
    // the operand planes of the next M^-1 p product, written while the row is hot: each lane re-reads exactly the
    // elements it stored above
    const float sc = pow2_lift(wmax(amax));
    const int KP = plane_stride(D);
    uint16_t* row = p_split + (size_t)c * 2 * KP;
    for (int i = lane; i < D / 4; i += 32) store_planes(row, KP, 4 * i, reinterpret_cast<const float4*>(p + ro)[i], sc);
    if (lane == 0) p_unscale[c] = 1.0f / sc;
  }
  acc = wsum(acc);
  if (lane == 0) logp_out[c] = 0.5f * acc + offset;
}

// Metropolis accept + select (hmc.py:158-163, proposal.py:214-235) for the dense path
__global__ void k_rows_accept(int C, int D, const uint32_t* __restrict__ keys, const float* __restrict__ e0,
                              const float* __restrict__ e1, float div_thr, const float* __restrict__ qw,
                              const float* __restrict__ gw, const float* __restrict__ lw, const float* q_in,
                              const float* g_in, const float* l_in, float* q_out, float* g_out, float* l_out, int L,
                              InfoPtrs info, int key_shared, uint32_t chain_offset) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (c >= C) return;
  const Key rk = key_shared ? fold_in(Key{keys[0], keys[1]}, chain_offset + (uint32_t)c) : Key{keys[2 * c], keys[2 * c + 1]};
  const Key ki = fold_in(rk, 1u);
  float delta = e0[c] - e1[c];
  if (isnan(delta)) delta = -__int_as_float(0x7f800000);
  const bool is_div = (-delta) > div_thr;
  float pa = expf(delta);
  pa = pa > 1.0f ? 1.0f : pa;
  const bool acc = uniform01(ki) < pa;
  const size_t ro = (size_t)c * D;
  if (acc || q_out != q_in) {
    const float4* sq = reinterpret_cast<const float4*>((acc ? qw : q_in) + ro);
    const float4* sg = reinterpret_cast<const float4*>((acc ? gw : g_in) + ro);
    for (int i = lane; i < D / 4; i += 32) {
      __stcs(reinterpret_cast<float4*>(q_out + ro) + i, __ldcs(sq + i));
      __stcs(reinterpret_cast<float4*>(g_out + ro) + i, __ldcs(sg + i));
    }
    if (lane == 0) l_out[c] = acc ? lw[c] : l_in[c];
  }
  if (lane == 0) {
    if (info.acceptance_rate) info.acceptance_rate[c] = pa;
    if (info.is_accepted) info.is_accepted[c] = acc;
    if (info.is_divergent) info.is_divergent[c] = is_div;
    if (info.energy) info.energy[c] = e1[c];
    if (info.num_integration_steps) info.num_integration_steps[c] = L;
  }
}
}  // namespace bjx

static inline dim3 g4(long long n4) { return dim3((unsigned)((n4 + 255) / 256)); }
static inline dim3 grow(int C) { return dim3((C + kRowWarps - 1) / kRowWarps); }

struct DenseWs {
  float *p, *v, *q, *g, *lw, *e0, *e1;
  uint16_t* xs[2];     // [C, 2, KP] binary16 operand planes of the momentum (PL_P) and position (PL_Q) rows
  float* unscale[2];   // [C] 2^-s_r of those planes
  float* rmax[2];      // [3, C] row maxima of p / q: previous production, current accumulator, next (cleared)
  float* mat_max;      // [4] max |a| of the constant matrices
  float* mat_unscale;  // [4] 2^-s_A
};
enum { MAT_IMM = 0, MAT_MSQRT = 1, MAT_PREC = 2, MAT_PRIOR = 3 };
enum { PL_P = 0, PL_Q = 1 };

// Every helper below works on the first n rows of its [C, D] / [C] arrays, all on the handle's stream: n = C, except for
// NUTS (bjx_dense_nuts.cuh), whose leaves run on the chains still expanding, compacted into the first n rows.

static int dense_ws(bjx_handle_t h, DenseWs& w) {
  const size_t C = h->cfg.n_chains, D = h->cfg.dim;
  const size_t row = ((C * D * sizeof(float)) + 255) & ~(size_t)255, vec = ((C * sizeof(float)) + 255) & ~(size_t)255;
  const size_t KP = plane_stride((int)D);
  const size_t xsb = ((C * 2 * KP * sizeof(uint16_t)) + 255) & ~(size_t)255;
  const size_t mat = ((D * 2 * KP * sizeof(uint16_t)) + 255) & ~(size_t)255;
  const size_t need = 4 * row + 11 * vec + 2 * xsb + 4 * mat + 256;
  int rc = bjx_grow(h, h->dense_block, h->dense_bytes, need, 1);
  if (rc) return rc;
  char* b = (char*)h->dense_block;
  w.p = (float*)b; w.v = (float*)(b + row); w.q = (float*)(b + 2 * row); w.g = (float*)(b + 3 * row);
  char* vb = b + 4 * row;
  w.lw = (float*)vb; w.e0 = (float*)(vb + vec); w.e1 = (float*)(vb + 2 * vec);
  w.unscale[PL_P] = (float*)(vb + 3 * vec); w.unscale[PL_Q] = (float*)(vb + 4 * vec);
  w.rmax[PL_P] = (float*)(vb + 5 * vec); w.rmax[PL_Q] = (float*)(vb + 8 * vec);  // 3 x vec each
  char* xb = vb + 11 * vec;
  w.xs[PL_P] = (uint16_t*)xb; w.xs[PL_Q] = (uint16_t*)(xb + xsb);
  for (int m = 0; m < 4; ++m) h->dense_mat_s[m] = (uint16_t*)(xb + 2 * xsb + m * mat);
  w.mat_max = (float*)(xb + 2 * xsb + 4 * mat);
  w.mat_unscale = w.mat_max + 4;
  if (h->dense_bytes_built != need) {  // fresh block: zero the plane pads, every split matrix must be rebuilt
    BJX_CUDA(cudaMemsetAsync(vb, 0, 11 * vec + 2 * xsb + 4 * mat, h->stream));
    for (int m = 0; m < 4; ++m) h->dense_mat_src[m] = nullptr;
    h->dense_bytes_built = need;
  }
  // (re)build the split copies of the constant matrices whose source changed (set_metric / set_target /
  // set_elliptical_prior)
  const float* src[4] = {h->metric_kind == BJX_METRIC_DENSE ? h->imm : nullptr,
                         h->metric_kind == BJX_METRIC_DENSE ? h->msqrt : nullptr,
                         h->cfg.target.kind == BJX_TARGET_DENSE_GAUSSIAN ? h->cfg.target.precision : nullptr,
                         h->ess_kind == BJX_METRIC_DENSE ? h->ess_prior + h->cfg.dim : nullptr};
  for (int m = 0; m < 4; ++m) {
    if (src[m] && (h->dense_mat_src[m] != src[m] || h->dense_mat_ver[m] != h->dense_version)) {
      BJX_CUDA(cudaMemsetAsync(w.mat_max + m, 0, sizeof(float), h->stream));
      k_absmax<<<sm_count(), 256, 0, h->stream>>>((long long)D * D / 4, src[m], w.mat_max + m);
      BJX_CHECK_LAUNCH("k_absmax");
      k_matrix_split2<<<g4((long long)D * D / 4), 256, 0, h->stream>>>((long long)D, (int)D, src[m], h->dense_mat_s[m],
                                                                      w.mat_max + m, w.mat_unscale + m);
      BJX_CHECK_LAUNCH("k_matrix_split2");
      h->dense_mat_src[m] = src[m];
      h->dense_mat_ver[m] = h->dense_version;
    }
  }
  return 0;
}

// What the product's epilogue emits besides Y: nothing, or the operand planes of Y as variable `var` (PL_P / PL_Q)
// whose row-maximum ring stands at `phase` (previous production in slot phase % 3).
struct PlanesOut {
  int var;    // -1: none
  int phase;
};

// Y[c,:] = alpha_c * (X . A^T)[c,:] + beta * Cin[c,:] for the first n rows, alpha_c = alpha * alpha_dev[c] (or alpha), A one
// of the handle's constant matrices (float32-accurate, bjx_gemm.cu).  X (when not null) is split exactly into the planes of
// variable `xvar` first; X == null: the planes of `xvar` are current.
// double_kick: Y = alpha_c acc + (alpha_c acc + Cin) instead (the two half kicks between consecutive leapfrog steps).
static int gemm(bjx_handle_t h, DenseWs& w, int n, const float* X, int xvar, int mat, float* Y, const float* Cin,
                float alpha, const float* alpha_dev, float beta, bool double_kick = false, PlanesOut po = PlanesOut{-1, 0}) {
  const int D = h->cfg.dim, C = h->cfg.n_chains;
  const int KP = plane_stride(D);
  if (X) {
    k_rows_split2<<<grow(n), kRowWarps * 32, 0, h->stream>>>(n, D, X, w.xs[xvar], w.unscale[xvar], nullptr, nullptr);
    BJX_CHECK_LAUNCH("k_rows_split2");
  }
  GemmCall g;
  g.x_planes = w.xs[xvar];
  g.a_planes = h->dense_mat_s[mat];
  g.Y = Y;
  g.Cin = Cin;
  g.planes_out = nullptr;
  g.M = n; g.N = D; g.K = D; g.KP = KP; g.KP_out = KP;
  g.epi.alpha = alpha;
  g.epi.alpha_dev = alpha_dev;
  g.epi.x_unscale = w.unscale[xvar];
  g.epi.mat_unscale = w.mat_unscale + mat;
  g.epi.beta = beta;
  g.epi.has_cin = Cin ? 1 : 0;
  g.epi.double_kick = double_kick ? 1 : 0;
  g.epi.planes = 0;
  g.epi.out_unscale = nullptr; g.epi.stale_max = nullptr; g.epi.next_max = nullptr; g.epi.zero_max = nullptr;
  if (po.var >= 0) {
    float* ring = w.rmax[po.var];
    g.planes_out = w.xs[po.var];
    g.epi.planes = 1;
    g.epi.out_unscale = w.unscale[po.var];
    g.epi.stale_max = ring + (size_t)(po.phase % 3) * C;
    g.epi.next_max = ring + (size_t)((po.phase + 1) % 3) * C;
    g.epi.zero_max = ring + (size_t)((po.phase + 2) % 3) * C;
  }
  const int rc = gemm_f16x3(g, h->stream);
  if (rc) return bjx_fail(h, BJX_E_UNSUPPORTED, "tensor-core product failed (stage " + std::to_string(rc) + ")");
  if (po.var >= 0) {  // rows whose lift left the exact window are re-split from Y (none in a stable trajectory)
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((n + 255) / 256);
    cfg.blockDim = dim3(256);
    cfg.stream = h->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    BJX_CUDA(cudaLaunchKernelEx(&cfg, k_planes_fixup, n, D, (const float*)Y, g.planes_out, g.epi.stale_max,
                                (const float*)g.epi.next_max, g.epi.out_unscale));
  }
  return 0;
}

// v = M^-1 p   (p_presplit: the planes of p are current)
static int dense_velocity(bjx_handle_t h, DenseWs& w, int n, const float* p, float* v, bool p_presplit = false) {
  const int D = h->cfg.dim;
  if (h->metric_kind == BJX_METRIC_DENSE) return gemm(h, w, n, p_presplit ? nullptr : p, PL_P, MAT_IMM, v, nullptr, 1.f, nullptr, 0.f);
  const bool per_chain = (h->metric_kind == BJX_METRIC_DIAG_PER_CHAIN);
  k_rows_scale<<<g4((long long)n * D / 4), 256, 0, h->stream>>>(n, D, h->imm, per_chain ? D : 0, p, v);
  BJX_CHECK_LAUNCH("k_rows_scale");
  return 0;
}

// g, logp = value_and_grad(q); optionally p += eh * g (once or twice).  q_presplit: the planes of q are current.
// split_p: also leave the exact planes of the kicked p (for the next M^-1 p product).
static int dense_grad(bjx_handle_t h, DenseWs& w, int n, const float* q, float* p, float eps, const float* eps_dev,
                      float* g, float* logp, int kicks = 1, bool split_p = false, bool q_presplit = false) {
  const int D = h->cfg.dim;
  const bjx_target_desc& t = h->cfg.target;
  uint16_t* ps = (split_p && p) ? w.xs[PL_P] : nullptr;
  if (t.kind == BJX_TARGET_DENSE_GAUSSIAN) {
    // g = -(q P): the sign rides on the product's epilogue
    int rc = gemm(h, w, n, q_presplit ? nullptr : q, PL_Q, MAT_PREC, g, nullptr, -1.f, nullptr, 0.f);
    if (rc) return rc;
    k_rows_grad_kick<2><<<grow(n), kRowWarps * 32, 0, h->stream>>>(n, D, q, g, nullptr, nullptr, t.logp_offset, p, eps, eps_dev,
                                                                 g, logp, kicks, ps, w.unscale[PL_P]);
  } else if (t.kind == BJX_TARGET_DIAG_GAUSSIAN) {
    k_rows_grad_kick<0><<<grow(n), kRowWarps * 32, 0, h->stream>>>(n, D, q, nullptr, t.inv_var, t.mean, t.logp_offset, p, eps,
                                                                 eps_dev, g, logp, kicks, ps, w.unscale[PL_P]);
  } else {
    return bjx_fail(h, BJX_E_UNSUPPORTED, "large-D dense path supports DENSE_GAUSSIAN and DIAG_GAUSSIAN targets");
  }
  BJX_CHECK_LAUNCH("k_rows_grad_kick");
  return 0;
}

static int dense_momentum(bjx_handle_t h, DenseWs& w, int n, const uint32_t* keys, float* p_out, bool split_first) {
  const int D = h->cfg.dim;
  const bool dense_m = (h->metric_kind == BJX_METRIC_DENSE);
  float* z = dense_m ? w.v : p_out;
  k_dense_normal<<<g4((long long)n * D / 4), 256, 0, h->stream>>>(n, D, keys, z, split_first ? 0 : -1, h->key_shared,
                                                                   h->chain_offset);
  BJX_CHECK_LAUNCH("k_dense_normal");
  if (dense_m) return gemm(h, w, n, z, PL_P, MAT_MSQRT, p_out, nullptr, 1.f, nullptr, 0.f);  // p = L^-T z
  const bool per_chain = (h->metric_kind == BJX_METRIC_DIAG_PER_CHAIN);
  k_rows_scale<<<g4((long long)n * D / 4), 256, 0, h->stream>>>(n, D, h->msqrt, per_chain ? D : 0, z, p_out);
  BJX_CHECK_LAUNCH("k_rows_scale");
  return 0;
}

static int dense_energy(bjx_handle_t h, DenseWs& w, int n, const float* p, const float* logp, float* e_out,
                        bool p_presplit = false) {
  const int D = h->cfg.dim;
  int rc = dense_velocity(h, w, n, p, w.v, p_presplit);
  if (rc) return rc;
  k_rows_energy<<<grow(n), kRowWarps * 32, 0, h->stream>>>(n, D, w.v, p, logp, e_out, 1.f);
  BJX_CHECK_LAUNCH("k_rows_energy");
  return 0;
}

// n_steps velocity-Verlet steps in place on all chains (integrators.py:104-150).  p_planes_after: leave the exact planes
// of the final p (the caller's next product is M^-1 p for the kinetic energy).
static int dense_leapfrog_core(bjx_handle_t h, DenseWs& w, float* q, float* p, float* logp, float* g, float eps,
                               const float* eps_dev, int n_steps, bool p_planes_after = false) {
  const int D = h->cfg.dim, C = h->cfg.n_chains;
  const long long n4 = (long long)C * D / 4;
  const bool dense_m = (h->metric_kind == BJX_METRIC_DENSE);
  const bool dense_t = (h->cfg.target.kind == BJX_TARGET_DENSE_GAUSSIAN);
  if (n_steps <= 0) return 0;
  if (dense_m && dense_t) {
    // BASELINE config 2.  Every product's epilogue writes the operand planes of the next product:
    //   q <- q + eps_c (p M^-1)            reads planes(p), Cin = q, emits planes(q)
    //   p <- p - (eps_c/2)(q P) twice       reads planes(q), Cin = p, emits planes(p)      (between two steps)
    // Only the opening half kick and the closing gradient / logp / half kick are row kernels.
    float *pr = w.rmax[PL_P], *qr = w.rmax[PL_Q];
    k_rows_open<<<grow(C), kRowWarps * 32, 0, h->stream>>>(C, D, p, g, q, eps, eps_dev, w.xs[PL_P], w.unscale[PL_P], pr, pr + C,
                                                          qr, qr + C);
    BJX_CHECK_LAUNCH("k_rows_open");
    int pphase = 0, qphase = 0;
    for (int s = 0; s < n_steps; ++s) {
      int rc = gemm(h, w, C, nullptr, PL_P, MAT_IMM, q, q, eps_dev ? 1.0f : eps * 1.0f, eps_dev, 1.f, false, PlanesOut{PL_Q, qphase++});
      if (rc) return rc;
      if (s + 1 < n_steps) {
        // Between two steps neither g nor logp is observable, only p += (eps_c/2) g twice (this step's second half kick
        // and the next step's first, integrators.py:134-141,235-239) with g = -(q P): both FMAs ride on the epilogue of
        // the gradient product, per-row factor -(eps_c * 0.5) (bit-identical to kicking with the stored gradient, since
        // the row lifts are powers of two).
        rc = gemm(h, w, C, nullptr, PL_Q, MAT_PREC, p, p, eps_dev ? -0.5f : -(eps * 0.5f), eps_dev, 1.f, true, PlanesOut{PL_P, pphase++});
        if (rc) return rc;
      } else {
        rc = dense_grad(h, w, C, q, p, eps, eps_dev, g, logp, 1, p_planes_after, true);
        if (rc) return rc;
      }
    }
    return 0;
  }
  k_rows_axpy<<<g4(n4), 256, 0, h->stream>>>(C, D, p, g, eps, eps_dev, 0.5f);  // first half kick p += (eps/2) g
  BJX_CHECK_LAUNCH("k_rows_axpy");
  bool p_presplit = false;
  for (int s = 0; s < n_steps; ++s) {
    int rc;
    if (dense_m) {
      // q = q + (eps_c * 1.0) * (p M^-1): the axpy rides on the product's epilogue
      rc = gemm(h, w, C, p_presplit ? nullptr : p, PL_P, MAT_IMM, q, q, eps_dev ? 1.0f : eps * 1.0f, eps_dev, 1.f);
      if (rc) return rc;
    } else {
      rc = dense_velocity(h, w, C, p, w.v);
      if (rc) return rc;
      k_rows_axpy<<<g4(n4), 256, 0, h->stream>>>(C, D, q, w.v, eps, eps_dev, 1.0f);
      BJX_CHECK_LAUNCH("k_rows_axpy");
    }
    const bool more = (s + 1 < n_steps);
    // g, logp at the new q; p += (eps/2) g; plus the next step's first half kick -- and, with a dense metric, the
    // operand planes of that step's M^-1 p product -- when one follows
    const bool want_planes = dense_m && (more || p_planes_after);
    rc = dense_grad(h, w, C, q, p, eps, eps_dev, g, logp, more ? 2 : 1, want_planes);
    if (rc) return rc;
    p_presplit = want_planes;
  }
  return 0;
}

int bjx_dense_velocity(bjx_handle_t h, const float* p, float* v) {
  DenseWs w;
  int rc = dense_ws(h, w);
  return rc ? rc : dense_velocity(h, w, h->cfg.n_chains, p, v);
}

// The elliptical slice prior's L z for every chain (bjx_ess.cu): z = normal(split(key_c, 4)[1], (D,)) and one
// float32-accurate product against the planes of L = chol(cov); *lz points at the result [C, D] in the workspace.
int bjx_dense_prior_product(bjx_handle_t h, const uint32_t* keys, const float** lz) {
  DenseWs w;
  int rc = dense_ws(h, w);
  if (rc) return rc;
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  k_dense_normal<<<g4((long long)C * D / 4), 256, 0, h->stream>>>(C, D, keys, w.v, 1, h->key_shared, h->chain_offset);
  BJX_CHECK_LAUNCH("k_dense_normal");
  *lz = w.p;
  return gemm(h, w, C, w.v, PL_P, MAT_PRIOR, w.p, nullptr, 1.f, nullptr, 0.f);
}

int bjx_dense_init_state(bjx_handle_t h, const float* q, float* logp_out, float* grad_out) {
  DenseWs w;
  int rc = dense_ws(h, w);
  return rc ? rc : dense_grad(h, w, h->cfg.n_chains, q, nullptr, 0.f, nullptr, grad_out, logp_out);
}

int bjx_dense_sample_momentum(bjx_handle_t h, const uint32_t* keys, float* p_out, bool split_first) {
  DenseWs w;
  int rc = dense_ws(h, w);
  return rc ? rc : dense_momentum(h, w, h->cfg.n_chains, keys, p_out, split_first);
}

int bjx_dense_energy(bjx_handle_t h, const float* p, const float* logp, float* e_out) {
  DenseWs w;
  int rc = dense_ws(h, w);
  return rc ? rc : dense_energy(h, w, h->cfg.n_chains, p, logp, e_out);
}

int bjx_dense_leapfrog(bjx_handle_t h, float* q, float* p, float* logp, float* g, float eps, const float* eps_dev,
                       int n_steps) {
  DenseWs w;
  int rc = dense_ws(h, w);
  return rc ? rc : dense_leapfrog_core(h, w, q, p, logp, g, eps, eps_dev, n_steps);
}

int bjx_dense_hmc_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, const float* g_in,
                       float* q_out, float* logp_out, float* g_out, float eps, const float* eps_dev, int L,
                       const InfoPtrs& info) {
  DenseWs w;
  int rc = dense_ws(h, w);
  if (rc) return rc;
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const size_t bytes = (size_t)C * D * sizeof(float);
  rc = dense_momentum(h, w, C, keys, w.p, true);  // hmc.py:299-302
  if (rc) return rc;
  if (info.momentum) BJX_CUDA(cudaMemcpyAsync(info.momentum, w.p, bytes, cudaMemcpyDeviceToDevice, h->stream));
  rc = dense_energy(h, w, C, w.p, logp_in, w.e0);  // hmc.py:159
  if (rc) return rc;
  BJX_CUDA(cudaMemcpyAsync(w.q, q_in, bytes, cudaMemcpyDeviceToDevice, h->stream));
  BJX_CUDA(cudaMemcpyAsync(w.g, g_in, bytes, cudaMemcpyDeviceToDevice, h->stream));
  BJX_CUDA(cudaMemcpyAsync(w.lw, logp_in, (size_t)C * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  const bool planes_after = (h->metric_kind == BJX_METRIC_DENSE) && L > 0;
  rc = dense_leapfrog_core(h, w, w.q, w.p, w.lw, w.g, eps, eps_dev, L, planes_after);  // trajectory.py:165
  if (rc) return rc;
  // kinetic energy of the (flipped) end momentum: (-p)^T M^-1 (-p) = p^T M^-1 p   (hmc.py:158-160)
  rc = dense_energy(h, w, C, w.p, w.lw, w.e1, planes_after);
  if (rc) return rc;
  if (info.proposal_position) BJX_CUDA(cudaMemcpyAsync(info.proposal_position, w.q, bytes, cudaMemcpyDeviceToDevice, h->stream));
  if (info.proposal_momentum) {  // flipped momentum (hmc.py:158)
    BJX_CUDA(cudaMemsetAsync(info.proposal_momentum, 0, bytes, h->stream));
    k_rows_axpy<<<g4((long long)C * D / 4), 256, 0, h->stream>>>(C, D, info.proposal_momentum, w.p, -1.0f, nullptr, 1.0f);
    BJX_CHECK_LAUNCH("k_rows_axpy");
  }
  k_rows_accept<<<grow(C), kRowWarps * 32, 0, h->stream>>>(C, D, keys, w.e0, w.e1, h->cfg.divergence_threshold, w.q, w.g, w.lw,
                                                          q_in, g_in, logp_in, q_out, g_out, logp_out, L, info, h->key_shared,
                                                          h->chain_offset);
  BJX_CHECK_LAUNCH("k_rows_accept");
  return 0;
}

#include "bjx_dense_nuts.cuh"
