// A standard normal inside a hard box at +-B (the bounded target of the reference's MCLMC NaN-handling tests,
// tests/mcmc/test_mclmc_nan_fix_969.py:45-47): a step that overshoots the box gives a NaN log-density, which MCLMC's
// handle_nans must detect and revert.
//
//   logp(x) = -1/2 sum_i x_i^2 + sum_i log(B - |x_i|)          theta = [B]
//   d/dx_i  = -x_i - s_i / (B - |x_i|),   s_i = 1 if x_i >= 0 else -1   (jax's derivative of |x|, 1 at 0)
#pragma once
namespace bjx_user {
template <class R>
struct Model {
  float B;

  __device__ __forceinline__ void init(const bjx::UserCtx& u) { B = __ldg(u.theta); }

  template <bool WANT_LOGP>
  __device__ __forceinline__ void value_and_grad(const bjx::UserCtx& u, const float (&q)[R::NS], float (&g)[R::NS],
                                                 float& logp) const {
    float sq = 0.f, lg = 0.f;
#pragma unroll
    for (int s = 0; s < R::NS; ++s) {
      if (R::idx(s, u.lane) >= u.D) {
        g[s] = 0.f;
        continue;
      }
      const float x = q[s];
      const float r = B - fabsf(x);
      g[s] = -x - (x >= 0.f ? 1.0f : -1.0f) / r;
      sq += x * x;
      lg += logf(r);
    }
    if (WANT_LOGP) logp = -0.5f * bjx::warp_sum(sq) + bjx::warp_sum(lg);
  }
};
}  // namespace bjx_user
