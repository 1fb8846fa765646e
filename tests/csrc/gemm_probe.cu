// Test probe: a host-only C entry point into the shipped dense-path product bjx::gemm_f16x3 (libbjx.so), so that the
// tests can call the kernel with any shape and epilogue its contract (bjx_gemm.h) allows, not only the ones the
// samplers use.  Includes bjx_gemm.h, so the GemmCall layout is the library's own.
#include "bjx_gemm.h"

extern "C" int bjx_probe_gemm_f16x3(const void* x_planes, const void* a_planes, void* Y, const void* Cin, void* planes_out,
                                    int M, int N, int K, int KP, int KP_out, float alpha, const void* alpha_dev,
                                    const void* x_unscale, const void* mat_unscale, float beta, int has_cin,
                                    int double_kick, int planes, void* out_unscale, const void* stale_max, void* next_max,
                                    void* zero_max, void* stream) {
  bjx::GemmCall g;
  g.x_planes = static_cast<const uint16_t*>(x_planes);
  g.a_planes = static_cast<const uint16_t*>(a_planes);
  g.Y = static_cast<float*>(Y);
  g.Cin = static_cast<const float*>(Cin);
  g.planes_out = static_cast<uint16_t*>(planes_out);
  g.M = M; g.N = N; g.K = K; g.KP = KP; g.KP_out = KP_out;
  g.epi.alpha = alpha;
  g.epi.alpha_dev = static_cast<const float*>(alpha_dev);
  g.epi.x_unscale = static_cast<const float*>(x_unscale);
  g.epi.mat_unscale = static_cast<const float*>(mat_unscale);
  g.epi.beta = beta;
  g.epi.has_cin = has_cin;
  g.epi.double_kick = double_kick;
  g.epi.planes = planes;
  g.epi.out_unscale = static_cast<float*>(out_unscale);
  g.epi.stale_max = static_cast<const float*>(stale_max);
  g.epi.next_max = static_cast<float*>(next_max);
  g.epi.zero_max = static_cast<float*>(zero_max);
  return bjx::gemm_f16x3(g, static_cast<cudaStream_t>(stream));
}
