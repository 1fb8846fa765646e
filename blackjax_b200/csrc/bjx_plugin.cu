// Translation unit of a user-defined target plug-in (include/bjx_user_target.h, bjx_plugin_load in include/bjx.h).
// Built once per target by blackjax_b200/plugin.py (or by hand):
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Xcompiler -fPIC -shared \
//        -I blackjax_b200/csrc -I include -DBJX_USER_SOURCE='"my_target.cuh"' [-DBJX_BUILD_SC=<size class>] \
//        blackjax_b200/csrc/bjx_plugin.cu -o libbjxt_my_target.so
//
// It holds every transition kernel of the path (init, leapfrog, HMC, multinomial HMC, generalized HMC, NUTS doubling,
// the decoupled NUTS sampler) instantiated around the user's bjx_user::Model, exactly as bjx_inst_*.cu does
// for the built-in targets, and exports the two symbols bjx_plugin_load resolves.
#ifndef BJX_USER_SOURCE
#error "define BJX_USER_SOURCE to the file that defines bjx_user::Model (or bjx_user::BigModel with -DBJX_PLUGIN_BIG=1)"
#endif

#if defined(BJX_PLUGIN_BIG) && BJX_PLUGIN_BIG
// ---- rows beyond a warp (1024 < dim <= 18432): CTA-per-chain kernels around bjx_user::BigModel ----------------------------
#include "bjx_big.cuh"
#include BJX_USER_SOURCE

extern "C" int bjx_plugin_built_for_abi(void) { return bjx::plugin_abi(); }
// 0 = launched; > 0 = the cudaError_t of the launch
extern "C" int bjx_plugin_launch_big(int kernel_id, const bjx::BigLaunchArgs* a) {
  return bjx::big_launch<BJX_TARGET_USER>(kernel_id, *a);
}
#else
#define BJX_INSTANTIATE_TK 4  // bjx::TK_USER
#include "bjx_row.cuh"
#include BJX_USER_SOURCE

#include "../../include/bjx.h"
#include "bjx_big.cuh"      // (plugin_abi)
#include "bjx_launch.cuh"

extern "C" int bjx_plugin_built_for_abi(void) { return bjx::plugin_abi(); }

// 0 = launched; -2 = this (kernel, row size, metric, integrator) variant was not built into the plug-in; > 0 = the
// cudaError_t of the launch (the plug-in has its own CUDA runtime instance, so it reports its own launch errors).
extern "C" int bjx_plugin_launch(int kernel_id, int sc, int dm, const bjx::LaunchArgs* a) {
  const int rc = bjx::Launcher<bjx::TK_USER>::launch(kernel_id, sc, dm != 0, *a);
  if (rc) return rc;
  return (int)cudaGetLastError();
}
#endif
