// Shared (cross-chain, cross-GPU) window adaptation, device resident, and the collective of the path.
//
// Reference semantics (blackjax/adaptation/staged_adaptation.py:153-171,906-966): ONE dual-averaging update per
// warm-up step fed with mean(acceptance_rate over ALL chains), and in slow windows the chain-pooled moment block
// (metric_buffers.py:396-420) merged into the window accumulator by Chan-Golub-LeVeque (metric_buffers.py:334-393);
// window end: regularised inverse mass matrix (mass_matrix.py:335-357), accumulator reset, dual averaging
// re-initialised at exp(log_step_avg) (staged_adaptation.py:233-249).  The reference's collective for the cross-device
// case is lax.psum over the "chains" axis (blackjax/eca.py:56-62); here it is ONE NCCL all-gather of the per-GPU
// summary blocks per warm-up step, followed by the same merge on every rank (no broadcast needed).
//
// Results do not depend on the GPU count: the chains of a rank are reduced in FIXED blocks of BJX_STAT_BLOCK_CHAINS
// chains (mean and centred second moment per block, deterministic tree), the blocks of all ranks are gathered in global
// chain order and merged sequentially, so 1 x 65536 chains and 2 x 32768 chains execute the same float operations.
// Everything (merge, dual averaging, mass-matrix finalisation, the per-chain step-size array the transition kernels read)
// stays on the device: no .item(), no host round trip per warm-up step.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>

#include "bjx_handle.h"
#include "bjx_internal.h"
#include "bjx_pooled_step.cuh"

namespace bjx {

constexpr int kStatBlock = BJX_STAT_BLOCK_CHAINS;
constexpr int kHdr = 16;  // scalar slots at the head of the adaptation state: PS_* (bjx_pooled_step.cuh), the rest unused

// ---- per-block chain-pooled statistics ------------------------------------------------------------------------
// grid (ceil(D/32), n_blocks), block (32, 8): block (bx, by) reduces columns [32 bx, +32) over chains [by*B, (by+1)*B)
// to mean and sum of squared deviations (two passes, shared-memory tree in a fixed order); bx == 0 also sums the
// acceptance rates of those chains.  out[by] = (sum accept, n, mean[D], M2[D]).
__global__ void k_block_stats(int C, int D, const float* __restrict__ x, const float* __restrict__ acc, float* __restrict__ out) {
  __shared__ float red[8][33];
  const int c0 = blockIdx.y * kStatBlock;
  const int c1 = min(C, c0 + kStatBlock);
  const int n = c1 - c0;
  const int col = blockIdx.x * 32 + threadIdx.x;
  float* o = out + (size_t)blockIdx.y * (2 + 2 * D);
  float a = 0.f;
  if (col < D)
    for (int c = c0 + threadIdx.y; c < c1; c += 8) a += x[(size_t)c * D + col];
  red[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += red[k][threadIdx.x];
    red[0][threadIdx.x] = s / (float)n;
  }
  __syncthreads();
  const float mean = red[0][threadIdx.x];
  __syncthreads();
  a = 0.f;
  if (col < D)
    for (int c = c0 + threadIdx.y; c < c1; c += 8) {
      const float d = x[(size_t)c * D + col] - mean;
      a = fmaf(d, d, a);
    }
  red[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && col < D) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += red[k][threadIdx.x];
    o[2 + col] = mean;
    o[2 + D + col] = s;
  }
  if (blockIdx.x == 0) {  // acceptance rates of the block's chains: 256 partial sums, fixed-order tree
    __syncthreads();
    const int t = threadIdx.y * 32 + threadIdx.x;
    float s = 0.f;
    for (int c = c0 + t; c < c1; c += 256) s += acc[c];
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (threadIdx.x == 0) red[threadIdx.y][0] = s;
    __syncthreads();
    if (t == 0) {
      float tot = 0.f;
      for (int k = 0; k < 8; ++k) tot += red[k][0];
      o[0] = tot;
      o[1] = (float)n;
    }
  }
}

// ---- merge + dual averaging + window bookkeeping: one CTA ---------------------------------------------------------
// state: header | w_mean [D] | w_m2 [D] (the window accumulator, its count in PS_WINDOW_N) | block records
__global__ void k_shared_adapt(int D, int nblk, const float* __restrict__ blocks, float* __restrict__ st, int stage, int window_end,
                               float target, float* __restrict__ imm, float* __restrict__ eps_hist) {
  const int S = 2 + 2 * D;
  const float w_n0 = st[PS_WINDOW_N];
  for (int d = threadIdx.x; d < D; d += blockDim.x) {  // threads own dimensions; each replays the scalar count recurrence
    float nn = blocks[1];
    float mean = blocks[2 + d], m2 = blocks[2 + D + d];
    for (int b = 1; b < nblk; ++b) {
      const float* g = blocks + (size_t)b * S;
      float fm, fc, nab;
      cgl_factors(nn, g[1], fm, fc, nab);
      const float delta = g[2 + d] - mean;
      mean = mean + delta * fm;
      m2 = m2 + g[2 + D + d] + delta * delta * fc;
      nn = nab;
    }
    if (stage == 1) {  // merge this step's pooled block into the window accumulator (staged_adaptation.py:283-297)
      float fm, fc, nab;
      cgl_factors(w_n0, nn, fm, fc, nab);
      const float delta = mean - st[kHdr + d];
      const float wm = st[kHdr + d] + delta * fm;
      const float w2 = st[kHdr + D + d] + m2 + delta * delta * fc;
      if (window_end) {  // mass_matrix.py:335-357, then reset
        const float cov = w2 / (nab - 1.f);
        const float denom = nab + 5.f;
        imm[d] = nab / denom * cov + 5.f / denom * 1e-3f;
        st[kHdr + d] = 0.f;
        st[kHdr + D + d] = 0.f;
      } else {
        st[kHdr + d] = wm;
        st[kHdr + D + d] = w2;
      }
    }
  }
  __syncthreads();  // every thread has read the window count
  if (threadIdx.x == 0) {
    const float n = pooled_step_size_update(nblk, blocks, S, st, window_end, target, eps_hist);
    if (stage == 1) {
      float fm, fc, wn_new;
      cgl_factors(w_n0, n, fm, fc, wn_new);
      st[PS_WINDOW_N] = window_end ? 0.f : wn_new;
    }
  }
}

__global__ void k_fill_from(int n, const float* __restrict__ src, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[0];
}
void launch_fill_from(int n, const float* src, float* dst, cudaStream_t s) {
  k_fill_from<<<(n + 255) / 256, 256, 0, s>>>(n, src, dst);
}
__global__ void k_adapt_init(int D, float* st, float eps0, float* imm) {
  for (int d = threadIdx.x; d < 2 * D; d += blockDim.x) st[kHdr + d] = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) imm[d] = 1.f;
  if (threadIdx.x == 0) {
    da_init(st + PS_DA, eps0);
    st[PS_EPS] = da_step_size(st + PS_DA);
    for (int k = PS_WINDOW_N; k < kHdr; ++k) st[k] = 0.f;
  }
}

// ---- NCCL, bound at run time (libbjx.so itself has no NCCL dependency: single-GPU users never load it) -----------
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string err;
};
static NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    // prefer a copy that is already in the process (PyTorch bundles one), else the system library
    api.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!api.lib) api.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!api.lib) api.lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!api.lib) {
      api.err = std::string("cannot load libnccl.so.2: ") + dlerror();
      return;
    }
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(api.lib, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(api.lib, "ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(api.lib, "ncclCommDestroy");
    api.AllGather = (decltype(api.AllGather))dlsym(api.lib, "ncclAllGather");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(api.lib, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather) api.err = "libnccl.so.2 lacks the expected symbols";
  });
  return api;
}
}  // namespace bjx

using namespace bjx;

static int nccl_fail(bjx_handle_t h, ncclResult_t r, const char* where) {
  NcclApi& a = nccl();
  return bjx_fail(h, BJX_E_UNSUPPORTED, std::string(where) + ": " + (a.GetErrorString ? a.GetErrorString(r) : "NCCL error"));
}

extern "C" int bjx_nccl_unique_id(void* id128_out) {
  NcclApi& a = nccl();
  if (!a.err.empty()) return bjx_fail(nullptr, BJX_E_UNSUPPORTED, a.err);
  if (!id128_out) return bjx_fail(nullptr, BJX_E_INVALID, "null argument");
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclResult_t r = a.GetUniqueId(reinterpret_cast<ncclUniqueId*>(id128_out));
  return r == ncclSuccess ? 0 : nccl_fail(nullptr, r, "ncclGetUniqueId");
}

extern "C" int bjx_nccl_comm_init_rank(const void* id128, int32_t n_ranks, int32_t rank, int32_t device, void** comm_out) {
  NcclApi& a = nccl();
  if (!a.err.empty()) return bjx_fail(nullptr, BJX_E_UNSUPPORTED, a.err);
  if (!id128 || !comm_out || n_ranks < 1 || rank < 0 || rank >= n_ranks) return bjx_fail(nullptr, BJX_E_INVALID, "bad argument");
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return bjx_cuda_fail(nullptr, e, "cudaSetDevice");
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t comm = nullptr;
  ncclResult_t r = a.CommInitRank(&comm, n_ranks, id, rank);
  if (r != ncclSuccess) return nccl_fail(nullptr, r, "ncclCommInitRank");
  *comm_out = comm;
  return 0;
}

extern "C" int bjx_nccl_comm_destroy(void* comm) {
  NcclApi& a = nccl();
  if (!a.err.empty() || !comm) return 0;
  ncclResult_t r = a.CommDestroy(reinterpret_cast<ncclComm_t>(comm));
  return r == ncclSuccess ? 0 : nccl_fail(nullptr, r, "ncclCommDestroy");
}

extern "C" int bjx_allgather_stats(bjx_handle_t h, void* nccl_comm, const float* block, int64_t count, float* gathered) {
  if (!h || !block || !gathered || count <= 0) return bjx_fail(h, BJX_E_INVALID, "bad argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  if (!nccl_comm) {  // one rank: the gathered array is the block
    if (gathered != block) BJX_CUDA(cudaMemcpyAsync(gathered, block, (size_t)count * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    return 0;
  }
  NcclApi& a = nccl();
  if (!a.err.empty()) return bjx_fail(h, BJX_E_UNSUPPORTED, a.err);
  ncclResult_t r = a.AllGather(block, gathered, (size_t)count, ncclFloat, reinterpret_cast<ncclComm_t>(nccl_comm), h->stream);
  return r == ncclSuccess ? 0 : nccl_fail(h, r, "ncclAllGather");
}

extern "C" int64_t bjx_adapt_shared_state_floats(int32_t n_chains_local, int32_t dim, int32_t n_ranks) {
  if (n_chains_local <= 0 || dim <= 0 || n_ranks <= 0) return 0;
  const int64_t blk = 2 + 2 * (int64_t)dim;
  return kHdr + 2 * (int64_t)dim + (int64_t)cov_stat_blocks(n_chains_local) * blk * (1 + n_ranks);
}

extern "C" int bjx_adapt_shared_init(bjx_handle_t h, float* state, float initial_step_size, float* step_size_chain_out, float* imm_out) {
  if (!h || !state || !step_size_chain_out || !imm_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (!(initial_step_size > 0.f)) return bjx_fail(h, BJX_E_INVALID, "initial_step_size must be positive");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  k_adapt_init<<<1, 256, 0, h->stream>>>(D, state, initial_step_size, imm_out);
  BJX_CHECK_LAUNCH("k_adapt_init");
  launch_fill_from(C, state + PS_EPS, step_size_chain_out, h->stream);
  BJX_CHECK_LAUNCH("k_fill_from");
  return bjx_set_metric(h, BJX_METRIC_DIAG, imm_out);
}

extern "C" int bjx_adapt_shared_update(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, float* state, const float* q,
                                       const float* acceptance_rate, int32_t stage, int32_t window_end, float target_acceptance,
                                       float* step_size_chain, float* imm, float* eps_history) {
  if (!h || !state || !q || !acceptance_rate || !step_size_chain || !imm) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (n_ranks < 1 || (n_ranks > 1 && !nccl_comm)) return bjx_fail(h, BJX_E_INVALID, "n_ranks > 1 needs a communicator");
  if (window_end && stage != 1) return bjx_fail(h, BJX_E_INVALID, "a window ends on a slow-stage step");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const int nb = cov_stat_blocks(C);
  const size_t blk = 2 + 2 * (size_t)D;
  float* local = state + kHdr + 2 * (size_t)D;
  float* gathered = local + (size_t)nb * blk;
  k_block_stats<<<dim3((D + 31) / 32, nb), dim3(32, 8), 0, h->stream>>>(C, D, q, acceptance_rate, local);
  BJX_CHECK_LAUNCH("k_block_stats");
  const float* merged_in = local;
  if (n_ranks > 1) {
    int rc = bjx_allgather_stats(h, nccl_comm, local, (int64_t)(nb * blk), gathered);
    if (rc) return rc;
    merged_in = gathered;
  }
  k_shared_adapt<<<1, 512, 0, h->stream>>>(D, nb * n_ranks, merged_in, state, stage, window_end, target_acceptance, imm, eps_history);
  BJX_CHECK_LAUNCH("k_shared_adapt");
  launch_fill_from(C, state + PS_EPS, step_size_chain, h->stream);
  BJX_CHECK_LAUNCH("k_fill_from");
  if (window_end) return bjx_set_metric(h, BJX_METRIC_DIAG, imm);  // mass_matrix_sqrt of the new metric, on the stream
  return 0;
}

extern "C" int bjx_adapt_shared_final(bjx_handle_t h, const float* state, float* step_size_out) {
  if (!h || !state || !step_size_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  launch_da(3, 1, const_cast<float*>(state), nullptr, 0.f, step_size_out, h->stream);  // exp(log_step_avg)
  BJX_CHECK_LAUNCH("k_da_final");
  return 0;
}

// =====================================================================================================================
// ChEES-HMC warm-up (blackjax/adaptation/chees_adaptation.py, mass_matrix_estimation=None): dual averaging on the
// harmonic mean of the acceptance probabilities (:341-360) and Adam ascent on log(trajectory length) along the ChEES
// gradient jitter * T * (|dx'|^2 - |dx|^2) <dx', p'> (:362-480), both from cross-chain statistics.  Same structure as
// the shared window adaptation above: fixed blocks of BJX_STAT_BLOCK_CHAINS chains, merged in global chain order after
// an all-gather (two per step: the centring means must be global before the per-chain dot products can be formed).
// =====================================================================================================================
namespace bjx {
constexpr int kChHdr = 32;
// header slots
enum { CH_EPS = 0, CH_LOG_EPS_MA, CH_T, CH_LOG_T_MA, CH_DA_LOGX, CH_DA_LOGX_AVG, CH_DA_STEP, CH_DA_ERR, CH_DA_MU, CH_AD_COUNT,
       CH_AD_MU, CH_AD_NU, CH_RGA, CH_STEP, CH_MAX_BITS, CH_JITTER_AMOUNT, CH_T_IDX, CH_L, CH_HM_SUM, CH_HM_N, CH_GRAD };

__device__ __forceinline__ float halton_f(int i, int max_bits) {  // dynamic_hmc.py:205-215
  float s = 0.f;
  for (int k = 0; k < max_bits; ++k) s += (float)(((i + 1) >> k) & 1) * (0.5f / (float)(1u << k));
  return s;
}

// per chain: w' = is_divergent ? 0 : acceptance, zeroed when the proposal row holds a non-finite entry (:239-247)
__global__ void k_chees_w(int C, int D, const float* __restrict__ prop_q, const float* __restrict__ acc,
                          const uint8_t* __restrict__ is_div, float* __restrict__ w) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  bool fin = true;
  for (int i = lane; i < D; i += 32) fin = fin && isfinite(prop_q[(size_t)c * D + i]);
  fin = __all_sync(0xffffffffu, fin);
  if (lane == 0) w[c] = (!is_div[c] && fin) ? acc[c] : 0.f;
}

// block (bx, by): columns [32 bx, +32) over chains of statistic block by.
// out[by] = (sum_{nd} 1/acc, n_nd, sum w', sum_c w'_c x_c [D], sum_c finite q_c [D], count of non-NaN q [D])
__global__ void k_chees_pass1(int C, int D, const float* __restrict__ prop_q, const float* __restrict__ init_q,
                              const float* __restrict__ acc, const uint8_t* __restrict__ is_div, const float* __restrict__ w,
                              float* __restrict__ out) {
  __shared__ float red[3][8][33];
  const int c0 = blockIdx.y * kStatBlock, c1 = min(C, c0 + kStatBlock);
  const int col = blockIdx.x * 32 + threadIdx.x;
  float* o = out + (size_t)blockIdx.y * (3 + 3 * (size_t)D);
  float sw = 0.f, sq = 0.f, cq = 0.f;
  if (col < D)
    for (int c = c0 + threadIdx.y; c < c1; c += 8) {
      const float x = prop_q[(size_t)c * D + col], q = init_q[(size_t)c * D + col];
      sw = fmaf(w[c], isfinite(x) ? x : 0.f, sw);
      if (!isnan(q)) { sq += q; cq += 1.f; }
    }
  red[0][threadIdx.y][threadIdx.x] = sw;
  red[1][threadIdx.y][threadIdx.x] = sq;
  red[2][threadIdx.y][threadIdx.x] = cq;
  __syncthreads();
  if (threadIdx.y == 0 && col < D) {
    float a = 0.f, b = 0.f, n = 0.f;
    for (int k = 0; k < 8; ++k) { a += red[0][k][threadIdx.x]; b += red[1][k][threadIdx.x]; n += red[2][k][threadIdx.x]; }
    o[3 + col] = a;
    o[3 + D + col] = b;
    o[3 + 2 * D + col] = n;
  }
  if (blockIdx.x == 0) {
    __syncthreads();
    const int t = threadIdx.y * 32 + threadIdx.x;
    float h = 0.f, n = 0.f, ws = 0.f;
    for (int c = c0 + t; c < c1; c += 256) {
      if (!is_div[c]) { h += 1.0f / acc[c]; n += 1.f; }
      ws += w[c];
    }
    for (int off = 16; off > 0; off >>= 1) {
      h += __shfl_xor_sync(0xffffffffu, h, off);
      n += __shfl_xor_sync(0xffffffffu, n, off);
      ws += __shfl_xor_sync(0xffffffffu, ws, off);
    }
    if (threadIdx.x == 0) { red[0][threadIdx.y][0] = h; red[1][threadIdx.y][0] = n; red[2][threadIdx.y][0] = ws; }
    __syncthreads();
    if (t == 0) {
      float a = 0.f, b = 0.f, c_ = 0.f;
      for (int k = 0; k < 8; ++k) { a += red[0][k][0]; b += red[1][k][0]; c_ += red[2][k][0]; }
      o[0] = a; o[1] = b; o[2] = c_;
    }
  }
}

// ---- diagonal-metric mode (mass_matrix_estimation="diagonal", chees_adaptation.py:61-237,758-1001) ----------------
// Its own state ("metric state", MmLayout below).  Header slots:
enum { MM_WSTEPS = 0, MM_CG, MM_THRESH, MM_ENGAGED, MM_LAMBDA, MM_WHITEN, MM_FLOOR };
constexpr int kMmHdr = 16;

// The diagonal Welford accumulator of the reference (mass_matrix.py:364-444, one row at a time) is kept as (n, mean, m2):
// each in-window step the k_block_stats blocks of the new positions are merged in global block order and the pooled
// block is merged into the accumulator (Chan-Golub-LeVeque; equal to the sequential fold in exact arithmetic).
// n = in-window steps * global chain count, formed in double (exact far beyond 2^24 samples).
__device__ __forceinline__ void mm_fold_diag(int D, int d, int nblk, int nbl, size_t R, size_t off, const float* __restrict__ blocks,
                                             float* __restrict__ ms) {
  const size_t S = 2 + 2 * (size_t)D;
  auto blk = [&](int b) { return blocks + (size_t)(b / nbl) * R + off + (size_t)(b % nbl) * S; };
  float nn = blk(0)[1], mean = blk(0)[2 + d], m2 = blk(0)[2 + D + d];
  for (int b = 1; b < nblk; ++b) {
    const float* g = blk(b);
    float fm, fc, nab;
    cgl_factors(nn, g[1], fm, fc, nab);
    const float delta = g[2 + d] - mean;
    mean = mean + delta * fm;
    m2 = m2 + g[2 + D + d] + delta * delta * fc;
    nn = nab;
  }
  const double na = (double)ms[MM_WSTEPS] * (double)ms[MM_CG], nb = (double)nn, ab = na + nb;
  const float fm = (float)(nb / ab), fc = (float)(na * nb / ab);
  const float delta = mean - ms[kMmHdr + d];
  ms[kMmHdr + d] = ms[kMmHdr + d] + delta * fm;
  ms[kMmHdr + D + d] = ms[kMmHdr + D + d] + m2 + delta * delta * fc;
}

// merge the pass-1 blocks in global order: proposal mean (weighted), initial mean (nanmean), harmonic-mean sums.  The
// payload is rank-major, R floats per rank, starting with the rank's nbl pass-1 blocks (the identity metric: R = nbl * S,
// so block b is at b * S).  The diagonal-metric payload follows them with the rank's nbl k_block_stats blocks of the new
// positions; with in_window these are folded into the diagonal accumulator of `ms`.
__global__ void k_chees_means(int D, int nblk, const float* __restrict__ blocks, float* __restrict__ st, int nbl, size_t R,
                              float* __restrict__ ms, int in_window) {
  const size_t S = 3 + 3 * (size_t)D;
  auto blk = [&](int b) { return blocks + (size_t)(b / nbl) * R + (size_t)(b % nbl) * S; };
  float* pm = st + kChHdr;
  float* qm = pm + D;
  float sw = 0.f;
  for (int b = 0; b < nblk; ++b) sw += blk(b)[2];
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float a = 0.f, q = 0.f, n = 0.f;
    for (int b = 0; b < nblk; ++b) {
      a += blk(b)[3 + d];
      q += blk(b)[3 + D + d];
      n += blk(b)[3 + 2 * D + d];
    }
    pm[d] = a / (sw + 1e-20f);
    qm[d] = q / n;
    if (in_window) mm_fold_diag(D, d, nblk, nbl, R, (size_t)nbl * S, blocks, ms);
  }
  if (threadIdx.x == 0) {
    float h = 0.f, n = 0.f;
    for (int b = 0; b < nblk; ++b) { h += blk(b)[0]; n += blk(b)[1]; }
    st[CH_HM_SUM] = h;
    st[CH_HM_N] = n;
  }
  __syncthreads();  // every thread has read the sample count
  if (in_window && threadIdx.x == 0) ms[MM_WSTEPS] += 1.f;
}

// per chain (one warp): (|x' - E x'|^2 - |x - E x|^2) <x' - E x', p'>, then its acceptance-weighted terms.
// kWhiten (chees_adaptation.py:449-458): x' - E x' and x - E x scaled by 1/sqrt(imm), the momentum by imm then 1/sqrt(imm);
// with imm = ones every scaling is exact, so the result is bit-identical to the raw expression.
template <bool kWhiten = false>
__global__ void k_chees_dots(int C, int D, const float* __restrict__ prop_q, const float* __restrict__ prop_p,
                             const float* __restrict__ init_q, const float* __restrict__ acc, const uint8_t* __restrict__ is_div,
                             const float* __restrict__ st, float* __restrict__ num, float* __restrict__ den,
                             const float* __restrict__ imm = nullptr) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  const float* pm = st + kChHdr;
  const float* qm = pm + D;
  float a = 0.f, b = 0.f, d = 0.f;
  for (int i = lane; i < D; i += 32) {
    if constexpr (kWhiten) {
      const float s = 1.0f / sqrtf(imm[i]);
      const float pc = (prop_q[(size_t)c * D + i] - pm[i]) * s;
      const float ic = (init_q[(size_t)c * D + i] - qm[i]) * s;
      a = fmaf(pc, pc, a);
      b = fmaf(ic, ic, b);
      d = fmaf(pc, (prop_p[(size_t)c * D + i] * imm[i]) * s, d);
    } else {
      const float pc = prop_q[(size_t)c * D + i] - pm[i];
      const float ic = init_q[(size_t)c * D + i] - qm[i];
      a = fmaf(pc, pc, a);
      b = fmaf(ic, ic, b);
      d = fmaf(pc, prop_p[(size_t)c * D + i], d);
    }
  }
  for (int off = 16; off > 0; off >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, off);
    b += __shfl_xor_sync(0xffffffffu, b, off);
    d += __shfl_xor_sync(0xffffffffu, d, off);
  }
  if (lane == 0) {
    const bool nd = !is_div[c];
    num[c] = nd ? acc[c] * ((a - b) * d) : 0.f;
    den[c] = nd ? acc[c] + 1e-20f : 0.f;
  }
}
// fixed-order sums of the two per-chain arrays over each statistic block -> out[by] = (sum num, sum den)
__global__ void k_chees_pass2(int C, const float* __restrict__ num, const float* __restrict__ den, float* __restrict__ out) {
  __shared__ float red[2][8];
  const int c0 = blockIdx.x * kStatBlock, c1 = min(C, c0 + kStatBlock);
  float a = 0.f, b = 0.f;
  for (int c = c0 + threadIdx.x; c < c1; c += 256) { a += num[c]; b += den[c]; }
  for (int off = 16; off > 0; off >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, off);
    b += __shfl_xor_sync(0xffffffffu, b, off);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float x = 0.f, y = 0.f;
    for (int k = 0; k < 8; ++k) { x += red[0][k]; y += red[1][k]; }
    out[2 * blockIdx.x] = x;
    out[2 * blockIdx.x + 1] = y;
  }
}

// the scalar update (chees_adaptation.py:341-360,470-511) and the next transition's step count.
// With a metric state `ms` whose length floor is on, the next transition consumes min(max(T, floor), max_leapfrog * eps)
// with floor = (pi/2) sqrt(lambda_max) once the diagonal estimate is engaged (_apply_length_floor, :192-236); T itself, the
// optimiser's state, is never floored.  lam_hist and eng_hist need `ms`.
__global__ void k_chees_finish(int nblk, const float* __restrict__ blocks2, float* __restrict__ st, float lr, float b1, float b2,
                               float target, float decay, float max_leapfrog, float* __restrict__ hist,
                               const float* __restrict__ ms, float* __restrict__ lam_hist, float* __restrict__ eng_hist) {
  if (threadIdx.x != 0) return;
  const int max_bits = (int)st[CH_MAX_BITS];
  const float jam = st[CH_JITTER_AMOUNT];
  const int rga = (int)st[CH_RGA];
  const float step = st[CH_STEP];
  float eps = st[CH_EPS], T = st[CH_T];
  // step size: dual averaging on target - harmonic mean of the non-divergent acceptance probabilities
  float hm = 1.0f / (st[CH_HM_SUM] / st[CH_HM_N]);
  if (!isfinite(hm)) hm = 0.f;
  float da[5];  // CH_DA_LOGX .. CH_DA_MU are a dual-averaging state; the update is kept only when the new step size is finite
  for (int k = 0; k < 5; ++k) da[k] = st[CH_DA_LOGX + k];
  float log_x = da[0];
  da_update_step(da, hm, target);
  if (isfinite(da_step_size(da))) {
    eps = da_step_size(da);
    log_x = da[0];
    for (int k = 0; k < 4; ++k) st[CH_DA_LOGX + k] = da[k];
  }
  const float uw = powf(step, -decay);
  const float log_eps_ma = (1.f - uw) * st[CH_LOG_EPS_MA] + uw * log_x;
  // trajectory length: Adam on log T along the ChEES gradient
  float num = 0.f, den = 0.f;
  for (int b = 0; b < nblk; ++b) { num += blocks2[2 * b]; den += blocks2[2 * b + 1]; }
  const float jit = halton_f(rga, max_bits) * jam + (1.f - jam);
  const float grad = (jit * T) * num / den;
  const float log_T = logf(T);
  float ad_mu = b1 * st[CH_AD_MU] + (1.f - b1) * grad;
  float ad_nu = b2 * st[CH_AD_NU] + (1.f - b2) * grad * grad;
  const float count = st[CH_AD_COUNT] + 1.f;
  const float mu_hat = ad_mu / (1.f - powf(b1, count));
  const float nu_hat = ad_nu / (1.f - powf(b2, count));
  float upd = -lr * (mu_hat / (sqrtf(nu_hat) + 1e-8f));
  upd = fminf(fmaxf(upd, -0.35f), 0.35f);
  if (isnan(-lr * (mu_hat / (sqrtf(nu_hat) + 1e-8f)))) upd = __int_as_float(0x7fc00000);
  float new_log_T = log_T;
  if (isfinite(log_T + upd)) {
    new_log_T = log_T + upd;
    st[CH_AD_MU] = ad_mu; st[CH_AD_NU] = ad_nu; st[CH_AD_COUNT] = count;
  }
  const float log_T_ma = (1.f - uw) * st[CH_LOG_T_MA] + uw * new_log_T;
  float newT = expf(log_T_ma);
  newT = fminf(fmaxf(newT, eps), max_leapfrog * eps);
  st[CH_EPS] = eps; st[CH_LOG_EPS_MA] = log_eps_ma; st[CH_T] = newT; st[CH_LOG_T_MA] = log_T_ma;
  st[CH_RGA] = (float)(rga + 1);
  st[CH_STEP] = step + 1.f;
  st[CH_GRAD] = grad;
  // next transition: ceil(jitter(i + 1) * T / eps) leapfrog steps (integration_steps_fn :775-779)
  const float jn = halton_f(rga + 1, max_bits) * jam + (1.f - jam);
  float consumed = newT;
  if (ms && ms[MM_FLOOR] != 0.f) {
    const float floor_v = ms[MM_ENGAGED] != 0.f ? 1.57079637f * sqrtf(ms[MM_LAMBDA]) : 0.f;
    consumed = fminf(fmaxf(newT, floor_v), max_leapfrog * eps);
  }
  st[CH_L] = ceilf(jn * (consumed / eps));
  const int t = (int)st[CH_T_IDX];
  if (hist) { hist[4 * t] = eps; hist[4 * t + 1] = newT; hist[4 * t + 2] = st[CH_L]; hist[4 * t + 3] = grad; }
  if (lam_hist) lam_hist[t] = ms[MM_LAMBDA];
  if (eng_hist) eng_hist[t] = ms[MM_ENGAGED];
  st[CH_T_IDX] = (float)(t + 1);
}
__global__ void k_chees_init(float* st, float eps0, int max_bits, float jitter_amount) {
  if (threadIdx.x != 0) return;
  for (int k = 0; k < kChHdr; ++k) st[k] = 0.f;
  st[CH_EPS] = eps0; st[CH_T] = eps0;
  da_init(st + CH_DA_LOGX, eps0);
  st[CH_STEP] = 1.f; st[CH_MAX_BITS] = (float)max_bits; st[CH_JITTER_AMOUNT] = jitter_amount;
  const float j0 = halton_f(0, max_bits) * jitter_amount + (1.f - jitter_amount);
  st[CH_L] = ceilf(j0 * (eps0 / eps0));
}
__global__ void k_fill_steps(int n, const float* __restrict__ src, int32_t* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (int32_t)src[0];
}

// ---- windowed covariance accumulator of the length floor (cgl_update_batch, metric_buffers.py:396-447) -------------
// Every statistic block b of BJX_STAT_BLOCK_CHAINS chains keeps its own (count, mean[D], m2[D, D]) over the window; per
// in-window step m2_b += X~_b^T X~_b + f delta delta^T with X~_b the block's rows centred on this step's block mean,
// delta = step mean - accumulated mean, f = n_a n_b / (n_a + n_b).  Only the lower triangle of m2_b is kept.
//
// k_cov_syrk: hand-written float32 SIMT SYRK.  grid (lower-triangular 64x64 output tiles, blocks), 256 threads, each
// thread a 4x4 register tile; the chain axis is staged through shared memory 16 rows at a time, centred (and zero-padded
// past the block's last chain or the last column) while it is staged, so every C and D <= 1024 takes the same code.  A
// 16-row chunk is summed in its own registers before it is added to the running tile (pairwise-style accumulation keeps
// the float32 error of a 4096-row block near 1e-7 of the diagonal).  The Chan update is the epilogue.
constexpr int kSyT = 64, kSyK = 16;
__global__ void __launch_bounds__(256) k_cov_syrk(int C, int D, const float* __restrict__ x, const float* __restrict__ bstats,
                                                   size_t bstride, float* __restrict__ cov, size_t cstride) {
  __shared__ __align__(16) float As[kSyK][kSyT];
  __shared__ __align__(16) float Bs[kSyK][kSyT];
  __shared__ float mu_i[kSyT], mu_j[kSyT];
  // lower-triangular tile index -> (ti, tj), ti >= tj
  const int p = blockIdx.x;
  int ti = (int)((sqrtf(8.f * (float)p + 1.f) - 1.f) * 0.5f);
  while (ti * (ti + 1) / 2 > p) --ti;
  while ((ti + 1) * (ti + 2) / 2 <= p) ++ti;
  const int tj = p - ti * (ti + 1) / 2;
  const int b = blockIdx.y;
  const int c0 = b * kStatBlock, c1 = min(C, c0 + kStatBlock);
  const float* mu = bstats + (size_t)b * bstride + 2;  // k_block_stats record: (sum accept, n, mean[D], M2[D])
  float* blk = cov + (size_t)b * cstride;              // (count, -, mean[D], m2[D*D])
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int i0 = ti * kSyT, j0 = tj * kSyT;
  if (tid < kSyT) {
    mu_i[tid] = (i0 + tid < D) ? mu[i0 + tid] : 0.f;
    mu_j[tid] = (j0 + tid < D) ? mu[j0 + tid] : 0.f;
  }
  __syncthreads();
  float acc[4][4], part[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) acc[r][s] = 0.f;
  const int lc = tid & 63, lk = tid >> 6;
  const bool iok = i0 + lc < D, jok = j0 + lc < D;
  for (int k0 = c0; k0 < c1; k0 += kSyK) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int k = lk + 4 * r, c = k0 + k;
      const bool cok = c < c1;
      As[k][lc] = (cok && iok) ? x[(size_t)c * D + i0 + lc] - mu_i[lc] : 0.f;
      Bs[k][lc] = (cok && jok) ? x[(size_t)c * D + j0 + lc] - mu_j[lc] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) part[r][s] = 0.f;
#pragma unroll
    for (int k = 0; k < kSyK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bb = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) part[r][s] = fmaf(av[r], bv[s], part[r][s]);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) acc[r][s] += part[r][s];
    __syncthreads();
  }
  // epilogue: Chan update against the block's accumulated mean (read before k_cov_mean_update rewrites it)
  float fm, fc, nab;
  cgl_factors(blk[0], (float)(c1 - c0), fm, fc, nab);
  const float* am = blk + 2;
  float* m2 = blk + 2 + D;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + ty * 4 + r;
    if (i >= D) continue;
    const float di = mu_i[ty * 4 + r] - am[i];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int j = j0 + tx * 4 + s;
      if (j > i || j >= D) continue;
      const float dj = mu_j[tx * 4 + s] - am[j];
      const size_t o = (size_t)i * D + j;
      m2[o] = (m2[o] + acc[r][s]) + di * dj * fc;
    }
  }
}
// count and mean of every block accumulator after the SYRK (one CTA per block: the count is read before it is rewritten)
__global__ void k_cov_mean_update(int C, int D, const float* __restrict__ bstats, size_t bstride, float* __restrict__ cov, size_t cstride) {
  const int b = blockIdx.x;
  const int c0 = b * kStatBlock, c1 = min(C, c0 + kStatBlock);
  float* blk = cov + (size_t)b * cstride;
  const float* mu = bstats + (size_t)b * bstride + 2;
  float fm, fc, nab;
  cgl_factors(blk[0], (float)(c1 - c0), fm, fc, nab);
  for (int d = threadIdx.x; d < D; d += blockDim.x) blk[2 + d] = blk[2 + d] + (mu[d] - blk[2 + d]) * fm;
  __syncthreads();
  if (threadIdx.x == 0) blk[0] = nab;
}

// merge the block accumulators in global order and whiten (_recompute_eig_state, :169-189):
// W = (m2 / max(count - 1, 1)) * s_i * s_j with s = 1 / sqrt(imm).  One thread per lower-triangle element, both halves written.
__global__ void k_cov_merge_whiten(int D, int nblk, const float* __restrict__ cov, size_t cstride, const float* __restrict__ imm,
                                   float* __restrict__ W, float* __restrict__ mean_out) {
  const int i = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > i) return;
  float n = 0.f, mi = 0.f, mj = 0.f, m2 = 0.f;
  for (int b = 0; b < nblk; ++b) {
    const float* blk = cov + (size_t)b * cstride;
    if (blk[0] == 0.f) continue;  // an empty block leaves the merge unchanged (cgl_merge_two's n_ab = 0 guard)
    float fm, fc, nab;
    cgl_factors(n, blk[0], fm, fc, nab);
    const float di = blk[2 + i] - mi, dj = blk[2 + j] - mj;
    m2 = m2 + blk[2 + D + (size_t)i * D + j] + di * dj * fc;
    mi = mi + di * fm;
    mj = mj + dj * fm;
    n = nab;
  }
  if (mean_out && j == 0) { mean_out[0] = n; mean_out[1 + i] = mi; }
  const float cv = m2 / fmaxf(n - 1.f, 1.f);
  if (imm) {
    const float w = cv * (1.0f / sqrtf(imm[i])) * (1.0f / sqrtf(imm[j]));
    W[(size_t)i * D + j] = w;
    W[(size_t)j * D + i] = w;
  } else {
    W[(size_t)i * D + j] = cv;
    W[(size_t)j * D + i] = cv;
  }
}

// one power iteration (_power_iteration_lambda_max, :147-166): v = x / ||x|| (norm guarded to 1 when 0; skipped for the
// warm start, which is already normalised), y = W v.  Every CTA forms v itself in a fixed order; CTA 0 stores it in v_out.
// 8 warps per CTA, one row per warp.
__global__ void __launch_bounds__(256) k_pow_iter(int D, const float* __restrict__ W, const float* __restrict__ x, int normalize,
                                                  float* __restrict__ v_out, float* __restrict__ y) {
  __shared__ float v[1024];
  __shared__ float red[8];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  float nrm = 1.f;
  if (normalize) {
    float s = 0.f;
    for (int d = tid; d < D; d += 256) s = fmaf(x[d], x[d], s);
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) red[w] = s;
    __syncthreads();
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += red[k];
    nrm = sqrtf(t);
    if (!(nrm > 0.f)) nrm = 1.f;
  }
  for (int d = tid; d < D; d += 256) v[d] = normalize ? x[d] / nrm : x[d];
  __syncthreads();
  if (v_out && blockIdx.x == 0)
    for (int d = tid; d < D; d += 256) v_out[d] = v[d];
  const int r = blockIdx.x * 8 + w;
  if (r >= D) return;
  float a = 0.f;
  for (int d = lane; d < D; d += 32) a = fmaf(W[(size_t)r * D + d], v[d], a);
  for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
  if (lane == 0) y[r] = a;
}
// lambda_max = max(v . W v, 1e-6) (_LENGTH_FLOOR_LAMBDA_EPS)
__global__ void k_pow_rayleigh(int D, const float* __restrict__ v, const float* __restrict__ y, float* __restrict__ ms) {
  __shared__ float red[8];
  const int tid = threadIdx.x;
  float s = 0.f;
  for (int d = tid; d < D; d += 256) s = fmaf(v[d], y[d], s);
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += red[k];
    ms[MM_LAMBDA] = fmaxf(t, 1e-6f);
  }
}

// the metric the next transition uses (_diagonal_mass_matrix_or_fallback, :75-90): max(m2 / (n - 1), 1e-20) once
// n >= max(64, int(2 sqrt(D))), ones before that
__global__ void k_mm_imm(int D, float* __restrict__ ms, float* __restrict__ imm) {
  const double n = (double)ms[MM_WSTEPS] * (double)ms[MM_CG];
  const bool engaged = n >= (double)ms[MM_THRESH];
  const float nm1 = (float)(n - 1.0);
  for (int d = threadIdx.x; d < D; d += blockDim.x) imm[d] = engaged ? fmaxf(ms[kMmHdr + D + d] / nm1, 1e-20f) : 1.f;
  __syncthreads();
  if (threadIdx.x == 0) ms[MM_ENGAGED] = engaged ? 1.f : 0.f;
}
__global__ void k_mm_init(int D, float* __restrict__ ms, float c_global, float thresh, int whiten, int floor_on, float* __restrict__ imm) {
  float* eig = ms + kMmHdr + 2 * (size_t)D;
  const float v0 = 1.0f / sqrtf((float)D);  // ones(D) / sqrt(D) (_eig_state_init, :142-144)
  for (int d = threadIdx.x; d < D; d += blockDim.x) { imm[d] = 1.f; eig[d] = v0; }
  if (threadIdx.x == 0) {
    ms[MM_CG] = c_global; ms[MM_THRESH] = thresh; ms[MM_LAMBDA] = 1.f;
    ms[MM_WHITEN] = (float)whiten; ms[MM_FLOOR] = (float)floor_on;
  }
}

// The launchers of the block statistics and the block covariance accumulators, shared by ChEES and MEADS-LRD (bjx_meads.cu).
int cov_stat_blocks(int C) { return (C + kStatBlock - 1) / kStatBlock; }
size_t cov_block_floats(int D) { return 2 + (size_t)D + (size_t)D * D; }
void launch_block_stats(int C, int D, const float* x, const float* acc, float* out, cudaStream_t s) {
  k_block_stats<<<dim3((D + 31) / 32, cov_stat_blocks(C)), dim3(32, 8), 0, s>>>(C, D, x, acc, out);
}
void launch_cov_fold(int C, int D, const float* q, const float* stats, float* cov, cudaStream_t s) {
  const int nb = cov_stat_blocks(C), tiles = (D + kSyT - 1) / kSyT;
  const size_t sstride = 2 + 2 * (size_t)D;
  k_cov_syrk<<<dim3(tiles * (tiles + 1) / 2, nb), 256, 0, s>>>(C, D, q, stats, sstride, cov, cov_block_floats(D));
  k_cov_mean_update<<<nb, 256, 0, s>>>(C, D, stats, sstride, cov, cov_block_floats(D));
}
void launch_cov_merge(int nblk, int D, const float* cov, const float* imm, float* out, float* count_mean, cudaStream_t s) {
  k_cov_merge_whiten<<<dim3((D + 255) / 256, D), 256, 0, s>>>(D, nblk, cov, cov_block_floats(D), imm, out, count_mean);
}
}  // namespace bjx

// =====================================================================================================================
// ChEES with mass_matrix_estimation="diagonal" (chees_adaptation.py:61-237,797-1001).  The metric state holds the diagonal
// accumulator, the power-iteration vectors, this step's payload for the first all-gather (the pass-1 blocks followed by the
// k_block_stats blocks of the new positions, so an ordinary step adds no collective) and, with the length floor, the
// per-block covariance accumulators and the whitened matrix of the last recompute.  Only recompute steps (every 32
// in-window steps, and the final parameters) move D x D data between GPUs: the block accumulators are all-gathered and
// merged in global block order on every rank (DESIGN.md section 7).
// =====================================================================================================================
namespace {
// The ChEES state of both modes: header, proposal mean[D], initial mean[D], the per-chain w, num and den [C], the pass-1
// blocks of this rank and of all ranks (the identity metric's payload; the diagonal metric gathers its own), and the
// pass-2 blocks (sum num, sum den) of this rank and of all ranks.
struct ChLayout {
  int nb;
  size_t S1;                                                     // pass-1 record stride
  size_t w, num, den, loc1, gat1, loc2, gat2, total;
};
ChLayout ch_layout(int C, int D, int n_ranks) {
  ChLayout L{};
  L.nb = cov_stat_blocks(C);
  L.S1 = 3 + 3 * (size_t)D;
  size_t o = kChHdr + 2 * (size_t)D;
  L.w = o; o += C;
  L.num = o; o += C;
  L.den = o; o += C;
  L.loc1 = o; o += (size_t)L.nb * L.S1;
  L.gat1 = o; o += (size_t)L.nb * L.S1 * n_ranks;
  L.loc2 = o; o += (size_t)L.nb * 2;
  L.gat2 = o; o += (size_t)L.nb * 2 * n_ranks;
  L.total = o;
  return L;
}

struct MmLayout {
  int nb;
  size_t S1, Sm, R, Sc;                                          // record strides; R = payload floats per rank
  size_t eig, u0, u1, pay_loc, pay_stats, W, cov_loc, pay_gat, cov_gat, total;
};
MmLayout mm_layout(int C, int D, int n_ranks, int options) {
  MmLayout L{};
  const size_t d = (size_t)D;
  const bool fl = options & BJX_CHEES_LENGTH_FLOOR;
  L.nb = cov_stat_blocks(C);
  L.S1 = 3 + 3 * d;
  L.Sm = 2 + 2 * d;
  L.R = (size_t)L.nb * (L.S1 + L.Sm);
  L.Sc = cov_block_floats(D);
  size_t o = kMmHdr + 2 * d;                                     // header, accumulator mean[D], m2[D]
  L.eig = o; o += d;
  L.u0 = o; o += d;
  L.u1 = o; o += d;
  L.pay_loc = o;                                                 // payload: pass-1 blocks, then the k_block_stats blocks
  L.pay_stats = o + (size_t)L.nb * L.S1; o += L.R;
  L.W = o; o += fl ? d * d : 0;
  L.cov_loc = o; o += fl ? (size_t)L.nb * L.Sc : 0;
  L.pay_gat = o; o += n_ranks > 1 ? L.R * n_ranks : 0;
  L.cov_gat = o; o += (fl && n_ranks > 1) ? (size_t)L.nb * L.Sc * n_ranks : 0;
  L.total = o;
  return L;
}

// merged block accumulators -> W (whitened by imm, or the plain covariance with imm = NULL); block order is global
int mm_cov_merge(bjx_handle_t h, void* comm, int n_ranks, const MmLayout& L, float* ms, const float* imm, float* W,
                 float* mean_out) {
  const float* cov = ms + L.cov_loc;
  if (n_ranks > 1) {
    int rc = bjx_allgather_stats(h, comm, ms + L.cov_loc, (int64_t)(L.nb * L.Sc), ms + L.cov_gat);
    if (rc) return rc;
    cov = ms + L.cov_gat;
  }
  launch_cov_merge(L.nb * n_ranks, h->cfg.dim, cov, imm, W, mean_out, h->stream);
  BJX_CHECK_LAUNCH("k_cov_merge_whiten");
  return 0;
}

// _recompute_eig_state: whiten by imm, `iters` power iterations warm-started from the stored eigenvector, lambda_max
int mm_recompute(bjx_handle_t h, void* comm, int n_ranks, const MmLayout& L, float* ms, const float* imm, int iters) {
  const int D = h->cfg.dim;
  int rc = mm_cov_merge(h, comm, n_ranks, L, ms, imm, ms + L.W, nullptr);
  if (rc) return rc;
  const float* W = ms + L.W;
  float* u[2] = {ms + L.u0, ms + L.u1};
  const int g = (D + 7) / 8;
  k_pow_iter<<<g, 256, 0, h->stream>>>(D, W, ms + L.eig, 0, nullptr, u[0]);
  for (int k = 1; k < iters; ++k) k_pow_iter<<<g, 256, 0, h->stream>>>(D, W, u[(k - 1) & 1], 1, nullptr, u[k & 1]);
  k_pow_iter<<<g, 256, 0, h->stream>>>(D, W, u[(iters - 1) & 1], 1, ms + L.eig, u[iters & 1]);
  k_pow_rayleigh<<<1, 256, 0, h->stream>>>(D, ms + L.eig, u[iters & 1], ms);
  BJX_CHECK_LAUNCH("k_pow_iter");
  return 0;
}

constexpr int kFloorIters = 5, kFloorFinalIters = 20;  // chees_adaptation.py:121-122 (the 32-step cadence is the caller's)

// One warm-up step of either mode.  The identity metric has no metric state (ms = NULL, options = 0, no window): its
// pass-1 payload is the state's.  The diagonal metric gathers the metric state's payload; its in-window steps fold the new
// positions into the diagonal accumulator (and, with the length floor, the covariance accumulators) and rewrite imm.
int chees_step(bjx_handle_t h, void* comm, int n_ranks, int options, float* state, float* ms, const float* init_q,
               const float* prop_q, const float* prop_p, const float* new_q, const float* acc, const uint8_t* is_div,
               float lr, float b1, float b2, float target, float decay, int max_lf, int in_window, int recompute,
               float* eps_c, int32_t* steps_c, float* hist, float* imm, float* lam_hist, float* eng_hist) {
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  const ChLayout L = ch_layout(C, D, n_ranks);
  const int nb = L.nb;
  MmLayout M{};
  float* pay = state + L.loc1;
  float* pay_gat = state + L.gat1;
  size_t R = (size_t)nb * L.S1;
  if (ms) {
    M = mm_layout(C, D, n_ranks, options);
    pay = ms + M.pay_loc;
    pay_gat = ms + M.pay_gat;
    R = M.R;
  }
  float* w = state + L.w;
  float* num = state + L.num;
  float* den = state + L.den;
  cudaStream_t s = h->stream;
  k_chees_w<<<(C + 7) / 8, 256, 0, s>>>(C, D, prop_q, acc, is_div, w);
  k_chees_pass1<<<dim3((D + 31) / 32, nb), dim3(32, 8), 0, s>>>(C, D, prop_q, init_q, acc, is_div, w, pay);
  BJX_CHECK_LAUNCH("k_chees_pass1");
  if (in_window) {
    launch_block_stats(C, D, new_q, acc, ms + M.pay_stats, s);
    BJX_CHECK_LAUNCH("k_block_stats");
  }
  const float* m1 = pay;
  if (n_ranks > 1) {
    int rc = bjx_allgather_stats(h, comm, pay, (int64_t)R, pay_gat);
    if (rc) return rc;
    m1 = pay_gat;
  }
  k_chees_means<<<1, 512, 0, s>>>(D, nb * n_ranks, m1, state, nb, R, ms, in_window);
  if (options & BJX_CHEES_WHITEN)  // the criterion of this step uses the metric of this step's transition
    k_chees_dots<true><<<(C + 7) / 8, 256, 0, s>>>(C, D, prop_q, prop_p, init_q, acc, is_div, state, num, den, imm);
  else
    k_chees_dots<<<(C + 7) / 8, 256, 0, s>>>(C, D, prop_q, prop_p, init_q, acc, is_div, state, num, den);
  k_chees_pass2<<<nb, 256, 0, s>>>(C, num, den, state + L.loc2);
  BJX_CHECK_LAUNCH("k_chees_pass2");
  const float* m2 = state + L.loc2;
  if (n_ranks > 1) {
    int rc = bjx_allgather_stats(h, comm, state + L.loc2, (int64_t)(nb * 2), state + L.gat2);
    if (rc) return rc;
    m2 = state + L.gat2;
  }
  if (in_window && (options & BJX_CHEES_LENGTH_FLOOR)) {
    launch_cov_fold(C, D, new_q, ms + M.pay_stats, ms + M.cov_loc, s);
    BJX_CHECK_LAUNCH("k_cov_syrk");
    if (recompute) {  // against the metric this step's transition used, before this step's fold engages (:898-903)
      int rc = mm_recompute(h, comm, n_ranks, M, ms, imm, kFloorIters);
      if (rc) return rc;
    }
  }
  if (in_window) {
    k_mm_imm<<<1, 1024, 0, s>>>(D, ms, imm);
    BJX_CHECK_LAUNCH("k_mm_imm");
  }
  k_chees_finish<<<1, 32, 0, s>>>(nb * n_ranks, m2, state, lr, b1, b2, target, decay, (float)max_lf, hist, ms, lam_hist,
                                  eng_hist);
  launch_fill_from(C, state + CH_EPS, eps_c, s);
  k_fill_steps<<<(C + 255) / 256, 256, 0, s>>>(C, state + CH_L, steps_c);
  BJX_CHECK_LAUNCH("k_chees_finish");
  if (in_window) return bjx_set_metric(h, BJX_METRIC_DIAG, imm);  // mass_matrix_sqrt of the new estimate, on the stream
  return 0;
}

// Final parameters (:958-1001), on the host: out[0] = exp(log eps_ma), out[1] = exp(log T_ma - log eps_ma).  With the
// length floor, 20 power iterations against the final metric (:971-978) come first and the floor is re-applied to
// exp(log T_ma), divided by exp(log eps_ma).  With a metric state, out[2] = floor clipped by the cap, out[3] = lambda_max.
int chees_final(bjx_handle_t h, void* comm, int n_ranks, int options, const float* state, float* ms, int max_lf,
                const float* imm, float* out) {
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const bool floor_on = options & BJX_CHEES_LENGTH_FLOOR;
  if (floor_on) {
    int rc = mm_recompute(h, comm, n_ranks, mm_layout(h->cfg.n_chains, h->cfg.dim, n_ranks, options), ms, imm,
                          kFloorFinalIters);
    if (rc) return rc;
  }
  float hst[kChHdr], hdr[kMmHdr];
  BJX_CUDA(cudaMemcpyAsync(hst, state, sizeof(hst), cudaMemcpyDeviceToHost, h->stream));
  if (ms) BJX_CUDA(cudaMemcpyAsync(hdr, ms, sizeof(hdr), cudaMemcpyDeviceToHost, h->stream));
  BJX_CUDA(cudaStreamSynchronize(h->stream));
  const float eps = expf(hst[CH_LOG_EPS_MA]);
  float n_lf = expf(hst[CH_LOG_T_MA] - hst[CH_LOG_EPS_MA]), clipped = 0.f;
  if (floor_on) {
    const bool engaged = hdr[MM_ENGAGED] != 0.f;
    const float floor_v = engaged ? 1.57079637f * sqrtf(hdr[MM_LAMBDA]) : 0.f;
    const float cap = (float)max_lf * eps;
    n_lf = fminf(fmaxf(expf(hst[CH_LOG_T_MA]), floor_v), cap) / eps;
    clipped = (engaged && floor_v > cap) ? 1.f : 0.f;
  }
  out[0] = eps;
  out[1] = n_lf;
  if (ms) {
    out[2] = clipped;
    out[3] = hdr[MM_LAMBDA];
  }
  return 0;
}
}  // namespace

extern "C" int64_t bjx_chees_state_floats(int32_t n_chains_local, int32_t dim, int32_t n_ranks) {
  if (n_chains_local <= 0 || dim <= 0 || n_ranks <= 0) return 0;
  return (int64_t)ch_layout(n_chains_local, dim, n_ranks).total;
}

extern "C" int bjx_chees_init(bjx_handle_t h, float* state, float step_size, int32_t max_bits, float jitter_amount,
                              float* step_size_chain_out, int32_t* steps_chain_out) {
  if (!h || !state || !step_size_chain_out || !steps_chain_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (!(step_size > 0.f) || max_bits < 1 || max_bits > 30) return bjx_fail(h, BJX_E_INVALID, "bad step_size / max_bits");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains;
  k_chees_init<<<1, 32, 0, h->stream>>>(state, step_size, max_bits, jitter_amount);
  BJX_CHECK_LAUNCH("k_chees_init");
  launch_fill_from(C, state + CH_EPS, step_size_chain_out, h->stream);
  k_fill_steps<<<(C + 255) / 256, 256, 0, h->stream>>>(C, state + CH_L, steps_chain_out);
  BJX_CHECK_LAUNCH("k_fill");
  return 0;
}

extern "C" int bjx_chees_update(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, float* state, const float* initial_position,
                                const float* proposal_position, const float* proposal_momentum, const float* acceptance_rate,
                                const uint8_t* is_divergent, float learning_rate, float b1, float b2, float target_acceptance,
                                float decay_rate, int32_t max_leapfrog_steps, float* step_size_chain, int32_t* steps_chain,
                                float* history) {
  if (!h || !state || !initial_position || !proposal_position || !proposal_momentum || !acceptance_rate || !is_divergent ||
      !step_size_chain || !steps_chain)
    return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (n_ranks < 1 || (n_ranks > 1 && !nccl_comm)) return bjx_fail(h, BJX_E_INVALID, "n_ranks > 1 needs a communicator");
  return chees_step(h, nccl_comm, n_ranks, 0, state, nullptr, initial_position, proposal_position, proposal_momentum, nullptr,
                    acceptance_rate, is_divergent, learning_rate, b1, b2, target_acceptance, decay_rate, max_leapfrog_steps,
                    0, 0, step_size_chain, steps_chain, history, nullptr, nullptr, nullptr);
}

extern "C" int bjx_chees_final(bjx_handle_t h, const float* state, float* out2) {
  if (!h || !state || !out2) return bjx_fail(h, BJX_E_INVALID, "null argument");
  return chees_final(h, nullptr, 1, 0, state, nullptr, 0, nullptr, out2);
}

extern "C" int64_t bjx_chees_metric_state_floats(int32_t n_chains_local, int32_t dim, int32_t n_ranks, int32_t options) {
  if (n_chains_local <= 0 || dim <= 0 || dim > 1024 || n_ranks <= 0) return 0;
  return (int64_t)mm_layout(n_chains_local, dim, n_ranks, options).total;
}

extern "C" int bjx_chees_metric_init(bjx_handle_t h, float* metric_state, int32_t n_ranks, int32_t options, float* imm_out) {
  if (!h || !metric_state || !imm_out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (n_ranks < 1 || (options & ~(BJX_CHEES_WHITEN | BJX_CHEES_LENGTH_FLOOR))) return bjx_fail(h, BJX_E_INVALID, "bad n_ranks / options");
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  if (D > 1024) return bjx_fail(h, BJX_E_UNSUPPORTED, "ChEES is built for dim <= 1024");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const MmLayout L = mm_layout(C, D, n_ranks, options);
  BJX_CUDA(cudaMemsetAsync(metric_state, 0, L.total * sizeof(float), h->stream));
  const int thresh = std::max(64, (int)(2.0 * std::sqrt((double)D)));  // _mass_matrix_engagement_threshold, :61-72
  k_mm_init<<<1, 256, 0, h->stream>>>(D, metric_state, (float)((double)C * n_ranks), (float)thresh,
                                       (options & BJX_CHEES_WHITEN) ? 1 : 0, (options & BJX_CHEES_LENGTH_FLOOR) ? 1 : 0, imm_out);
  BJX_CHECK_LAUNCH("k_mm_init");
  return bjx_set_metric(h, BJX_METRIC_DIAG, imm_out);
}

extern "C" int bjx_chees_update_metric(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, int32_t options, float* state,
                                       float* metric_state, const float* initial_position, const float* proposal_position,
                                       const float* proposal_momentum, const float* new_position, const float* acceptance_rate,
                                       const uint8_t* is_divergent, float learning_rate, float b1, float b2,
                                       float target_acceptance, float decay_rate, int32_t max_leapfrog_steps, int32_t in_window,
                                       int32_t recompute, float* step_size_chain, int32_t* steps_chain, float* history,
                                       float* imm, float* lambda_history, float* engaged_history) {
  if (!h || !state || !metric_state || !initial_position || !proposal_position || !proposal_momentum || !new_position ||
      !acceptance_rate || !is_divergent || !step_size_chain || !steps_chain || !imm)
    return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (n_ranks < 1 || (n_ranks > 1 && !nccl_comm)) return bjx_fail(h, BJX_E_INVALID, "n_ranks > 1 needs a communicator");
  if (recompute && !(in_window && (options & BJX_CHEES_LENGTH_FLOOR)))
    return bjx_fail(h, BJX_E_INVALID, "recompute needs an in-window step and the length floor");
  if (h->cfg.dim > 1024) return bjx_fail(h, BJX_E_UNSUPPORTED, "ChEES is built for dim <= 1024");
  return chees_step(h, nccl_comm, n_ranks, options, state, metric_state, initial_position, proposal_position,
                    proposal_momentum, new_position, acceptance_rate, is_divergent, learning_rate, b1, b2, target_acceptance,
                    decay_rate, max_leapfrog_steps, in_window, recompute, step_size_chain, steps_chain, history, imm,
                    lambda_history, engaged_history);
}

extern "C" int bjx_chees_final_metric(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, int32_t options, const float* state,
                                      float* metric_state, int32_t max_leapfrog_steps, const float* imm, float* out4_host) {
  if (!h || !state || !metric_state || !imm || !out4_host) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (n_ranks < 1 || (n_ranks > 1 && !nccl_comm)) return bjx_fail(h, BJX_E_INVALID, "n_ranks > 1 needs a communicator");
  if (h->cfg.dim > 1024) return bjx_fail(h, BJX_E_UNSUPPORTED, "ChEES is built for dim <= 1024");
  return chees_final(h, nccl_comm, n_ranks, options, state, metric_state, max_leapfrog_steps, imm, out4_host);
}

extern "C" int bjx_chees_metric_fold_covariance(bjx_handle_t h, int32_t options, float* metric_state, const float* q) {
  if (!h || !metric_state || !q) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (!(options & BJX_CHEES_LENGTH_FLOOR)) return bjx_fail(h, BJX_E_INVALID, "the covariance accumulator needs the length floor");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  if (D > 1024) return bjx_fail(h, BJX_E_UNSUPPORTED, "ChEES is built for dim <= 1024");
  const MmLayout L = mm_layout(C, D, 1, options);
  // k_block_stats also sums an acceptance array over each block; q stands in for it (that sum is not read here)
  launch_block_stats(C, D, q, q, metric_state + L.pay_stats, h->stream);
  BJX_CHECK_LAUNCH("k_block_stats");
  launch_cov_fold(C, D, q, metric_state + L.pay_stats, metric_state + L.cov_loc, h->stream);
  BJX_CHECK_LAUNCH("k_cov_syrk");
  return 0;
}

extern "C" int bjx_chees_metric_covariance(bjx_handle_t h, void* nccl_comm, int32_t n_ranks, int32_t options, float* metric_state,
                                           float* out) {
  if (!h || !metric_state || !out) return bjx_fail(h, BJX_E_INVALID, "null argument");
  if (n_ranks < 1 || (n_ranks > 1 && !nccl_comm)) return bjx_fail(h, BJX_E_INVALID, "n_ranks > 1 needs a communicator");
  if (!(options & BJX_CHEES_LENGTH_FLOOR)) return bjx_fail(h, BJX_E_INVALID, "the covariance accumulator needs the length floor");
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  if (D > 1024) return bjx_fail(h, BJX_E_UNSUPPORTED, "ChEES is built for dim <= 1024");
  const MmLayout L = mm_layout(C, D, n_ranks, options);
  return mm_cov_merge(h, nccl_comm, n_ranks, L, metric_state, nullptr, out + 1 + D, out);
}
