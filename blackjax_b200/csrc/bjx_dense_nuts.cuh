// NUTS on the tensor-core dense path (dense metric and / or dense Gaussian target, 128 < D <= 1024).  Included at the end of
// bjx_dense.cu (it uses that file's product / gradient helpers).
//
// The generalized U-turn test and the kinetic energy need M^-1 p for every leaf (metrics.py:263-304), so a leaf costs two
// metric products (the half-step velocity and the full-step velocity) plus the target's gradient product.  Products want
// many rows, so the chains that run doubling d advance through its 2^d leaves IN LOCK STEP, compacted into the first n rows
// of the working arrays (gathered when the doubling starts, scattered back when it ends):
//   per doubling   k_dn_begin   direction / keys (trajectory.py:645-655), gather the endpoint that moves, first half kick
//   per leaf       velocity product -> q += eps v -> gradient (+ product) + second half kick -> velocity product ->
//                  k_dn_leaf: energy, progressive sampling (proposal.py:118-143), checkpoints and the iterative U-turn test
//                  (termination.py:56-104) with the checkpoints' cached velocities, next half kick
//   per doubling   k_dn_end     biased proposal update (proposal.py:146-176), merge, full-trajectory U-turn
//                  (trajectory.py:672-717) with the endpoints' cached velocities, compaction of the chains that go on
// A chain whose sub-tree stops early (divergence / U-turn) freezes its endpoint at that leaf and idles (its rows keep
// flowing through the products; nothing of it is read again) until the doubling ends.  The host reads ONE integer per
// doubling (the number of chains that go on: it sizes the products of the next doubling).
namespace bjx {

struct DnWs {
  float *cq, *cp, *cg, *cv, *cps;   // compact rows [C, D]: moving state, its velocity, sub-tree momentum sum
  float *ck_p, *ck_s, *ck_v;        // checkpoints [depth][C, D] (compact row index)
  float *left_v, *right_v;          // per chain: M^-1 p of the trajectory endpoints
  float *clogp, *ceps, *sub_weight, *sub_slpa, *sub_logp, *sub_energy, *u_prop;  // compact scalars [C]
  int *cn, *cdone, *cdir;
  uint32_t* ctk;                    // [C, 2] trajectory key of the running doubling
};

__device__ __forceinline__ float dn_dot(const float* a, const float* b, int D, int lane) {
  float acc = 0.f;
  for (int i = lane; i < D / 4; i += 32) {
    const float4 x = reinterpret_cast<const float4*>(a)[i], y = reinterpret_cast<const float4*>(b)[i];
    acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc); acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
  }
  return wsum(acc);
}
__device__ __forceinline__ void dn_copy(float* dst, const float* src, int D, int lane) {
  for (int i = lane; i < D / 4; i += 32) reinterpret_cast<float4*>(dst)[i] = reinterpret_cast<const float4*>(src)[i];
}
// p <- p + eh * g in place, and (planes != null) the exact operand planes of the kicked row
__device__ __forceinline__ void dn_kick(float* p, const float* g, float eh, int D, int lane, uint16_t* planes, float* unscale) {
  float amax = 0.f;
  for (int i = lane; i < D / 4; i += 32) {
    float4 pv = reinterpret_cast<const float4*>(p)[i];
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    pv.x = fmaf(eh, gv.x, pv.x); pv.y = fmaf(eh, gv.y, pv.y); pv.z = fmaf(eh, gv.z, pv.z); pv.w = fmaf(eh, gv.w, pv.w);
    reinterpret_cast<float4*>(p)[i] = pv;
    amax = max4(amax, pv);
  }
  if (planes) {
    const float sc = pow2_lift(wmax(amax));
    const int KP = plane_stride(D);
    for (int i = lane; i < D / 4; i += 32) store_planes(planes, KP, 4 * i, reinterpret_cast<const float4*>(p)[i], sc);
    if (lane == 0) *unscale = 1.0f / sc;
  }
}
// is_turning(p_l, p_r, p_sum) with the endpoint velocities given (metrics.py:272-304): rho = p_sum - (p_r + p_l)/2
__device__ __forceinline__ bool dn_turning(const float* pl, const float* vl, const float* pr, const float* vr, const float* psum,
                                           const float* sub_a, const float* sub_b, int D, int lane) {
  // p_sum = psum (sub_a == null) or psum - sub_a + sub_b (the checkpoint form, termination.py:96-103)
  float al = 0.f, ar = 0.f;
  for (int i = lane; i < D / 4; i += 32) {
    const float4 a = reinterpret_cast<const float4*>(pl)[i], b = reinterpret_cast<const float4*>(pr)[i];
    float4 s = reinterpret_cast<const float4*>(psum)[i];
    if (sub_a) {
      const float4 x = reinterpret_cast<const float4*>(sub_a)[i], y = reinterpret_cast<const float4*>(sub_b)[i];
      s = make_float4(s.x - x.x + y.x, s.y - x.y + y.y, s.z - x.z + y.z, s.w - x.w + y.w);
    }
    const float4 u = reinterpret_cast<const float4*>(vl)[i], w = reinterpret_cast<const float4*>(vr)[i];
    const float r0 = s.x - (b.x + a.x) / 2.0f, r1 = s.y - (b.y + a.y) / 2.0f, r2 = s.z - (b.z + a.z) / 2.0f,
                r3 = s.w - (b.w + a.w) / 2.0f;
    al = fmaf(u.x, r0, al); al = fmaf(u.y, r1, al); al = fmaf(u.z, r2, al); al = fmaf(u.w, r3, al);
    ar = fmaf(w.x, r0, ar); ar = fmaf(w.y, r1, ar); ar = fmaf(w.z, r2, ar); ar = fmaf(w.w, r3, ar);
  }
  al = wsum(al);
  ar = wsum(ar);
  return (al <= 0.f) || (ar <= 0.f);
}

// nuts.py:133-136,278-294 after the momentum draw (ws.left_p) and its velocity (dn.left_v) are in place
__global__ void k_dn_init(int C, int D, NutsWs ws, DnWs dn, const uint32_t* __restrict__ keys, int key_shared,
                          uint32_t chain_offset, const uint32_t* __restrict__ keyint_override, const float* q_in,
                          const float* logp_in, const float* g_in, float* q_out, float* logp_out, float* g_out, float* mom_out) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (c >= C) return;
  const size_t ro = (size_t)c * D;
  const float kin = 0.5f * dn_dot(dn.left_v + ro, ws.left_p + ro, D, lane);
  dn_copy(ws.right_p + ro, ws.left_p + ro, D, lane);
  dn_copy(dn.right_v + ro, dn.left_v + ro, D, lane);
  dn_copy(ws.psum + ro, ws.left_p + ro, D, lane);
  dn_copy(ws.left_q + ro, q_in + ro, D, lane);
  dn_copy(ws.right_q + ro, q_in + ro, D, lane);
  dn_copy(ws.left_g + ro, g_in + ro, D, lane);
  dn_copy(ws.right_g + ro, g_in + ro, D, lane);
  if (mom_out) dn_copy(mom_out + ro, ws.left_p + ro, D, lane);
  if (q_out != q_in) {
    dn_copy(q_out + ro, q_in + ro, D, lane);
    dn_copy(g_out + ro, g_in + ro, D, lane);
  }
  if (lane == 0) {
    const float logp0 = logp_in[c];
    const float h0 = -logp0 + kin;
    Key ki;
    if (keyint_override) {
      ki = Key{keyint_override[2 * c], keyint_override[2 * c + 1]};
    } else {
      const Key rk = key_shared ? fold_in(Key{keys[0], keys[1]}, chain_offset + (uint32_t)c) : Key{keys[2 * c], keys[2 * c + 1]};
      ki = fold_in(rk, 1u);
    }
    if (q_out != q_in) logp_out[c] = logp0;
    ws.left_logp[c] = logp0;
    ws.right_logp[c] = logp0;
    ws.h0[c] = h0;
    ws.prop_energy[c] = h0;
    ws.prop_weight[c] = 0.f;
    ws.prop_slpa[c] = -__int_as_float(0x7f800000);
    ws.n_states[c] = 0;
    ws.step[c] = 0;
    ws.is_div[c] = 0;
    ws.is_turn[c] = 0;
    ws.key_int[2 * c] = ki.a;
    ws.key_int[2 * c + 1] = ki.b;
  }
}

// start of doubling d for compact row r (chain list[r]): keys, direction, gather the moving endpoint, first half kick
__global__ void k_dn_begin(int n, int D, int d, NutsWs ws, DnWs dn, const int* __restrict__ list, float eps,
                           const float* __restrict__ eps_dev, uint16_t* __restrict__ p_planes, float* __restrict__ p_unscale) {
  const int lane = threadIdx.x & 31, r = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (r >= n) return;
  const int c = list ? list[r] : r;
  const size_t ro = (size_t)c * D, rr = (size_t)r * D;
  const Key ki{ws.key_int[2 * c], ws.key_int[2 * c + 1]};
  const Key sub = fold_in(ki, (uint32_t)d);             // trajectory.py:645-650
  const int dir = (uniform01(fold_in(sub, 0u)) < 0.5f) ? 1 : -1;
  const Key tk = fold_in(sub, 1u);
  const float ec = (float)dir * (eps_dev ? eps_dev[c] : eps);
  dn_copy(dn.cq + rr, (dir > 0 ? ws.right_q : ws.left_q) + ro, D, lane);
  dn_copy(dn.cp + rr, (dir > 0 ? ws.right_p : ws.left_p) + ro, D, lane);
  dn_copy(dn.cg + rr, (dir > 0 ? ws.right_g : ws.left_g) + ro, D, lane);
  __syncwarp();
  dn_kick(dn.cp + rr, dn.cg + rr, ec * 0.5f, D, lane, p_planes ? p_planes + (size_t)r * 2 * plane_stride(D) : nullptr,
          p_unscale + r);
  if (lane == 0) {
    dn.cdir[r] = dir;
    dn.ceps[r] = ec;
    dn.ctk[2 * r] = tk.a;
    dn.ctk[2 * r + 1] = tk.b;
    dn.u_prop[r] = uniform01(fold_in(sub, 2u));
    dn.cn[r] = 0;
    dn.cdone[r] = 0;
    dn.sub_weight[r] = -__int_as_float(0x7f800000);
    dn.sub_slpa[r] = -__int_as_float(0x7f800000);
    dn.sub_logp[r] = 0.f;
    dn.sub_energy[r] = 0.f;
  }
}

// leaf i of the running doubling (trajectory.py:318-372) for compact row r; (cq, cp, cg, clogp) hold the new state, cv = M^-1 cp
__global__ void k_dn_leaf(int n, int D, int i, int last, int C, NutsWs ws, DnWs dn, const int* __restrict__ list, float div_thr,
                          uint16_t* __restrict__ p_planes, float* __restrict__ p_unscale) {
  const int lane = threadIdx.x & 31, r = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (r >= n) return;
  if (dn.cdone[r]) return;
  const int c = list ? list[r] : r;
  const size_t ro = (size_t)c * D, rr = (size_t)r * D;
  const float* p = dn.cp + rr;
  const float* v = dn.cv + rr;
  float* ps = dn.cps + rr;
  const float logp = dn.clogp[r];
  const float e_new = -logp + 0.5f * dn_dot(v, p, D, lane);
  const float w_new = safe_energy_diff(ws.h0[c], e_new);    // proposal.py:94-98
  const float slpa_new = fminf(w_new, 0.f);
  const bool is_div = (-w_new) > div_thr;
  float sub_weight = dn.sub_weight[r], sub_slpa = dn.sub_slpa[r];
  bool take;
  if (i == 0) {
    dn_copy(ps, p, D, lane);
    take = true;
    sub_weight = w_new;
    sub_slpa = slpa_new;
  } else {
    for (int k = lane; k < D / 4; k += 32) {
      float4 a = reinterpret_cast<float4*>(ps)[k];
      const float4 b = reinterpret_cast<const float4*>(p)[k];
      a.x = a.x + b.x; a.y = a.y + b.y; a.z = a.z + b.z; a.w = a.w + b.w;
      reinterpret_cast<float4*>(ps)[k] = a;
    }
    const Key tk{dn.ctk[2 * r], dn.ctk[2 * r + 1]};
    const float u_leaf = uniform01(fold_in(tk, (uint32_t)i));
    take = u_leaf < expit_f(w_new - sub_weight);
    sub_weight = logaddexp_f(sub_weight, w_new);            // proposal.py:124-127
    sub_slpa = logaddexp_f(sub_slpa, slpa_new);
  }
  __syncwarp();
  if (take) {
    dn_copy(ws.sub_prop_q + ro, dn.cq + rr, D, lane);
    dn_copy(ws.sub_prop_g + ro, dn.cg + rr, D, lane);
  }
  // termination.py:75-84 checkpoint index range of leaf i
  const int idx_max = __popc((unsigned)i >> 1);
  const int idx_min = idx_max - __popc((~(unsigned)i & ((unsigned)i + 1u)) - 1u) + 1;
  const size_t lvl = (size_t)C * D;
  if ((i & 1) == 0) {  // termination.py:66-72
    dn_copy(dn.ck_p + idx_max * lvl + rr, p, D, lane);
    dn_copy(dn.ck_s + idx_max * lvl + rr, ps, D, lane);
    dn_copy(dn.ck_v + idx_max * lvl + rr, v, D, lane);
  }
  __syncwarp();
  bool turning = false;
  for (int k = idx_max; k >= idx_min && !turning; --k)  // termination.py:96-103: is_turning(ckpt_p, p, ps - ckpt_s + ckpt_p)
    turning = dn_turning(dn.ck_p + k * lvl + rr, dn.ck_v + k * lvl + rr, p, v, ps, dn.ck_s + k * lvl + rr, dn.ck_p + k * lvl + rr,
                         D, lane);
  const bool stop = is_div || turning;
  const int dir = dn.cdir[r];
  if (stop || i == last) {  // this leaf is the new endpoint of the merged trajectory (trajectory.py:376-385,697-704)
    dn_copy((dir > 0 ? ws.right_q : ws.left_q) + ro, dn.cq + rr, D, lane);
    dn_copy((dir > 0 ? ws.right_p : ws.left_p) + ro, p, D, lane);
    dn_copy((dir > 0 ? ws.right_g : ws.left_g) + ro, dn.cg + rr, D, lane);
    dn_copy((dir > 0 ? dn.right_v : dn.left_v) + ro, v, D, lane);
  } else {  // the next leaf's first half kick (integrators.py:235-239) and the operand planes of its velocity product
    __syncwarp();
    dn_kick(dn.cp + rr, dn.cg + rr, dn.ceps[r] * 0.5f, D, lane,
            p_planes ? p_planes + (size_t)r * 2 * plane_stride(D) : nullptr, p_unscale + r);
  }
  if (lane == 0) {
    dn.sub_weight[r] = sub_weight;
    dn.sub_slpa[r] = sub_slpa;
    if (take) {
      dn.sub_logp[r] = logp;
      dn.sub_energy[r] = e_new;
    }
    dn.cn[r] = i + 1;
    if (stop || i == last) {
      if (dir > 0) ws.right_logp[c] = logp; else ws.left_logp[c] = logp;
    }
    if (stop) dn.cdone[r] = is_div ? 1 : 2;
    // a sub-tree that diverges AND turns at the same leaf reports both (trajectory.py:340-371)
    if (stop && is_div && turning) dn.cdone[r] = 3;
  }
}

// end of doubling d (trajectory.py:672-717)
__global__ void k_dn_end(int n, int D, int d, int max_doublings, NutsWs ws, DnWs dn, const int* __restrict__ list,
                         int* __restrict__ list_out, int* __restrict__ counter_out, float* q_out, float* logp_out, float* g_out) {
  const int lane = threadIdx.x & 31, r = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (r >= n) return;
  const int c = list ? list[r] : r;
  const size_t ro = (size_t)c * D, rr = (size_t)r * D;
  const int done = dn.cdone[r];
  const bool sub_div = (done & 1) != 0, sub_term = (done & 2) != 0;
  const bool bad = sub_div || sub_term;
  const float sub_weight = dn.sub_weight[r];
  float prop_weight = ws.prop_weight[c];
  bool take2 = false;
  if (!bad) take2 = dn.u_prop[r] < clip_max1(expf(sub_weight - prop_weight));  // proposal.py:155-156
  if (take2) {
    dn_copy(q_out + ro, ws.sub_prop_q + ro, D, lane);
    dn_copy(g_out + ro, ws.sub_prop_g + ro, D, lane);
  }
  for (int k = lane; k < D / 4; k += 32) {  // merge_trajectories (trajectory.py:102-125)
    float4 a = reinterpret_cast<float4*>(ws.psum + ro)[k];
    const float4 b = reinterpret_cast<const float4*>(dn.cps + rr)[k];
    a.x = a.x + b.x; a.y = a.y + b.y; a.z = a.z + b.z; a.w = a.w + b.w;
    reinterpret_cast<float4*>(ws.psum + ro)[k] = a;
  }
  __syncwarp();
  const bool turning = dn_turning(ws.left_p + ro, dn.left_v + ro, ws.right_p + ro, dn.right_v + ro, ws.psum + ro, nullptr, nullptr,
                                  D, lane);                                        // :706-710
  const bool is_turn = sub_term || turning;                                        // :715
  const bool run_next = (d + 1 < max_doublings) && !sub_div && !is_turn;
  if (lane == 0) {
    if (!bad) prop_weight = logaddexp_f(prop_weight, sub_weight);
    ws.prop_weight[c] = prop_weight;
    ws.prop_slpa[c] = logaddexp_f(ws.prop_slpa[c], dn.sub_slpa[r]);
    ws.n_states[c] += dn.cn[r];
    ws.step[c] = d + 1;
    if (take2) {
      logp_out[c] = dn.sub_logp[r];
      ws.prop_energy[c] = dn.sub_energy[r];
    }
    ws.is_div[c] = sub_div;
    ws.is_turn[c] = is_turn;
    if (run_next) list_out[atomicAdd(counter_out, 1)] = c;
  }
}

static int dn_ws(bjx_handle_t h, DnWs& dn) {
  const size_t C = h->cfg.n_chains, D = h->cfg.dim, depth = h->cfg.max_tree_depth;
  const size_t row = ((C * D * sizeof(float)) + 255) & ~(size_t)255, vec = ((C * sizeof(float)) + 255) & ~(size_t)255;
  const size_t need = (7 + depth) * row + 12 * vec + 256;
  int rc = bjx_grow(h, h->dn_block, h->dn_bytes, need, 1);
  if (rc) return rc;
  char* b = (char*)h->dn_block;
  auto take = [&](size_t bytes) { char* r = b; b += bytes; return r; };
  dn.cq = (float*)take(row); dn.cp = (float*)take(row); dn.cg = (float*)take(row); dn.cv = (float*)take(row);
  dn.cps = (float*)take(row); dn.left_v = (float*)take(row); dn.right_v = (float*)take(row);
  dn.ck_v = (float*)take(depth * row);
  dn.ck_p = h->ws.ckpt_p;      // the warp kernels' checkpoint arrays ([C, depth, D] there, [depth][C, D] here: same size)
  dn.ck_s = h->ws.ckpt_sum;
  dn.clogp = (float*)take(vec); dn.ceps = (float*)take(vec); dn.sub_weight = (float*)take(vec); dn.sub_slpa = (float*)take(vec);
  dn.sub_logp = (float*)take(vec); dn.sub_energy = (float*)take(vec); dn.u_prop = (float*)take(vec);
  dn.cn = (int*)take(vec); dn.cdone = (int*)take(vec); dn.cdir = (int*)take(vec);
  dn.ctk = (uint32_t*)take(2 * vec);
  return 0;
}

}  // namespace bjx

using namespace bjx;

int bjx_dense_nuts_step(bjx_handle_t h, const uint32_t* keys, const float* q_in, const float* logp_in, const float* g_in,
                        float* q_out, float* logp_out, float* g_out, float step_size, const float* step_size_dev,
                        int max_num_doublings, InfoPtrs info, const float* momentum_override,
                        const uint32_t* key_integrator_override) {
  BJX_CUDA(cudaSetDevice(h->cfg.device));
  const int C = h->cfg.n_chains, D = h->cfg.dim;
  int rc = bjx_ensure_nuts_ws(h);
  if (rc) return rc;
  DenseWs w;
  rc = dense_ws(h, w);
  if (rc) return rc;
  DnWs dn;
  rc = dn_ws(h, dn);
  if (rc) return rc;
  NutsWs& ws = h->ws;
  cudaStream_t st = h->stream;
  const bool dense_m = (h->metric_kind == BJX_METRIC_DENSE);
  BJX_CUDA(cudaMemsetAsync(ws.counters, 0, 64 * sizeof(int), st));
  // momentum draw (nuts.py:136) and its velocity
  if (momentum_override) {
    BJX_CUDA(cudaMemcpyAsync(ws.left_p, momentum_override, (size_t)C * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
  } else {
    rc = dense_momentum(h, w, C, keys, ws.left_p, true);
    if (rc) return rc;
  }
  rc = dense_velocity(h, w, C, ws.left_p, dn.left_v);
  if (rc) return rc;
  k_dn_init<<<grow(C), kRowWarps * 32, 0, st>>>(C, D, ws, dn, keys, h->key_shared, h->chain_offset, key_integrator_override, q_in,
                                                logp_in, g_in, q_out, logp_out, g_out, info.momentum);
  BJX_CHECK_LAUNCH("k_dn_init");

  int n = C;
  const int* list = nullptr;
  int64_t launches = 0;
  for (int d = 0; d < max_num_doublings && n > 0; ++d) {
    uint16_t* planes = dense_m ? w.xs[PL_P] : nullptr;
    k_dn_begin<<<grow(n), kRowWarps * 32, 0, st>>>(n, D, d, ws, dn, list, step_size, step_size_dev, planes, w.unscale[PL_P]);
    BJX_CHECK_LAUNCH("k_dn_begin");
    const int leaves = 1 << d;
    for (int i = 0; i < leaves; ++i) {
      // half-step velocity, position update (integrators.py:199-203,242)
      rc = dense_velocity(h, w, n, dn.cp, w.v, dense_m);
      if (rc) return rc;
      k_rows_axpy<<<g4((long long)n * D / 4), 256, 0, st>>>(n, D, dn.cq, w.v, 0.f, dn.ceps, 1.0f);
      BJX_CHECK_LAUNCH("k_rows_axpy");
      // gradient, log density, second half kick (and the planes of the full-step momentum)
      rc = dense_grad(h, w, n, dn.cq, dn.cp, 0.f, dn.ceps, dn.cg, dn.clogp, 1, dense_m, false);
      if (rc) return rc;
      // full-step velocity: kinetic energy and the U-turn tests of this leaf
      rc = dense_velocity(h, w, n, dn.cp, dn.cv, dense_m);
      if (rc) return rc;
      k_dn_leaf<<<grow(n), kRowWarps * 32, 0, st>>>(n, D, i, leaves - 1, C, ws, dn, list, h->cfg.divergence_threshold, planes,
                                                    w.unscale[PL_P]);
      BJX_CHECK_LAUNCH("k_dn_leaf");
      ++launches;
    }
    int* list_out = (d & 1) ? ws.list_b : ws.list_a;
    k_dn_end<<<grow(n), kRowWarps * 32, 0, st>>>(n, D, d, max_num_doublings, ws, dn, list, list_out, ws.counters + 1 + d, q_out,
                                                 logp_out, g_out);
    BJX_CHECK_LAUNCH("k_dn_end");
    if (d + 1 < max_num_doublings) {  // the one host read per doubling: how many chains go on
      BJX_CUDA(cudaMemcpyAsync(h->h_flag, ws.counters + 1 + d, sizeof(int), cudaMemcpyDeviceToHost, st));
      BJX_CUDA(cudaStreamSynchronize(st));
      n = h->h_flag[0];
      list = list_out;
    }
  }
  k_nuts_finish<<<(C + 255) / 256, 256, 0, st>>>(C, ws, info);
  BJX_CHECK_LAUNCH("k_nuts_finish");
  h->last_leaf_launches = launches;
  h->last_depth = -1;
  return 0;
}
