// Evaluation recorder (Trainer.evaluate_trace): per-step trajectories of chosen slots (ic3_trace_step) and counts of
// where agents open their communication gate (ic3_comm_map_step), both read from the evaluation loop's one lock-step of
// scratch between policy step t and env step t.
#include <algorithm>

#include "ic3_common.cuh"

namespace {

// What both kernels need of the environment: where the positions and (traffic junction) the alive mask and routes live.
struct EvalEnv {
  int B, N, NA, rows, width, npos, pp;
  const int32_t* loc;        // [B, rows, 2]
  const uint8_t* alive;      // [B, N] traffic junction, NULL for predator-prey (every row is in the environment)
  const int32_t* route_id;   // [B, N] traffic junction
};

struct EvalArgs {
  EvalEnv env;
  ic3_eval_step_io io;
};

int eval_check(const ic3_eval_step_io* io, EvalEnv* env) {
  if (!io) return IC3_E_NULL;
  const bool pp = io->pp_env && io->pp_state, tj = io->tj_env && io->tj_state;
  if (pp == tj) return IC3_E_NULL;
  if (!io->t_ep || !io->halted || !io->action) return IC3_E_NULL;
  if (io->nheads < 1 || io->nheads > IC3_MAX_HEADS || io->logp_cols < io->nheads) return IC3_E_RANGE;
  if (io->max_steps < 1 || io->max_steps > 32767) return IC3_E_RANGE;
  if (io->comm_col >= io->logp_cols || io->comm_col < -1) return IC3_E_RANGE;
  if (pp) {
    const ic3_pp_cfg& c = *io->pp_env;
    if (!io->pp_state->loc) return IC3_E_NULL;
    if (c.B < 1 || c.N < 1 || c.N >= IC3_MAX_AGENTS || c.dim < 1 || c.dim > 181) return IC3_E_RANGE;
    *env = EvalEnv{c.B, c.N, ic3_pp_agents(c), c.N + 1, c.dim, c.dim * c.dim, 1, io->pp_state->loc, nullptr, nullptr};
  } else {
    const ic3_tj_cfg& c = *io->tj_env;
    if (!io->tj_state->loc || !io->tj_state->alive || !io->tj_state->route_id) return IC3_E_NULL;
    if (c.B < 1 || c.N < 1 || c.N > IC3_MAX_AGENTS || c.h < 1 || c.w < 1 || c.h > 32767 || c.w > 32767)
      return IC3_E_RANGE;
    *env = EvalEnv{c.B, c.N, c.N, c.N, c.w, c.h * c.w, 0, io->tj_state->loc, io->tj_state->alive,
                   io->tj_state->route_id};
  }
  return IC3_OK;
}

// One warp per recorded slot, lane = agent row / position row (both <= 32).
__global__ void __launch_bounds__(256) trace_step_kernel(EvalArgs a, ic3_eval_trace tr, int t) {
  const EvalEnv& v = a.env;
  const ic3_eval_step_io& io = a.io;
  const int k = (int)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)), lane = threadIdx.x & 31;
  if (k >= tr.K) return;
  const int e = tr.slots[k];
  if (e < 0 || e >= v.B) {
    if (lane == 0) atomicOr(io.err, IC3_ERR_TRACE_SLOT);
    return;
  }
  const int K = tr.K, NA = v.NA, nh = io.nheads;
  if (t < tr.T) {                                    // row t: the state entering step t and the policy's outputs
    const size_t row = (size_t)t * K + k;
    const bool ok = io.halted[e] == 0;
    if (lane < v.rows) {
      const int32_t* l = v.loc + ((size_t)e * v.rows + lane) * 2;
      tr.loc[(row * v.rows + lane) * 2] = ok ? (int16_t)l[0] : (int16_t)0;
      tr.loc[(row * v.rows + lane) * 2 + 1] = ok ? (int16_t)l[1] : (int16_t)0;
    }
    if (lane < NA) {
      const size_t a_ = (size_t)e * NA + lane, o = row * NA + lane;
      tr.alive[o] = ok ? (v.alive ? v.alive[a_] : (uint8_t)1) : (uint8_t)0;
      tr.value[o] = ok ? io.value[a_] : 0.f;
      for (int j = 0; j < nh; ++j) tr.action[o * nh + j] = ok ? (int8_t)io.action[a_ * nh + j] : (int8_t)0;
      if (tr.comm_prob) tr.comm_prob[o] = ok ? expf(io.logp[a_ * io.logp_cols + io.comm_col]) : 0.f;
      if (tr.route_id) tr.route_id[o] = ok ? (int16_t)v.route_id[a_] : (int16_t)0;
    }
    if (lane == 0) {
      tr.t_ep[row] = ok ? (int16_t)io.t_ep[e] : (int16_t)0;
      tr.valid[row] = ok ? 1 : 0;
    }
  }
  if (t > 0) {                                       // row t - 1: what env step t - 1 did
    const size_t row = (size_t)(t - 1) * K + k;
    const bool ok = tr.valid[row] != 0;              // written by the previous call
    if (lane < v.rows) {
      const int32_t* l = io.out_loc + ((size_t)e * v.rows + lane) * 2;
      tr.loc_next[(row * v.rows + lane) * 2] = ok ? (int16_t)l[0] : (int16_t)0;
      tr.loc_next[(row * v.rows + lane) * 2 + 1] = ok ? (int16_t)l[1] : (int16_t)0;
    }
    if (lane < NA) tr.reward[row * NA + lane] = ok ? io.reward[(size_t)e * NA + lane] : 0.f;
    if (lane == 0) {
      tr.done[row] = ok ? io.fresh[e] : (uint8_t)0;
      tr.success[row] = ok ? io.out_success[e] : (uint8_t)0;
    }
  }
}

// One thread per agent row; counts are privatised per CTA (PRIV: 32-bit shared counters, added to the global 64-bit
// ones at the end; otherwise straight global atomics for maps too large for shared memory).
template <bool PRIV>
__global__ void __launch_bounds__(256) comm_map_kernel(EvalArgs a, unsigned long long* __restrict__ counts, int ncount) {
  extern __shared__ uint32_t s_cnt[];
  const EvalEnv& v = a.env;
  const ic3_eval_step_io& io = a.io;
  const bool gate = io.comm_col >= 0;
  const int S = io.max_steps, P = v.npos;
  // block offsets of the layout documented in the header
  const int o_open = P, o_vt = gate ? 2 * P : P, o_ot = o_vt + S, o_vr = gate ? o_vt + 2 * S : o_vt + S, o_or = o_vr + 2;
  if (PRIV) {
    for (int i = threadIdx.x; i < ncount; i += blockDim.x) s_cnt[i] = 0;
    __syncthreads();
  }
  auto add = [&](int idx) {
    if (PRIV) atomicAdd(&s_cnt[idx], 1u);
    else atomicAdd(&counts[idx], 1ull);
  };
  const int nf = v.pp ? v.N : v.NA;                  // friendly rows: the predators / every car
  const long long R = (long long)v.B * v.NA;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(r / v.NA), i = (int)(r - (long long)e * v.NA);
    if (i >= nf || io.halted[e]) continue;
    if (v.alive && !v.alive[(size_t)e * v.N + i]) continue;
    const int32_t* l = v.loc + ((size_t)e * v.rows + i) * 2;
    const int cell = l[0] * v.width + l[1];
    const int te = io.t_ep[e];
    const bool open = gate && io.action[(size_t)r * io.nheads + io.nheads - 1] != 0;
    if (cell >= 0 && cell < P) {
      add(cell);
      if (open) add(o_open + cell);
    }
    if (te >= 0 && te < S) {
      add(o_vt + te);
      if (open) add(o_ot + te);
    }
    if (v.pp) {
      const int32_t* q = v.loc + ((size_t)e * v.rows + v.N) * 2;
      const int on = (l[0] == q[0] && l[1] == q[1]) ? 1 : 0;
      add(o_vr + on);
      if (open) add(o_or + on);
    }
  }
  if (PRIV) {
    __syncthreads();
    for (int i = threadIdx.x; i < ncount; i += blockDim.x)
      if (s_cnt[i]) atomicAdd(&counts[i], (unsigned long long)s_cnt[i]);
  }
}

constexpr int kMapCtas = 264;                        // 2 per SM of an H100 SXM: few global flushes, every SM busy
constexpr size_t kMapSmemMax = 96 * 1024;

}  // namespace

extern "C" int ic3_trace_step(const ic3_eval_step_io* io, const ic3_eval_trace* tr, int32_t t, void* stream) {
  EvalArgs a;
  int rc = eval_check(io, &a.env);
  if (rc) return rc;
  if (!tr || !io->err || !tr->slots || !tr->loc || !tr->loc_next || !tr->alive || !tr->action || !tr->value ||
      !tr->reward || !tr->t_ep || !tr->done || !tr->success || !tr->valid)
    return IC3_E_NULL;
  if (!io->value || !io->reward || !io->fresh || !io->out_loc || !io->out_success) return IC3_E_NULL;
  if (io->comm_col >= 0 && (!io->logp || !tr->comm_prob)) return IC3_E_NULL;
  if (io->comm_col < 0 && tr->comm_prob) return IC3_E_ARG;
  if (a.env.pp ? tr->route_id != nullptr : !tr->route_id) return a.env.pp ? IC3_E_ARG : IC3_E_NULL;
  if (tr->T < 1 || tr->K < 1 || t < 0 || t > tr->T) return IC3_E_RANGE;
  a.io = *io;
  const int per = 256 / 32;
  trace_step_kernel<<<(tr->K + per - 1) / per, 256, 0, (cudaStream_t)stream>>>(a, *tr, t);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

extern "C" int ic3_comm_map_step(const ic3_eval_step_io* io, uint64_t* counts, void* stream) {
  EvalArgs a;
  int rc = eval_check(io, &a.env);
  if (rc) return rc;
  if (!counts) return IC3_E_NULL;
  a.io = *io;
  const bool gate = io->comm_col >= 0;
  const int ncount = (gate ? 2 : 1) * (a.env.npos + io->max_steps) + (a.env.pp ? (gate ? 4 : 2) : 0);
  const long long R = (long long)a.env.B * a.env.NA;
  const int grid = (int)std::min<long long>((R + 255) / 256, kMapCtas);
  const size_t smem = (size_t)ncount * sizeof(uint32_t);
  unsigned long long* c = reinterpret_cast<unsigned long long*>(counts);
  cudaStream_t s = (cudaStream_t)stream;
  if (smem <= kMapSmemMax) {
    if (smem > 48 * 1024) {
      const cudaError_t e = cudaFuncSetAttribute(comm_map_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 (int)kMapSmemMax);
      if (e != cudaSuccess) return (int)e;
    }
    comm_map_kernel<true><<<grid, 256, smem, s>>>(a, c, ncount);
  } else {
    comm_map_kernel<false><<<grid, 256, 0, s>>>(a, c, ncount);
  }
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}
