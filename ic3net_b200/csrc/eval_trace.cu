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

// ---- messages (ic3_trace_comm_step / ic3_message_map_step) -------------------------------------------------------

struct CommArgs {
  EvalEnv env;
  ic3_eval_step_io io;
  ic3_eval_comm_io cm;
};

int comm_check(const ic3_eval_step_io* io, const ic3_eval_comm_io* cm, CommArgs* a) {
  int rc = eval_check(io, &a->env);
  if (rc) return rc;
  if (!cm || !cm->h || !cm->alive || !cm->fresh || (cm->hard && !cm->comm)) return IC3_E_NULL;
  if (cm->H < 16 || cm->H > 1024 || cm->H % 16) return IC3_E_RANGE;
  if (cm->comm_avg < 0 || cm->comm_avg > 1 || cm->hard < 0 || cm->hard > 1) return IC3_E_RANGE;
  a->io = *io;
  a->cm = *cm;
  return IC3_OK;
}

// The gates of one slot, computed by a whole warp (lane j reads row j): bit j of g = g_j, of live = the row's message
// is its h (alive and not fresh); den = S's divisor.
struct SlotGates {
  uint32_t g, live;
  double den;
};

__device__ __forceinline__ SlotGates slot_gates(const ic3_eval_comm_io& cm, int e, int NA, int lane) {
  const bool fr = cm.fresh[e] != 0;
  bool al = false, cmj = false;
  if (lane < NA) {
    al = fr || cm.alive[(size_t)e * NA + lane] != 0;
    cmj = cm.hard ? (!fr && cm.comm[(size_t)e * NA + lane] != 0) : true;
  }
  const uint32_t alive = __ballot_sync(0xffffffffu, al), g = __ballot_sync(0xffffffffu, al && cmj);
  const int n_alive = __popc(alive);
  return SlotGates{g, fr ? 0u : alive, (cm.comm_avg && n_alive > 1) ? (double)(n_alive - 1) : 1.0};
}

// The messages of one column: m[j] = h_j for a live row, else 0 (all loads issued together); returns
// sum_j g_j m_j in float64, in agent order.
__device__ __forceinline__ double load_messages(const ic3_eval_comm_io& cm, const SlotGates& s, int e, int NA, int col,
                                                float (&m)[IC3_MAX_AGENTS]) {
#pragma unroll
  for (int j = 0; j < IC3_MAX_AGENTS; ++j)
    m[j] = (j < NA && (s.live >> j & 1u)) ? cm.h[((size_t)e * NA + j) * cm.H + col] : 0.f;
  double tot = 0.0;
#pragma unroll
  for (int j = 0; j < IC3_MAX_AGENTS; ++j)
    if (j < NA && (s.g >> j & 1u)) tot += (double)m[j];
  return tot;
}

// S_k of one column from the column's gated sum
__device__ __forceinline__ float received(const SlotGates& s, int k, double tot, float mk) {
  return (s.g >> k & 1u) ? (float)((tot - (double)mk) / s.den) : 0.f;
}

// One CTA of 128 threads per recorded slot, thread = column.
__global__ void __launch_bounds__(128) trace_comm_kernel(CommArgs a, ic3_eval_trace tr, float* __restrict__ msg_h,
                                                         uint8_t* __restrict__ msg_gate, float* __restrict__ msg_in,
                                                         int t) {
  const EvalEnv& v = a.env;
  const ic3_eval_comm_io& cm = a.cm;
  const int k = blockIdx.x, NA = v.NA, H = cm.H, lane = threadIdx.x & 31;
  const int e = tr.slots[k];
  if (e < 0 || e >= v.B) {
    if (threadIdx.x == 0) atomicOr(a.io.err, IC3_ERR_TRACE_SLOT);
    return;
  }
  const size_t row = ((size_t)t * tr.K + k) * NA;
  const bool ok = a.io.halted[e] == 0;
  const SlotGates s = ok ? slot_gates(cm, e, NA, lane) : SlotGates{0u, 0u, 1.0};
  for (int j = threadIdx.x; j < NA; j += blockDim.x) msg_gate[row + j] = (uint8_t)(s.g >> j & 1u);
  for (int col = threadIdx.x; col < H; col += blockDim.x) {
    float m[IC3_MAX_AGENTS];
    const double tot = load_messages(cm, s, e, NA, col, m);
#pragma unroll
    for (int j = 0; j < IC3_MAX_AGENTS; ++j) {
      if (j >= NA) break;
      msg_h[(row + j) * H + col] = m[j];
      msg_in[(row + j) * H + col] = received(s, j, tot, m[j]);
    }
  }
}

__device__ __forceinline__ long long fixed32(float v) { return llrintf(v * 4294967296.f); }

// Warp per slot, CTA y owns columns [16y, 16y + 16): lanes 0-15 add the sent messages of those columns, lanes 16-31
// the received ones, so each h element is loaded by one warp once; lane i first reads row i's keys, which the row loop
// takes by shuffle.  PRIV: the CTA's [R][32] slice (and, for y == 0, the senders counts) is summed in shared memory and
// flushed once with global atomics; otherwise global atomics.
template <bool PRIV>
__global__ void __launch_bounds__(1024) message_map_kernel(CommArgs a, unsigned long long* __restrict__ sums, int R) {
  extern __shared__ unsigned long long s_sum[];      // [R][32], then senders [R]
  const EvalEnv& v = a.env;
  const ic3_eval_step_io& io = a.io;
  const ic3_eval_comm_io& cm = a.cm;
  const int H = cm.H, NA = v.NA, S = io.max_steps, P = v.npos;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int role = lane >> 4, col = blockIdx.y * 16 + (lane & 15);
  const bool counts = blockIdx.y == 0 && lane == 0;
  const int nsh = R * 32 + (blockIdx.y == 0 ? R : 0);
  unsigned long long* g_blk = sums + (size_t)role * R * H + col;     // [R, H] block of this lane, at its column
  unsigned long long* g_cnt = sums + (size_t)2 * R * H;
  if (PRIV) {
    for (int i = threadIdx.x; i < nsh; i += blockDim.x) s_sum[i] = 0ull;
    __syncthreads();
  }
  auto add = [&](int key, long long val) {
    if (!val) return;
    if (PRIV) atomicAdd(&s_sum[key * 32 + lane], (unsigned long long)val);
    else atomicAdd(&g_blk[(size_t)key * H], (unsigned long long)val);
  };
  auto count = [&](int key) {
    if (PRIV) atomicAdd(&s_sum[R * 32 + key], 1ull);
    else atomicAdd(&g_cnt[key], 1ull);
  };
  const int nf = v.pp ? v.N : NA;
  for (int e = blockIdx.x * nwarp + warp; e < v.B; e += gridDim.x * nwarp) {
    if (io.halted[e]) continue;                      // warp-uniform
    const SlotGates s = slot_gates(cm, e, NA, lane);
    float m[IC3_MAX_AGENTS];
    const double tot = load_messages(cm, s, e, NA, col, m);
    // row `lane`'s keys: cell (or -1), prey flag (or -1); -2 = not counted
    int my_cell = -2, my_on = -1;
    if (lane < nf && (!v.alive || v.alive[(size_t)e * v.N + lane])) {
      const int32_t* l = v.loc + ((size_t)e * v.rows + lane) * 2;
      const int c = l[0] * v.width + l[1];
      my_cell = (c >= 0 && c < P) ? c : -1;
      if (v.pp) {
        const int32_t* q = v.loc + ((size_t)e * v.rows + v.N) * 2;
        my_on = (l[0] == q[0] && l[1] == q[1]) ? 1 : 0;
      }
    }
    const int te = io.t_ep[e];
    const bool in_t = te >= 0 && te < S;
#pragma unroll
    for (int i = 0; i < IC3_MAX_AGENTS; ++i) {
      if (i >= nf) break;
      const int cell = __shfl_sync(0xffffffffu, my_cell, i), on = __shfl_sync(0xffffffffu, my_on, i);
      if (cell == -2) continue;
      const bool open = s.g >> i & 1u;
      if (role == 0 && !open) continue;
      const long long val = fixed32(role == 0 ? m[i] : received(s, i, tot, m[i]));
      if (cell >= 0) add(cell, val);
      if (in_t) add(P + te, val);
      if (on >= 0) add(P + S + on, val);
      if (counts && open) {
        if (cell >= 0) count(cell);
        if (in_t) count(P + te);
        if (on >= 0) count(P + S + on);
      }
    }
  }
  if (PRIV) {
    __syncthreads();
    for (int i = threadIdx.x; i < R * 32; i += blockDim.x) {
      const unsigned long long val = s_sum[i];
      const int l = i & 31;
      if (val) atomicAdd(&sums[(size_t)(l >> 4) * R * H + (size_t)(i >> 5) * H + blockIdx.y * 16 + (l & 15)], val);
    }
    if (blockIdx.y == 0)
      for (int i = threadIdx.x; i < R; i += blockDim.x)
        if (s_sum[R * 32 + i]) atomicAdd(&g_cnt[i], s_sum[R * 32 + i]);
  }
}

constexpr int kMsgCtas = 132;                        // one 1024-thread CTA per SM of an H100 SXM
constexpr int kMsgThreads = 1024;
constexpr size_t kMsgSmemMax = 200 * 1024;

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

extern "C" int ic3_trace_comm_step(const ic3_eval_step_io* io, const ic3_eval_comm_io* cm, const ic3_eval_trace* tr,
                                   float* msg_h, uint8_t* msg_gate, float* msg_in, int32_t t, void* stream) {
  CommArgs a;
  int rc = comm_check(io, cm, &a);
  if (rc) return rc;
  if (!tr || !tr->slots || !io->err || !msg_h || !msg_gate || !msg_in) return IC3_E_NULL;
  if (tr->T < 1 || tr->K < 1 || t < 0 || t >= tr->T) return IC3_E_RANGE;
  trace_comm_kernel<<<tr->K, 128, 0, (cudaStream_t)stream>>>(a, *tr, msg_h, msg_gate, msg_in, t);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

extern "C" int ic3_message_map_step(const ic3_eval_step_io* io, const ic3_eval_comm_io* cm, int64_t* sums,
                                    void* stream) {
  CommArgs a;
  int rc = comm_check(io, cm, &a);
  if (rc) return rc;
  if (!sums) return IC3_E_NULL;
  const int R = a.env.npos + io->max_steps + (a.env.pp ? 2 : 0);
  const int ny = cm->H / 16;
  const int nx = (int)std::max<long long>(1, std::min<long long>((a.env.B + 31) / 32, std::max(1, kMsgCtas / ny)));
  const dim3 grid(nx, ny);
  const size_t smem = (size_t)R * 33 * sizeof(unsigned long long);
  unsigned long long* s_ = reinterpret_cast<unsigned long long*>(sums);
  cudaStream_t s = (cudaStream_t)stream;
  if (smem <= kMsgSmemMax) {
    if (smem > 48 * 1024) {
      const cudaError_t e = cudaFuncSetAttribute(message_map_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 (int)kMsgSmemMax);
      if (e != cudaSuccess) return (int)e;
    }
    message_map_kernel<true><<<grid, kMsgThreads, smem, s>>>(a, s_, R);
  } else {
    message_map_kernel<false><<<grid, kMsgThreads, 0, s>>>(a, s_, R);
  }
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}
