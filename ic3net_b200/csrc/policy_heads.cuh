// Value / action heads, log-softmax and inverse-CDF sampling for one agent row, executed by
// one warp (reference: comm.py:228-239, action_utils.py:32-36).  Shared by the fp32 SIMT
// policy kernel (policy.cu), the tensor-core policy path (policy_tc.cu) and the Random policy
// step (random_policy.cu).
#pragma once
#include "ic3_common.cuh"

// log-softmax + inverse-CDF sampling of one head; logits live one per lane
// (lane off+a holds logit a).  Every lane of the warp executes this.
__device__ __forceinline__ void head_logp_sample(float mylogit, int off, int na, float u, bool do_sample,
                                                 float& mylogp, int& action) {
  float m = -INFINITY;
  for (int a = 0; a < na; ++a) m = fmaxf(m, __shfl_sync(IC3_FULL_MASK, mylogit, off + a));
  float s = 0.f;
  for (int a = 0; a < na; ++a) s += expf(__shfl_sync(IC3_FULL_MASK, mylogit, off + a) - m);
  const float lse = m + logf(s);
  mylogp = mylogit - lse;
  action = na - 1;
  if (do_sample) {
    float cdf = 0.f;
    bool found = false;
    for (int a = 0; a < na; ++a) {
      cdf += expf(__shfl_sync(IC3_FULL_MASK, mylogp, off + a));
      if (!found && cdf > u) {
        action = a;
        found = true;
      }
    }
  }
}

// hv[m] = h'[row][lane + 32*m].  grow = global agent row, e = env, i = agent in env.
template <int H>
__device__ __forceinline__ void heads_for_row(const ic3_policy_cfg& cfg, const float* __restrict__ head_w,
                                              const float* __restrict__ head_b, const float (&hv)[H / 32],
                                              size_t grow, int e, int i, int lane, const uint32_t* tick,
                                              const uint32_t* draws, float* __restrict__ value,
                                              float* __restrict__ logp, int32_t* __restrict__ action) {
  int atot = 0;
  for (int k = 0; k < cfg.nheads; ++k) atot += cfg.head_dim[k];
  const int nout = 1 + atot;
  float mylogit = 0.f;
  for (int o = 0; o < nout; ++o) {
    float part = 0.f;
#pragma unroll
    for (int m = 0; m < H / 32; ++m) part = fmaf(hv[m], __ldg(head_w + (size_t)o * H + lane + 32 * m), part);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) part += __shfl_xor_sync(IC3_FULL_MASK, part, s);
    if (lane == o) mylogit = part + __ldg(head_b + o);
  }
  if (lane == 0) value[grow] = mylogit;
  uint4 w = make_uint4(0, 0, 0, 0);
  const bool do_sample = action != nullptr;
  if (do_sample && !draws)
    w = ic3_draw24(cfg.seed, cfg.env_id0 + (uint32_t)e, tick ? tick[e] : 0u, IC3_STREAM_ACTION, (uint32_t)i);
  int off = 1;
  for (int k = 0; k < cfg.nheads; ++k) {
    const int na = cfg.head_dim[k];
    uint32_t u24 = 0;
    if (do_sample) u24 = draws ? draws[grow * cfg.nheads + k] : ic3_word(w, k);
    float mylogp;
    int act;
    head_logp_sample(mylogit, off, na, (float)u24 * 5.9604644775390625e-08f, do_sample, mylogp, act);
    if (lane >= off && lane < off + na) logp[grow * atot + (off - 1) + (lane - off)] = mylogp;
    if (do_sample && lane == 0) action[grow * cfg.nheads + k] = act;
    off += na;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Finishing the heads from the per-slot partial logits of the tensor-core LSTM epilogue (fixed summation order ->
// deterministic): value, log-softmax per head, inverse-CDF sampling of ONE agent row by ONE thread.  Used by
// heads_finish_kernel (policy_tc).
// ---------------------------------------------------------------------------------------------------------------
constexpr int IC3_HEAD_PAD = 8;    // outputs (value + action logits) the fused epilogue supports
constexpr int IC3_HEAD_NSLOT = 8;  // partial-logit slots per row

struct HeadsFinish {
  const float* partial;   // [R][IC3_HEAD_NSLOT][IC3_HEAD_PAD]
  const float* head_b;    // [1 + sum(na)]
  int nheads;
  int head_dim[IC3_MAX_HEADS];
  uint64_t seed;
  uint32_t env_id0;
  const uint32_t* tick;   // [B] or NULL
  const uint32_t* draws;  // [R, nheads] or NULL
  float* value;           // [R]
  float* logp;            // [R, sum(na)]
  int32_t* action;        // [R, nheads] or NULL (no sampling)
};

// Log-softmax per head and inverse-CDF sampling of ONE agent row by ONE thread (action_utils.py:32-36): logit[1 + j] is
// action logit j, heads concatenated (logit[0], the value, is not read), 1 + atot <= IC3_HEAD_PAD.  Head k samples with
// word k of the action stream (env_id0 + e, tick[e], IC3_STREAM_ACTION, i) or draws[row, k]; action == NULL: no
// sampling.  Shared by the tensor-core heads (heads_finish_row) and the Random policy step (random_policy.cu).
__device__ __forceinline__ void heads_logp_sample_row(const float (&logit)[IC3_HEAD_PAD], int nheads,
                                                      const int* head_dim, int atot, uint64_t seed, uint32_t env_id0,
                                                      const uint32_t* tick, const uint32_t* draws, long row, int e,
                                                      int i, float* logp, int32_t* action) {
  const bool do_sample = action != nullptr;
  uint4 d24 = make_uint4(0, 0, 0, 0);
  if (do_sample && !draws)
    d24 = ic3_draw24(seed, env_id0 + (uint32_t)e, tick ? tick[e] : 0u, IC3_STREAM_ACTION, (uint32_t)i);
  int off = 1;
  for (int k = 0; k < nheads; ++k) {
    const int na = head_dim[k];
    float m = -INFINITY;
#pragma unroll
    for (int o = 1; o < IC3_HEAD_PAD; ++o)
      if (o >= off && o < off + na) m = fmaxf(m, logit[o]);
    float ssum = 0.f;
#pragma unroll
    for (int o = 1; o < IC3_HEAD_PAD; ++o)
      if (o >= off && o < off + na) ssum += expf(logit[o] - m);
    const float lse = m + logf(ssum);
    uint32_t u24 = 0;
    if (do_sample) u24 = draws ? draws[(size_t)row * nheads + k] : ic3_word(d24, k);
    const float u = (float)u24 * 5.9604644775390625e-08f;
    float cdf = 0.f;
    int act = na - 1;
    bool found = false;
#pragma unroll
    for (int o = 1; o < IC3_HEAD_PAD; ++o) {
      if (o >= off && o < off + na) {
        const float lp = logit[o] - lse;
        logp[(size_t)row * atot + (o - 1)] = lp;
        cdf += expf(lp);
        if (!found && cdf > u) {
          act = o - off;
          found = true;
        }
      }
    }
    if (do_sample) action[(size_t)row * nheads + k] = act;
    off += na;
  }
}

__device__ __forceinline__ void heads_finish_row(const HeadsFinish& f, long row, int e, int i) {
  float logit[IC3_HEAD_PAD];
  const float4* p4 = reinterpret_cast<const float4*>(f.partial + (size_t)row * IC3_HEAD_NSLOT * IC3_HEAD_PAD);
  {
    float4 a = p4[0], b = p4[1];
#pragma unroll
    for (int sl = 1; sl < IC3_HEAD_NSLOT; ++sl) {
      const float4 c = p4[2 * sl], d = p4[2 * sl + 1];
      a.x += c.x; a.y += c.y; a.z += c.z; a.w += c.w;
      b.x += d.x; b.y += d.y; b.z += d.z; b.w += d.w;
    }
    logit[0] = a.x; logit[1] = a.y; logit[2] = a.z; logit[3] = a.w;
    logit[4] = b.x; logit[5] = b.y; logit[6] = b.z; logit[7] = b.w;
  }
  int atot = 0;
  for (int k = 0; k < f.nheads; ++k) atot += f.head_dim[k];
#pragma unroll
  for (int o = 0; o < IC3_HEAD_PAD; ++o) logit[o] += (o < 1 + atot) ? __ldg(f.head_b + o) : 0.f;
  f.value[row] = logit[0];
  heads_logp_sample_row(logit, f.nheads, f.head_dim, atot, f.seed, f.env_id0, f.tick, f.draws, row, e, i, f.logp,
                        f.action);
}
