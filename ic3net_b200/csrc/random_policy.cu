// models.Random (reference models.py:45-56) + select_action (action_utils.py:32-36) for a batch of environments: one
// thread per agent row draws the value and the action logits from Philox stream 4, takes the log-softmax of each head
// and samples the actions from the action stream with the policy kernels' own code (policy_heads.cuh).
#include "policy_heads.cuh"

namespace {

constexpr float kTwoM24 = 5.9604644775390625e-08f;   // 2^-24
constexpr float kTwoM23 = 1.1920928955078125e-07f;   // 2^-23

// cfg is a __grid_constant__: heads_logp_sample_row reads head_dim through a pointer, which would otherwise copy the
// whole struct to the stack
__global__ void __launch_bounds__(128) random_policy_kernel(const __grid_constant__ ic3_policy_cfg cfg,
                                                            const uint32_t* __restrict__ tick,
                                                            const uint32_t* __restrict__ random_draws,
                                                            const uint32_t* __restrict__ draws,
                                                            float* __restrict__ value, float* __restrict__ logp,
                                                            int32_t* __restrict__ action) {
  const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= (long)cfg.B * cfg.N) return;
  const int e = (int)(row / cfg.N), i = (int)(row - (long)e * cfg.N);
  int atot = 0;
  for (int k = 0; k < cfg.nheads; ++k) atot += cfg.head_dim[k];
  const int nblk = (2 * atot + 4) / 4;              // blocks holding words 0 .. 2 atot
  const uint32_t tk = tick ? tick[e] : 0u;
  uint32_t u[IC3_RANDOM_WORDS];
#pragma unroll
  for (int b = 0; b < IC3_RANDOM_WORDS / 4; ++b) {
    uint4 w = make_uint4(0, 0, 0, 0);
    if (b < nblk) {
      if (random_draws) {
        const uint32_t* p = random_draws + (size_t)row * IC3_RANDOM_WORDS + 4 * b;
        w = make_uint4(p[0] & 0xFFFFFFu, p[1] & 0xFFFFFFu, p[2] & 0xFFFFFFu, p[3] & 0xFFFFFFu);
      } else {
        w = ic3_draw24(cfg.seed, cfg.env_id0 + (uint32_t)e, tk, IC3_STREAM_RANDOM_POLICY, 4u * (uint32_t)i + b);
      }
    }
    u[4 * b] = w.x;
    u[4 * b + 1] = w.y;
    u[4 * b + 2] = w.z;
    u[4 * b + 3] = w.w;
  }
  value[row] = (float)u[0] * kTwoM24;               // torch.rand: a 24-bit uniform, exact in fp32
  // torch.randn per head: Box-Muller on (0, 1] x [0, 1).  (u + 1) 2^-24 and the cospi argument 2 u 2^-24 are exact,
  // and logf / sqrtf / cospif are the accurate library functions, so each logit is within a few ulp of the float64
  // value (cosf(2 pi u) would add the rounding of its argument, up to 2.4e-7 absolute, times |r| <= 5.8).
  float logit[IC3_HEAD_PAD];
  logit[0] = 0.f;
#pragma unroll
  for (int j = 0; j < IC3_HEAD_PAD - 1; ++j) {
    float z = 0.f;
    if (j < atot) {
      const float r = sqrtf(-2.f * logf((float)(u[1 + 2 * j] + 1u) * kTwoM24));
      z = r * cospif((float)u[2 + 2 * j] * kTwoM23);
    }
    logit[1 + j] = z;
  }
  heads_logp_sample_row(logit, cfg.nheads, cfg.head_dim, atot, cfg.seed, cfg.env_id0, tick, draws, row, e, i, logp,
                        action, false);
}

}  // namespace

extern "C" int ic3_random_policy_step(const ic3_policy_cfg* cfg, const ic3_policy_io* io, const uint32_t* random_draws,
                                      void* stream) {
  if (!cfg || !io) return IC3_E_NULL;
  if (cfg->greedy) return IC3_E_ARG;                 // an argmax over the uniform policy's logits means nothing
  if (cfg->B <= 0 || cfg->N <= 0 || cfg->N > IC3_MAX_AGENTS) return IC3_E_RANGE;
  if (cfg->nheads < 1 || cfg->nheads > IC3_MAX_HEADS) return IC3_E_RANGE;
  int tot = 1;
  for (int k = 0; k < cfg->nheads; ++k) {
    if (cfg->head_dim[k] < 1 || cfg->head_dim[k] > IC3_MAX_HEAD_DIM) return IC3_E_RANGE;
    tot += cfg->head_dim[k];
  }
  if (tot > IC3_HEAD_PAD) return IC3_E_RANGE;       // value + logits of one row in registers
  if (!io->value || !io->logp) return IC3_E_NULL;
  const long rows = (long)cfg->B * cfg->N;
  random_policy_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      *cfg, io->tick, random_draws, io->draws, io->value, io->logp, io->action);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}
