// Back-propagation through time of the rollout loss (Trainer.compute_grad, reference trainer.py:128-225) as
// hand-written sm_90a kernels (H = 128).  One call of ic3_bptt_step differentiates ONE lock-step iteration t of
// the recorded rollout for all env slots; the host walks t = T-1 .. 0.  With comm_passes P > 1 a step is P backward
// units (t, P-1) .. (t, 0), each the chain below on its pass's weight image (heads on the last pass only), after the
// states entering passes 1 .. P-1 have been re-run from the record (ic3_tc_pass_states).  Per unit:
//
//   heads      d(loss)/d(value, logits) from the records (advantages, log-probs, actions, masks), the value /
//              action-head weight gradients, the three loss sums                               [bptt_heads_kernel]
//   scale      power-of-two scale of this step's gate gradients for the fp16 hi/lo operand split [bptt_scale_kernel]
//   prep       [x | S | h_{t-1}] operand image (the forward's own kernel, fed from the records) + the sparse
//              observation pattern P + the comm gate factors                                    [prep_kernel<.., BWD>]
//   gates      wgmma: gate pre-activations re-computed exactly like the forward (K = 384), LSTM cell backward in
//              the epilogue -> d gates (fp16 hi/lo image), d c_{t-1}                            [bptt_gates_kernel]
//   dgrad      wgmma: [dS | dh] = d gates . [W_ih C | W_hh]   (K = 512, N = 256)              [bptt_dgrad_kernel]
//   comm       backward of the gated hidden-state mean + episode-start / detach cuts -> d h_{t-1} [bptt_comm_kernel]
//   wgrad      wgmma: G += (d gates)^T . [x | S | h | P]  -- both operands MN-major views of the images the other
//              kernels already wrote, contraction over the agent rows; per-role accumulators    [bptt_wgrad_kernel]
//
// After the last step ic3_bptt_finish folds G into the parameter gradients (float64):
//   dW_hh = G_h,  dW_ih = G_x + G_S C^T + g1 c_b^T,  db_ih = db_hh = g1,  dC = W_ih^T G_S,  dc_b = W_ih^T g1,
//   d encoder = W_ih^T (d gates)^T P scattered back through the observation layout (one-hot class per window cell
//   of the agent position, count / scalar features), with g1 = column of ones of P.
//
// The tanh recurrence without communication (models.RNN with rnn_type 'MLP': the IC / IRIC baselines, run by the SIMT
// policy kernel), h' = tanh(z), z = affine1(obs) + affine2(h), is the same chain with one 128-column "gate" block:
//   tanh       dz = (dh + W_heads^T dout) (1 - h'^2), h' from the record -> dz image (no GEMM)     [bptt_tanh_kernel]
//   dgrad      dh_{t-1} = dz . W_f (K = 128)                                                      [bptt_dgrad_kernel<4>]
//   comm       the episode-start cut only (no_comm)                                               [bptt_comm_kernel]
//   wgrad      G += dz^T . [h | P]  (slice 0 narrowed to the h block of the operand image)          [bptt_wgrad_kernel]
// and ic3_bptt_finish folds  d affine2.weight = G_h,  d affine2.bias = d affine1.bias = g1,  d affine1.weight = dz^T P
// scattered through the observation layout (the fold above with W_ih^T replaced by the identity).
//
// Arithmetic of the three GEMMs: the forward's fp16 hi/lo split (3 MMAs, fp32 accumulate).  d gates of a step are
// scaled by a power of two s_t chosen from an upper bound of their magnitude (so hi stays below 2^14 and lo keeps
// 2^-35 of the step's largest element); products are unscaled when they leave the accumulator registers.
#include <cuda.h>

#include "ff_grad_tc.h"
#include "policy_tc_kernels.cuh"

namespace {

constexpr int BP_HEADS = HEAD_PAD;                 // value + action logits handled by the fused heads backward (<= 8)
constexpr int DG_TILE_HALFS = 2 * 64 * 16 * 64;    // d gates image per tile: [hi, lo][cg 64][rg 16][8][8]
constexpr int DG_PART_HALFS = 64 * 16 * 64;
constexpr int WG_MAX_NP = 512;                     // columns of P the weight-gradient kernel can hold (4 warpgroups x 128 in registers)

struct BpttScalars {      // device-resident scalars of the recursion
  unsigned dhmax;         // bits of max |dh| entering the next step to be processed (atomicMax on non-negative floats)
  unsigned dcmax;
  unsigned hbound[2];     // bound of the heads' contribution to |dh| of step t, slot t & 1 (heads of step t - 1 run early)
  float cmax;             // max |c| over the whole record (set by the host once per compute_grad)
  float scale[2];         // s_t, indexed by t & 1: the weight-gradient kernel of step t runs on a side stream while
  float inv_scale[2];     // 1 / s_t          the main stream already prepares step t - 1
};

// ------------------------------------------------------------------------------------------------------------------
// heads: d loss / d outputs of step t  (trainer.py:176-220, utils.py:42-46)
// ------------------------------------------------------------------------------------------------------------------
struct HeadsArgs {
  int R, N, nheads, atot;
  int head_dim[IC3_MAX_HEADS];
  float value_coeff, entr;
  const float* logp;          // [R, atot]
  const int32_t* action;      // [R, nheads]
  const float* value;         // [R]
  const float* ret;           // [R]
  const float* adv;           // [R]
  const uint8_t* alive_post;  // [R]
  const uint8_t* valid;       // [B] or NULL
  const float* h_new;         // [R, H] h'_t
  const float* head_w;        // packed [1 + atot, H]
  float* dout;                // [R, 8]
  float* gw_part;             // [nblocks][8][H]  per-block partial sums of d head weights (block-private, += every step)
  double* gs_part;            // [nblocks][8 + 3] per-block: d head biases (8), action_loss, value_loss, entropy
  BpttScalars* sc;
  int q;                      // t & 1
  // upstream form (ic3_policy_step_backward): d loss / d (log-probs, value) given by the caller, NULL = zero
  const float* dlogp;         // [R, atot]
  const float* dvalue;        // [R]
};

constexpr int HB_ROWS = 256;   // rows per block of the heads kernel

// <= 40 registers: one CTA of this kernel fits beside a resident bptt_gates_kernel CTA (288 threads x 168 registers), so it
// overlaps the tensor-core kernels of the previous step when launched ahead on the side stream (ic3_bptt_prepare)
// UPSTREAM = false: d outputs from the records (the rollout loss).  UPSTREAM = true: from the caller's upstream gradients,
//   dout_0 = dvalue,  dlogit_j = dlogp_j - p_j sum_k dlogp_k per head (log_softmax backward, p = exp of the saved
//   log-probs); no loss sums.  Everything after d outputs (bound, bias / weight partials) is shared.
template <bool UPSTREAM>
__global__ void __launch_bounds__(256, 6) bptt_heads_kernel(HeadsArgs a) {
  __shared__ __align__(16) float s_dout[HB_ROWS][BP_HEADS];
  __shared__ float s_wmax[BP_HEADS];
  __shared__ double s_red[8][BP_HEADS + 3];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row = blockIdx.x * HB_ROWS + tid;
  const int nout = 1 + a.atot;
  if (tid < BP_HEADS) {
    float m = 0.f;
    if (tid < nout)
      for (int k = 0; k < TC_H; ++k) m = fmaxf(m, fabsf(__ldg(a.head_w + (size_t)tid * TC_H + k)));
    s_wmax[tid] = m;
  }
  float d[BP_HEADS];
#pragma unroll
  for (int o = 0; o < BP_HEADS; ++o) d[o] = 0.f;
  double al = 0.0, vl = 0.0, en = 0.0;
  if (UPSTREAM && row < a.R) {
    d[0] = a.dvalue ? a.dvalue[row] : 0.f;
    int off = 0;
    for (int m = 0; a.dlogp && m < a.nheads; ++m) {
      const int na = a.head_dim[m];
      const float* dl = a.dlogp + (size_t)row * a.atot + off;
      float sum = 0.f;
      for (int j = 0; j < na; ++j) sum += dl[j];
      for (int j = 0; j < na; ++j) {
        const float pj = __expf(a.logp[(size_t)row * a.atot + off + j]);
        if (1 + off + j < BP_HEADS) d[1 + off + j] = fmaf(-pj, sum, dl[j]);
      }
      off += na;
    }
    *reinterpret_cast<float4*>(a.dout + (size_t)row * BP_HEADS) = make_float4(d[0], d[1], d[2], d[3]);
    *reinterpret_cast<float4*>(a.dout + (size_t)row * BP_HEADS + 4) = make_float4(d[4], d[5], d[6], d[7]);
  }
  if (!UPSTREAM && row < a.R) {
    const float alive = a.alive_post[row] ? 1.f : 0.f;
    const float vmask = (a.valid == nullptr || a.valid[row / a.N]) ? 1.f : 0.f;
    const float value = a.value[row], ret = a.ret[row], adv = a.adv[row];
    d[0] = 2.f * a.value_coeff * alive * (value - ret);                       // trainer.py:205-208
    vl = (double)((value - ret) * (value - ret) * alive);
    float lp_taken = 0.f;
    int off = 0;
    for (int m = 0; m < a.nheads; ++m) {
      const int na = a.head_dim[m];
      const int act = a.action[(size_t)row * a.nheads + m];
      float Hm = 0.f;
      for (int j = 0; j < na; ++j) {
        const float lp = a.logp[(size_t)row * a.atot + off + j];
        Hm -= lp * __expf(lp);
      }
      en += (double)(Hm * vmask);                                             // trainer.py:211-216 (not alive-masked)
      for (int j = 0; j < na; ++j) {
        const float lp = a.logp[(size_t)row * a.atot + off + j];
        const float pj = __expf(lp);
        float g = (-adv * alive) * ((j == act ? 1.f : 0.f) - pj);             // d(-A logp[act]) / d logit_j
        if (a.entr > 0.f) g += a.entr * pj * (lp + Hm) * vmask;               // d(-entr * H) / d logit_j
        if (1 + off + j < BP_HEADS) d[1 + off + j] = g;
        if (j == act) lp_taken += lp;
      }
      off += na;
    }
    al = (double)(-adv * lp_taken * alive);                                   // trainer.py:198-201
    *reinterpret_cast<float4*>(a.dout + (size_t)row * BP_HEADS) = make_float4(d[0], d[1], d[2], d[3]);
    *reinterpret_cast<float4*>(a.dout + (size_t)row * BP_HEADS + 4) = make_float4(d[4], d[5], d[6], d[7]);
  }
#pragma unroll
  for (int o = 0; o < BP_HEADS; ++o) s_dout[tid][o] = d[o];
  __syncthreads();
  // bound of the heads' contribution to |dh| of a row: sum_o |dout_o| max_u |W[o][u]|
  float hb = 0.f;
#pragma unroll
  for (int o = 0; o < BP_HEADS; ++o) hb += fabsf(d[o]) * s_wmax[o];
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) hb = fmaxf(hb, __shfl_xor_sync(IC3_FULL_MASK, hb, s));
  if (lane == 0 && hb > 0.f) atomicMax(&a.sc->hbound[a.q], __float_as_uint(hb));
  // block sums: bias gradients + losses (double)
  double v[BP_HEADS + 3];
#pragma unroll
  for (int o = 0; o < BP_HEADS; ++o) v[o] = (double)d[o];
  v[BP_HEADS] = al; v[BP_HEADS + 1] = vl; v[BP_HEADS + 2] = en;
#pragma unroll
  for (int o = 0; o < BP_HEADS + 3; ++o) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v[o] += __shfl_xor_sync(IC3_FULL_MASK, v[o], s);
    if (lane == 0) s_red[warp][o] = v[o];
  }
  __syncthreads();
  if (tid < BP_HEADS + 3) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s_red[w][tid];
    a.gs_part[(size_t)blockIdx.x * (BP_HEADS + 3) + tid] += t;
  }
  // head weight gradients: thread = (hidden unit u, half of the block's rows); fixed summation order
  const int u = tid & (TC_H - 1), half = tid >> 7;
  float acc[BP_HEADS];
#pragma unroll
  for (int o = 0; o < BP_HEADS; ++o) acc[o] = 0.f;
  const int r0 = blockIdx.x * HB_ROWS + half * (HB_ROWS / 2);
  const int nr = min(HB_ROWS / 2, a.R - r0);                 // rows of this half that exist (<= 0: none)
  const float* hp = a.h_new + (size_t)r0 * TC_H + u;
  int r = 0;
  for (; r + 8 <= nr; r += 8) {                               // 8 independent loads in flight per thread
    float hv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) hv[q] = __ldg(hp + (size_t)(r + q) * TC_H);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 d0 = *reinterpret_cast<const float4*>(&s_dout[half * (HB_ROWS / 2) + r + q][0]);
      const float4 d1 = *reinterpret_cast<const float4*>(&s_dout[half * (HB_ROWS / 2) + r + q][4]);
      acc[0] = fmaf(d0.x, hv[q], acc[0]); acc[1] = fmaf(d0.y, hv[q], acc[1]);
      acc[2] = fmaf(d0.z, hv[q], acc[2]); acc[3] = fmaf(d0.w, hv[q], acc[3]);
      acc[4] = fmaf(d1.x, hv[q], acc[4]); acc[5] = fmaf(d1.y, hv[q], acc[5]);
      acc[6] = fmaf(d1.z, hv[q], acc[6]); acc[7] = fmaf(d1.w, hv[q], acc[7]);
    }
  }
  for (; r < nr; ++r) {
    const float hv = __ldg(hp + (size_t)r * TC_H);
    const float* dr = s_dout[half * (HB_ROWS / 2) + r];
#pragma unroll
    for (int o = 0; o < BP_HEADS; ++o) acc[o] = fmaf(dr[o], hv, acc[o]);
  }
  __shared__ float s_acc[BP_HEADS][TC_H];
  if (half == 1) {
#pragma unroll
    for (int o = 0; o < BP_HEADS; ++o) s_acc[o][u] = acc[o];
  }
  __syncthreads();
  if (half == 0) {
    float* gp = a.gw_part + (size_t)blockIdx.x * BP_HEADS * TC_H;
#pragma unroll
    for (int o = 0; o < BP_HEADS; ++o) gp[o * TC_H + u] += acc[o] + s_acc[o][u];
  }
}

// s_t = 2^e with  bound * s_t in (2^13, 2^14]:  |d gate| <= (|dc| + |dh|) * max(1, |c_prev| / 4)
__global__ void bptt_scale_kernel(BpttScalars* sc, int q) {
  const float dh = __uint_as_float(sc->dhmax) + __uint_as_float(sc->hbound[q]);
  const float dc = __uint_as_float(sc->dcmax);
  const float bound = (dh + dc) * fmaxf(1.f, 0.25f * sc->cmax);
  float s = 1.f;
  if (bound > 0.f && isfinite(bound)) {
    int e;
    frexpf(bound, &e);                       // bound = m * 2^e, m in [0.5, 1)
    e = 14 - e;
    e = e > 100 ? 100 : (e < -100 ? -100 : e);
    s = ldexpf(1.f, e);
  }
  sc->scale[q] = s;
  sc->inv_scale[q] = 1.f / s;
  sc->dhmax = 0u;
  sc->dcmax = 0u;
  sc->hbound[q] = 0u;
}

// ic3_policy_step_backward: the recursion's inputs from the caller's upstream gradients.  dh = dh_new, dc = dc_new (NULL:
// zero), and the maxima the scale kernel reads are reduced here on the device instead of coming from the host:
// dhmax = max |dh_new|, dcmax = max |dc_new|, cmax = max |c_prev| + cadd (cadd = passes - 1, see ic3_bptt_begin).  The
// scalars were zeroed before; the maxima are non-negative, so their bit patterns order like the values.
__global__ void bptt_upstream_kernel(size_t n4, const float4* __restrict__ dh_new, const float4* __restrict__ dc_new,
                                     const float4* __restrict__ c_prev, float4* __restrict__ dh, float4* __restrict__ dc,
                                     float cadd, BpttScalars* sc) {
  float mh = 0.f, mc = 0.f, mp = 0.f;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 h = dh_new ? dh_new[i] : z;
    dh[i] = h;
    mh = fmaxf(mh, fmaxf(fmaxf(fabsf(h.x), fabsf(h.y)), fmaxf(fabsf(h.z), fabsf(h.w))));
    if (dc) {
      const float4 c = dc_new ? dc_new[i] : z;
      dc[i] = c;
      mc = fmaxf(mc, fmaxf(fmaxf(fabsf(c.x), fabsf(c.y)), fmaxf(fabsf(c.z), fabsf(c.w))));
    }
    if (c_prev) {
      const float4 c = c_prev[i];
      mp = fmaxf(mp, fmaxf(fmaxf(fabsf(c.x) + cadd, fabsf(c.y) + cadd), fmaxf(fabsf(c.z) + cadd, fabsf(c.w) + cadd)));
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    mh = fmaxf(mh, __shfl_xor_sync(IC3_FULL_MASK, mh, s));
    mc = fmaxf(mc, __shfl_xor_sync(IC3_FULL_MASK, mc, s));
    mp = fmaxf(mp, __shfl_xor_sync(IC3_FULL_MASK, mp, s));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&sc->dhmax, __float_as_uint(mh));
    atomicMax(&sc->dcmax, __float_as_uint(mc));
    atomicMax(reinterpret_cast<unsigned*>(&sc->cmax), __float_as_uint(mp));
  }
}

// ------------------------------------------------------------------------------------------------------------------
// gates: forward gate GEMM re-computed + LSTM cell backward in the epilogue
// ------------------------------------------------------------------------------------------------------------------
struct GatesArgs {
  int R, N;
  const float* c_prev;      // [R, H] c_{t-1}
  const uint8_t* fresh;     // [B] step t starts an episode: h_{t-1} = c_{t-1} = 0 and nothing flows further back
  const uint8_t* cut;       // [B] or NULL: (h', c') of step t were detached (trainer.py:56-60): incoming dh, dc are dropped
  const float* dout;        // [R, 8]
  float* dh;                // [R, H] in: d loss / d h'_t from later steps
  float* dc;                // [R, H] in: d loss / d c'_t;  out: d loss / d c_{t-1}
  __half* dg_img;           // d gates image
  BpttScalars* sc;
  int q;                    // t & 1
  int32_t* err;
};

// sigmoid / tanh of the four gates of a hidden unit with the forward's arithmetic (lstm_cell4): same SFU
// approximations, so the re-computed activations are the ones the rollout used.
__device__ __forceinline__ void gates4(const float (&v)[16], const float* s_bias4, int bstride, float (&gi)[4], float (&gf)[4],
                                       float (&gg)[4], float (&go)[4]) {
  constexpr float SG = -INV_SCALE * LOG2E;
  constexpr float TMAX = 30.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 b = *reinterpret_cast<const float4*>(s_bias4 + j * bstride);
    const float ai = 1.f + ex2_fast(fminf(fmaf(v[4 * j + 0], SG, b.x), TMAX));
    const float af = 1.f + ex2_fast(fminf(fmaf(v[4 * j + 1], SG, b.y), TMAX));
    const float ag = 1.f + ex2_fast(fminf(fmaf(v[4 * j + 2], 2.f * SG, b.z), TMAX));
    const float ao = 1.f + ex2_fast(fminf(fmaf(v[4 * j + 3], SG, b.w), TMAX));
    const float p1 = ai * af, p2 = ag * ao;
    const float r = rcp_fast(p1 * p2);
    const float r1 = r * p2, r2 = r * p1;
    gi[j] = r1 * af;
    gf[j] = r1 * ai;
    gg[j] = fmaf(2.f, r2 * ao, -1.f);
    go[j] = r2 * ag;
  }
}

__device__ __forceinline__ float tanh_fwd(float c) {      // tanh(c') as the forward computes it
  const float b = 1.f + ex2_fast(fminf(c * (-2.f * LOG2E), 30.f));
  return fmaf(2.f, rcp_fast(b), -1.f);
}

// 4 values -> hi / lo fp16 halves (x * scale = hi + lo).  hi = x * scale truncated to 11 significant bits by an
// integer mask -- exactly representable in fp16, so no conversion back is needed -- and lo = the exact remainder rounded
// to fp16 (|lo| < 2^-10 |hi|): 21-22 significant bits, two values per conversion instruction.
__device__ __forceinline__ uint2 pack4_hi_lo(const float (&x)[4], float scale, uint2& lo) {
  uint32_t h[2], l[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float a = x[2 * j] * scale, b = x[2 * j + 1] * scale;       // power of two: exact
    const float ah = __uint_as_float(__float_as_uint(a) & 0xFFFFE000u), bh = __uint_as_float(__float_as_uint(b) & 0xFFFFE000u);
    const __half2 hh = __floats2half2_rn(ah, bh);
    const __half2 ll = __floats2half2_rn(a - ah, b - bh);
    h[j] = *reinterpret_cast<const uint32_t*>(&hh);
    l[j] = *reinterpret_cast<const uint32_t*>(&ll);
  }
  lo = make_uint2(l[0], l[1]);
  return make_uint2(h[0], h[1]);
}

// Same ring and MMAs as lstm_tc_kernel (warp 8 producer, two consumer warpgroups of 64 rows); the epilogue of a
// thread covers units 2j + (lane % 4) / 2 of one row (gather_gates).
__global__ void __launch_bounds__(TC_P_THREADS, 1) bptt_gates_kernel(GatesArgs g, const __half* __restrict__ a_img,
                                                                    const __half* __restrict__ b_img,
                                                                    const float* __restrict__ bias_cat, int nitems,
                                                                    const float* __restrict__ head_w, int nout) {
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGE_P * STAGE_BYTES);
  float* s_hw = reinterpret_cast<float*>(smem + NSTAGE_P * STAGE_BYTES + 256);   // head weights, unit-major [128][8]
  float* s_bias = s_hw + TC_H * HEAD_PAD;
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + NSTAGE_P);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE_P; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, MMA_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  load_scaled_bias(s_bias, bias_cat);
  for (int idx = threadIdx.x; idx < TC_H * HEAD_PAD; idx += blockDim.x) {
    const int u = idx / HEAD_PAD, o = idx - u * HEAD_PAD;
    s_hw[idx] = o < nout ? __ldg(head_w + (size_t)o * TC_H + u) : 0.f;
  }
  __syncthreads();
  const uint32_t smem_base = smem_u32(smem);

  if (warp == MMA_WARPS) {
    if (lane == 0) {
      const unsigned char* a = reinterpret_cast<const unsigned char*>(a_img);
      const unsigned char* b = reinterpret_cast<const unsigned char*>(b_img);
      ring_producer<TC_NCHUNK>(
          smem_base, bar_full, bar_empty, blockIdx.x, nitems, gridDim.x, (size_t)A_TILE_HALFS,
          [=](int item, int c) { return a + (size_t)(item >> 1) * TC_NCHUNK * A_CHUNK_BYTES + (size_t)c * (A_CHUNK_BYTES / 2); },
          [=](int item, int c) { return b + (size_t)((item & 1) * TC_NCHUNK + c) * B_CHUNK_BYTES; }, g.err);
    }
    return;
  }
  const int wg = warp >> 2, w4 = warp & 3;
  const bool odd = lane & 1, hl = (lane >> 1) & 1;
  const float scale = g.sc->scale[g.q];
  float d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0.f;
  uint32_t li = 0;
  bool ok = true;
  float dcm = 0.f;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++li) {
    wg_gemm_item<TC_NCHUNK>(d, smem_base, wg * 1024, bar_full, bar_empty, li, lane, ok, g.err);
    const int tile = item >> 1, nh = item & 1;
    const int rt = wg * 64 + w4 * 16 + (lane >> 2) + (odd ? 8 : 0);      // row inside the tile
    const int row = tile * TC_M + rt;
    const bool inrange = row < g.R;
    bool fr = false, ct = false;
    if (inrange) {
      const int e = row / g.N;
      fr = g.fresh && g.fresh[e] != 0;
      ct = g.cut && g.cut[e] != 0;
    }
    float dsum[HEAD_PAD];      // d outputs of this row (value + logits)
    {
      float4 d0 = make_float4(0.f, 0.f, 0.f, 0.f), d1 = d0;
      if (inrange) {
        d0 = *reinterpret_cast<const float4*>(g.dout + (size_t)row * BP_HEADS);
        d1 = *reinterpret_cast<const float4*>(g.dout + (size_t)row * BP_HEADS + 4);
      }
      dsum[0] = d0.x; dsum[1] = d0.y; dsum[2] = d0.z; dsum[3] = d0.w;
      dsum[4] = d1.x; dsum[5] = d1.y; dsum[6] = d1.z; dsum[7] = d1.w;
    }
    const bool ld_c = inrange && !fr, ld_d = inrange && !ct;
    const int ub = nh * (TC_NH / 4) + hl;            // unit of j = 0; unit of j = ub + 2j
    const size_t rbase = (size_t)row * TC_H;
    // d gates image, column 4u + gate: core matrix (column group u / 2, row group rt / 8), columns 4 (u & 1) + gate
    __half* img = g.dg_img + (size_t)tile * DG_TILE_HALFS + (size_t)(rt >> 3) * 64 + (lane >> 2) * 8 + hl * 4 +
                  (size_t)nh * 32 * 1024;
#pragma unroll
    for (int j0 = 0; j0 < 32; j0 += 4) {
      float v[16];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        float gq[4];
        gather_gates(d, j0 + jj, odd, gq);
        v[4 * jj + 0] = gq[0]; v[4 * jj + 1] = gq[1]; v[4 * jj + 2] = gq[2]; v[4 * jj + 3] = gq[3];
      }
      float gi[4], gf[4], gg[4], go[4];
      gates4(v, s_bias + 4 * (ub + 2 * j0), 8, gi, gf, gg, go);
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int u = ub + 2 * (j0 + jj);
        float dg[4] = {0.f, 0.f, 0.f, 0.f};
        if (ok && inrange) {
          const float cp = ld_c ? g.c_prev[rbase + u] : 0.f;
          float dh = ld_d ? g.dh[rbase + u] : 0.f;
          const float dc = ld_d ? g.dc[rbase + u] : 0.f;
          // heads: dh += sum_o dout_o W_o[u]
          const float4 w0 = *reinterpret_cast<const float4*>(&s_hw[u * HEAD_PAD]);
          const float4 w1 = *reinterpret_cast<const float4*>(&s_hw[u * HEAD_PAD + 4]);
          dh = fmaf(dsum[0], w0.x, dh); dh = fmaf(dsum[1], w0.y, dh); dh = fmaf(dsum[2], w0.z, dh); dh = fmaf(dsum[3], w0.w, dh);
          dh = fmaf(dsum[4], w1.x, dh); dh = fmaf(dsum[5], w1.y, dh); dh = fmaf(dsum[6], w1.z, dh); dh = fmaf(dsum[7], w1.w, dh);
          const float cn = fmaf(gf[jj], cp, gi[jj] * gg[jj]);
          const float tc = tanh_fwd(cn);
          const float dct = fmaf(dh * go[jj], 1.f - tc * tc, dc);
          dg[0] = dct * gg[jj] * gi[jj] * (1.f - gi[jj]);
          dg[1] = dct * cp * gf[jj] * (1.f - gf[jj]);
          dg[2] = dct * gi[jj] * (1.f - gg[jj] * gg[jj]);
          dg[3] = dh * tc * go[jj] * (1.f - go[jj]);
          const float dcp = fr ? 0.f : dct * gf[jj];
          dcm = fmaxf(dcm, fabsf(dcp));
          g.dc[rbase + u] = dcp;
        }
        // rows past R and a broken pipeline write zeros: the other GEMMs read whole tiles
        uint2 lo;
        const uint2 hi = pack4_hi_lo(dg, scale, lo);
        __half* p0 = img + (size_t)(j0 + jj) * 1024;
        *reinterpret_cast<uint2*>(p0) = hi;
        *reinterpret_cast<uint2*>(p0 + DG_PART_HALFS) = lo;
      }
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) dcm = fmaxf(dcm, __shfl_xor_sync(IC3_FULL_MASK, dcm, s));
  if (lane == 0 && dcm > 0.f) atomicMax(&g.sc->dcmax, __float_as_uint(dcm));
}

// ------------------------------------------------------------------------------------------------------------------
// tanh cell backward: dz = (dh + W_heads^T dout) (1 - h'^2), elementwise.  h' is the record the forward wrote (its own
// tanhf value), so nothing is re-computed and no GEMM is needed.  The dz image has the d gates image's layout with 128
// columns (column = hidden unit): [tile][hi, lo][cg 16][rg 16][8][8].  Thread = (row, 8 consecutive units = one column
// group); rows past R (up to whole tiles) write zeros, the GEMMs read whole tiles.
// ------------------------------------------------------------------------------------------------------------------
constexpr int DZ_TILE_HALFS = 2 * 16 * 16 * 64;
constexpr int DZ_PART_HALFS = 16 * 16 * 64;
constexpr int TZ_ROWS = 16;                        // rows per 256-thread block

struct TanhArgs {
  int R, N, nrows;          // nrows: R rounded up to whole tiles
  const uint8_t* cut;       // [B] or NULL: h' of step t was detached (trainer.py:56-60): the incoming dh is dropped
  const float* dout;        // [R, 8]
  const float* h_new;       // [R, H] h'_t
  const float* dh;          // [R, H] d loss / d h'_t from later steps
  const float* head_w;      // packed [nout, H]
  int nout;
  __half* dz_img;
  const BpttScalars* sc;
  int q;                    // t & 1
};

__global__ void __launch_bounds__(256) bptt_tanh_kernel(TanhArgs a) {
  __shared__ __align__(16) float s_hw[HEAD_PAD][TC_H];
  for (int idx = threadIdx.x; idx < HEAD_PAD * TC_H; idx += blockDim.x) {
    const int o = idx / TC_H, u = idx - o * TC_H;
    s_hw[o][u] = o < a.nout ? __ldg(a.head_w + (size_t)o * TC_H + u) : 0.f;
  }
  __syncthreads();
  const int cg = threadIdx.x & 15;
  const int row = blockIdx.x * TZ_ROWS + (threadIdx.x >> 4);
  if (row >= a.nrows) return;
  float dz[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) dz[k] = 0.f;
  if (row < a.R) {
    const bool ct = a.cut && a.cut[row / a.N] != 0;
    const float4 d0 = *reinterpret_cast<const float4*>(a.dout + (size_t)row * BP_HEADS);
    const float4 d1 = *reinterpret_cast<const float4*>(a.dout + (size_t)row * BP_HEADS + 4);
    const float dsum[HEAD_PAD] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
    const size_t base = (size_t)row * TC_H + 8 * cg;
    const float4 h0 = *reinterpret_cast<const float4*>(a.h_new + base);
    const float4 h1 = *reinterpret_cast<const float4*>(a.h_new + base + 4);
    float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0;
    if (!ct) {
      g0 = *reinterpret_cast<const float4*>(a.dh + base);
      g1 = *reinterpret_cast<const float4*>(a.dh + base + 4);
    }
    const float hv[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
    float dh[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    // heads: dh += sum_o dout_o W_o[u], in output order (as bptt_gates_kernel)
#pragma unroll
    for (int o = 0; o < HEAD_PAD; ++o) {
      const float4 w0 = *reinterpret_cast<const float4*>(&s_hw[o][8 * cg]);
      const float4 w1 = *reinterpret_cast<const float4*>(&s_hw[o][8 * cg + 4]);
      dh[0] = fmaf(dsum[o], w0.x, dh[0]); dh[1] = fmaf(dsum[o], w0.y, dh[1]);
      dh[2] = fmaf(dsum[o], w0.z, dh[2]); dh[3] = fmaf(dsum[o], w0.w, dh[3]);
      dh[4] = fmaf(dsum[o], w1.x, dh[4]); dh[5] = fmaf(dsum[o], w1.y, dh[5]);
      dh[6] = fmaf(dsum[o], w1.z, dh[6]); dh[7] = fmaf(dsum[o], w1.w, dh[7]);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) dz[k] = dh[k] * (1.f - hv[k] * hv[k]);
  }
  const float scale = a.sc->scale[a.q];
  const float v4[2][4] = {{dz[0], dz[1], dz[2], dz[3]}, {dz[4], dz[5], dz[6], dz[7]}};
  uint2 lo0, lo1;
  const uint2 hi0 = pack4_hi_lo(v4[0], scale, lo0);
  const uint2 hi1 = pack4_hi_lo(v4[1], scale, lo1);
  const int tile = row / TC_M, rt = row - tile * TC_M;
  __half* p = a.dz_img + (size_t)tile * DZ_TILE_HALFS + (size_t)(cg * 16 + (rt >> 3)) * 64 + (rt & 7) * 8;
  *reinterpret_cast<uint4*>(p) = make_uint4(hi0.x, hi0.y, hi1.x, hi1.y);
  *reinterpret_cast<uint4*>(p + DZ_PART_HALFS) = make_uint4(lo0.x, lo0.y, lo1.x, lo1.y);
}

// ------------------------------------------------------------------------------------------------------------------
// dgrad: [dS | dh_direct] = d gates . [W_ih C | W_hh]        (M = rows, K = 512 gate columns, N = 256)
// tanh cell: [0 | dh_direct] = dz . [0 | W_f]                 (K = 128 units, the S half of the weight image is zero)
// ------------------------------------------------------------------------------------------------------------------
constexpr int DGR_NCHUNK = 16;                       // 512 gate columns / 32
constexpr int DGR_NCHUNK_TANH = 4;                   // 128 units / 32
constexpr int DGR_STAGE = A_CHUNK_BYTES + B_CHUNK_BYTES;   // 16 KB (hi + lo of 32 columns x 128 rows) + 32 KB

// weight image of the dgrad GEMM: element (n = S / h feature, k = gate column j) = scaled forward weight
// [W_ih ; W_ih C ; W_hh] (j, 128 + n): [chunk 16][hi, lo][kcore 4][ncore 32][8][8]
__host__ __device__ __forceinline__ size_t w2_img_off(int k, int n, int part) {
  const int c = k >> 5, kk = k & 31;
  return ((((size_t)(c * 2 + part) * 4 + (kk >> 3)) * 32 + (n >> 3)) * 8 + (n & 7)) * 8 + (kk & 7);
}
constexpr size_t W2_IMG_HALFS = (size_t)DGR_NCHUNK * 2 * 4 * 32 * 64;     // 262144 halfs = 512 KB

__global__ void bptt_pack_w2_kernel(const __half* __restrict__ b_img, __half* __restrict__ w2) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;      // (n, j)
  if (idx >= 256 * 512) return;
  const int n = idx >> 9, j = idx & 511;
  const int nh = j >> 8, col = j & 255;
#pragma unroll
  for (int part = 0; part < 2; ++part) w2[w2_img_off(j, n, part)] = b_img[b_img_off(nh, 128 + n, col, part)];
}

// the tanh cell's image, from the packed f_wT (f_wT[k][n] = f.weight[n][k]): element (n, k = unit u) = SCALE_B *
// f.weight[u][n - 128] for n >= 128, zero for the S half n < 128; same hi/lo split as the forward's weight images
constexpr size_t W2_IMG_HALFS_TANH = (size_t)DGR_NCHUNK_TANH * 2 * 4 * 32 * 64;

__global__ void bptt_pack_w2_tanh_kernel(const float* __restrict__ f_wT, __half* __restrict__ w2) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;      // (n, k)
  if (idx >= 256 * TC_H) return;
  const int n = idx >> 7, k = idx & 127;
  __half hi, lo;
  split_f16(n < TC_H ? 0.f : f_wT[(size_t)(n - TC_H) * TC_H + k], SCALE_B, hi, lo);
  w2[w2_img_off(k, n, 0)] = hi;
  w2[w2_img_off(k, n, 1)] = lo;
}

struct DgradArgs {
  int R;
  const float* gs;       // [R] g / den
  float* dSs;            // [R, H]  out: gs * dS  (NULL: not stored, the tanh cell)
  float* dh_direct;      // [R, H]  out
  const BpttScalars* sc;
  int q;
  int32_t* err;
};

// NCHUNK = K / 32: the d gates image of a tile is [hi, lo][K / 8 column groups][rg 16][8][8]
template <int NCHUNK>
__global__ void __launch_bounds__(TC_P_THREADS, 1) bptt_dgrad_kernel(DgradArgs g, const __half* __restrict__ dg_img,
                                                                    const __half* __restrict__ w2_img, int ntiles) {
  static_assert(DGR_STAGE == STAGE_BYTES, "dgrad shares the stage layout of the gate GEMM");
  constexpr size_t PART_BYTES = (size_t)NCHUNK * 32 * TC_M * 2, TILE_BYTES = 2 * PART_BYTES;
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGE_P * DGR_STAGE);
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + NSTAGE_P);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE_P; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, MMA_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t smem_base = smem_u32(smem);

  if (warp == MMA_WARPS) {
    if (lane == 0) {
      // 32 gate columns = 4 column groups = 8 KB per part, contiguous in the d gates image
      const unsigned char* a = reinterpret_cast<const unsigned char*>(dg_img);
      const unsigned char* b = reinterpret_cast<const unsigned char*>(w2_img);
      ring_producer<NCHUNK>(
          smem_base, bar_full, bar_empty, blockIdx.x, ntiles, gridDim.x, PART_BYTES,
          [=](int tile, int c) { return a + (size_t)tile * TILE_BYTES + (size_t)c * 8192; },
          [=](int, int c) { return b + (size_t)c * B_CHUNK_BYTES; }, g.err);
    }
    return;
  }
  const int wg = warp >> 2, w4 = warp & 3;
  const float unscale = g.sc->inv_scale[g.q] * (1.f / SCALE_B);
  float d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0.f;
  uint32_t li = 0;
  bool ok = true;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++li) {
    wg_gemm_item<NCHUNK>(d, smem_base, wg * 1024, bar_full, bar_empty, li, lane, ok, g.err);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = tile * TC_M + wg * 64 + w4 * 16 + (lane >> 2) + 8 * i;
      if (!ok || row >= g.R) continue;
      const float fs = g.dSs ? unscale * g.gs[row] : 0.f;
      // columns 0..127 -> gs * dS, 128..255 -> dh_direct
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        if (j < 16 && !g.dSs) continue;
        const float f = j < 16 ? fs : unscale;
        float* dst = (j < 16 ? g.dSs + (size_t)row * TC_H + col : g.dh_direct + (size_t)row * TC_H + col - 128);
        *reinterpret_cast<float2*>(dst) = make_float2(d[4 * j + 2 * i] * f, d[4 * j + 2 * i + 1] * f);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// comm: backward of S_k = (g_k / den) (sum_j g_j h_j - g_k h_k)  (comm.py:181-205) + the cuts of the recursion
//   dh_{t-1}[j] = keep * (dh_direct[j] + g_j (sum_k dSs[k] - g_j dSs[j])),  dSs = (g / den) dS,  keep = 1 - fresh_t
// One warp per environment, lane = 4 hidden units.
// ------------------------------------------------------------------------------------------------------------------
struct CommArgs {
  int B, N;
  const float* dSs;
  const float* dh_direct;
  const float* gr;          // [R]
  const uint8_t* fresh;     // [B]
  int no_comm;              // comm_mask_zero
  float* dh;                // [R, H] out
  BpttScalars* sc;
};

__global__ void __launch_bounds__(256) bptt_comm_kernel(CommArgs a) {
  const int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  float m = 0.f;
  if (e < a.B) {
    const bool fr = a.fresh && a.fresh[e] != 0;
    const size_t base = (size_t)e * a.N;
    float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!fr && !a.no_comm) {
      for (int k = 0; k < a.N; ++k) {
        const float4 d = *(reinterpret_cast<const float4*>(a.dSs + (base + k) * TC_H) + lane);
        tot.x += d.x; tot.y += d.y; tot.z += d.z; tot.w += d.w;
      }
    }
    for (int j = 0; j < a.N; ++j) {
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
      if (!fr) {
        o = *(reinterpret_cast<const float4*>(a.dh_direct + (base + j) * TC_H) + lane);
        if (!a.no_comm) {
          const float gj = a.gr[base + j];
          if (gj != 0.f) {
            const float4 d = *(reinterpret_cast<const float4*>(a.dSs + (base + j) * TC_H) + lane);
            o.x += gj * (tot.x - gj * d.x); o.y += gj * (tot.y - gj * d.y);
            o.z += gj * (tot.z - gj * d.z); o.w += gj * (tot.w - gj * d.w);
          }
        }
      }
      *(reinterpret_cast<float4*>(a.dh + (base + j) * TC_H) + lane) = o;
      m = fmaxf(m, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(IC3_FULL_MASK, m, s));
  if (lane == 0 && m > 0.f) atomicMax(&a.sc->dhmax, __float_as_uint(m));
}

// ------------------------------------------------------------------------------------------------------------------
// wgrad: G[gate column j][feature n] += sum_rows dgates[row][j] * F[row][n],  F = [x | S | h] (hi/lo) and P (exact)
// Both operands are MN-major views of images written for the other GEMMs; a pipeline stage is a 32-row slab
// gathered by tensor copies (cp.async.bulk.tensor) whose box re-packs it as [group][4 row groups][8][8].
// CTA role = (block of 128 gate columns mb, feature slice sl, row-tile subset); the two CTAs of a role split the
// gate columns (64 each).  Consumer warpgroup w accumulates features [128 w, 128 w + 128) of the slice in registers
// for the whole launch and adds them into the role's private fp32 partial at the end (no atomics; the partials of
// all roles are summed in float64 by ic3_bptt_finish).
// ------------------------------------------------------------------------------------------------------------------
constexpr int WG_CONSUMERS = 4;                   // consumer warpgroups: up to 512 feature columns
constexpr int WG_THREADS = WG_CONSUMERS * 128 + 32;   // + producer warp
constexpr int WG_DG_BYTES = 16 * 4 * 128;       // 8 KB: 16 column groups x 4 row groups, one part
constexpr int WG_A_BYTES = 48 * 4 * 128;        // 24 KB: 48 feature groups x 4 row groups, one part
constexpr int WG_STAGE0 = 2 * WG_DG_BYTES + 2 * WG_A_BYTES;   // 64 KB
constexpr int WG_NSTAGE0 = 3;
constexpr int WG_NSTAGE1 = 4;

struct WgradArgs {
  int ntiles;
  int np;                // columns of P (multiple of 16, <= WG_MAX_NP)
  int j0, j1;            // row-tile subsets of slice 0 / slice 1 ((gate blocks) * (j0 + j1) roles)
  int h_only;            // slice 0 = the h block of the operand image alone (tanh cell: G_h is all it needs)
  float* partial;        // [nroles][512 columns max][128] fp32, role-private
  const BpttScalars* sc;
  int q;
  int32_t* err;
};

__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4,
                                            uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// d (+)= dg^T . F for an MN-major 64-column block of dg and an NW-column block of F (NW = 16 .. 128, multiple of 16)
template <int NW>
__device__ __forceinline__ void wgmma_mn(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  static_assert(NW % 16 == 0 && NW >= 16 && NW <= 128, "feature block width");
  if constexpr (NW == 16) wgmma_m64n16_mn(d, da, db, acc);
  else if constexpr (NW == 32) wgmma_m64n32_mn(d, da, db, acc);
  else if constexpr (NW == 48) wgmma_m64n48_mn(d, da, db, acc);
  else if constexpr (NW == 64) wgmma_m64n64_mn(d, da, db, acc);
  else if constexpr (NW == 80) wgmma_m64n80_mn(d, da, db, acc);
  else if constexpr (NW == 96) wgmma_m64n96_mn(d, da, db, acc);
  else if constexpr (NW == 112) wgmma_m64n112_mn(d, da, db, acc);
  else wgmma_m64n128_mn(d, da, db, acc);
}

__device__ __forceinline__ unsigned char* wgrad_smem() {
  extern __shared__ __align__(1024) unsigned char wg_smem[];
  return wg_smem;
}

struct WgradRole {
  int role, mh, sl, nstage, stage_bytes, a_bytes, nchunks, n0;   // a_bytes: one part of the slice-0 features
  uint32_t bar_full, bar_empty;
};

// One consumer warpgroup of bptt_wgrad_kernel: the slab loop for its NW feature columns (SPLIT: x|S|h as hi/lo, three
// products per k-step; otherwise the exact P columns, two), then the flush into the role's partial.  The block width
// is a template parameter chosen once per warpgroup: inside a loop every MMA has the same accumulator footprint, which
// keeps ptxas from inserting warpgroup arrives and serialising the MMAs (it does when the width is switched per MMA).
template <int NW, bool SPLIT>
__device__ __forceinline__ void wgrad_consumer(const WgradArgs g, const WgradRole r, int w4, int lane) {
  float d[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  bool ok = true;
  const uint32_t sbase = smem_u32(wgrad_smem());
  // MN-major no-swizzle: LBO = stride between the two 8-row (K) groups of one MMA = 128 B,
  //                      SBO = stride between 8-element M / N groups = 4 row groups x 128 B = 512 B
  wgmma_fence_regs(d);
  for (int ch = 0; ch < r.nchunks; ++ch) {
    const int s = ch % r.nstage;
    if (ok) ok = mbar_wait(r.bar_full + 8 * s, (ch / r.nstage) & 1, g.err);
    wgmma_fence();
    const uint32_t st = sbase + s * r.stage_bytes;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {               // 16 rows = 2 row groups per MMA
      const uint64_t dg_hi = make_desc(st + r.mh * 8 * 512 + ks * 256, 128, 512);
      const uint64_t dg_lo = make_desc(st + WG_DG_BYTES + r.mh * 8 * 512 + ks * 256, 128, 512);
      const uint32_t accum = (ch | ks) != 0;
      const uint32_t f = st + 2 * WG_DG_BYTES + (r.n0 / 8) * 512 + ks * 256;
      wgmma_mn<NW>(d, dg_hi, make_desc(f, 128, 512), accum);
      wgmma_mn<NW>(d, dg_lo, make_desc(f, 128, 512), 1);
      if (SPLIT) wgmma_mn<NW>(d, dg_hi, make_desc(f + r.a_bytes, 128, 512), 1);
    }
    wgmma_commit();
    wgmma_wait<1>();                               // the MMAs of slab ch - 1 have read their stage
    if (ch > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(r.bar_empty + 8 * ((ch - 1) % r.nstage));
    }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  __syncwarp();
  if (lane == 0) mbar_arrive(r.bar_empty + 8 * ((r.nchunks - 1) % r.nstage));
  if (!ok) return;
  // flush: fragment (m, n) -> partial[n][m]; slice 0: x|S|h products carry SCALE_A * s_t, slice 1 (P exact) only s_t
  const float unscale = g.sc->inv_scale[g.q] * (SPLIT ? 1.f / SCALE_A : 1.f);
  float* part = g.partial + (size_t)r.role * 512 * 128;
  const int m = r.mh * 64 + w4 * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < NW / 8; ++j) {
    const int n = r.n0 + 8 * j + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c) part[(size_t)(n + c) * 128 + m + 8 * i] += d[4 * j + 2 * i + c] * unscale;
  }
}

__global__ void __launch_bounds__(WG_THREADS, 1) bptt_wgrad_kernel(WgradArgs g, const __grid_constant__ CUtensorMap map_dg,
                                                                  const __grid_constant__ CUtensorMap map_a,
                                                                  const __grid_constant__ CUtensorMap map_p) {
  unsigned char* smem = wgrad_smem();
  __shared__ uint64_t bars[2 * WG_NSTAGE1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // role
  const int role = blockIdx.x >> 1, mh = blockIdx.x & 1;    // mh: which 64 of the role's 128 gate columns
  const int per_mb = g.j0 + g.j1;
  const int mb = role / per_mb, rj = role - mb * per_mb;
  const int sl = rj < g.j0 ? 0 : 1;
  const int jj = sl == 0 ? rj : rj - g.j0, jn = sl == 0 ? g.j0 : g.j1;
  const int nstage = sl == 0 && !g.h_only ? WG_NSTAGE0 : WG_NSTAGE1;
  const int p_bytes = g.np * 64;                    // np/8 groups x 4 row groups x 128 B
  const int a_bytes = g.h_only ? WG_A_BYTES / 3 : WG_A_BYTES;
  const int stage_bytes = sl == 0 ? 2 * WG_DG_BYTES + 2 * a_bytes : 2 * WG_DG_BYTES + p_bytes;
  const int ncols = sl == 0 ? (g.h_only ? 128 : 384) : g.np;
  const int nact = (ncols + 127) / 128;             // consumer warpgroups with columns
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + WG_NSTAGE1);
  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_NSTAGE1; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 4 * nact);      // one release per warp of the active warpgroups
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nmine = (g.ntiles - jj + jn - 1) / jn;      // tiles jj, jj + jn, ...
  const int nchunks = nmine > 0 ? nmine * 4 : 0;         // 32-row slabs

  if (warp == WG_CONSUMERS * 4) {
    // ===== producer =====
    if (lane != 0) return;
    bool ok = true;
    const uint32_t smem_base = smem_u32(smem);
    for (int ch = 0; ch < nchunks && ok; ++ch) {
      const int tile = jj + (ch >> 2) * jn, rc = ch & 3;
      const int s = ch % nstage;
      ok = mbar_wait(bar_empty + 8 * s, ((ch / nstage) & 1) ^ 1, g.err);
      const uint32_t dst = smem_base + s * stage_bytes;
      mbar_expect_tx(bar_full + 8 * s, stage_bytes);
      tma_load_5d(dst, &map_dg, 0, 4 * rc, 16 * mb, 0, tile, bar_full + 8 * s);
      tma_load_5d(dst + WG_DG_BYTES, &map_dg, 0, 4 * rc, 16 * mb, 1, tile, bar_full + 8 * s);
      if (sl == 0) {                                // h_only: the box is the 16 groups of h, from feature group 32
        const int g0 = g.h_only ? 32 : 0;
        tma_load_5d(dst + 2 * WG_DG_BYTES, &map_a, 0, 4 * rc, g0, 0, tile, bar_full + 8 * s);
        tma_load_5d(dst + 2 * WG_DG_BYTES + a_bytes, &map_a, 0, 4 * rc, g0, 1, tile, bar_full + 8 * s);
      } else {
        tma_load_4d(dst + 2 * WG_DG_BYTES, &map_p, 0, 4 * rc, 0, tile, bar_full + 8 * s);
      }
    }
    return;
  }
  const int w = warp >> 2, w4 = warp & 3;
  if (w >= nact || nchunks == 0) return;
  const WgradRole r{role, mh, sl, nstage, stage_bytes, a_bytes, nchunks, 128 * w, bar_full, bar_empty};
  if (sl == 0) {
    wgrad_consumer<128, true>(g, r, w4, lane);
    return;
  }
  switch (min(128, ncols - r.n0) >> 4) {           // width of this warpgroup's block of P columns
    case 1: wgrad_consumer<16, false>(g, r, w4, lane); break;
    case 2: wgrad_consumer<32, false>(g, r, w4, lane); break;
    case 3: wgrad_consumer<48, false>(g, r, w4, lane); break;
    case 4: wgrad_consumer<64, false>(g, r, w4, lane); break;
    case 5: wgrad_consumer<80, false>(g, r, w4, lane); break;
    case 6: wgrad_consumer<96, false>(g, r, w4, lane); break;
    case 7: wgrad_consumer<112, false>(g, r, w4, lane); break;
    default: wgrad_consumer<128, false>(g, r, w4, lane); break;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// finish
// ------------------------------------------------------------------------------------------------------------------
// G[j][n] = sum over the CTAs of (mb = j / 128, slice(n)) of partial[cta][n_local][j % 128]   (float64)
// ng gate columns (512; tanh cell 128), nc0 slice-0 feature columns (x | S | h = 384; tanh cell h = 128)
__global__ void bptt_reduce_partials_kernel(const float* __restrict__ partial, int ng, int nc0, int j0, int j1,
                                            double* __restrict__ G, int ncols_total) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;     // (n, j): j fastest -> coalesced partial reads
  if (idx >= ng * ncols_total) return;
  const int n = idx / ng, j = idx - n * ng;
  const int mb = j >> 7, m = j & 127;
  const int sl = n < nc0 ? 0 : 1, nl = sl == 0 ? n : n - nc0;
  const int per_mb = j0 + j1;
  const int first = mb * per_mb + (sl == 0 ? 0 : j0), cnt = sl == 0 ? j0 : j1;
  double acc = 0.0;
  for (int c = 0; c < cnt; ++c) acc += (double)partial[((size_t)(first + c) * 512 + nl) * 128 + m];
  G[(size_t)j * ncols_total + n] = acc;
}

// out[m][n] (+)= sum_k A[k * lda + m] * B[k * ldb + n]   (float64, tiny matrices: once per update)
__global__ void small_gemm_tn_kernel(int M, int Nn, int K, const double* __restrict__ A, int lda, const double* __restrict__ Bm,
                                     int ldb, double* __restrict__ out, int ldo, int accumulate) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * Nn) return;
  const int m = idx / Nn, n = idx - m * Nn;
  double acc = 0.0;
  for (int k = 0; k < K; ++k) acc += A[(size_t)k * lda + m] * Bm[(size_t)k * ldb + n];
  if (accumulate) out[(size_t)m * ldo + n] += acc;
  else out[(size_t)m * ldo + n] = acc;
}

struct FinishArgs {
  int O, nheads, atot, npos, np, WW;
  int head_dim[IC3_MAX_HEADS];
  const double* G;          // [512][NC] rows = gate column j = 4u + gate
  int NC;
  const double* Y;          // [128][ldy]  W_ih^T Q  (tanh cell: Q itself, the P block of G)
  int ldy;
  const double* GSC;        // [512][128] G_S C^T
  const double* dC;         // [128][128] W_ih^T G_S
  const float* c_b;
  float* g_w_ih; float* g_w_hh; float* g_b_ih; float* g_b_hh; float* g_c_w; float* g_c_b;
  float* g_enc_w; float* g_enc_b; float* g_value_w; float* g_value_b;
  float* g_head_w[IC3_MAX_HEADS]; float* g_head_b[IC3_MAX_HEADS];
  float* g_f_w; float* g_f_b;                               // tanh cell: affine2
  const float* gw_part; const double* gs_part; int nhb;     // heads partials
  double* losses;            // [3] out
  ic3_pp_cfg pp; ic3_tj_cfg tj; int is_tj;
  int ones_col;              // column of P holding the constant 1
};

// LSTM / comm parameter gradients: thread = (LSTM row r = gate * H + u, k)
__global__ void bptt_finish_lstm_kernel(FinishArgs f) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < 512 * TC_H) {
    const int r = idx >> 7, k = idx & 127;
    const int gate = r >> 7, u = r & 127, j = 4 * u + gate;
    const double* Gj = f.G + (size_t)j * f.NC;
    const double g1 = Gj[384 + f.ones_col];                   // sum over rows of d gates (bias gradient)
    f.g_w_hh[idx] += (float)Gj[256 + k];
    f.g_w_ih[idx] += (float)(Gj[k] + f.GSC[(size_t)j * TC_H + k] + g1 * (double)f.c_b[k]);
    if (k == 0) {
      f.g_b_ih[r] += (float)g1;
      f.g_b_hh[r] += (float)g1;
    }
  }
  if (idx < TC_H * TC_H) f.g_c_w[idx] += (float)f.dC[idx];     // [k][m]
}

// tanh cell: d affine2.weight[u][k] = G_h[u][k], d affine2.bias[u] = g1[u]  (G = [h | P], rows = unit u)
__global__ void bptt_finish_tanh_kernel(FinishArgs f) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= TC_H * TC_H) return;
  const int u = idx >> 7, k = idx & 127;
  const double* Gu = f.G + (size_t)u * f.NC;
  f.g_f_w[idx] += (float)Gu[k];
  if (k == 0) f.g_f_b[u] += (float)Gu[TC_H + f.ones_col];
}

// encoder window-cell features per update: W^2 cells x V classes (+ the two TJ scalars)
__host__ __device__ inline int finish_enc_items(const FinishArgs& f) {
  const int W = f.is_tj ? 2 * f.tj.vision + 1 : 2 * f.pp.vision + 1;
  return W * W * (f.is_tj ? f.tj.vocab : f.pp.dim * f.pp.dim + 4) + (f.is_tj ? 2 : 0);
}

// encoder / comm-bias gradients.  Thread = (encoder feature, hidden unit k).  Each feature column of the encoder
// weight [H][O] is written by exactly one thread, which adds up the P columns that feed it (position one-hot columns
// whose window cell holds that class, count and scalar columns) in a fixed order: no atomics, so the gradient is
// bit-identical from run to run.
__global__ void bptt_finish_misc_kernel(FinishArgs f) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int k = idx & 127;
  const double* Yk = f.Y + (size_t)k * f.ldy;
  if (idx < TC_H) {
    const double y1 = Yk[f.ones_col];
    if (f.g_c_b) f.g_c_b[k] += (float)y1;      // W_ih^T g1 (NULL: the tanh RNN's frozen zero C bias gets nothing)
    f.g_enc_b[k] += (float)y1;
  }
  const int W = f.is_tj ? 2 * f.tj.vision + 1 : 2 * f.pp.vision + 1;
  const int WW = W * W;
  const int V = f.is_tj ? f.tj.vocab : f.pp.dim * f.pp.dim + 4;
  const int item = idx >> 7;
  if (item >= finish_enc_items(f)) return;
  if (item >= WW * V) {                        // TJ scalars: last_act; route id ratio (hi + lo columns)
    if (item == WW * V) f.g_enc_w[(size_t)k * f.O] += (float)Yk[f.npos + WW];
    else f.g_enc_w[(size_t)k * f.O + 1] += (float)(Yk[f.npos + WW + 1] + Yk[f.npos + WW + 2]);
    return;
  }
  const int w = item / V, c = item - w * V;    // window cell w, class c
  const int dy = w / W, dx = w - dy * W;
  double y = 0.0;
  bool fed = false;
  if (!f.is_tj) {
    const int D = f.pp.dim, v = f.pp.vision;
    if (c < D * D) {                           // a grid cell: the one position whose window cell w it is
      const int pr = c / D + v - dy, pc = c % D + v - dx;
      if (pr >= 0 && pr < D && pc >= 0 && pc < D) {
        y = Yk[pr * D + pc];
        fed = true;
      }
    } else if (c == V - 3) {                   // outside the grid: every position whose window cell w leaves it
      for (int pos = 0; pos < f.npos; ++pos) {
        const int rr = pos / D - v + dy, cc = pos % D - v + dx;
        if (rr < 0 || rr >= D || cc < 0 || cc >= D) {
          y += Yk[pos];
          fed = true;
        }
      }
    } else if (c >= V - 2) {                   // prey (V - 2) / predator (V - 1) count of window cell w
      y = Yk[f.npos + 2 * w + (c == V - 1 ? 1 : 0)];
      fed = true;
    }
  } else {
    const int v = f.tj.vision;
    for (int pos = 0; pos < f.npos; ++pos) {   // every position whose window cell w holds class c
      const int rr = pos / f.tj.w - v + dy, cc = pos % f.tj.w - v + dx;
      const int cls = (rr >= 0 && rr < f.tj.h && cc >= 0 && cc < f.tj.w) ? f.tj.grid[rr * f.tj.w + cc] : f.tj.outside_cls;
      if (cls == c) {
        y += Yk[pos];
        fed = true;
      }
    }
    if (c == f.tj.car_cls) {                   // car count of window cell w
      y += Yk[f.npos + w];
      fed = true;
    }
  }
  if (fed) f.g_enc_w[(size_t)k * f.O + (f.is_tj ? 2 : 0) + w * V + c] += (float)y;
}

__global__ void bptt_finish_heads_kernel(FinishArgs f) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;     // (o, u)
  if (idx < BP_HEADS * TC_H) {
    const int o = idx >> 7, u = idx & 127;
    double acc = 0.0;
    for (int b = 0; b < f.nhb; ++b) acc += (double)f.gw_part[((size_t)b * BP_HEADS + o) * TC_H + u];
    if (o == 0) {
      f.g_value_w[u] += (float)acc;
    } else {
      int off = 1;
      for (int m = 0; m < f.nheads; ++m) {
        if (o < off + f.head_dim[m]) {
          f.g_head_w[m][(size_t)(o - off) * TC_H + u] += (float)acc;
          break;
        }
        off += f.head_dim[m];
      }
    }
  }
  if (idx < BP_HEADS + 3) {
    double acc = 0.0;
    for (int b = 0; b < f.nhb; ++b) acc += f.gs_part[(size_t)b * (BP_HEADS + 3) + idx];
    if (idx >= BP_HEADS) {
      f.losses[idx - BP_HEADS] = acc;
    } else if (idx == 0) {
      f.g_value_b[0] += (float)acc;
    } else {
      int off = 1;
      for (int m = 0; m < f.nheads; ++m) {
        if (idx < off + f.head_dim[m]) {
          f.g_head_b[m][idx - off] += (float)acc;
          break;
        }
        off += f.head_dim[m];
      }
    }
  }
}

// double copies of the fp32 weights the finishing GEMMs need: W_ih in gate-column order [j][k], C [n][k]
__global__ void bptt_weights_f64_kernel(const float* __restrict__ w_ih, const float* __restrict__ c_w, double* __restrict__ wj,
                                        double* __restrict__ cw) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < 512 * TC_H) {
    const int j = idx >> 7, k = idx & 127;
    const int u = j >> 2, gate = j & 3;
    wj[idx] = (double)w_ih[(size_t)(gate * TC_H + u) * TC_H + k];
  }
  if (idx < TC_H * TC_H) cw[idx] = (double)c_w[idx];
}

// G_S C^T: out[j][k] = sum_m G[j][128 + m] * C[k][m]   -> small_gemm_tn wants A[k'][m'] layout; do it directly
__global__ void bptt_gsc_kernel(const double* __restrict__ G, int NC, const double* __restrict__ cw, double* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 512 * TC_H) return;
  const int j = idx >> 7, k = idx & 127;
  double acc = 0.0;
  for (int m = 0; m < TC_H; ++m) acc += G[(size_t)j * NC + 128 + m] * cw[(size_t)k * TC_H + m];
  out[idx] = acc;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// image of core matrices [tile][(part)][group][rg 16][64 halfs]: box = [64][4 row groups][ngroups_box][1]([1])
int make_image_map(CUtensorMap* map, void* base, int ntiles, int nparts, int ngroups, int box_groups) {
  EncodeTiledFn fn = encode_tiled();
  if (!fn) return IC3_E_UNSUPPORTED;
  if (nparts > 0) {
    cuuint64_t dims[5] = {64, 16, (cuuint64_t)ngroups, (cuuint64_t)nparts, (cuuint64_t)ntiles};
    cuuint64_t strides[4] = {128, 2048, (cuuint64_t)ngroups * 2048, (cuuint64_t)nparts * ngroups * 2048};
    cuuint32_t box[5] = {64, 4, (cuuint32_t)box_groups, 1, 1};
    cuuint32_t es[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? IC3_OK : IC3_E_RANGE;
  }
  cuuint64_t dims[4] = {64, 16, (cuuint64_t)ngroups, (cuuint64_t)ntiles};
  cuuint64_t strides[3] = {128, 2048, (cuuint64_t)ngroups * 2048};
  cuuint32_t box[4] = {64, 4, (cuuint32_t)box_groups, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? IC3_OK : IC3_E_RANGE;
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Side stream of the weight-gradient kernel + the events that order it against the main stream (IC3_BPTT_OVERLAP=0
// keeps everything on the caller's stream).
struct BpttStreams {
  cudaStream_t side;
  cudaEvent_t gates_done[2], wgrad_done[2], prep_done[2], main_done[2];
  bool overlap;
  int prepared_t[2];         // lock-step index whose heads / operand images occupy buffer set q (-1: none)
};

BpttStreams* bptt_streams() {
  static BpttStreams ss;
  static int state = 0;      // 0 = not created, 1 = ok, -1 = failed
  if (state == 0) {
    const char* e = getenv("IC3_BPTT_OVERLAP");
    ss.overlap = !(e && atoi(e) == 0);
    ss.prepared_t[0] = ss.prepared_t[1] = -1;
    bool ok = cudaStreamCreateWithFlags(&ss.side, cudaStreamNonBlocking) == cudaSuccess;
    for (int k = 0; k < 2 && ok; ++k) {
      ok = cudaEventCreateWithFlags(&ss.gates_done[k], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&ss.wgrad_done[k], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&ss.prep_done[k], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&ss.main_done[k], cudaEventDisableTiming) == cudaSuccess;
    }
    state = ok ? 1 : -1;
  }
  return state == 1 ? &ss : nullptr;
}

// The persistent tensor-core kernels leave ~30 KB of an SM's shared memory unused; with the carve-out pinned to the
// maximum (instead of the smallest configuration that fits the kernel) one CTA of the look-ahead kernels (operand images,
// heads gradient) can be resident beside them.
template <typename K>
cudaError_t prefer_max_smem(K kern) {
  return cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

struct Layout {         // of the workspace, in bytes
  size_t a_img, p_img, dg_img, img_stride, w2_img, hc_pass, tc_ws, dout, dSs, dh_direct, gs, gr, partial, part_stride, dout0,
      gw_part, gs_part, sc, G, Y, GSC, dC, wj, cw, losses, total;
  int ntiles, np, npos, WW, j0, j1, ncta_wg, nhb;
  int P;                // comm passes: backward units per lock-step
  int tanh;             // the tanh recurrence without communication (models.RNN, rnn_type 'MLP')
  int ng, nc0;          // gate columns (512; tanh 128) and slice-0 feature columns of G (x | S | h = 384; tanh h = 128)
};

int plan_layout(const ic3_policy_cfg* cfg, int npos, int WW, int is_tj, Layout* L) {
  // the LSTM-cell policies of the tensor-core path, 1 .. IC3_MAX_PASSES comm passes; the tanh recurrence with one pass
  // and no communication (comm_mask_zero, no hard attention: the IC / IRIC baselines of the SIMT path)
  if (cfg->x_tanh || cfg->h_from_x || cfg->passes > IC3_MAX_PASSES) return IC3_E_UNSUPPORTED;
  const bool tanh_cell = cfg->cell == IC3_CELL_TANH && cfg->passes <= 1 && cfg->comm_mask_zero && !cfg->hard_attn;
  if (cfg->cell != IC3_CELL_LSTM && !tanh_cell) return IC3_E_UNSUPPORTED;
  L->tanh = tanh_cell;
  L->ng = tanh_cell ? TC_H : 4 * TC_H;
  L->nc0 = tanh_cell ? TC_H : 3 * TC_H;
  L->P = cfg->passes > 1 ? cfg->passes : 1;
  const long R = (long)cfg->B * cfg->N;
  L->ntiles = (int)((R + TC_M - 1) / TC_M);
  L->npos = npos;
  L->WW = WW;
  const int used = npos + (is_tj ? WW + 4 : 2 * WW + 1);
  L->np = (used + 15) / 16 * 16;
  if (L->np > WG_MAX_NP) return IC3_E_UNSUPPORTED;
  const int nmb = L->ng / 128;             // gate-column blocks
  const int per_mb = sm_count() / (2 * nmb);   // nmb gate-column blocks x per_mb roles x 2 CTAs: one CTA per SM
  if (per_mb < 2) return IC3_E_UNSUPPORTED;
  // MMA cycles per 16 rows: slice 0 = 3 * (128 + 86) for x | S | h (a third of it for the h block alone), slice 1 =
  // 2 * (n0 + n1 shapes) -> split the CTAs accordingly
  const double c0 = 3.0 * (128 + 86) * L->nc0 / 384.0;
  const double c1 = 2.0 * (L->np > 256 ? 128 + 0.5 * (L->np - 256) + 22 : 0.5 * L->np + 22);
  int j0 = (int)(per_mb * c0 / (c0 + c1) + 0.5);
  if (j0 < 1) j0 = 1;
  if (j0 > per_mb - 1) j0 = per_mb - 1;
  L->j0 = j0;
  L->j1 = per_mb - j0;
  L->ncta_wg = nmb * per_mb;               // roles (weight-gradient partials); the kernel runs two CTAs per role
  L->nhb = (int)((R + HB_ROWS - 1) / HB_ROWS);
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 1023) / 1024 * 1024; return o; };
  // two sets of operand images (step parity): the weight-gradient kernel of step t reads set t & 1 on the side stream
  // while the main stream fills the other set for step t - 1
  L->a_img = take((size_t)L->ntiles * A_TILE_HALFS * 2);
  L->p_img = take((size_t)L->ntiles * (L->np / 8) * 16 * 128);
  L->dg_img = take((size_t)L->ntiles * (tanh_cell ? DZ_TILE_HALFS : DG_TILE_HALFS) * 2);
  L->img_stride = off;
  take(off);                                   // second set: same sizes, same order
  L->w2_img = take((size_t)L->P * (tanh_cell ? W2_IMG_HALFS_TANH : W2_IMG_HALFS) * 2);   // one dgrad weight image per pass
  // comm_passes > 1: (h, c) after passes 0 .. P-2 of the step being differentiated (re-run from the record by
  // ic3_tc_pass_states), and the scratch of that re-run (operand image, head partials)
  ic3_policy_cfg one_pass = *cfg;
  one_pass.passes = 1;
  L->hc_pass = take(L->P > 1 ? (size_t)(L->P - 1) * 2 * R * TC_H * 4 : 0);
  L->tc_ws = take(L->P > 1 ? (size_t)ic3_tc_workspace_bytes(&one_pass) : 0);
  L->dout = take((size_t)2 * L->ntiles * TC_M * BP_HEADS * 4);         // [2]: heads of step t - 1 run while step t reads
  L->dSs = take(tanh_cell ? 0 : (size_t)L->ntiles * TC_M * TC_H * 4);
  L->dh_direct = take((size_t)L->ntiles * TC_M * TC_H * 4);
  L->gs = take((size_t)2 * L->ntiles * TC_M * 4);                       // [2] by step parity, like the images
  L->gr = take((size_t)2 * L->ntiles * TC_M * 4);
  // weight-gradient partials per pass: the S block and the constant column of G belong to pass p's C_modules[p]
  L->part_stride = (size_t)L->ncta_wg * 512 * 128 * 4;
  L->partial = take((size_t)L->P * L->part_stride);
  L->dout0 = take(L->P > 1 ? (size_t)L->ntiles * TC_M * BP_HEADS * 4 : 0);   // zeros: no heads after passes < P-1
  L->gw_part = take((size_t)L->nhb * BP_HEADS * TC_H * 4);
  L->gs_part = take((size_t)L->nhb * (BP_HEADS + 3) * 8);
  L->sc = take(sizeof(BpttScalars));
  const int NC = L->nc0 + L->np;
  L->G = take((size_t)L->ng * NC * 8);
  // the LSTM cell's folds through W_ih and C (the tanh cell reads its G directly)
  const int lstm = tanh_cell ? 0 : 1;
  L->Y = take(lstm * (size_t)TC_H * L->np * 8);
  L->GSC = take(lstm * (size_t)512 * TC_H * 8);
  L->dC = take(lstm * (size_t)TC_H * TC_H * 8);
  L->wj = take(lstm * (size_t)512 * TC_H * 8);
  L->cw = take(lstm * (size_t)TC_H * TC_H * 8);
  L->losses = take(3 * 8);
  L->total = off;
  return IC3_OK;
}

int env_geometry(const ic3_bptt_plan* p, int* npos, int* WW, int* is_tj) {
  if (p->pp_env) {
    const int W = 2 * p->pp_env->vision + 1;
    *npos = p->pp_env->dim * p->pp_env->dim;
    *WW = W * W;
    *is_tj = 0;
  } else if (p->tj_env) {
    const int W = 2 * p->tj_env->vision + 1;
    *npos = p->tj_env->h * p->tj_env->w;
    *WW = W * W;
    *is_tj = 1;
  } else {
    return IC3_E_NULL;
  }
  if (*WW > PREP_MAX_WW) return IC3_E_UNSUPPORTED;
  return IC3_OK;
}

// The recorded env state of ic3_bptt_step_io / ic3_ff_grad_io: the fields the backward reads must be set.
int records_check(const ic3_pp_state* pp, const ic3_tj_state* tj, int is_tj) {
  if (is_tj) return tj && tj->loc && tj->alive && tj->last_act && tj->route_id ? IC3_OK : IC3_E_NULL;
  return pp && pp->loc ? IC3_OK : IC3_E_NULL;
}

}  // namespace

extern "C" uint64_t ic3_bptt_workspace_bytes(const ic3_bptt_plan* p) {
  if (!p || !p->cfg || p->cfg->H != TC_H) return 0;
  int npos, WW, is_tj;
  if (env_geometry(p, &npos, &WW, &is_tj)) return 0;
  // the operand images sum the class terms apart from the counts (ic3_policy_cfg.obs_vocab): the environment's own
  // layout hint is required
  if (p->cfg->obs_vocab == 0 || (is_tj ? ic3_tj_layout_check(p->tj_env, p->cfg) : ic3_pp_layout_check(p->pp_env, p->cfg)))
    return 0;
  Layout L;
  if (plan_layout(p->cfg, npos, WW, is_tj, &L)) return 0;
  int nout = 1;
  for (int k = 0; k < p->cfg->nheads; ++k) nout += p->cfg->head_dim[k];
  if (nout > BP_HEADS) return 0;
  return (uint64_t)L.total;
}

// Zero the accumulators and scalars (partial .. end of the workspace) and build the dgrad weight image(s).
static int bptt_reset(const ic3_bptt_plan* p, const Layout& L, cudaStream_t s) {
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  cudaError_t e = cudaMemsetAsync(ws + L.partial, 0, L.total - L.partial, s);   // partial .. end: all accumulators / scalars
  if (e != cudaSuccess) return (int)e;
  if (L.tanh) {                                // SIMT-packed weights: no forward image, the dgrad image comes from f_wT
    bptt_pack_w2_tanh_kernel<<<(256 * TC_H + 255) / 256, 256, 0, s>>>(p->w->f_wT, reinterpret_cast<__half*>(ws + L.w2_img));
    IC3_LAUNCH_CHECK();
  }
  for (int ps = 0; ps < L.P && !L.tanh; ++ps) {   // w->lstm_img holds the forward image of every pass, back to back
    bptt_pack_w2_kernel<<<(256 * 512 + 255) / 256, 256, 0, s>>>(
        reinterpret_cast<const __half*>(p->w->lstm_img) + (size_t)ps * B_IMG_HALFS,
        reinterpret_cast<__half*>(ws + L.w2_img) + (size_t)ps * W2_IMG_HALFS);
    IC3_LAUNCH_CHECK();
  }
  BpttStreams* ss = bptt_streams();
  if (!ss) return IC3_E_UNSUPPORTED;
  ss->prepared_t[0] = ss->prepared_t[1] = -1;
  return IC3_OK;
}

// Start of a compute_grad: zero the accumulators and both operand-image sets, build the dgrad weight image, set max |c|.
extern "C" int ic3_bptt_begin(const ic3_bptt_plan* p, float cmax, void* stream) {
  if (!p || !p->cfg || !p->w || !p->workspace) return IC3_E_NULL;
  int npos, WW, is_tj;
  int rc = env_geometry(p, &npos, &WW, &is_tj);
  if (rc) return rc;
  Layout L;
  rc = plan_layout(p->cfg, npos, WW, is_tj, &L);
  if (rc) return rc;
  if (L.tanh && !p->w->f_wT) return IC3_E_NULL;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  rc = bptt_reset(p, L, s);
  if (rc) return rc;
  cudaError_t e = cudaMemsetAsync(ws + L.a_img, 0, L.w2_img - L.a_img, s);      // both image sets
  if (e != cudaSuccess) return (int)e;
  BpttStreams* ss = bptt_streams();
  BpttScalars init;
  memset(&init, 0, sizeof(init));
  // the cell states entering passes 1 .. P-1 are not in the record: each pass changes |c| by at most 1
  // (|f c + i g| <= |c| + 1), so |c^p| <= |c_{t-1}| + p bounds them
  init.cmax = L.P > 1 ? cmax + (float)(L.P - 1) : cmax;
  init.scale[0] = init.scale[1] = 1.f;
  init.inv_scale[0] = init.inv_scale[1] = 1.f;
  e = cudaMemcpyAsync(ws + L.sc, &init, sizeof(init), cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return (int)e;
  // the look-ahead kernels of the first two steps (side stream) must see the zeroed accumulators -- and everything the
  // caller enqueued before this call (returns, advantages, the rollout records)
  for (int k = 0; k < 2; ++k) {
    e = cudaEventRecord(ss->main_done[k], s);
    if (e != cudaSuccess) return (int)e;
  }
  return IC3_OK;
}

// Recursion-independent part of a backward unit (step t, comm pass ps): the operand images of the pass (prep) from
// the state h_in entering it, and -- for the last pass only -- d loss / d outputs from the records (heads).  Runs on
// `s` into buffer set q (parity of the unit counter t * P + ps).
// up != NULL: the heads take the caller's upstream gradients (ic3_policy_step_backward) instead of the records.
static int bptt_prepare_on(const ic3_bptt_plan* p, const ic3_bptt_step_io* io, const Layout& L, int npos, int is_tj,
                           cudaStream_t s, int q, int ps, const float* h_in, const ic3_policy_bwd_io* up) {
  const ic3_policy_cfg* cfg = p->cfg;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  const int R = cfg->B * cfg->N;
  int atot = 0;
  for (int k = 0; k < cfg->nheads; ++k) atot += cfg->head_dim[k];
  BpttScalars* sc = reinterpret_cast<BpttScalars*>(ws + L.sc);
  const size_t rows_pad = (size_t)L.ntiles * TC_M;
  __half* a_img = reinterpret_cast<__half*>(ws + L.a_img + (size_t)q * L.img_stride);
  __half* p_img = reinterpret_cast<__half*>(ws + L.p_img + (size_t)q * L.img_stride);
  // ---- operand images of pass ps of step t from the records ----
  ic3_policy_io pio;
  memset(&pio, 0, sizeof(pio));
  pio.h = h_in; pio.c = io->c_prev; pio.comm_action = io->comm; pio.alive = io->alive; pio.fresh = io->fresh;
  pio.err = io->err;
  pio.pass_index = ps;                 // a fresh slot's zero state and silent first pass apply to pass 0 only
  PrepSrc src;
  memset(&src, 0, sizeof(src));
  // tanh cell: x is no operand of its GEMMs (the x block of the image stays zero), so it needs no table
  src.wT = p->w->enc_wT; src.bias = p->w->enc_b; src.split = cfg->obs_vocab > 0; src.table = L.tanh ? nullptr : p->x_table;
  src.wflags = p->w->flags;
  if ((!src.table && !L.tanh) || !src.split) return IC3_E_NULL;
  PrepBwd bw;
  bw.p_img = p_img;
  bw.gs = reinterpret_cast<float*>(ws + L.gs) + (size_t)q * rows_pad;
  bw.gr = reinterpret_cast<float*>(ws + L.gr) + (size_t)q * rows_pad;
  bw.npg = L.np / 8;
  bw.npos = npos;
  const int ntiles = L.ntiles;
  if (!is_tj) {
    src.pp = *p->pp_env;
    src.pps = *io->pp_state;
    prep_kernel<XSRC_PP, true, true><<<2 * ntiles, PREP_THREADS, prep_T_bytes(cfg->N), s>>>(*cfg, pio, a_img, src, bw);
    IC3_LAUNCH_CHECK();
  } else {
    src.tj = *p->tj_env;
    src.tjs = *io->tj_state;
    prep_kernel<XSRC_TJ, true, true><<<2 * ntiles, PREP_THREADS, prep_T_bytes(cfg->N), s>>>(*cfg, pio, a_img, src, bw);
    IC3_LAUNCH_CHECK();
  }
  if (ps != L.P - 1) return IC3_OK;    // heads and loss act on the last pass's h'
  // ---- heads ----
  HeadsArgs ha;
  memset(&ha, 0, sizeof(ha));
  ha.R = R; ha.N = cfg->N; ha.nheads = cfg->nheads; ha.atot = atot;
  for (int k = 0; k < IC3_MAX_HEADS; ++k) ha.head_dim[k] = cfg->head_dim[k];
  ha.value_coeff = p->value_coeff; ha.entr = p->entr;
  ha.logp = io->logp; ha.action = io->action; ha.value = io->value; ha.ret = io->ret; ha.adv = io->adv;
  ha.alive_post = io->alive_post; ha.valid = io->valid; ha.h_new = io->h_new; ha.head_w = p->w->head_w;
  ha.dout = reinterpret_cast<float*>(ws + L.dout) + (size_t)q * rows_pad * BP_HEADS;
  ha.gw_part = reinterpret_cast<float*>(ws + L.gw_part);
  ha.gs_part = reinterpret_cast<double*>(ws + L.gs_part);
  ha.sc = sc;
  ha.q = q;
  if (up) {
    ha.dlogp = up->dlogp; ha.dvalue = up->dvalue;
    bptt_heads_kernel<true><<<L.nhb, 256, 0, s>>>(ha);
  } else {
    bptt_heads_kernel<false><<<L.nhb, 256, 0, s>>>(ha);
  }
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

static int bptt_common(const ic3_bptt_plan* p, const ic3_bptt_step_io* io, Layout* L, int* npos, int* is_tj) {
  if (!p || !io || !p->cfg || !p->w || !p->workspace) return IC3_E_NULL;
  if (!io->h_prev || !io->h_new || !io->logp || !io->action || !io->value || !io->ret || !io->adv || !io->alive_post ||
      !io->dh)
    return IC3_E_NULL;
  if (p->cfg->H != TC_H) return IC3_E_UNSUPPORTED;
  int WW;
  int rc = env_geometry(p, npos, &WW, is_tj);
  if (rc) return rc;
  rc = plan_layout(p->cfg, *npos, WW, *is_tj, L);
  if (rc) return rc;
  if (!L->tanh && (!io->c_prev || !io->dc)) return IC3_E_NULL;     // the tanh cell has no c
  if (p->cfg->hard_attn && !io->comm) return IC3_E_NULL;
  if (records_check(io->pp_state, io->tj_state, *is_tj)) return IC3_E_NULL;
  int nout = 1;
  for (int k = 0; k < p->cfg->nheads; ++k) nout += p->cfg->head_dim[k];
  return nout > BP_HEADS ? IC3_E_UNSUPPORTED : IC3_OK;
}

// Optional: launch the recursion-independent kernels of step io->t (heads, operand images) AHEAD of ic3_bptt_step(t),
// on the library's side stream, so that they overlap the tensor-core kernels of step t + 1 (which leave one CTA slot
// per SM free).  `stream` is the stream ic3_bptt_step will be called on.  Without this call (or with
// IC3_BPTT_OVERLAP=0) ic3_bptt_step runs them itself.
// comm_passes > 1: a no-op.  The units (t, p) of a step alternate the two buffer sets, so the set the look-ahead of
// step t - 1 would fill is the one unit (t, 1) uses, and the operand images of passes >= 1 need the re-run pass
// states; ic3_bptt_step then prepares every unit inline (the weight-gradient kernels still run on the side stream).
extern "C" int ic3_bptt_prepare(const ic3_bptt_plan* p, const ic3_bptt_step_io* io, void* stream) {
  Layout L;
  int npos, is_tj;
  int rc = bptt_common(p, io, &L, &npos, &is_tj);
  if (rc) return rc;
  BpttStreams* ss = bptt_streams();
  if (!ss) return IC3_E_UNSUPPORTED;
  if (!ss->overlap || L.P > 1) return IC3_OK;       // ic3_bptt_step will do it inline
  const int q = io->t & 1;
  // buffer set q was last used by step t + 2: its main-stream kernels (gates / dgrad / comm read A, dout, gs, gr) and
  // its weight-gradient kernel (side stream, already ordered before this call)
  cudaError_t e = cudaStreamWaitEvent(ss->side, ss->main_done[q], 0);
  if (e != cudaSuccess) return (int)e;
  rc = bptt_prepare_on(p, io, L, npos, is_tj, ss->side, q, 0, io->h_prev, nullptr);
  if (rc) return rc;
  e = cudaEventRecord(ss->prep_done[q], ss->side);
  if (e != cudaSuccess) return (int)e;
  ss->prepared_t[q] = io->t;
  return IC3_OK;
}

// One backward unit: comm pass ps of step io->t, entered with state (h_in, c_in), on buffer set q.  The incoming
// io->dh / io->dc are d loss / d (h, c) leaving the pass; they are replaced by d loss / d (h_in, c_in).
static int bptt_unit(const ic3_bptt_plan* p, const ic3_bptt_step_io* io, const Layout& L, int npos, int is_tj,
                     cudaStream_t s, int q, int ps, const float* h_in, const float* c_in, const ic3_policy_bwd_io* up) {
  int rc;
  const ic3_policy_cfg* cfg = p->cfg;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  const int R = cfg->B * cfg->N;
  int nout = 1;
  for (int k = 0; k < cfg->nheads; ++k) nout += cfg->head_dim[k];
  BpttScalars* sc = reinterpret_cast<BpttScalars*>(ws + L.sc);
  const size_t rows_pad = (size_t)L.ntiles * TC_M;
  const int ntiles = L.ntiles;
  const bool first = ps == 0, last = ps == L.P - 1;
  __half* a_img = reinterpret_cast<__half*>(ws + L.a_img + (size_t)q * L.img_stride);
  __half* dg_img = reinterpret_cast<__half*>(ws + L.dg_img + (size_t)q * L.img_stride);
  BpttStreams* ss = bptt_streams();
  if (!ss) return IC3_E_UNSUPPORTED;
  // buffer set q (images, scale) was last read by the weight-gradient kernel of unit u + 2 (side stream)
  cudaError_t se = cudaStreamWaitEvent(s, ss->wgrad_done[q], 0);
  if (se != cudaSuccess) return (int)se;
  if (L.P == 1 && ss->prepared_t[q] == io->t) {    // heads + images were launched ahead (ic3_bptt_prepare)
    se = cudaStreamWaitEvent(s, ss->prep_done[q], 0);
    if (se != cudaSuccess) return (int)se;
    ss->prepared_t[q] = -1;
  } else {
    rc = bptt_prepare_on(p, io, L, npos, is_tj, s, q, ps, h_in, up);
    if (rc) return rc;
  }
  bptt_scale_kernel<<<1, 1, 0, s>>>(sc, q);
  IC3_LAUNCH_CHECK();

  // ---- tanh cell: dz image (takes the place of the gate GEMM) ----
  if (L.tanh) {
    TanhArgs ta;
    ta.R = R; ta.N = cfg->N; ta.nrows = ntiles * TC_M; ta.cut = io->cut;
    ta.dout = reinterpret_cast<const float*>(ws + L.dout) + (size_t)q * rows_pad * BP_HEADS;
    ta.h_new = io->h_new; ta.dh = io->dh; ta.head_w = (const float*)p->w->head_w; ta.nout = nout;
    ta.dz_img = dg_img; ta.sc = sc; ta.q = q;
    bptt_tanh_kernel<<<ntiles * (TC_M / TZ_ROWS), 256, 0, s>>>(ta);
    IC3_LAUNCH_CHECK();
    se = cudaEventRecord(ss->gates_done[q], s);
    if (se != cudaSuccess) return (int)se;
  }
  // ---- gates ----
  if (!L.tanh) {
    static bool cfgd = false;
    const size_t smem = NSTAGE_P * STAGE_BYTES + 256 + TC_H * HEAD_PAD * sizeof(float) + 4 * TC_H * sizeof(float);
    if (!cfgd) {
      cudaError_t e = cudaFuncSetAttribute(bptt_gates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return (int)e;
      prefer_max_smem(bptt_gates_kernel);
      cfgd = true;
    }
    // the episode start zeroes the state entering pass 0; the detach cut drops what reaches the step's output (the
    // last pass) from later steps; heads act on the last pass only (passes before it read a zero d outputs block)
    GatesArgs ga;
    ga.R = R; ga.N = cfg->N; ga.c_prev = c_in; ga.fresh = first ? io->fresh : nullptr; ga.cut = last ? io->cut : nullptr;
    ga.dout = last ? reinterpret_cast<const float*>(ws + L.dout) + (size_t)q * rows_pad * BP_HEADS
                   : reinterpret_cast<const float*>(ws + L.dout0);
    ga.dh = io->dh; ga.dc = io->dc; ga.dg_img = dg_img; ga.sc = sc;
    ga.q = q;
    ga.err = io->err;
    const int nitems = 2 * ntiles;
    const int grid = nitems < sm_count() ? nitems : sm_count();
    bptt_gates_kernel<<<grid, TC_P_THREADS, smem, s>>>(
        ga, a_img, reinterpret_cast<const __half*>(p->w->lstm_img) + (size_t)ps * B_IMG_HALFS,
        (const float*)p->w->bias_cat + (size_t)ps * 4 * TC_H, nitems, (const float*)p->w->head_w, nout);
    IC3_LAUNCH_CHECK();
    se = cudaEventRecord(ss->gates_done[q], s);
    if (se != cudaSuccess) return (int)se;
  }
  // ---- dgrad ----
  {
    static bool cfgd = false;
    const size_t smem = NSTAGE_P * DGR_STAGE + 256;
    if (!cfgd) {
      for (auto kern : {bptt_dgrad_kernel<DGR_NCHUNK>, bptt_dgrad_kernel<DGR_NCHUNK_TANH>}) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
        prefer_max_smem(kern);
      }
      cfgd = true;
    }
    DgradArgs da;
    da.R = R; da.gs = reinterpret_cast<const float*>(ws + L.gs) + (size_t)q * rows_pad;
    da.dSs = L.tanh ? nullptr : reinterpret_cast<float*>(ws + L.dSs);
    da.dh_direct = reinterpret_cast<float*>(ws + L.dh_direct); da.sc = sc; da.q = q; da.err = io->err;
    const int grid = ntiles < sm_count() ? ntiles : sm_count();
    const __half* w2 = reinterpret_cast<const __half*>(ws + L.w2_img);
    if (L.tanh)
      bptt_dgrad_kernel<DGR_NCHUNK_TANH><<<grid, TC_P_THREADS, smem, s>>>(da, dg_img, w2, ntiles);
    else
      bptt_dgrad_kernel<DGR_NCHUNK><<<grid, TC_P_THREADS, smem, s>>>(da, dg_img, w2 + (size_t)ps * W2_IMG_HALFS, ntiles);
    IC3_LAUNCH_CHECK();
  }
  // ---- comm backward -> dh_{t-1} ----
  {
    CommArgs ca;
    ca.B = cfg->B; ca.N = cfg->N; ca.dSs = reinterpret_cast<const float*>(ws + L.dSs);
    ca.dh_direct = reinterpret_cast<const float*>(ws + L.dh_direct); ca.gr = reinterpret_cast<const float*>(ws + L.gr) + (size_t)q * rows_pad;
    ca.fresh = first ? io->fresh : nullptr; ca.no_comm = cfg->comm_mask_zero || cfg->N < 2; ca.dh = io->dh; ca.sc = sc;
    bptt_comm_kernel<<<(cfg->B + 7) / 8, 256, 0, s>>>(ca);
    IC3_LAUNCH_CHECK();
    se = cudaEventRecord(ss->main_done[q], s);          // buffer set q may be refilled for unit u - 2 once wgrad(u) is done too
    if (se != cudaSuccess) return (int)se;
  }
  // ---- weight gradients: on the side stream, overlapping the small kernels of this and the next step ----
  {
    static bool cfgd = false;
    static CUtensorMap map_dg[2], map_a[2], map_p[2];
    static void* key_ws = nullptr;
    static int key_tiles = 0, key_np = 0, key_tanh = 0;
    const size_t smem1 = (size_t)WG_NSTAGE1 * (2 * WG_DG_BYTES + (size_t)L.np * 64);
    const size_t smem = (size_t)WG_NSTAGE0 * WG_STAGE0 > smem1 ? (size_t)WG_NSTAGE0 * WG_STAGE0 : smem1;
    if (!cfgd) {
      cudaError_t e = cudaFuncSetAttribute(bptt_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      if (e != cudaSuccess) return (int)e;
      prefer_max_smem(bptt_wgrad_kernel);
      prefer_max_smem(bptt_heads_kernel<false>);
      prefer_max_smem(bptt_heads_kernel<true>);
      prefer_max_smem(bptt_comm_kernel);
      prefer_max_smem(prep_kernel<XSRC_PP, true, true>);
      prefer_max_smem(prep_kernel<XSRC_TJ, true, true>);
      cfgd = true;
    }
    if (smem > 200 * 1024) return IC3_E_UNSUPPORTED;
    if (key_ws != p->workspace || key_tiles != ntiles || key_np != L.np || key_tanh != L.tanh) {
      for (int k = 0; k < 2; ++k) {
        rc = make_image_map(&map_dg[k], ws + L.dg_img + (size_t)k * L.img_stride, ntiles, 2, L.ng / 8, 16);
        if (rc) return rc;
        // tanh cell: the box is the h block alone (16 of the 48 feature groups)
        rc = make_image_map(&map_a[k], ws + L.a_img + (size_t)k * L.img_stride, ntiles, 2, 48, L.tanh ? 16 : 48);
        if (rc) return rc;
        rc = make_image_map(&map_p[k], ws + L.p_img + (size_t)k * L.img_stride, ntiles, 0, L.np / 8, L.np / 8);
        if (rc) return rc;
      }
      key_ws = p->workspace; key_tiles = ntiles; key_np = L.np; key_tanh = L.tanh;
    }
    WgradArgs wa;
    wa.ntiles = ntiles; wa.np = L.np; wa.j0 = L.j0; wa.j1 = L.j1; wa.h_only = L.tanh;
    wa.partial = reinterpret_cast<float*>(ws + L.partial + (size_t)ps * L.part_stride); wa.sc = sc; wa.q = q; wa.err = io->err;
    cudaStream_t ws_stream = ss->overlap ? ss->side : s;
    if (ss->overlap) {
      se = cudaStreamWaitEvent(ws_stream, ss->gates_done[q], 0);
      if (se != cudaSuccess) return (int)se;
    }
    bptt_wgrad_kernel<<<2 * L.ncta_wg, WG_THREADS, smem, ws_stream>>>(wa, map_dg[q], map_a[q], map_p[q]);
    IC3_LAUNCH_CHECK();
    se = cudaEventRecord(ss->wgrad_done[q], ws_stream);
    if (se != cudaSuccess) return (int)se;
  }
  return IC3_OK;
}

// Step t = the units (t, P-1) .. (t, 0).  With P > 1 comm passes the states entering passes 1 .. P-1 are re-run first
// from the record (h_{t-1}, c_{t-1}) with the rollout's own kernels (ic3_tc_pass_states).
static int bptt_step_on(const ic3_bptt_plan* p, const ic3_bptt_step_io* io, const Layout& L, int npos, int is_tj,
                        cudaStream_t s, const ic3_policy_bwd_io* up) {
  int rc;
  if (L.P == 1) return bptt_unit(p, io, L, npos, is_tj, s, io->t & 1, 0, io->h_prev, io->c_prev, up);
  const ic3_policy_cfg* cfg = p->cfg;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  const size_t RH = (size_t)cfg->B * cfg->N * TC_H;
  float* h_pass = reinterpret_cast<float*>(ws + L.hc_pass);     // [P-1][R][H]: state after pass 0 .. P-2
  float* c_pass = h_pass + (size_t)(L.P - 1) * RH;
  ic3_policy_io pio;
  memset(&pio, 0, sizeof(pio));
  pio.h = io->h_prev; pio.c = io->c_prev; pio.comm_action = io->comm; pio.alive = io->alive; pio.fresh = io->fresh;
  pio.err = io->err; pio.x_table = p->x_table;
  pio.workspace = ws + L.tc_ws;
  if (!is_tj) {
    pio.pp_env = p->pp_env; pio.pp_state = io->pp_state;
  } else {
    pio.tj_env = p->tj_env; pio.tj_state = io->tj_state;
  }
  rc = ic3_tc_pass_states(cfg, p->w, &pio, L.P - 1, h_pass, c_pass, s);
  if (rc) return rc;
  for (int ps = L.P - 1; ps >= 0; --ps) {
    const int q = (io->t * L.P + ps) & 1;                 // unit counter parity: consecutive units alternate sets
    const float* h_in = ps == 0 ? io->h_prev : h_pass + (size_t)(ps - 1) * RH;
    const float* c_in = ps == 0 ? io->c_prev : c_pass + (size_t)(ps - 1) * RH;
    rc = bptt_unit(p, io, L, npos, is_tj, s, q, ps, h_in, c_in, up);
    if (rc) return rc;
  }
  return IC3_OK;
}

extern "C" int ic3_bptt_step(const ic3_bptt_plan* p, const ic3_bptt_step_io* io, void* stream) {
  Layout L;
  int npos, is_tj;
  int rc = bptt_common(p, io, &L, &npos, &is_tj);
  if (rc) return rc;
  return bptt_step_on(p, io, L, npos, is_tj, (cudaStream_t)stream, nullptr);
}

// After step 0: fold the accumulators into the parameter gradients (added to what the buffers hold) and return the
// three loss sums (action_loss, value_loss, entropy) in losses[3] (device, float64).
extern "C" int ic3_bptt_finish(const ic3_bptt_plan* p, const ic3_policy_params* params, const ic3_policy_params* grads,
                               double* losses, void* stream) {
  if (!p || !params || !grads || !losses || !p->cfg || !p->workspace) return IC3_E_NULL;
  const ic3_policy_cfg* cfg = p->cfg;
  int npos, WW, is_tj;
  int rc = env_geometry(p, &npos, &WW, &is_tj);
  if (rc) return rc;
  Layout L;
  rc = plan_layout(cfg, npos, WW, is_tj, &L);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  if (BpttStreams* ss = bptt_streams()) {       // the last weight-gradient kernels may still run on the side stream
    for (int k = 0; k < 2; ++k) {
      cudaError_t e = cudaStreamWaitEvent(s, ss->wgrad_done[k], 0);
      if (e != cudaSuccess) return (int)e;
    }
  }
  const int NC = L.nc0 + L.np;
  double* G = reinterpret_cast<double*>(ws + L.G);
  double* Y = reinterpret_cast<double*>(ws + L.Y);
  double* GSC = reinterpret_cast<double*>(ws + L.GSC);
  double* dC = reinterpret_cast<double*>(ws + L.dC);
  double* wj = reinterpret_cast<double*>(ws + L.wj);
  double* cw = reinterpret_cast<double*>(ws + L.cw);
  FinishArgs f;
  memset(&f, 0, sizeof(f));
  int atot = 0;
  for (int k = 0; k < cfg->nheads; ++k) atot += cfg->head_dim[k];
  f.O = cfg->O; f.nheads = cfg->nheads; f.atot = atot; f.npos = npos; f.np = L.np; f.WW = WW;
  for (int k = 0; k < IC3_MAX_HEADS; ++k) f.head_dim[k] = cfg->head_dim[k];
  f.G = G; f.NC = NC; f.Y = Y; f.ldy = L.np; f.GSC = GSC; f.dC = dC;
  f.g_w_ih = const_cast<float*>(grads->w_ih); f.g_w_hh = const_cast<float*>(grads->w_hh);
  f.g_b_ih = const_cast<float*>(grads->b_ih); f.g_b_hh = const_cast<float*>(grads->b_hh);
  f.g_enc_w = const_cast<float*>(grads->encoder_w); f.g_enc_b = const_cast<float*>(grads->encoder_b);
  f.g_value_w = const_cast<float*>(grads->value_w); f.g_value_b = const_cast<float*>(grads->value_b);
  for (int k = 0; k < IC3_MAX_HEADS; ++k) {
    f.g_head_w[k] = const_cast<float*>(grads->head_w[k]);
    f.g_head_b[k] = const_cast<float*>(grads->head_b[k]);
  }
  f.gw_part = reinterpret_cast<const float*>(ws + L.gw_part);
  f.gs_part = reinterpret_cast<const double*>(ws + L.gs_part);
  f.nhb = L.nhb;
  f.losses = losses;
  f.is_tj = is_tj;
  if (is_tj) f.tj = *p->tj_env;
  else f.pp = *p->pp_env;
  f.ones_col = npos + (is_tj ? WW + 3 : 2 * WW);     // the constant column of P is its last used column
  if (L.tanh) {
    // G = [G_h | Q]: affine2 from G_h and g1; affine1 through the observation layout with Y = Q (d x = dz)
    f.g_f_w = const_cast<float*>(grads->f_w_pass[0]);
    f.g_f_b = const_cast<float*>(grads->f_b_pass[0]);
    if (!f.g_f_w || !f.g_f_b) return IC3_E_NULL;
    bptt_reduce_partials_kernel<<<(L.ng * NC + 255) / 256, 256, 0, s>>>(
        reinterpret_cast<const float*>(ws + L.partial), L.ng, L.nc0, L.j0, L.j1, G, NC);
    IC3_LAUNCH_CHECK();
    bptt_finish_tanh_kernel<<<(TC_H * TC_H + 255) / 256, 256, 0, s>>>(f);
    IC3_LAUNCH_CHECK();
    f.Y = G + L.nc0;
    f.ldy = NC;
    f.g_c_b = nullptr;
    bptt_finish_misc_kernel<<<(finish_enc_items(f) * 128 + 255) / 256, 256, 0, s>>>(f);
    IC3_LAUNCH_CHECK();
  }
  // One fold per comm pass, in pass order, each ADDING its share: pass p's partials hold G_x, G_h and the P columns of
  // its units (summed over the passes by the additions) and its own S block / constant column, which go with
  // C_modules[p] (share_weights: every pass adds into the one module's gradient buffers).
  for (int ps = 0; ps < L.P && !L.tanh; ++ps) {
    const bool own = ps > 0;                           // pass 0 is c_w / c_b, as in ic3_policy_pack
    const float* c_w = own && params->c_w_pass[ps] ? params->c_w_pass[ps] : params->c_w;
    const float* c_b = own && params->c_b_pass[ps] ? params->c_b_pass[ps] : params->c_b;
    const float* g_c_w = own && grads->c_w_pass[ps] ? grads->c_w_pass[ps] : grads->c_w;
    const float* g_c_b = own && grads->c_b_pass[ps] ? grads->c_b_pass[ps] : grads->c_b;
    if (!c_w || !c_b || !g_c_w || !g_c_b) return IC3_E_NULL;
    bptt_reduce_partials_kernel<<<(L.ng * NC + 255) / 256, 256, 0, s>>>(
        reinterpret_cast<const float*>(ws + L.partial + (size_t)ps * L.part_stride), L.ng, L.nc0, L.j0, L.j1, G, NC);
    IC3_LAUNCH_CHECK();
    bptt_weights_f64_kernel<<<(512 * TC_H + 255) / 256, 256, 0, s>>>(params->w_ih, c_w, wj, cw);
    IC3_LAUNCH_CHECK();
    // Y[k][n] = sum_j W_ih[j][k] Q[j][n],  Q = G[:, 384:]
    small_gemm_tn_kernel<<<(TC_H * L.np + 255) / 256, 256, 0, s>>>(TC_H, L.np, 512, wj, TC_H, G + 384, NC, Y, L.np, 0);
    IC3_LAUNCH_CHECK();
    // dC[k][m] = sum_j W_ih[j][k] G_S[j][m]
    small_gemm_tn_kernel<<<(TC_H * TC_H + 255) / 256, 256, 0, s>>>(TC_H, TC_H, 512, wj, TC_H, G + 128, NC, dC, TC_H, 0);
    IC3_LAUNCH_CHECK();
    bptt_gsc_kernel<<<(512 * TC_H + 255) / 256, 256, 0, s>>>(G, NC, cw, GSC);
    IC3_LAUNCH_CHECK();
    f.c_b = c_b;
    f.g_c_w = const_cast<float*>(g_c_w); f.g_c_b = const_cast<float*>(g_c_b);
    bptt_finish_lstm_kernel<<<(512 * TC_H + 255) / 256, 256, 0, s>>>(f);
    IC3_LAUNCH_CHECK();
    bptt_finish_misc_kernel<<<(finish_enc_items(f) * 128 + 255) / 256, 256, 0, s>>>(f);
    IC3_LAUNCH_CHECK();
  }
  bptt_finish_heads_kernel<<<(BP_HEADS * TC_H + 255) / 256, 256, 0, s>>>(f);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

namespace {
// the parameter / gradient pointers ic3_bptt_finish reads for the plan's cell
int finish_args_check(const ic3_policy_cfg* cfg, const Layout& L, const ic3_policy_params* params,
                      const ic3_policy_params* grads) {
  if (!grads->encoder_w || !grads->encoder_b || !grads->value_w || !grads->value_b) return IC3_E_NULL;
  for (int k = 0; k < cfg->nheads; ++k)
    if (!grads->head_w[k] || !grads->head_b[k]) return IC3_E_NULL;
  if (L.tanh) return grads->f_w_pass[0] && grads->f_b_pass[0] ? IC3_OK : IC3_E_NULL;
  if (!params->w_ih || !params->c_w || !params->c_b || !grads->w_ih || !grads->w_hh || !grads->b_ih || !grads->b_hh ||
      !grads->c_w || !grads->c_b)
    return IC3_E_NULL;
  return IC3_OK;
}
}  // namespace

// The backward of one ic3_policy_step under caller-given upstream gradients: the BPTT unit chain of ic3_bptt_step with
// the heads in their upstream form, between a reset of the accumulators and ic3_bptt_finish.  dh_prev / dc_prev carry
// the recursion (in: d / d (h', c'), out: d / d (h, c)).  No host synchronisation: the operand-scale bound is reduced on
// the device (bptt_upstream_kernel).  The operand images are not cleared: the preparation, gate and tanh kernels write
// every row of every tile they cover, padding rows included.
extern "C" int ic3_policy_step_backward(const ic3_bptt_plan* p, const ic3_policy_bwd_io* io,
                                        const ic3_policy_params* params, const ic3_policy_params* grads, void* stream) {
  if (!p || !io || !params || !grads || !p->cfg || !p->w || !p->workspace) return IC3_E_NULL;
  const ic3_policy_cfg* cfg = p->cfg;
  if (cfg->H != TC_H) return IC3_E_UNSUPPORTED;
  int npos, WW, is_tj;
  int rc = env_geometry(p, &npos, &WW, &is_tj);
  if (rc) return rc;
  if (cfg->obs_vocab == 0 || (is_tj ? ic3_tj_layout_check(p->tj_env, cfg) : ic3_pp_layout_check(p->pp_env, cfg)))
    return IC3_E_UNSUPPORTED;
  Layout L;
  rc = plan_layout(cfg, npos, WW, is_tj, &L);
  if (rc) return rc;
  int nout = 1;
  for (int k = 0; k < cfg->nheads; ++k) nout += cfg->head_dim[k];
  if (nout > BP_HEADS) return IC3_E_UNSUPPORTED;
  if (!io->h_prev || !io->h_new || !io->logp || !io->dh_prev) return IC3_E_NULL;
  if (!L.tanh && (!io->c_prev || !io->dc_prev || !p->x_table || !p->w->lstm_img || !p->w->bias_cat)) return IC3_E_NULL;
  if (L.tanh && !p->w->f_wT) return IC3_E_NULL;
  if (!p->w->head_w || !p->w->enc_wT || !p->w->enc_b) return IC3_E_NULL;
  if (cfg->hard_attn && !io->comm) return IC3_E_NULL;
  rc = records_check(io->pp_state, io->tj_state, is_tj);
  if (rc) return rc;
  rc = finish_args_check(cfg, L, params, grads);
  if (rc) return rc;

  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  rc = bptt_reset(p, L, s);
  if (rc) return rc;
  const size_t n4 = (size_t)cfg->B * cfg->N * TC_H / 4;
  const size_t nblk = (n4 + 255) / 256, cap = (size_t)4 * sm_count();
  bptt_upstream_kernel<<<(int)(nblk < cap ? nblk : cap), 256, 0, s>>>(
      n4, reinterpret_cast<const float4*>(io->dh_new), L.tanh ? nullptr : reinterpret_cast<const float4*>(io->dc_new),
      L.tanh ? nullptr : reinterpret_cast<const float4*>(io->c_prev), reinterpret_cast<float4*>(io->dh_prev),
      L.tanh ? nullptr : reinterpret_cast<float4*>(io->dc_prev), (float)(L.P - 1),
      reinterpret_cast<BpttScalars*>(ws + L.sc));
  IC3_LAUNCH_CHECK();
  ic3_bptt_step_io st;
  memset(&st, 0, sizeof(st));
  st.h_prev = io->h_prev; st.c_prev = L.tanh ? nullptr : io->c_prev; st.h_new = io->h_new;
  st.comm = io->comm; st.alive = io->alive; st.pp_state = io->pp_state; st.tj_state = io->tj_state;
  st.logp = io->logp; st.dh = io->dh_prev; st.dc = L.tanh ? nullptr : io->dc_prev; st.err = io->err;
  rc = bptt_step_on(p, &st, L, npos, is_tj, s, io);
  if (rc) return rc;
  return ic3_bptt_finish(p, params, grads, reinterpret_cast<double*>(ws + L.losses), s);
}

// ==================================================================================================================
// Non-recurrent tanh policies (models.MLP, CommNet / IC3Net without --recurrent): ic3_ff_grad_*.  No state crosses a
// step, so a chunk of K consecutive lock-steps is one batch of K*B env slots.  Per chunk:
//   records   the chunk's env records, slots of valid = 0 given an empty state                   [ff_records_kernel]
//   desc      observation pattern of every row (position, counts / scalars, constant)           [ff_desc_kernel]
//   forward   index encoder + the SIMT step's pass-state form (ic3_policy_ff_states): tanh(x), h_1 .. h_P, S_0 .. S_{P-1}
//   heads     d loss / d (value, logits), head weight gradients, loss sums                       [bptt_heads_kernel]
//   pass p    dz = g (1 - h_{p+1}^2), dx += dz, g = dz F_p + comm^T(dz C_p)  (tiles of whole envs)
//             G_F += dz^T h_p, G_C += dz^T S_p, g_b += sum dz  (fixed row blocks)
//   encoder   dpre = (dx + g) (1 - tanh(x)^2);  Y += dpre^T P
// The pass and encoder products run on the tensor cores (ff_grad_tc.cu; ic3_ff_grad_begin packs their weight images).
// ic3_ff_grad_finish sums the row-block partials in float64 and folds Y through the observation layout like the BPTT
// finish (bptt_finish_misc_kernel).  Every sum has a fixed order.
// ==================================================================================================================
namespace {

constexpr int FF_NB = 256;         // row blocks of the weight-gradient sums (fixed: the partition does not depend on the card)

struct FfGeom {
  int npos, WW, is_tj, np, npad, ne;   // positions, window cells, env kind, pattern columns, padded to 128, columns >= npos
  int P, comm, R;                      // passes, communication on, max rows
  size_t x, hs, ss, g, dx, dz, dout, pos, ext, rloc, rroute, ralive, rlast, apost, fpart, cpart, bpart, ypart,
      gw_part, gs_part, sc, Y, total;
  size_t tc;                           // weight images and operand-scale words (ff_grad_tc.cu)
  int nhb;
};

int ff_geometry(const ic3_ff_grad_plan* p, FfGeom* G) {
  if (!p || !p->cfg) return IC3_E_NULL;
  const ic3_policy_cfg* cfg = p->cfg;
  if (cfg->H != TC_H || cfg->cell != IC3_CELL_TANH || !cfg->x_tanh || !cfg->h_from_x) return IC3_E_UNSUPPORTED;
  if (cfg->passes < 0 || cfg->passes > IC3_MAX_PASSES) return IC3_E_UNSUPPORTED;
  if (cfg->N < 1 || cfg->N > IC3_MAX_AGENTS || cfg->B < 1 || cfg->nheads < 1 || cfg->nheads > IC3_MAX_HEADS)
    return IC3_E_RANGE;
  int nout = 1;
  for (int k = 0; k < cfg->nheads; ++k) nout += cfg->head_dim[k];
  if (nout > BP_HEADS) return IC3_E_UNSUPPORTED;
  if (!!p->pp_env == !!p->tj_env) return IC3_E_NULL;
  int W;
  if (p->pp_env) {
    W = 2 * p->pp_env->vision + 1;
    G->npos = p->pp_env->dim * p->pp_env->dim;
    G->is_tj = 0;
    // the index encoder's limits (ic3_pp_encoder_index)
    if (cfg->O != W * W * (G->npos + 4) || ic3_pp_agents(*p->pp_env) != cfg->N || p->pp_env->N >= IC3_MAX_AGENTS ||
        ic3_pp_layout_check(p->pp_env, cfg))
      return IC3_E_RANGE;
  } else {
    W = 2 * p->tj_env->vision + 1;
    G->npos = p->tj_env->h * p->tj_env->w;
    G->is_tj = 1;
    if (cfg->O != 2 + W * W * p->tj_env->vocab || p->tj_env->N != cfg->N || ic3_tj_layout_check(p->tj_env, cfg))
      return IC3_E_RANGE;
    if (!p->tj_env->grid) return IC3_E_NULL;
  }
  G->WW = W * W;
  if (G->WW > PREP_MAX_WW) return IC3_E_UNSUPPORTED;
  G->ne = G->is_tj ? G->WW + 4 : 2 * G->WW + 1;
  G->np = G->npos + G->ne;
  if ((G->np + 15) / 16 * 16 > WG_MAX_NP) return IC3_E_UNSUPPORTED;
  G->npad = (G->np + 127) / 128 * 128;
  G->P = cfg->passes > 1 ? cfg->passes : 1;
  G->comm = !cfg->comm_mask_zero;
  if ((long)p->max_rows < (long)cfg->B * cfg->N) return IC3_E_RANGE;
  G->R = p->max_rows;
  const size_t R = (size_t)G->R, RH = R * TC_H * 4, HH = (size_t)TC_H * TC_H * 4;
  G->nhb = (int)((R + HB_ROWS - 1) / HB_ROWS);
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 1023) / 1024 * 1024; return o; };
  G->x = take(RH);
  G->hs = take((size_t)(G->P + 1) * RH);
  G->ss = take(G->comm ? (size_t)G->P * RH : 0);
  G->g = take(RH);
  G->dx = take(RH);
  G->dz = take(RH);
  G->dout = take(R * BP_HEADS * 4);
  G->pos = take(R * 4);
  G->ext = take(R * G->ne * 4);
  // the chunk's env records with the slots of valid = 0 replaced by an empty state (their recorded state is stale)
  G->rloc = take(R * 16);                    // predator-prey [K*B, N_pred + 1, 2] or traffic junction [K*B*N, 2]
  G->rroute = take(R * 4);
  G->ralive = take(R);
  G->rlast = take(R);
  G->apost = take(R);                        // alive_post AND valid: what the heads backward reads
  G->tc = take(ic3_ff_grad_tc_bytes(G->P, G->comm));
  // accumulators, zeroed by ic3_ff_grad_begin (fpart .. end)
  G->fpart = take((size_t)G->P * FF_NB * HH);
  G->cpart = take(G->comm ? (size_t)G->P * FF_NB * HH : 0);
  G->bpart = take((size_t)G->P * FF_NB * TC_H * 4);
  G->ypart = take((size_t)FF_NB * TC_H * G->npad * 4);
  G->gw_part = take((size_t)G->nhb * BP_HEADS * TC_H * 4);
  G->gs_part = take((size_t)G->nhb * (BP_HEADS + 3) * 8);
  G->sc = take(sizeof(BpttScalars));
  G->Y = take((size_t)TC_H * G->npad * 8);
  G->total = off;
  return IC3_OK;
}

// Observation pattern of every row (the columns of prep_kernel's P image): pos = one-hot column of the agent position
// (-1: no class term -- a dead car, or a slot with valid = 0), ext = [prey, predator count per window cell, 1]
// (predator-prey) or [car count per window cell, last_act, route ratio, 0, 1] (traffic junction).  Rows of slots with
// valid = 0 get an all-zero pattern and never index the grid.
struct DescArgs {
  int R, N, ne, is_tj;
  ic3_pp_cfg pp; ic3_tj_cfg tj;
  const int32_t* pp_loc; const int32_t* tj_loc; const uint8_t* tj_alive; const uint8_t* tj_last_act;
  const int32_t* tj_route_id; const uint8_t* valid;
  int32_t* pos; float* ext;
};

__global__ void __launch_bounds__(256) ff_desc_kernel(DescArgs a) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= a.R) return;
  const int e = row / a.N, i = row - e * a.N;
  float* x = a.ext + (size_t)row * a.ne;
  for (int c = 0; c < a.ne; ++c) x[c] = 0.f;
  if (a.valid && !a.valid[e]) {
    a.pos[row] = -1;
    return;
  }
  if (!a.is_tj) {
    const int D = a.pp.dim, v = a.pp.vision, W = 2 * v + 1, NP = a.pp.N;
    const int* l = a.pp_loc + (size_t)e * (NP + 1) * 2;
    a.pos[row] = l[2 * i] * D + l[2 * i + 1];
    for (int w = 0; w < W * W; ++w) {
      const int rr = l[2 * i] - v + w / W, cc = l[2 * i + 1] - v + w % W;
      if (rr < 0 || rr >= D || cc < 0 || cc >= D) continue;
      int npred = 0;
      for (int j = 0; j < NP; ++j) npred += (l[2 * j] == rr && l[2 * j + 1] == cc);
      x[2 * w] = (float)(l[2 * NP] == rr && l[2 * NP + 1] == cc);
      x[2 * w + 1] = (float)npred;
    }
    x[2 * W * W] = 1.f;
  } else {
    const int v = a.tj.vision, W = 2 * v + 1, N = a.N;
    x[W * W + 3] = 1.f;
    if (!a.tj_alive[row]) {                      // dead car: all-zero observation
      a.pos[row] = -1;
      return;
    }
    const int* l = a.tj_loc + (size_t)e * N * 2;
    a.pos[row] = l[2 * i] * a.tj.w + l[2 * i + 1];
    for (int w = 0; w < W * W; ++w) {
      const int rr = l[2 * i] - v + w / W, cc = l[2 * i + 1] - v + w % W;
      if (rr < 0 || rr >= a.tj.h || cc < 0 || cc >= a.tj.w) continue;
      int cnt = 0;
      for (int j = 0; j < N; ++j) cnt += (l[2 * j] == rr && l[2 * j + 1] == cc);
      x[w] = (float)cnt;
    }
    x[W * W] = (float)a.tj_last_act[row];
    x[W * W + 1] = (float)a.tj_route_id[row] / (float)(a.tj.npath - 1);
  }
}

// Per agent row of a chunk: the env records the forward re-run reads, with every slot of valid = 0 given an empty
// state (all agents at (0, 0); traffic junction: no car alive), and alive_post masked by valid, so that such a slot
// indexes nothing from its stale records and contributes exactly zero.
struct RecArgs {
  int R, N, NP, is_tj;
  ic3_pp_state pps; ic3_tj_state tjs;          // the records (ic3_ff_grad_io)
  const uint8_t* alive_post; const uint8_t* valid;
  int32_t* loc; int32_t* route; uint8_t* alive; uint8_t* last; uint8_t* apost;
};

__global__ void __launch_bounds__(256) ff_records_kernel(RecArgs a) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= a.R) return;
  const int e = row / a.N, i = row - e * a.N;
  const bool ok = !a.valid || a.valid[e];
  a.apost[row] = ok && a.alive_post[row] ? 1 : 0;
  if (!a.is_tj) {
    if (i <= a.NP) {                           // rows 0 .. NP of env e carry its N_pred + 1 positions
      const size_t o = ((size_t)e * (a.NP + 1) + i) * 2;
      a.loc[o] = ok ? a.pps.loc[o] : 0;
      a.loc[o + 1] = ok ? a.pps.loc[o + 1] : 0;
    }
    if (i == a.N - 1 && a.NP >= a.N) {         // N_pred + 1 > N rows: the prey's position goes with the last row
      const size_t o = ((size_t)e * (a.NP + 1) + a.NP) * 2;
      a.loc[o] = ok ? a.pps.loc[o] : 0;
      a.loc[o + 1] = ok ? a.pps.loc[o + 1] : 0;
    }
  } else {
    a.loc[2 * (size_t)row] = ok ? a.tjs.loc[2 * (size_t)row] : 0;
    a.loc[2 * (size_t)row + 1] = ok ? a.tjs.loc[2 * (size_t)row + 1] : 0;
    a.alive[row] = ok ? a.tjs.alive[row] : 0;
    a.last[row] = ok ? a.tjs.last_act[row] : 0;
    a.route[row] = ok ? a.tjs.route_id[row] : 0;
  }
}

// grad[i] += sum_blk part[blk][i] (float64, block order), i < n
__global__ void ff_reduce_add_kernel(const float* __restrict__ part, size_t stride, int n, float* __restrict__ grad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc = 0.0;
  for (int b = 0; b < FF_NB; ++b) acc += (double)part[(size_t)b * stride + i];
  grad[i] += (float)acc;
}

// Y[n][c] = sum_blk ypart[blk][n][c]
__global__ void ff_reduce_y_kernel(const float* __restrict__ part, int n, double* __restrict__ Y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc = 0.0;
  for (int b = 0; b < FF_NB; ++b) acc += (double)part[(size_t)b * n + i];
  Y[i] = acc;
}

}  // namespace

extern "C" uint64_t ic3_ff_grad_workspace_bytes(const ic3_ff_grad_plan* p) {
  FfGeom G;
  if (ff_geometry(p, &G)) return 0;
  return (uint64_t)G.total;
}

extern "C" int ic3_ff_grad_begin(const ic3_ff_grad_plan* p, void* stream) {
  FfGeom G;
  int rc = ff_geometry(p, &G);
  if (rc) return rc;
  if (!p->w || !p->workspace || !p->w->f_wT || (G.comm && !p->w->c_wT)) return IC3_E_NULL;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  cudaError_t e = cudaMemsetAsync(ws + G.fpart, 0, G.total - G.fpart, s);
  if (e != cudaSuccess) return (int)e;
  return ic3_ff_grad_tc_pack(G.P, G.comm, p->w->f_wT, p->w->c_wT, ws + G.tc, s);
}

extern "C" int ic3_ff_grad_chunk(const ic3_ff_grad_plan* p, const ic3_ff_grad_io* io, void* stream) {
  FfGeom G;
  int rc = ff_geometry(p, &G);
  if (rc) return rc;
  if (!io || !p->w || !p->workspace || !p->w->head_w) return IC3_E_NULL;
  const ic3_policy_cfg* cfg = p->cfg;
  if (io->nsteps < 1 || (long)io->nsteps * cfg->B * cfg->N > (long)G.R) return IC3_E_RANGE;
  if (!io->fresh || !io->logp || !io->action || !io->value || !io->ret || !io->adv || !io->alive_post) return IC3_E_NULL;
  if (cfg->hard_attn && !io->comm) return IC3_E_NULL;
  if (records_check(io->pp_state, io->tj_state, G.is_tj)) return IC3_E_NULL;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  const int Bk = io->nsteps * cfg->B, N = cfg->N, R = Bk * N;
  const size_t RHs = (size_t)R * TC_H;             // floats of one [R, H] block of this chunk
  float* x = reinterpret_cast<float*>(ws + G.x);
  float* hs = reinterpret_cast<float*>(ws + G.hs);
  float* ss = G.comm ? reinterpret_cast<float*>(ws + G.ss) : nullptr;
  float* g = reinterpret_cast<float*>(ws + G.g);
  float* dx = reinterpret_cast<float*>(ws + G.dx);
  float* dz = reinterpret_cast<float*>(ws + G.dz);
  float* dout = reinterpret_cast<float*>(ws + G.dout);
  int32_t* pos = reinterpret_cast<int32_t*>(ws + G.pos);
  float* ext = reinterpret_cast<float*>(ws + G.ext);
  RecArgs ra;
  memset(&ra, 0, sizeof(ra));
  ra.R = R; ra.N = N; ra.NP = G.is_tj ? N : p->pp_env->N; ra.is_tj = G.is_tj;
  if (G.is_tj) ra.tjs = *io->tj_state;
  else ra.pps = *io->pp_state;
  ra.alive_post = io->alive_post; ra.valid = io->valid;
  ra.loc = reinterpret_cast<int32_t*>(ws + G.rloc); ra.route = reinterpret_cast<int32_t*>(ws + G.rroute);
  ra.alive = ws + G.ralive; ra.last = ws + G.rlast; ra.apost = ws + G.apost;
  ff_records_kernel<<<(R + 255) / 256, 256, 0, s>>>(ra);
  IC3_LAUNCH_CHECK();
  const int32_t* pp_loc = G.is_tj ? nullptr : ra.loc;
  const int32_t* tj_loc = G.is_tj ? ra.loc : nullptr;
  // observation pattern
  DescArgs d;
  memset(&d, 0, sizeof(d));
  d.R = R; d.N = N; d.ne = G.ne; d.is_tj = G.is_tj;
  if (G.is_tj) d.tj = *p->tj_env;
  else d.pp = *p->pp_env;
  d.pp_loc = pp_loc; d.tj_loc = tj_loc; d.tj_alive = ra.alive; d.tj_last_act = ra.last;
  d.tj_route_id = ra.route; d.valid = io->valid; d.pos = pos; d.ext = ext;
  ff_desc_kernel<<<(R + 255) / 256, 256, 0, s>>>(d);
  IC3_LAUNCH_CHECK();
  // forward: x from the recorded env state (the K steps as K*B env slots), then every pass state
  ic3_policy_cfg ccfg = *cfg;
  ccfg.B = Bk;
  if (G.is_tj) {
    ic3_tj_cfg env = *p->tj_env;
    env.B = Bk;
    ic3_tj_state st;
    memset(&st, 0, sizeof(st));
    st.loc = const_cast<int32_t*>(tj_loc); st.alive = ra.alive; st.last_act = ra.last; st.route_id = ra.route;
    rc = ic3_tj_encoder_index(&env, &st, &ccfg, p->w, x, stream);
  } else {
    ic3_pp_cfg env = *p->pp_env;
    env.B = Bk;
    ic3_pp_state st;
    memset(&st, 0, sizeof(st));
    st.loc = const_cast<int32_t*>(pp_loc);
    rc = ic3_pp_encoder_index(&env, &st, &ccfg, p->w, x, stream);
  }
  if (rc) return rc;
  // pass blocks of this chunk: [p][R][H] with the chunk's own R (packed at the front of the capacity)
  ic3_policy_io pio;
  memset(&pio, 0, sizeof(pio));
  pio.x = x; pio.comm_action = cfg->hard_attn ? io->comm : nullptr; pio.alive = io->alive; pio.fresh = io->fresh;
  rc = ic3_policy_ff_states(&ccfg, p->w, &pio, hs, ss, stream);
  if (rc) return rc;
  // heads of the last pass
  int atot = 0;
  for (int k = 0; k < cfg->nheads; ++k) atot += cfg->head_dim[k];
  HeadsArgs h;
  memset(&h, 0, sizeof(h));
  h.R = R; h.N = N; h.nheads = cfg->nheads; h.atot = atot;
  for (int k = 0; k < IC3_MAX_HEADS; ++k) h.head_dim[k] = cfg->head_dim[k];
  h.value_coeff = p->value_coeff; h.entr = p->entr;
  h.logp = io->logp; h.action = io->action; h.value = io->value; h.ret = io->ret; h.adv = io->adv;
  h.alive_post = ra.apost; h.valid = io->valid;
  h.h_new = hs + (size_t)G.P * RHs;
  h.head_w = p->w->head_w;
  h.dout = dout;
  h.gw_part = reinterpret_cast<float*>(ws + G.gw_part);
  h.gs_part = reinterpret_cast<double*>(ws + G.gs_part);
  h.sc = reinterpret_cast<BpttScalars*>(ws + G.sc);
  h.q = 0;
  bptt_heads_kernel<false><<<(R + HB_ROWS - 1) / HB_ROWS, 256, 0, s>>>(h);
  IC3_LAUNCH_CHECK();
  FfGradTcChunk c;
  memset(&c, 0, sizeof(c));
  c.R = R; c.N = N; c.Bk = Bk; c.P = G.P; c.comm = G.comm; c.hard_attn = cfg->hard_attn; c.comm_avg = cfg->comm_avg;
  c.nout = 1 + atot; c.npos = G.npos; c.ne = G.ne; c.npad = G.npad; c.is_tj = G.is_tj;
  c.hs = hs; c.ss = ss; c.dout = dout; c.head_w = p->w->head_w;
  c.fresh = io->fresh; c.comm_action = cfg->hard_attn ? io->comm : nullptr; c.alive = io->alive; c.valid = io->valid;
  c.g = g; c.dx = dx; c.dz = dz; c.pos = pos; c.ext = ext;
  c.fpart = reinterpret_cast<float*>(ws + G.fpart);
  c.cpart = G.comm ? reinterpret_cast<float*>(ws + G.cpart) : nullptr;
  c.bpart = reinterpret_cast<float*>(ws + G.bpart);
  c.ypart = reinterpret_cast<float*>(ws + G.ypart);
  c.nb = FF_NB;
  c.tc = ws + G.tc;
  return ic3_ff_grad_tc_chunk(&c, s);
}

extern "C" int ic3_ff_grad_finish(const ic3_ff_grad_plan* p, const ic3_policy_params* params, const ic3_policy_params* grads,
                                  double* losses, void* stream) {
  FfGeom G;
  int rc = ff_geometry(p, &G);
  if (rc) return rc;
  if (!params || !grads || !losses || !p->workspace) return IC3_E_NULL;
  if (!grads->encoder_w || !grads->encoder_b || !grads->value_w || !grads->value_b) return IC3_E_NULL;
  const ic3_policy_cfg* cfg = p->cfg;
  for (int k = 0; k < cfg->nheads; ++k)
    if (!grads->head_w[k] || !grads->head_b[k]) return IC3_E_NULL;
  for (int ps = 0; ps < G.P; ++ps) {
    const float* g_c_w = ps > 0 && grads->c_w_pass[ps] ? grads->c_w_pass[ps] : grads->c_w;
    const float* g_c_b = ps > 0 && grads->c_b_pass[ps] ? grads->c_b_pass[ps] : grads->c_b;
    if (!grads->f_w_pass[ps] || !grads->f_b_pass[ps] || !g_c_b || (G.comm && !g_c_w)) return IC3_E_NULL;
  }
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* ws = reinterpret_cast<unsigned char*>(p->workspace);
  const size_t HH = (size_t)TC_H * TC_H;
  // pass by pass, in order: with share_weights every pass adds into the one module's buffers
  for (int ps = 0; ps < G.P; ++ps) {
    float* g_c_w = const_cast<float*>(ps > 0 && grads->c_w_pass[ps] ? grads->c_w_pass[ps] : grads->c_w);
    float* g_c_b = const_cast<float*>(ps > 0 && grads->c_b_pass[ps] ? grads->c_b_pass[ps] : grads->c_b);
    const float* fp = reinterpret_cast<const float*>(ws + G.fpart) + (size_t)ps * FF_NB * HH;
    const float* bp = reinterpret_cast<const float*>(ws + G.bpart) + (size_t)ps * FF_NB * TC_H;
    ff_reduce_add_kernel<<<(int)(HH / 256), 256, 0, s>>>(fp, HH, (int)HH, const_cast<float*>(grads->f_w_pass[ps]));
    IC3_LAUNCH_CHECK();
    ff_reduce_add_kernel<<<1, TC_H, 0, s>>>(bp, TC_H, TC_H, const_cast<float*>(grads->f_b_pass[ps]));
    IC3_LAUNCH_CHECK();
    ff_reduce_add_kernel<<<1, TC_H, 0, s>>>(bp, TC_H, TC_H, g_c_b);      // c_b enters beside f_b: the same sum
    IC3_LAUNCH_CHECK();
    if (G.comm) {
      const float* cp = reinterpret_cast<const float*>(ws + G.cpart) + (size_t)ps * FF_NB * HH;
      ff_reduce_add_kernel<<<(int)(HH / 256), 256, 0, s>>>(cp, HH, (int)HH, g_c_w);
      IC3_LAUNCH_CHECK();
    }
  }
  // encoder through the observation layout, then the heads
  double* Y = reinterpret_cast<double*>(ws + G.Y);
  const int ny = TC_H * G.npad;
  ff_reduce_y_kernel<<<(ny + 255) / 256, 256, 0, s>>>(reinterpret_cast<const float*>(ws + G.ypart), ny, Y);
  IC3_LAUNCH_CHECK();
  FinishArgs f;
  memset(&f, 0, sizeof(f));
  int atot = 0;
  for (int k = 0; k < cfg->nheads; ++k) atot += cfg->head_dim[k];
  f.O = cfg->O; f.nheads = cfg->nheads; f.atot = atot; f.npos = G.npos; f.np = G.npad; f.WW = G.WW;
  for (int k = 0; k < IC3_MAX_HEADS; ++k) f.head_dim[k] = cfg->head_dim[k];
  f.Y = Y; f.ldy = G.npad;
  f.g_enc_w = const_cast<float*>(grads->encoder_w); f.g_enc_b = const_cast<float*>(grads->encoder_b);
  f.g_c_b = nullptr;
  f.g_value_w = const_cast<float*>(grads->value_w); f.g_value_b = const_cast<float*>(grads->value_b);
  for (int k = 0; k < IC3_MAX_HEADS; ++k) {
    f.g_head_w[k] = const_cast<float*>(grads->head_w[k]);
    f.g_head_b[k] = const_cast<float*>(grads->head_b[k]);
  }
  f.gw_part = reinterpret_cast<const float*>(ws + G.gw_part);
  f.gs_part = reinterpret_cast<const double*>(ws + G.gs_part);
  f.nhb = G.nhb;
  f.losses = losses;
  f.is_tj = G.is_tj;
  if (G.is_tj) f.tj = *p->tj_env;
  else f.pp = *p->pp_env;
  f.ones_col = G.np - 1;
  bptt_finish_misc_kernel<<<(finish_enc_items(f) * 128 + 255) / 256, 256, 0, s>>>(f);
  IC3_LAUNCH_CHECK();
  bptt_finish_heads_kernel<<<(BP_HEADS * TC_H + 255) / 256, 256, 0, s>>>(f);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}
