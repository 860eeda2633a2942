// Policy step of the tanh policies without a recurrent LSTM cell on the Hopper tensor cores, H = 128, in two forms:
//  - non-recurrent (models.MLP and CommNet / IC3Net without --recurrent: comm.py:127-129, 179-224, models.py:23-25):
//      x~ = tanh(x),  h_0 = x~
//      pass p:  S_p = gated mean of h_p over the env's other agents (zero with comm_mask_zero)
//               h_{p+1} = tanh(x~ + c_b,p + S_p . C_p^T + h_p . F_p^T + f_b,p)
//  - recurrent (models.RNN with the vanilla recurrence, the IC and IRIC baselines: models.py:83-85): one pass without
//    communication, x~ = x and h_0 = the previous step's h (zero for slots starting an episode)
//  then value / action heads, log-softmax and sampling of h_P.
//
// One launch per pass.  The pass's weight image -- the fp16 hi/lo split of 256 * F_p (and of 256 * C_p unless
// comm_mask_zero) in the no-swizzle K-major core-matrix layout, 64 KB per matrix -- stays in shared memory for the whole
// launch; only activations stream.  With communication the two products are one K = 256 contraction of [h | S] against
// [F_p ; C_p] into the same 64 x 128 accumulator.  Persistent CTAs of one warpgroup loop over 64-row tiles: two CTAs
// per SM and 64 consecutive rows per tile without communication, one CTA per SM and whole envs per tile with it
// (floor(64 / N) envs, padding rows at the end):
//   A  x~ of the thread's accumulator fragment (tanh on the SFU unless recurrent), kept in registers for C; gate and
//      divisor per row
//   A  h_p -> hi/lo fp16 (x 16) into the core-matrix layout in shared memory; with communication one thread per
//      (env, column quad) also sums the gated rows (T) and writes S = g (T - h) / den into the S image
//   B  8 k-steps x 3 wgmma m64n128k16 (hi.hi + lo.hi + hi.lo, tc_common.cuh) per product, fp32 accumulator
//   C  h_{p+1} = tanh((x~ + c_b) + acc / 4096 + f_b) on the SFU -> HBM; last pass: also as fp32 over the A image
//   D  last pass: heads of the tile's rows from shared memory, one warp per row (policy_heads.cuh)
// Between passes h travels through a workspace buffer in place (a tile reads only its own rows, before it writes them).
// The pass-state form (ic3_policy_ff_states) is the non-recurrent kernel with tanh(x), S_p and h_{p+1} written out and
// no heads.
#include "ic3_common.cuh"
#include "policy_heads.cuh"
#include "policy_internal.h"
#include "tc_common.cuh"

namespace {

constexpr int FT_H = 128;
constexpr int FT_M = 64;                          // rows per tile: one warpgroup
constexpr int FT_THREADS = 128;
constexpr int FT_W_PART = FT_H * FT_H * 2;        // bytes of the hi (or lo) half of one weight matrix's image
constexpr int FT_A_PART = FT_M * FT_H * 2;        // bytes of the hi (or lo) half of a tile's h (or S) image
constexpr int FT_HP_LD = FT_H + 8;                // fp32 h' tile, rows padded: the fragment's float2 stores hit every bank once
constexpr int FT_HP_BYTES = FT_M * FT_HP_LD * 4;
static_assert(IC3_FF_IMG_BYTES(1, 0) == 2 * FT_W_PART && IC3_FF_IMG_BYTES(1, 1) == 4 * FT_W_PART,
              "weight image size of the header");

template <bool COMM>
struct FtLayout {
  static constexpr int NMAT = COMM ? 2 : 1;                               // F (and C)
  static constexpr int W_BYTES = NMAT * 2 * FT_W_PART;
  static constexpr int A_IMG = NMAT * 2 * FT_A_PART;                      // [h hi, h lo (, S hi, S lo)]
  static constexpr int A_BYTES = A_IMG > FT_HP_BYTES ? A_IMG : FT_HP_BYTES;   // the h' tile overlays the A image
  static constexpr size_t SMEM = (size_t)W_BYTES + A_BYTES + 2 * FT_H * sizeof(float) + 2 * FT_M * sizeof(float);
};

// weight image of one matrix part, in halfs: [k >> 3][n >> 3][n & 7][k & 7]  (W[n][k]: K-major B operand of h . W^T)
__host__ __device__ __forceinline__ size_t ft_w_off(int n, int k) {
  return ((size_t)(k >> 3) * (FT_H / 8) + (n >> 3)) * 64 + (n & 7) * 8 + (k & 7);
}
// A image of one part, in halfs: row rl, float4 column q (k = 4q .. 4q + 3)
__device__ __forceinline__ size_t ft_a_off(int rl, int q) {
  return (size_t)((q >> 1) * (FT_M / 8) + (rl >> 3)) * 64 + (rl & 7) * 8 + (q & 1) * 4;
}

// one thread per (n, k) of one weight matrix: its hi and lo parts
__global__ void ff_tc_pack_kernel(const float* __restrict__ wm, __half* __restrict__ part, int32_t* __restrict__ flags) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;      // (n, k)
  if (idx >= FT_H * FT_H) return;
  const int n = idx / FT_H, k = idx - n * FT_H;
  const float w = wm[idx];
  __half hi, lo;
  split_f16(w, SCALE_B, hi, lo);
  if (flags && !(fabsf(w) * SCALE_B < 65504.f)) atomicOr(flags, IC3_ERR_FP16_RANGE);   // also catches NaN
  part[ft_w_off(n, k)] = hi;
  part[FT_W_PART / 2 + ft_w_off(n, k)] = lo;
}

struct FfTcArgs {
  ic3_policy_cfg cfg;
  ic3_policy_io io;      // x, comm_action, alive, fresh; heads: tick, draws, value, logp, action, err
  const __half* w_img;   // this pass's image
  const float* f_b;      // this pass's biases
  const float* c_b;      // recurrent form: bias of the (zero) comm projection, x + C(0) = x + c_b as the SIMT kernel adds it
  const float* head_w;
  const float* head_b;
  const int32_t* wflags;
  const float* h_in;     // h_p, or NULL on pass 0 (h_0 = tanh(x)); recurrent form: io.h; may alias h_out
  float* h_out;          // h_{p+1}
  float* st_x;           // pass-state form, pass 0: tanh(x), else NULL
  float* st_s;           // pass-state form: S_p, else NULL
  int heads;             // last pass of the step: heads and sampling
  int epb, ntiles;       // with communication: envs per tile; tiles
};

__device__ __forceinline__ float4 tanh4(float4 v) {
  return make_float4(tanh_fast(v.x), tanh_fast(v.y), tanh_fast(v.z), tanh_fast(v.w));
}

template <bool COMM, bool RECUR>
__global__ void __launch_bounds__(FT_THREADS, COMM ? 1 : 2) ff_tc_kernel(FfTcArgs a) {
  static_assert(!(COMM && RECUR), "the recurrent form has no communication");
  using L = FtLayout<COMM>;
  extern __shared__ __align__(1024) unsigned char smem[];
  __half* s_a = reinterpret_cast<__half*>(smem + L::W_BYTES);
  float* s_hp = reinterpret_cast<float*>(smem + L::W_BYTES);
  float* s_fb = reinterpret_cast<float*>(smem + L::W_BYTES + L::A_BYTES);
  float* s_cb = s_fb + FT_H;
  float* s_gate = s_cb + FT_H;
  float* s_den = s_gate + FT_M;
  const ic3_policy_cfg& cfg = a.cfg;
  const ic3_policy_io& io = a.io;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int N = cfg.N, B = cfg.B;
  if (blockIdx.x == 0 && tid == 0 && a.wflags && io.err && *a.wflags) atomicOr(io.err, *a.wflags);
  for (int i = tid; i < L::W_BYTES / 16; i += FT_THREADS)
    reinterpret_cast<uint4*>(smem)[i] = __ldg(reinterpret_cast<const uint4*>(a.w_img) + i);
  s_fb[tid] = __ldg(a.f_b + tid);
  s_cb[tid] = __ldg(a.c_b + tid);
  const uint32_t smem_base = smem_u32(smem);
  // K-major, no swizzle: LBO = distance of K-adjacent core matrices, SBO = distance of 8-row groups (tc_common.cuh)
  const uint64_t dA = make_desc(smem_base + L::W_BYTES, (FT_M / 8) * 128, 128);
  const uint64_t dB = make_desc(smem_base, (FT_H / 8) * 128, 128);
  const int fr = lane >> 2, fc = 2 * (lane & 3);       // accumulator fragment: rows 16 warp + fr + 8 i, columns 8 j + fc + {0, 1}
  // the recurrent form is a rollout step: heads, no pass states
  const bool heads = RECUR || a.heads;
  float* const st_x = RECUR ? nullptr : a.st_x;
  float* const st_s = RECUR ? nullptr : a.st_s;
  // h_p of row `row`, float4 column q (plain loads: h_in may alias h_out)
  auto load_h = [&](long row, int q) -> float4 {
    if (RECUR) {     // an episode start enters with h = 0 whatever io.h holds (trainer.py:50-51)
      if (io.fresh && io.fresh[row / N]) return make_float4(0.f, 0.f, 0.f, 0.f);
      return *(reinterpret_cast<const float4*>(a.h_in + row * FT_H) + q);
    }
    if (a.h_in) return *(reinterpret_cast<const float4*>(a.h_in + row * FT_H) + q);
    return tanh4(__ldg(reinterpret_cast<const float4*>(io.x + row * FT_H) + q));
  };
  auto range_check = [&](const float4& v) {
    const float m = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
    if (!(m * SCALE_A < 65504.f) && io.err) atomicOr(io.err, IC3_ERR_FP16_RANGE);
  };

  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    // with communication a tile holds whole envs; without, 64 consecutive rows (each row's product is its own)
    const int e0 = COMM ? tile * a.epb : 0;
    const long row0 = COMM ? (long)e0 * N : (long)tile * FT_M;
    const int nrows = COMM ? min(a.epb, B - e0) * N : (int)min((long)FT_M, (long)B * N - row0);
    // ---- A: x~ of this thread's fragment; gate and divisor per row (as policy_step_kernel) -------------
    float2 xv[32];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int rl = 16 * warp + fr + 8 * i;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float2 v = make_float2(0.f, 0.f);
        if (rl < nrows) v = __ldg(reinterpret_cast<const float2*>(io.x + (row0 + rl) * FT_H + 8 * j + fc));
        xv[16 * i + j] = RECUR ? v : make_float2(tanh_fast(v.x), tanh_fast(v.y));
      }
    }
    if (COMM && tid < FT_M) {
      const int r = tid;
      float g = 0.f, den = 1.f;
      if (r < nrows) {
        const int el = r / N, e = e0 + el, i = r - el * N;
        const bool fr0 = io.fresh && io.fresh[e];
        int n_alive = N, al = 1;                      // comm.py:102-107
        if (io.alive && !fr0) {
          n_alive = 0;
          for (int j = 0; j < N; ++j) n_alive += io.alive[(size_t)e * N + j] != 0;
          al = io.alive[(size_t)e * N + i] != 0;
        }
        int cm = 1;
        if (cfg.hard_attn) cm = fr0 ? 0 : (io.comm_action[(size_t)e * N + i] != 0);   // comm.py:171-175
        g = (float)(al * cm);
        if (cfg.comm_avg && n_alive > 1) den = (float)(n_alive - 1);                   // comm.py:194-196
      }
      s_gate[r] = g;
      s_den[r] = den;
    }
    if (COMM) __syncthreads();
    // ---- A: h (and S) -> operand image ----------------------------------------------------------------
    if (!COMM) {
      // warp item = 8 rows x 4 float4 columns: every store instruction writes two whole 128-byte core matrices
#pragma unroll 4
      for (int item = warp; item < (FT_M / 8) * 8; item += FT_THREADS / 32) {
        const int rl = (item & 7) * 8 + (lane & 7), q = (item >> 3) * 4 + (lane >> 3);
        float4 hv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rl < nrows) {
          hv = load_h(row0 + rl, q);
          if (st_x) *(reinterpret_cast<float4*>(st_x + (row0 + rl) * FT_H) + q) = hv;
          if (st_s) *(reinterpret_cast<float4*>(st_s + (row0 + rl) * FT_H) + q) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        range_check(hv);
        store_split4(s_a, ft_a_off(rl, q), FT_A_PART / 2 + ft_a_off(rl, q), hv, SCALE_A);
      }
    } else {
      // thread item = (env of the tile, float4 column): T = sum of the gated rows, then S = g (T - h) / den
      // (comm.py:181-205; the sum over j != k of the SIMT kernel, taken as the total minus the row's own term)
      __half* s_s = s_a + FT_A_PART;                  // S image: parts 2, 3 (in halfs: 2 * FT_A_PART / 2)
      const int nenv = nrows / N;
      for (int it = tid; it < nenv * (FT_H / 4); it += FT_THREADS) {
        const int el = it >> 5, q = it & 31, rb = el * N;
        float4 T = make_float4(0.f, 0.f, 0.f, 0.f);
        // rows in groups of 4 with every load issued before the group is used: 4 loads in flight per thread
        for (int j0 = 0; j0 < N; j0 += 4) {
          float4 hv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u)
            if (j0 + u < N) hv[u] = load_h(row0 + rb + j0 + u, q);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (j0 + u >= N) break;
            const int rl = rb + j0 + u;
            if (st_x) *(reinterpret_cast<float4*>(st_x + (row0 + rl) * FT_H) + q) = hv[u];
            if (s_gate[rl] != 0.f) { T.x += hv[u].x; T.y += hv[u].y; T.z += hv[u].z; T.w += hv[u].w; }
            range_check(hv[u]);
            store_split4(s_a, ft_a_off(rl, q), FT_A_PART / 2 + ft_a_off(rl, q), hv[u], SCALE_A);
          }
        }
        for (int k0 = 0; k0 < N; k0 += 4) {
          float4 hv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u)
            if (k0 + u < N && s_gate[rb + k0 + u] != 0.f) hv[u] = load_h(row0 + rb + k0 + u, q);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (k0 + u >= N) break;
            const int rl = rb + k0 + u;
            float4 sv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (s_gate[rl] != 0.f) {
              const float d = s_den[rl];
              sv = make_float4((T.x - hv[u].x) / d, (T.y - hv[u].y) / d, (T.z - hv[u].z) / d, (T.w - hv[u].w) / d);
            }
            if (st_s) *(reinterpret_cast<float4*>(st_s + (row0 + rl) * FT_H) + q) = sv;
            range_check(sv);
            store_split4(s_s, ft_a_off(rl, q), FT_A_PART / 2 + ft_a_off(rl, q), sv, SCALE_A);
          }
        }
      }
      // padding rows at the end of the tile enter as zero
      for (int it = nrows * (FT_H / 4) + tid; it < FT_M * (FT_H / 4); it += FT_THREADS) {
        const int rl = it >> 5, q = it & 31;
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        store_split4(s_a, ft_a_off(rl, q), FT_A_PART / 2 + ft_a_off(rl, q), z, SCALE_A);
        store_split4(s_s, ft_a_off(rl, q), FT_A_PART / 2 + ft_a_off(rl, q), z, SCALE_A);
      }
    }
    fence_proxy_async();          // the image (and, first tile, the weights) was written through the generic proxy
    __syncthreads();

    // ---- B: acc = (16 h) . (256 F)^T (+ (16 S) . (256 C)^T) -------------------------------------------
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    wgmma_fence_regs(d);
    wgmma_fence();
#pragma unroll
    for (int m = 0; m < L::NMAT; ++m) {
#pragma unroll
      for (int ks = 0; ks < FT_H / 16; ++ks) {
        const uint64_t da_hi = dA + ((m * 2 * FT_A_PART + ks * 2 * (FT_M / 8) * 128) >> 4), da_lo = da_hi + (FT_A_PART >> 4);
        const uint64_t db_hi = dB + ((m * 2 * FT_W_PART + ks * 2 * (FT_H / 8) * 128) >> 4), db_lo = db_hi + (FT_W_PART >> 4);
        wgmma_m64n128_kk(d, da_hi, db_hi, (m | ks) != 0);
        wgmma_m64n128_kk(d, da_lo, db_hi, 1);
        wgmma_m64n128_kk(d, da_hi, db_lo, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    __syncthreads();              // every warp's MMAs have read the A image: h' may overwrite it

    // ---- C: h' = tanh((x~ + c_b) + acc / 4096 + f_b) --------------------------------------------------
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int rl = 16 * warp + fr + 8 * i;
      const long row = row0 + rl;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = 8 * j + fc;
        const float2 fb = *reinterpret_cast<const float2*>(s_fb + col), cb = *reinterpret_cast<const float2*>(s_cb + col);
        float2 hn;
        hn.x = tanh_fast((xv[16 * i + j].x + cb.x) + fmaf(d[4 * j + 2 * i + 0], INV_SCALE, fb.x));
        hn.y = tanh_fast((xv[16 * i + j].y + cb.y) + fmaf(d[4 * j + 2 * i + 1], INV_SCALE, fb.y));
        if (rl < nrows) *reinterpret_cast<float2*>(a.h_out + row * FT_H + col) = hn;
        if (heads) *reinterpret_cast<float2*>(s_hp + rl * FT_HP_LD + col) = hn;
      }
    }
    if (!heads) continue;       // the next tile's image writes follow the MMA barrier above
    __syncthreads();

    // ---- D: heads, log-softmax, sampling (comm.py:228-239, action_utils.py:32-36) --------------------
    for (int rl = warp; rl < nrows; rl += FT_THREADS / 32) {
      float hv[FT_H / 32];
#pragma unroll
      for (int m = 0; m < FT_H / 32; ++m) hv[m] = s_hp[rl * FT_HP_LD + lane + 32 * m];
      const long row = row0 + rl;
      const int e = (int)(row / N), i = (int)(row - (long)e * N);
      heads_for_row<FT_H>(cfg, a.head_w, a.head_b, hv, (size_t)row, e, i, lane, io.tick, io.draws, io.value, io.logp,
                          io.action);
    }
    __syncthreads();              // the heads have read h' before the next tile's image replaces it
  }
}

template <bool COMM, bool RECUR>
int ff_tc_launch(const FfTcArgs& a, cudaStream_t s) {
  const size_t smem = FtLayout<COMM>::SMEM;
  int grid = 0;
  const int rc = ic3_persistent_grid((const void*)ff_tc_kernel<COMM, RECUR>, FT_THREADS, smem, a.ntiles, &grid);
  if (rc) return rc;
  ff_tc_kernel<COMM, RECUR><<<grid, FT_THREADS, smem, s>>>(a);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

// The passes of one step.  st_h == NULL: the rollout form (h between passes in `carry`, the last pass into io->h_out
// with heads); else the pass-state form (st_h [P + 1][R][H], st_s [P][R][H] or NULL, no heads).
int ff_tc_run(const ic3_policy_cfg* cfg, const ic3_policy_packed* w, const ic3_policy_io* io, float* carry, float* st_h,
              float* st_s, cudaStream_t s) {
  const int P = cfg->passes > 1 ? cfg->passes : 1;
  const bool comm = !cfg->comm_mask_zero, recur = !cfg->h_from_x;
  const size_t RH = (size_t)cfg->B * cfg->N * FT_H;
  FfTcArgs a;
  a.cfg = *cfg;
  a.io = *io;
  a.head_w = w->head_w;
  a.head_b = w->head_b;
  a.wflags = w->flags;
  a.epb = FT_M / cfg->N;
  a.ntiles = comm ? (cfg->B + a.epb - 1) / a.epb : (int)((RH / FT_H + FT_M - 1) / FT_M);
  const size_t img_pass = IC3_FF_IMG_BYTES(1, comm ? 1 : 0);
  for (int ps = 0; ps < P; ++ps) {
    a.w_img = reinterpret_cast<const __half*>(reinterpret_cast<const unsigned char*>(w->ff_img) + ps * img_pass);
    a.f_b = w->f_b + (size_t)ps * FT_H;
    a.c_b = w->c_b + (size_t)ps * FT_H;
    if (st_h) {
      a.h_in = ps == 0 ? nullptr : st_h + ps * RH;
      a.h_out = st_h + (ps + 1) * RH;
      a.st_x = ps == 0 ? st_h : nullptr;
      a.st_s = st_s ? st_s + ps * RH : nullptr;
      a.heads = 0;
    } else {
      a.h_in = ps > 0 ? carry : recur ? io->h : nullptr;
      a.h_out = ps == P - 1 ? io->h_out : carry;
      a.st_x = a.st_s = nullptr;
      a.heads = ps == P - 1;
    }
    const int rc = comm ? ff_tc_launch<true, false>(a, s) : recur ? ff_tc_launch<false, true>(a, s)
                                                                  : ff_tc_launch<false, false>(a, s);
    if (rc) return rc;
  }
  return IC3_OK;
}

}  // namespace

bool ic3_ff_tc_capable(const ic3_policy_cfg* cfg) {
  if (cfg->cell != IC3_CELL_TANH || cfg->H != FT_H) return false;
  if (!cfg->x_tanh && !cfg->h_from_x)     // the tanh RNN: one pass without communication
    return cfg->passes <= 1 && cfg->comm_mask_zero && !cfg->hard_attn;
  return cfg->x_tanh && cfg->h_from_x && cfg->N <= IC3_MAX_AGENTS && cfg->passes <= IC3_MAX_PASSES;
}

uint64_t ic3_ff_tc_workspace_bytes(const ic3_policy_cfg* cfg) {
  // one [R, H] buffer carries h from pass to pass; one pass (the tanh RNN's too) needs none, and reports a nominal
  // 16 bytes: a non-NULL workspace is what selects the tensor-core path
  if (cfg->passes <= 1) return 16;
  return (uint64_t)cfg->B * cfg->N * FT_H * sizeof(float);
}

int ic3_ff_tc_pack(const ic3_policy_cfg* cfg, const ic3_policy_params* p, const ic3_policy_packed* out, cudaStream_t s) {
  if (!ic3_ff_tc_capable(cfg)) return IC3_E_UNSUPPORTED;
  const int P = cfg->passes > 1 ? cfg->passes : 1, nmat = cfg->comm_mask_zero ? 1 : 2;
  for (int ps = 0; ps < P; ++ps) {
    const float* c_w = (ps > 0 && p->c_w_pass[ps]) ? p->c_w_pass[ps] : p->c_w;     // as pack_kernel
    if (!p->f_w_pass[ps] || !c_w) return IC3_E_NULL;
  }
  if (out->flags) {
    cudaError_t e = cudaMemsetAsync(out->flags, 0, sizeof(int32_t), s);
    if (e != cudaSuccess) return (int)e;
  }
  __half* img = reinterpret_cast<__half*>(out->ff_img);
  for (int ps = 0; ps < P; ++ps)
    for (int m = 0; m < nmat; ++m) {        // parts [pass][F hi, F lo (, C hi, C lo)]
      const float* wm = m == 0 ? p->f_w_pass[ps] : ((ps > 0 && p->c_w_pass[ps]) ? p->c_w_pass[ps] : p->c_w);
      ff_tc_pack_kernel<<<FT_H * FT_H / 256, 256, 0, s>>>(wm, img + (size_t)(ps * nmat + m) * FT_W_PART, out->flags);
      IC3_LAUNCH_CHECK();
    }
  return IC3_OK;
}

int ic3_ff_tc_policy_step(const ic3_policy_cfg* cfg, const ic3_policy_packed* w, const ic3_policy_io* io, cudaStream_t s) {
  if (!ic3_ff_tc_capable(cfg)) return IC3_E_UNSUPPORTED;
  if (!io->x || !io->workspace || !w->ff_img || !w->f_b) return IC3_E_NULL;
  ic3_prof_mark(0, s);
  ic3_prof_mark(1, s);
  const int rc = ff_tc_run(cfg, w, io, reinterpret_cast<float*>(io->workspace), nullptr, nullptr, s);
  if (rc) return rc;
  ic3_prof_mark(2, s);
  ic3_prof_mark(3, s);
  return IC3_OK;
}

int ic3_ff_tc_states(const ic3_policy_cfg* cfg, const ic3_policy_packed* w, const ic3_policy_io* io, float* st_h,
                     float* st_s, cudaStream_t s) {
  if (!ic3_ff_tc_capable(cfg)) return IC3_E_UNSUPPORTED;
  if (!io->x || !w->ff_img || !w->f_b || !st_h) return IC3_E_NULL;
  return ff_tc_run(cfg, w, io, nullptr, st_h, st_s, s);
}
