// Kernels of the wgmma policy path (see policy_tc.cu for the overview).  Included by policy_tc.cu (rollout
// forward) and bptt_tc.cu (backward), each inside its own anonymous namespace.
#pragma once
#include <cuda_fp16.h>

#include <cstdlib>
#include <cstring>

#include "ic3_common.cuh"
#include "policy_heads.cuh"
#include "policy_internal.h"
#include "tc_common.cuh"

namespace {

constexpr int TC_H = 128;
constexpr int TC_K = 384;               // [x | S | h]
constexpr int TC_KC = 32;               // K per pipeline stage
constexpr int TC_NCHUNK = TC_K / TC_KC; // 12
constexpr int TC_M = 128;               // rows per tile
constexpr int TC_NH = 256;              // gate columns per CTA (64 hidden units x i,f,g,o)
constexpr int A_CHUNK_BYTES = 2 * TC_M * TC_KC * 2;   // hi + lo = 16384
constexpr int B_CHUNK_BYTES = 2 * TC_NH * TC_KC * 2;  // 32768
constexpr int STAGE_BYTES = A_CHUNK_BYTES + B_CHUNK_BYTES;
constexpr int A_TILE_HALFS = TC_NCHUNK * A_CHUNK_BYTES / 2;   // 98304

// ---- image addressing (in halfs) ---------------------------------------------------------
// A image: [tile][part = hi, lo][fg = k >> 3 (48)][rg = r >> 3 (16)][r & 7][k & 7].  Uniform strides in both
// directions (feature group 2048 B, row group 128 B), so the SAME bytes serve as a K-major operand of the
// forward / backward GEMMs that contract over features (a pipeline chunk of 32 features = 4 consecutive feature
// groups = one contiguous 8 KB piece per part) and as an MN-major operand of the weight-gradient GEMM that
// contracts over rows (bptt_tc.cu).
__host__ __device__ __forceinline__ size_t a_img_off(int tile, int k, int r, int part) {
  return (size_t)tile * A_TILE_HALFS + (size_t)part * (A_TILE_HALFS / 2) + ((size_t)(k >> 3) * 16 + (r >> 3)) * 64 + (r & 7) * 8 +
         (k & 7);
}
__host__ __device__ __forceinline__ size_t b_img_off(int nh, int k, int n, int part) {
  const int c = k >> 5, kk = k & 31;
  return ((((((size_t)(nh * TC_NCHUNK + c) * 2 + part) * 4 + (kk >> 3)) * 32 + (n >> 3)) * 8 + (n & 7)) * 8) + (kk & 7);
}

constexpr size_t B_IMG_HALFS = (size_t)2 * TC_NCHUNK * B_CHUNK_BYTES / 2;   // one weight image, in halfs

// ---- weight images (once per optimizer step) ------------------------------------------------
__global__ void pack_tc_kernel(ic3_policy_params p, __half* __restrict__ img, float* __restrict__ bias_cat,
                               int32_t* __restrict__ flags) {
  const int H = TC_H;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;      // (col, k)
  if (idx < 4 * H * TC_K) {
    const int col = idx / TC_K, k = idx - col * TC_K;
    const int u = col >> 2, g = col & 3, row = g * H + u;       // column 4*u+gate <- LSTMCell row g*H+u
    double w;
    if (k < H) {
      w = p.w_ih[(size_t)row * H + k];
    } else if (k < 2 * H) {                                     // (W_ih . C)[row][k-H]
      double acc = 0.0;
      for (int m = 0; m < H; ++m) acc += (double)p.w_ih[(size_t)row * H + m] * (double)p.c_w[(size_t)m * H + (k - H)];
      w = acc;
    } else {
      w = p.w_hh[(size_t)row * H + (k - 2 * H)];
    }
    __half hi, lo;
    split_f16((float)w, SCALE_B, hi, lo);
    if (flags && !(fabs(w) * SCALE_B < 65504.0)) atomicOr(flags, IC3_ERR_FP16_RANGE);   // also catches NaN
    const int nh = col >> 8, n = col & 255;
    img[b_img_off(nh, k, n, 0)] = hi;
    img[b_img_off(nh, k, n, 1)] = lo;
  }
  if (idx < 4 * H) {
    const int u = idx >> 2, g = idx & 3, row = g * H + u;
    double acc = (double)p.b_ih[row] + (double)p.b_hh[row];
    for (int m = 0; m < H; ++m) acc += (double)p.w_ih[(size_t)row * H + m] * (double)p.c_b[m];
    bias_cat[idx] = (float)acc;
  }
}

// ---- operand A image: x | S | h (every step) ---------------------------------------------------
// One CTA per 128-row tile.  Phase 1 forms, per environment touching the tile, the gated sum
// T = sum_j g_j h_j (comm.py:181-205) in shared memory (environments may straddle tiles: their
// other rows are read straight from global memory); phase 2 streams the tile: a warp item is
// 8 rows x 4 float4 columns so every store instruction writes two complete 128-byte core
// matrices, with S_k = g_k (T - h_k) / (n_alive - 1).
constexpr int PREP_ROWS = 64;      // rows per CTA (half a tile): 2 x more CTAs in flight than tiles
constexpr int PREP_THREADS = 160;  // 40 registers x 160 threads -> 10 CTAs/SM: the 1280 half-tile CTAs of a c2 step form ONE wave on 132 SMs (1320 slots; 256 threads: 8 CTAs/SM = 1056 slots, a second wave of 224 CTAs)
__host__ __device__ inline size_t prep_T_bytes(int N) { return (size_t)(PREP_ROWS / N + 2) * TC_H * sizeof(float); }
constexpr int PREP_MAX_WW = 25;    // window cells (vision <= 2) the fused index encoder supports
constexpr int PREP_X_BYTES = PREP_ROWS * TC_H * 4;   // shared-memory x tile of the fused index encoder

// Where the encoder output x comes from: a [R,H] fp32 tensor, or -- fused index encoder -- straight from the
// environment state (same sum, same order as *_encoder_index_kernel / encoder_dense_kernel -> bit-identical x).
enum { XSRC_TENSOR = 0, XSRC_PP = 1, XSRC_TJ = 2 };
struct PrepSrc {
  ic3_pp_cfg pp;
  ic3_pp_state pps;
  ic3_tj_cfg tj;
  ic3_tj_state tjs;
  const float* wT;     // encoder.weight^T [O, H]
  const float* bias;   // [H]
  const float* table;  // [positions, H] class part of the sum per agent position (ic3_*_encoder_table) or NULL
  int split;           // ic3_policy_cfg.obs_vocab > 0: class terms and count / scalar terms are summed separately
  const int32_t* wflags;   // ic3_policy_packed.flags (weight range check of the pack kernel) or NULL
};

__device__ __forceinline__ void fma4(float4& a, float v, const float4 w) {
  a.x = fmaf(v, w.x, a.x); a.y = fmaf(v, w.y, a.y); a.z = fmaf(v, w.z, a.z); a.w = fmaf(v, w.w, a.w);
}

// accumulate into `a` when sel, else into `b` (both stay in registers)
__device__ __forceinline__ void fma4_sel(bool sel, float4& a, float4& b, float v, const float4 w) {
  if (sel) fma4(a, v, w);
  else fma4(b, v, w);
}

// TAB: the class part of x comes from the per-position table (src.table); the fused encoder then needs neither
// the x tile in shared memory nor the class feature indices, only the sparse count terms of each row.
// Extra outputs of the operand-preparation kernel when it runs inside the backward pass (bptt_tc.cu):
//   p_img  "feature" operand of the weight-gradient GEMM, [tile][pg = column >> 3][rg 16][8 rows][8 columns] fp16:
//          the NON-ZERO pattern of the observation row as exact small numbers -- one-hot agent position (columns
//          [0, npos)), the count features of the window cells, the scalar features, and a constant 1 (bias column);
//          d(loss)/d(encoder weights) = (d gates)^T . P folded with W_ih afterwards, so the [R, O] observation is
//          never materialised in the backward pass either
//   gs, gr per-row comm gate factors g / den and g of comm.py:181-205 (needed by the comm backward)
struct PrepBwd {
  __half* p_img;
  float* gs;
  float* gr;
  int npg;      // column groups of P (columns padded to a multiple of 16)
  int npos;     // positions (dim*dim or h*w): first column after the one-hot block
};

template <int XSRC, bool TAB, bool BWD = false>
__global__ void __launch_bounds__(256) prep_kernel(ic3_policy_cfg cfg, ic3_policy_io io, __half* __restrict__ img,
                                                   PrepSrc src, PrepBwd bw) {
  static_assert(!(TAB && XSRC == XSRC_TENSOR), "the table belongs to the fused index encoder");
  static_assert(!BWD || TAB, "the backward pass uses the per-position table form of the encoder (table NULL: x = 0)");
  __shared__ float s_gate[PREP_ROWS + 64];
  __shared__ float s_den[PREP_ROWS + 64];
  // s_T: gated hidden-state sum of every environment touching this CTA's rows, [PREP_ROWS / N + 2][H] floats at the
  // start of the dynamic shared memory (sized by the launcher: a static [34][H] array would cap the kernel at 8 CTAs/SM)
  // fused index encoder: per (row, window cell) the feature index of the one-hot class and the counts
  __shared__ int s_feat[(XSRC == XSRC_TENSOR || TAB) ? 1 : PREP_ROWS * PREP_MAX_WW];
  __shared__ int s_cnt[XSRC == XSRC_TENSOR ? 1 : PREP_ROWS * PREP_MAX_WW];
  __shared__ unsigned s_mask[TAB ? PREP_ROWS : 1];    // window cells of the row that hold a count
  __shared__ int s_pos[TAB ? PREP_ROWS : 1];          // table row of the agent (-1: observation is all zero)
  __shared__ float s_la[XSRC == XSRC_TJ ? PREP_ROWS : 1], s_ri[XSRC == XSRC_TJ ? PREP_ROWS : 1];
  __shared__ int s_live[XSRC == XSRC_TJ ? PREP_ROWS : 1];
  extern __shared__ __align__(16) float s_dyn[];
  float (*s_T)[TC_H] = reinterpret_cast<float (*)[TC_H]>(s_dyn);
  float* s_x = s_dyn + (size_t)(PREP_ROWS / cfg.N + 2) * TC_H;   // [PREP_ROWS][H] encoder output (index sources without table)
  const int N = cfg.N;
  const int R = cfg.B * N;
  const int tile = blockIdx.x >> 1, hb = blockIdx.x & 1;
  const int row0 = tile * TC_M + hb * PREP_ROWS;
  if (TAB) {
    if (threadIdx.x < PREP_ROWS) s_mask[threadIdx.x] = 0u;
    __syncthreads();
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && src.wflags && io.err && *src.wflags) atomicOr(io.err, *src.wflags);
  for (int w = threadIdx.x; w < PREP_ROWS + 64; w += blockDim.x) {
    const int row = row0 - 32 + w;
    float g = 0.f, den = 1.f;
    if (row >= 0 && row < R) {
      const int e = row / N, i = row - e * N;
      const bool fr = io.fresh && io.fresh[e];
      int n_alive = N, al = 1;
      if (io.alive && !fr) {                       // comm.py:102-104
        n_alive = 0;
        for (int j = 0; j < N; ++j) n_alive += io.alive[(size_t)e * N + j] != 0;
        al = io.alive[(size_t)e * N + i] != 0;
      }
      int cm = 1;
      if (cfg.hard_attn) cm = fr ? 0 : (io.comm_action[(size_t)e * N + i] != 0);   // comm.py:171-175
      // episode start: every agent of the env has h = 0 (trainer.py:50-51) -> nothing to send in the first comm pass
      g = (fr && io.pass_index == 0) ? 0.f : (float)(al * cm);
      if (cfg.comm_avg && n_alive > 1) den = (float)(n_alive - 1);                  // comm.py:194-196
    }
    s_gate[w] = g;
    s_den[w] = den;
  }
  if (XSRC == XSRC_PP) {          // predator_prey_env.py:188-210
    const int D = src.pp.dim, v = src.pp.vision, W = 2 * v + 1, WW = W * W, V = D * D + 4;
    const int NP = src.pp.N;      // predators; agent row NP (present with enemy_comm: N == NP + 1) is the prey
    for (int p = threadIdx.x; p < PREP_ROWS * WW; p += blockDim.x) {
      const int rl = p / WW, w = p - rl * WW, row = row0 + rl;
      int feat = 0, cnt = 0;
      if (row < R) {
        const int e = row / N, i = row - e * N;
        const int* l = src.pps.loc + (size_t)e * (NP + 1) * 2;
        const int dy = w / W, dx = w - dy * W;
        const int rr = l[2 * i] - v + dy, cc = l[2 * i + 1] - v + dx;
        if (rr >= 0 && rr < D && cc >= 0 && cc < D) {
          int npred = 0;
          for (int j = 0; j < NP; ++j) npred += (l[2 * j] == rr && l[2 * j + 1] == cc);
          const int nprey = (l[2 * NP] == rr && l[2 * NP + 1] == cc);
          feat = w * V + rr * D + cc;
          cnt = npred | (nprey << 8);
        } else {
          feat = w * V + V - 3;                          // OUTSIDE class
        }
        if (TAB && w == 0) s_pos[rl] = l[2 * i] * D + l[2 * i + 1];
      } else if (TAB && w == 0) {
        s_pos[rl] = -1;
      }
      if (!TAB) s_feat[rl * WW + w] = feat;
      s_cnt[rl * WW + w] = cnt;
      if (TAB && cnt) atomicOr(&s_mask[rl], 1u << w);
    }
  } else if (XSRC == XSRC_TJ) {   // traffic_junction_env.py:321-366
    const int v = src.tj.vision, W = 2 * v + 1, WW = W * W, V = src.tj.vocab;
    for (int rl = threadIdx.x; rl < PREP_ROWS; rl += blockDim.x) {
      const int row = row0 + rl;
      int live = 0;
      float la = 0.f, ri = 0.f;
      if (row < R) {
        live = src.tjs.alive[row] != 0;
        la = (float)src.tjs.last_act[row];
        ri = (float)src.tjs.route_id[row] / (float)(src.tj.npath - 1);
      }
      s_live[rl] = live; s_la[rl] = la; s_ri[rl] = ri;
    }
    for (int p = threadIdx.x; p < PREP_ROWS * WW; p += blockDim.x) {
      const int rl = p / WW, w = p - rl * WW, row = row0 + rl;
      int feat = 0, cnt = 0;
      if (row < R) {
        const int e = row / N;
        const int* l = src.tjs.loc + (size_t)e * N * 2;
        const int i = row - e * N;
        const int dy = w / W, dx = w - dy * W;
        const int rr = l[2 * i] - v + dy, cc = l[2 * i + 1] - v + dx;
        int cls = src.tj.outside_cls;
        if (rr >= 0 && rr < src.tj.h && cc >= 0 && cc < src.tj.w) {
          cls = src.tj.grid[rr * src.tj.w + cc];
          for (int j = 0; j < N; ++j) cnt += (l[2 * j] == rr && l[2 * j + 1] == cc);
        }
        feat = 2 + w * V + cls;
        if (TAB && w == 0) s_pos[rl] = src.tjs.alive[row] ? l[2 * i] * src.tj.w + l[2 * i + 1] : -1;
        if (TAB && !src.tjs.alive[row]) cnt = 0;         // dead car: all-zero observation
      } else if (TAB && w == 0) {
        s_pos[rl] = -1;
      }
      if (!TAB) s_feat[rl * WW + w] = feat;
      s_cnt[rl * WW + w] = cnt;
      if (TAB && cnt) atomicOr(&s_mask[rl], 1u << w);
    }
  }
  __syncthreads();
  if (XSRC != XSRC_TENSOR && !TAB) {
    // comm.py:119 on the one-hot observation, never materialised: warp per row, lane = 4 consecutive hidden
    // units, every weight-row read is one coalesced 512-byte request; x lands in shared memory.
    // xv = bias + class terms, x2 = count / scalar terms when the layout hint asks for separate sums (else they join
    // xv, in feature order).  (With the per-position table this whole phase is skipped: TAB specialisation below.)
    const int gw = threadIdx.x >> 5, gl = threadIdx.x & 31;
    const float4* wq = reinterpret_cast<const float4*>(src.wT) + gl;
    const bool split = src.split != 0;
    for (int rl = gw; rl < PREP_ROWS; rl += (blockDim.x >> 5)) {
      float4 xv = __ldg(reinterpret_cast<const float4*>(src.bias) + gl);
      float4 x2 = make_float4(0.f, 0.f, 0.f, 0.f);
      const int row = row0 + rl;
      if (row < R) {
        if (XSRC == XSRC_PP) {
          const int W = 2 * src.pp.vision + 1, WW = W * W, V = src.pp.dim * src.pp.dim + 4;
          for (int w = 0; w < WW; ++w) {
            const int feat = s_feat[rl * WW + w], cnt = s_cnt[rl * WW + w];
            fma4(xv, 1.f, __ldg(wq + (size_t)feat * (TC_H / 4)));
            if (cnt >> 8) fma4_sel(split, x2, xv, (float)(cnt >> 8), __ldg(wq + (size_t)(w * V + V - 2) * (TC_H / 4)));     // PREY
            if (cnt & 255) fma4_sel(split, x2, xv, (float)(cnt & 255), __ldg(wq + (size_t)(w * V + V - 1) * (TC_H / 4)));  // PREDATOR
          }
        } else if (s_live[rl]) {
          const int W = 2 * src.tj.vision + 1, WW = W * W, V = src.tj.vocab;
          if (s_la[rl] != 0.f) fma4_sel(split, x2, xv, s_la[rl], __ldg(wq));
          if (s_ri[rl] != 0.f) fma4_sel(split, x2, xv, s_ri[rl], __ldg(wq + (TC_H / 4)));
          for (int w = 0; w < WW; ++w) {
            const int feat = s_feat[rl * WW + w], cnt = s_cnt[rl * WW + w];
            fma4(xv, 1.f, __ldg(wq + (size_t)feat * (TC_H / 4)));
            if (cnt) fma4_sel(split, x2, xv, (float)cnt, __ldg(wq + (size_t)(2 + w * V + src.tj.car_cls) * (TC_H / 4)));
          }
        }
      }
      xv.x += x2.x; xv.y += x2.y; xv.z += x2.z; xv.w += x2.w;
      *reinterpret_cast<float4*>(&s_x[rl * TC_H + 4 * gl]) = xv;
    }
  }
  const int e_first = row0 / N;
  const int last_row = min(R, row0 + PREP_ROWS) - 1;
  const bool want_s = !cfg.comm_mask_zero && N >= 2 && last_row >= row0;
  if (want_s) {
    const int nenv = last_row / N - e_first + 1;
    for (int idx = threadIdx.x; idx < nenv * (TC_H / 4); idx += blockDim.x) {
      const int el = idx >> 5, q = idx & 31;
      const int base = (e_first + el) * N;
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int j = 0; j < N; ++j) {
        if (s_gate[base + j - row0 + 32] != 0.f) {
          const float4 o = __ldg(reinterpret_cast<const float4*>(io.h + (size_t)(base + j) * TC_H) + q);
          t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w;
        }
      }
      *reinterpret_cast<float4*>(&s_T[el][4 * q]) = t;
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (BWD) {
    // row factors of the comm backward
    for (int rl = threadIdx.x; rl < PREP_ROWS; rl += blockDim.x) {
      const int row = row0 + rl;
      if (row < R) {
        bw.gs[row] = s_gate[rl + 32] / s_den[rl + 32];
        bw.gr[row] = s_gate[rl + 32];
      }
    }
    // P image of this CTA's 8 row groups: one core matrix (8 rows x 8 columns, 128 B) per warp iteration,
    // lane = (row r8 = lane >> 2, column pair 2 * (lane & 3)) -> every store instruction writes one whole core matrix
    const int WW = XSRC == XSRC_PP ? (2 * src.pp.vision + 1) * (2 * src.pp.vision + 1)
                                   : (2 * src.tj.vision + 1) * (2 * src.tj.vision + 1);
    const int r8 = lane >> 2, c2 = (lane & 3) * 2;
    for (int cm = warp; cm < bw.npg * 8; cm += (blockDim.x >> 5)) {
      const int pg = cm >> 3, rgl = cm & 7;
      const int rl = rgl * 8 + r8, row = row0 + rl;
      float v[2] = {0.f, 0.f};
      if (row < R) {
        const int pos = s_pos[rl];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int col = pg * 8 + c2 + j;
          if (col < bw.npos) {
            v[j] = (col == pos) ? 1.f : 0.f;
          } else {
            const int idx = col - bw.npos;
            if (XSRC == XSRC_PP) {        // [prey count, predator count] per window cell, then the constant
              if (idx < 2 * WW) {
                const int cnt = s_cnt[rl * WW + (idx >> 1)];
                v[j] = (float)((idx & 1) ? (cnt & 255) : (cnt >> 8));
              } else if (idx == 2 * WW) {
                v[j] = 1.f;
              }
            } else if (XSRC == XSRC_TJ) { // car count per window cell, last_act, route id ratio (hi, lo), the constant
              if (idx < WW) v[j] = pos >= 0 ? (float)s_cnt[rl * WW + idx] : 0.f;
              else if (idx == WW) v[j] = pos >= 0 ? s_la[rl] : 0.f;
              else if (idx == WW + 1) v[j] = pos >= 0 ? __half2float(__float2half_rn(s_ri[rl])) : 0.f;
              else if (idx == WW + 2) v[j] = pos >= 0 ? s_ri[rl] - __half2float(__float2half_rn(s_ri[rl])) : 0.f;
              else if (idx == WW + 3) v[j] = 1.f;
            }
          }
        }
      }
      const size_t off = (((size_t)tile * bw.npg + pg) * 16 + (hb * 8 + rgl)) * 64 + r8 * 8 + c2;
      *reinterpret_cast<__half2*>(bw.p_img + off) = __floats2half2_rn(v[0], v[1]);
    }
  }
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const size_t tile_base = (size_t)tile * A_TILE_HALFS;
#pragma unroll 2
  for (int item = warp; item < 64; item += (blockDim.x >> 5)) {
    const int rcl = item & 7, qg = item >> 3;
    const int r8 = lane & 7, q = qg * 4 + (lane >> 3);
    const int rl = rcl * 8 + r8;                 // row inside this CTA's 64 rows
    const int rc = hb * 8 + rcl;                 // 8-row group inside the 128-row tile
    const int row = row0 + rl;
    float4 xv = zero4, hv = zero4, sv = zero4;
    if (row < R) {
      const int e = row / N;
      const bool fr = io.fresh && io.fresh[e] && io.pass_index == 0;     // zero state: first comm pass only
      if (XSRC == XSRC_TENSOR) {
        xv = __ldg(reinterpret_cast<const float4*>(io.x + (size_t)row * TC_H) + q);
      } else if (!TAB) {
        xv = *reinterpret_cast<const float4*>(&s_x[rl * TC_H + 4 * q]);
      } else if (!BWD || src.table) {   // backward of the tanh cell: no table, x is no operand of its GEMMs (zero)
        // x = table[position] + (count / scalar terms in feature order): the same additions as the gather above
        const int pos = s_pos[rl];
        xv = __ldg(reinterpret_cast<const float4*>(pos >= 0 ? src.table + (size_t)pos * TC_H : src.bias) + q);
        float4 x2 = zero4;
        const float4* wq = reinterpret_cast<const float4*>(src.wT) + q;
        if (XSRC == XSRC_PP) {
          const int W = 2 * src.pp.vision + 1, WW = W * W, V = src.pp.dim * src.pp.dim + 4;
          for (unsigned m = s_mask[rl]; m; m &= m - 1) {
            const int w = __ffs(m) - 1, cnt = s_cnt[rl * WW + w];
            if (cnt >> 8) fma4(x2, (float)(cnt >> 8), __ldg(wq + (size_t)(w * V + V - 2) * (TC_H / 4)));     // PREY
            if (cnt & 255) fma4(x2, (float)(cnt & 255), __ldg(wq + (size_t)(w * V + V - 1) * (TC_H / 4)));  // PREDATOR
          }
        } else if (pos >= 0) {
          const int W = 2 * src.tj.vision + 1, WW = W * W, V = src.tj.vocab;
          if (s_la[rl] != 0.f) fma4(x2, s_la[rl], __ldg(wq));
          if (s_ri[rl] != 0.f) fma4(x2, s_ri[rl], __ldg(wq + (TC_H / 4)));
          for (unsigned m = s_mask[rl]; m; m &= m - 1) {
            const int w = __ffs(m) - 1;
            fma4(x2, (float)s_cnt[rl * WW + w], __ldg(wq + (size_t)(2 + w * V + src.tj.car_cls) * (TC_H / 4)));
          }
        }
        xv.x += x2.x; xv.y += x2.y; xv.z += x2.z; xv.w += x2.w;
      }
      if (!fr) hv = __ldg(reinterpret_cast<const float4*>(io.h + (size_t)row * TC_H) + q);
      if (want_s && s_gate[rl + 32] != 0.f) {      // gate 1 => own h is part of T
        const float4 t = *reinterpret_cast<const float4*>(&s_T[e - e_first][4 * q]);
        const float inv = 1.f / s_den[rl + 32];
        sv.x = (t.x - hv.x) * inv; sv.y = (t.y - hv.y) * inv; sv.z = (t.z - hv.z) * inv; sv.w = (t.w - hv.w) * inv;
      }
    }
    {   // operand split range (|a| * 16 must stay inside fp16): flag instead of silently saturating to inf
      const float m = fmaxf(fmaxf(fmaxf(fabsf(xv.x), fabsf(xv.y)), fmaxf(fabsf(xv.z), fabsf(xv.w))),
                            fmaxf(fmaxf(fmaxf(fabsf(hv.x), fabsf(hv.y)), fmaxf(fabsf(hv.z), fabsf(hv.w))),
                                  fmaxf(fmaxf(fabsf(sv.x), fabsf(sv.y)), fmaxf(fabsf(sv.z), fabsf(sv.w)))));
      if (!(m * SCALE_A < 65504.f) && io.err) atomicOr(io.err, IC3_ERR_FP16_RANGE);
    }
    // k = sec*128 + 4q  ->  feature group fg = sec*16 + (q >> 1), k & 7 = 4 * (q & 1)
    const size_t cell = tile_base + (size_t)(((q >> 1) * 16 + rc) * 64 + r8 * 8 + (q & 1) * 4);
    constexpr size_t LO = A_TILE_HALFS / 2, SEC = 16 * 1024;      // lo half of the tile; 16 feature groups per section
    store_split4(img, cell + 0 * SEC, cell + 0 * SEC + LO, xv, SCALE_A);
    store_split4(img, cell + 1 * SEC, cell + 1 * SEC + LO, sv, SCALE_A);
    store_split4(img, cell + 2 * SEC, cell + 2 * SEC + LO, hv, SCALE_A);
  }
}

// Gate non-linearities on the SFU, one ex2.approx (2^-22 rel.) + one rcp.approx (1 ulp) each, well inside the
// 1e-5 budget of the hidden state (tests/test_gpu_policy.py, tests/test_gpu_rollout.py).  The epilogue is the
// pacing stage of the kernel, so the forms are chosen for instruction count: the argument arrives already scaled
// by -log2(e) (folded into the accumulator scale and the shared-memory bias copy), and both functions are
// 1 / (1 + 2^t), see lstm_cell4 (ex2_fast, rcp_fast, LOG2E: tc_common.cuh).

// Gate biases pre-multiplied like the accumulator scale: (i, f, o) * -log2(e), g * -2 log2(e); [4H] in shared memory.
__device__ __forceinline__ void load_scaled_bias(float* s_bias, const float* __restrict__ bias_cat) {
  for (int idx = threadIdx.x; idx < 4 * TC_H; idx += blockDim.x)
    s_bias[idx] = __ldg(bias_cat + idx) * ((idx & 3) == 2 ? -2.f * LOG2E : -LOG2E);
}

// LSTM cell of 4 hidden units from 16 accumulator columns (v[4j + gate] of unit j): LSTMCell semantics of comm.py:194.
// The biases of unit j are the float4 at s_bias4 + j * bstride.
// The SFU (16 lanes/clk/SM) is the scarcest pipe of the epilogue, so reciprocals are shared: the four gates of a
// unit are 1/(1+2^t) with ONE rcp of the product of the four denominators (each 1/a recovered with FMA-pipe
// multiplies), and the four tanh(c') of the group share one more -- 6.25 SFU ops per hidden unit instead of 10.
// Exponents are clamped at 30 (denominators <= 2^30+1, products <= 2^121: no overflow); the clamp changes a
// sigmoid by < 1e-9.
__device__ __forceinline__ void lstm_cell4(const float (&v)[16], const float (&co)[4], const float* s_bias4, int bstride,
                                           float (&cn)[4], float (&hn)[4]) {
  constexpr float SG = -INV_SCALE * LOG2E;
  constexpr float TMAX = 30.f;
  float go[4], bc[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 b = *reinterpret_cast<const float4*>(s_bias4 + j * bstride);
    const float ai = 1.f + ex2_fast(fminf(fmaf(v[4 * j + 0], SG, b.x), TMAX));
    const float af = 1.f + ex2_fast(fminf(fmaf(v[4 * j + 1], SG, b.y), TMAX));
    const float ag = 1.f + ex2_fast(fminf(fmaf(v[4 * j + 2], 2.f * SG, b.z), TMAX));
    const float ao = 1.f + ex2_fast(fminf(fmaf(v[4 * j + 3], SG, b.w), TMAX));
    const float p1 = ai * af, p2 = ag * ao;
    const float r = rcp_fast(p1 * p2);
    const float r1 = r * p2, r2 = r * p1;              // 1 / (ai af), 1 / (ag ao)
    const float gi = r1 * af, gf = r1 * ai;            // sigmoid(i), sigmoid(f)
    const float gg = fmaf(2.f, r2 * ao, -1.f);         // tanh(g) = 2 sigmoid(2g) - 1
    go[j] = r2 * ag;                                   // sigmoid(o)
    cn[j] = fmaf(gf, co[j], gi * gg);
    bc[j] = 1.f + ex2_fast(fminf(cn[j] * (-2.f * LOG2E), TMAX));
  }
  const float q1 = bc[0] * bc[1], q2 = bc[2] * bc[3];
  const float r = rcp_fast(q1 * q2);
  const float r1 = r * q2, r2 = r * q1;
  hn[0] = go[0] * fmaf(2.f, r1 * bc[1], -1.f);         // o * tanh(c')
  hn[1] = go[1] * fmaf(2.f, r1 * bc[0], -1.f);
  hn[2] = go[2] * fmaf(2.f, r2 * bc[3], -1.f);
  hn[3] = go[3] * fmaf(2.f, r2 * bc[2], -1.f);
}

// ---- the tensor-core kernel -----------------------------------------------------------------------
// Persistent, one CTA per SM, warp-specialised:
//   warp 8          producer: ring of NSTAGE_P (A 16 KB + B 32 KB) stages filled by cp.async.bulk, running ahead
//                   across work items
//   warps 0-7       two consumer warpgroups; warpgroup g owns rows 64g .. 64g+63 of the tile: 3 x wgmma
//                   (64 x 256 x 16) per k-step into 128 fp32 registers per thread, then the LSTM cell of its rows
// Work item = (128-row tile, 256-column half); item 2t and 2t+1 share the A tile (second read hits L2).
constexpr int NSTAGE_P = 4;
constexpr int HEAD_PAD = IC3_HEAD_PAD;   // outputs (value + action logits) the fused epilogue supports
constexpr int MMA_WARPS = 8;             // two consumer warpgroups
constexpr int TC_P_THREADS = MMA_WARPS * 32 + 32;   // + producer warp
constexpr int NSLOT = IC3_HEAD_NSLOT;    // partial-logit slots per row: (column half, lane parity of the unit, unit half)

// Consumer side of the ring for one work item: NCHUNK stages of 32 K, 2 k-steps x 3 products (hi.hi + lo.hi +
// hi.lo) each.  A stage goes back to the producer (one arrival per consumer warp) once the MMAs reading it are done;
// the MMAs of the next stage are already in flight by then.  a_row: byte offset of this warpgroup's 64 rows in A.
template <int NCHUNK>
__device__ __forceinline__ void wg_gemm_item(float (&d)[128], uint32_t smem_base, uint32_t a_row, uint32_t bar_full,
                                             uint32_t bar_empty, uint32_t li, int lane, bool& ok, int32_t* err) {
  static_assert(NCHUNK % NSTAGE_P == 0, "stage index must be a function of the chunk index alone");
  const uint64_t dA = make_desc(smem_base + a_row, 2048, 128), dB = make_desc(smem_base + A_CHUNK_BYTES, 4096, 128);
  wgmma_fence_regs(d);
#pragma unroll
  for (int c = 0; c < NCHUNK; ++c) {
    const uint32_t s = c % NSTAGE_P;
    // after a watchdog timeout the MMAs are still issued (on stale data) so that the warpgroup stays converged
    if (ok) ok = mbar_wait(bar_full + 8 * s, (li * (NCHUNK / NSTAGE_P) + c / NSTAGE_P) & 1, err);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < TC_KC / 16; ++ks) {
      const uint64_t da_hi = dA + ((s * STAGE_BYTES + ks * 4096) >> 4);
      const uint64_t da_lo = dA + ((s * STAGE_BYTES + A_CHUNK_BYTES / 2 + ks * 4096) >> 4);
      const uint64_t db_hi = dB + ((s * STAGE_BYTES + ks * 8192) >> 4);
      const uint64_t db_lo = dB + ((s * STAGE_BYTES + B_CHUNK_BYTES / 2 + ks * 8192) >> 4);
      wgmma_m64n256_kk(d, da_hi, db_hi, (c | ks) != 0);
      wgmma_m64n256_kk(d, da_lo, db_hi, 1);
      wgmma_m64n256_kk(d, da_hi, db_lo, 1);
    }
    wgmma_commit();
    wgmma_wait<1>();                       // the MMAs of chunk c - 1 have read their stage
    if (c > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * ((c - 1) % NSTAGE_P));
    }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  __syncwarp();
  if (lane == 0) mbar_arrive(bar_empty + 8 * ((NCHUNK - 1) % NSTAGE_P));
}

// Producer of the ring: for every work item, NCHUNK stages of (A hi 8 KB, A lo 8 KB, B 32 KB).  a_src(item, c) /
// b_src(item, c) give the sources of the A part (its lo half follows at a_lo_off) and of the B chunk.
template <int NCHUNK, typename ASrc, typename BSrc>
__device__ __forceinline__ void ring_producer(uint32_t smem_base, uint32_t bar_full, uint32_t bar_empty, int item0,
                                              int nitems, int stride, size_t a_lo_off, ASrc a_src, BSrc b_src,
                                              int32_t* err) {
  uint32_t li = 0;
  bool ok = true;
  for (int item = item0; item < nitems && ok; item += stride, ++li) {
#pragma unroll
    for (int c = 0; c < NCHUNK; ++c) {
      if (!ok) break;
      const uint32_t s = c % NSTAGE_P;
      ok = mbar_wait(bar_empty + 8 * s, ((li * (NCHUNK / NSTAGE_P) + c / NSTAGE_P) & 1) ^ 1, err);
      const uint32_t dst = smem_base + s * STAGE_BYTES;
      const unsigned char* a = a_src(item, c);
      mbar_expect_tx(bar_full + 8 * s, STAGE_BYTES);
      bulk_g2s(dst, a, A_CHUNK_BYTES / 2, bar_full + 8 * s);                                    // hi
      bulk_g2s(dst + A_CHUNK_BYTES / 2, a + a_lo_off, A_CHUNK_BYTES / 2, bar_full + 8 * s);      // lo
      bulk_g2s(dst + A_CHUNK_BYTES, b_src(item, c), B_CHUNK_BYTES, bar_full + 8 * s);
    }
  }
}

// The accumulator columns of a (row, hidden unit) are 4u + gate, so a thread's fragment holds two gates of a unit
// for two rows; one exchange with the neighbouring lane gives each thread all four gates of units 2j + (lane % 4) / 2
// (j = 0 .. 31) of ONE row: row 16w + lane / 4 + 8 (lane & 1) of the warpgroup's 64.
__device__ __forceinline__ void gather_gates(const float (&d)[128], int j, bool odd, float (&g)[4]) {
  const float s0 = odd ? d[4 * j + 0] : d[4 * j + 2];
  const float s1 = odd ? d[4 * j + 1] : d[4 * j + 3];
  const float r0 = __shfl_xor_sync(IC3_FULL_MASK, s0, 1), r1 = __shfl_xor_sync(IC3_FULL_MASK, s1, 1);
  g[0] = odd ? r0 : d[4 * j + 0];
  g[1] = odd ? r1 : d[4 * j + 1];
  g[2] = odd ? d[4 * j + 2] : r0;
  g[3] = odd ? d[4 * j + 3] : r1;
}

// Units 2j and 2j + 2 (this lane) / 2j + 1 and 2j + 3 (lane ^ 2) of the same row: one exchange, then each lane
// stores two adjacent units.
__device__ __forceinline__ void pair_store2(float* rowp, int j, bool hi_lane, float a, float b, bool st) {
  const float r = __shfl_xor_sync(IC3_FULL_MASK, hi_lane ? a : b, 2);
  const float2 v = hi_lane ? make_float2(r, b) : make_float2(a, r);
  if (st) *reinterpret_cast<float2*>(rowp + 2 * j + (hi_lane ? 2 : 0)) = v;
}
// The inverse: each lane loads two adjacent units, one exchange gives a = unit 2j + hi_lane, b = unit 2j + 2 + hi_lane.
__device__ __forceinline__ void pair_load2(const float* rowp, int j, bool hi_lane, bool ld, float& a, float& b) {
  const float2 v = ld ? *reinterpret_cast<const float2*>(rowp + 2 * j + (hi_lane ? 2 : 0)) : make_float2(0.f, 0.f);
  const float r = __shfl_xor_sync(IC3_FULL_MASK, hi_lane ? v.x : v.y, 2);
  a = hi_lane ? r : v.x;
  b = hi_lane ? v.y : r;
}

// Epilogue of one work item of a consumer thread: LSTM cell of its 32 units from the accumulators, h'/c' stores,
// partial head logits (slot = column half, unit parity, unit half; fixed order -> deterministic).
__device__ __forceinline__ void epilogue_item(const ic3_policy_cfg& cfg, const ic3_policy_io& io, const float* s_bias,
                                              const float* s_hw, float* __restrict__ partial, const float (&d)[128],
                                              int tile, int nh, int wg, int w4, int lane, bool ok) {
  const int R = cfg.B * cfg.N;
  const bool odd = lane & 1, hl = (lane >> 1) & 1;
  const int row = tile * TC_M + wg * 64 + w4 * 16 + (lane >> 2) + (odd ? 8 : 0);
  const bool st = ok && row < R;
  bool fr = false;
  if (row < R && io.fresh && io.pass_index == 0) fr = io.fresh[row / cfg.N] != 0;
  const int ub = nh * (TC_NH / 4) + hl;             // unit of j = 0; unit of j = ub + 2j
  const float* crow = io.c + (size_t)row * TC_H + nh * (TC_NH / 4);
  float part[2][HEAD_PAD];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int o = 0; o < HEAD_PAD; ++o) part[h][o] = 0.f;
#pragma unroll
  for (int j0 = 0; j0 < 32; j0 += 4) {             // 4 units per cell call
    float v[16], co[4], cn[4], hn[4];
    pair_load2(crow, j0, hl, row < R && !fr, co[0], co[1]);         // c of units ub + 2 (j0 .. j0 + 3)
    pair_load2(crow, j0 + 2, hl, row < R && !fr, co[2], co[3]);
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      float g[4];
      gather_gates(d, j0 + jj, odd, g);
      v[4 * jj + 0] = g[0]; v[4 * jj + 1] = g[1]; v[4 * jj + 2] = g[2]; v[4 * jj + 3] = g[3];
    }
    lstm_cell4(v, co, s_bias + 4 * (ub + 2 * j0), 8, cn, hn);
    if (partial) {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int u = ub + 2 * (j0 + jj);
        const float4 w0 = *reinterpret_cast<const float4*>(&s_hw[u * HEAD_PAD]);
        const float4 w1 = *reinterpret_cast<const float4*>(&s_hw[u * HEAD_PAD + 4]);
        float* p = part[j0 >= 16];
        p[0] = fmaf(hn[jj], w0.x, p[0]); p[1] = fmaf(hn[jj], w0.y, p[1]);
        p[2] = fmaf(hn[jj], w0.z, p[2]); p[3] = fmaf(hn[jj], w0.w, p[3]);
        p[4] = fmaf(hn[jj], w1.x, p[4]); p[5] = fmaf(hn[jj], w1.y, p[5]);
        p[6] = fmaf(hn[jj], w1.z, p[6]); p[7] = fmaf(hn[jj], w1.w, p[7]);
      }
    }
    float* co_row = io.c_out + (size_t)row * TC_H + nh * (TC_NH / 4);
    float* ho_row = io.h_out + (size_t)row * TC_H + nh * (TC_NH / 4);
#pragma unroll
    for (int pr = 0; pr < 2; ++pr) {
      pair_store2(co_row, j0 + 2 * pr, hl, cn[2 * pr], cn[2 * pr + 1], st);
      pair_store2(ho_row, j0 + 2 * pr, hl, hn[2 * pr], hn[2 * pr + 1], st);
    }
  }
  if (partial && st) {
    float4* p = reinterpret_cast<float4*>(partial + ((size_t)row * NSLOT + nh * 4 + hl * 2) * HEAD_PAD);
    p[0] = make_float4(part[0][0], part[0][1], part[0][2], part[0][3]);
    p[1] = make_float4(part[0][4], part[0][5], part[0][6], part[0][7]);
    p[2] = make_float4(part[1][0], part[1][1], part[1][2], part[1][3]);
    p[3] = make_float4(part[1][4], part[1][5], part[1][6], part[1][7]);
  }
}

__global__ void __launch_bounds__(TC_P_THREADS, 1) lstm_tc_kernel(ic3_policy_cfg cfg, ic3_policy_io io,
                                                                 const __half* __restrict__ a_img,
                                                                 const __half* __restrict__ b_img,
                                                                 const float* __restrict__ bias_cat, int nitems,
                                                                 const float* __restrict__ head_w, int nout,
                                                                 float* __restrict__ partial) {
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGE_P * STAGE_BYTES);
  // head weights, unit-major [128][8] (zero padded): the epilogue folds value/action-head dot products
  // of its hidden units into per-slot partial logits (partial != nullptr  <=>  nout <= 8)
  float* s_hw = reinterpret_cast<float*>(smem + NSTAGE_P * STAGE_BYTES + 256);
  float* s_bias = s_hw + TC_H * HEAD_PAD;
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + NSTAGE_P);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE_P; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, MMA_WARPS);   // one release per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  load_scaled_bias(s_bias, bias_cat);
  if (partial) {
    for (int idx = threadIdx.x; idx < TC_H * HEAD_PAD; idx += blockDim.x) {
      const int u = idx / HEAD_PAD, o = idx - u * HEAD_PAD;
      s_hw[idx] = o < nout ? __ldg(head_w + (size_t)o * TC_H + u) : 0.f;
    }
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
          [=](int item, int c) { return b + (size_t)((item & 1) * TC_NCHUNK + c) * B_CHUNK_BYTES; }, io.err);
    }
  } else {
    const int wg = warp >> 2, w4 = warp & 3;
    float d[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0.f;
    uint32_t li = 0;
    bool ok = true;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x, ++li) {
      wg_gemm_item<TC_NCHUNK>(d, smem_base, wg * 1024, bar_full, bar_empty, li, lane, ok, io.err);
      epilogue_item(cfg, io, s_bias, s_hw, partial, d, item >> 1, item & 1, wg, w4, lane, ok);
    }
  }
}

// ---- heads + sampling from h' (comm.py:228-239, action_utils.py:32-36) -----------------------------
// P lanes per agent row (P = pow2 >= 1 + sum(na)), lane o of a group computes output o as a full
// 128-long dot product (h row broadcast inside the group, weight rows L1-resident), then the
// log-softmax / inverse-CDF sampling runs inside the group with width-P shuffles.
template <int P>
__global__ void __launch_bounds__(256) heads_kernel(ic3_policy_cfg cfg, ic3_policy_packed w, ic3_policy_io io) {
  constexpr int RPW = 32 / P;
  const int lane = threadIdx.x & 31, o = lane % P;
  const long R = (long)cfg.B * cfg.N;
  const long row = ((long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + lane / P;
  const bool live = row < R;
  int atot = 0;
  for (int k = 0; k < cfg.nheads; ++k) atot += cfg.head_dim[k];
  const int nout = 1 + atot;
  // head weights k-major in shared memory: the P lanes of a group read P consecutive floats,
  // every group reads the same addresses -> one broadcast wavefront per load
  __shared__ float s_w[TC_H * P];
  for (int idx = threadIdx.x; idx < TC_H * P; idx += blockDim.x) {
    const int k = idx / P, oo = idx - k * P;
    s_w[idx] = oo < nout ? __ldg(w.head_w + (size_t)oo * TC_H + k) : 0.f;
  }
  __syncthreads();
  float logit = 0.f;
  if (live) {
    const float4* hp = reinterpret_cast<const float4*>(io.h_out + (size_t)row * TC_H);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 8
    for (int q = 0; q < TC_H / 4; ++q) {
      const float4 hv = hp[q];
      a0 = fmaf(hv.x, s_w[(4 * q + 0) * P + o], a0);
      a1 = fmaf(hv.y, s_w[(4 * q + 1) * P + o], a1);
      a2 = fmaf(hv.z, s_w[(4 * q + 2) * P + o], a2);
      a3 = fmaf(hv.w, s_w[(4 * q + 3) * P + o], a3);
    }
    logit = (a0 + a1) + (a2 + a3) + (o < nout ? __ldg(w.head_b + o) : 0.f);
  }
  if (live && o == 0) io.value[row] = logit;
  const bool do_sample = io.action != nullptr;
  const bool greedy = cfg.greedy != 0;    // argmax: neither the action stream nor draws is read
  const int e = live ? (int)(row / cfg.N) : 0, i = live ? (int)(row - (long)e * cfg.N) : 0;
  uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
  if (do_sample && !greedy && !io.draws) {
    if (o == 0 && live) {
      const uint4 d = ic3_draw24(cfg.seed, cfg.env_id0 + (uint32_t)e, io.tick ? io.tick[e] : 0u, IC3_STREAM_ACTION, (uint32_t)i);
      w0 = d.x; w1 = d.y; w2 = d.z; w3 = d.w;
    }
    w0 = __shfl_sync(IC3_FULL_MASK, w0, 0, P); w1 = __shfl_sync(IC3_FULL_MASK, w1, 0, P);
    w2 = __shfl_sync(IC3_FULL_MASK, w2, 0, P); w3 = __shfl_sync(IC3_FULL_MASK, w3, 0, P);
  }
  int off = 1;
  for (int k = 0; k < cfg.nheads; ++k) {
    const int na = cfg.head_dim[k];
    float m = -INFINITY;
    for (int a = 0; a < na; ++a) m = fmaxf(m, __shfl_sync(IC3_FULL_MASK, logit, off + a, P));
    float s = 0.f;
    for (int a = 0; a < na; ++a) s += expf(__shfl_sync(IC3_FULL_MASK, logit, off + a, P) - m);
    const float mylogp = logit - (m + logf(s));
    uint32_t u24 = 0;
    if (do_sample && !greedy) {
      if (io.draws) u24 = live ? io.draws[(size_t)row * cfg.nheads + k] : 0u;
      else u24 = k == 0 ? w0 : (k == 1 ? w1 : (k == 2 ? w2 : w3));
    }
    const float u = (float)u24 * 5.9604644775390625e-08f;
    int act = na - 1;
    if (do_sample && greedy) {
      for (int a = na - 1; a >= 0; --a)
        if (__shfl_sync(IC3_FULL_MASK, logit, off + a, P) == m) act = a;
    } else if (do_sample) {
      float cdf = 0.f;
      bool found = false;
      for (int a = 0; a < na; ++a) {
        cdf += expf(__shfl_sync(IC3_FULL_MASK, mylogp, off + a, P));
        if (!found && cdf > u) {
          act = a;
          found = true;
        }
      }
    }
    if (live && o >= off && o < off + na) io.logp[(size_t)row * atot + (off - 1) + (o - off)] = mylogp;
    if (live && do_sample && o == 0) io.action[(size_t)row * cfg.nheads + k] = act;
    off += na;
  }
}

// Finish the heads from the NSLOT per-slot partial logits (fixed summation order -> deterministic):
// value, log-softmax per head, inverse-CDF sampling.  One thread per agent row.
__global__ void __launch_bounds__(128) heads_finish_kernel(ic3_policy_cfg cfg, ic3_policy_packed w, ic3_policy_io io,
                                                            const float* __restrict__ partial) {
  const long row = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= (long)cfg.B * cfg.N) return;
  HeadsFinish f;
  f.partial = partial; f.head_b = w.head_b; f.nheads = cfg.nheads;
#pragma unroll
  for (int k = 0; k < IC3_MAX_HEADS; ++k) f.head_dim[k] = cfg.head_dim[k];
  f.seed = cfg.seed; f.env_id0 = cfg.env_id0; f.tick = io.tick; f.draws = io.draws;
  f.value = io.value; f.logp = io.logp; f.action = io.action; f.greedy = cfg.greedy;
  const int e = (int)(row / cfg.N), i = (int)(row - (long)e * cfg.N);
  heads_finish_row(f, row, e, i);
}

}  // namespace
