// Backward of the non-recurrent tanh policies (models.MLP, CommNet / IC3Net without --recurrent) on the Hopper tensor
// cores: ic3_ff_grad_* with plan->impl == IC3_FF_GRAD_TC.  The forward re-run, the observation pattern, the heads
// backward and the float64 finish are those of the SIMT path (bptt_tc.cu); this file replaces its three fp32 SIMT
// stages.  Per chunk, for p = P-1 .. 0:
//   dgrad   dz = g (1 - h_{p+1}^2) (g of the last pass: dout . W_heads), dx += dz, then one wgmma product
//           [dz F_p | dz C_p] (N = 128 without communication, 256 with it) over 128-row tiles of whole envs; the comm
//           scatter  g += gate (sum_{m != row} gs_m dS_m)  runs in the epilogue from shared memory.  On pass 0 the
//           epilogue writes dpre = (dx + g) (1 - tanh(x)^2) instead of g.                        [fgt_dgrad_kernel]
//   wgrad   G_F += dz^T h_p, G_C += dz^T S_p (both operands MN-major, contraction over the rows of a fixed row block),
//           g_b += sum dz                                                                       [fgt_wgrad_kernel]
// then the encoder: Y += dpre^T P with the P tile built in shared memory from (pos, ext)          [fgt_wgrad_kernel<PAT>]
//
// Arithmetic: the fp16 hi/lo split with three MMAs (hi.hi + lo.hi + hi.lo, fp32 accumulate) of the forward kernels.
// 3xTF32 would keep about the same 22 significant bits, but the fp16 MMA issues at twice the TF32 rate; fp16's narrow
// exponent range is handled by power-of-two operand scales:
//   weights   one scale for all passes, from max |F|, |C| (max * s in [2^13, 2^14))               [fgt_wmax_kernel]
//   dz (dgrad A operand)   per 128-row tile, from the tile's own max |dz|
//   dz, dpre (weight-gradient A operands)   per chunk and pass, from max |dz| / max |dpre| that the dgrad kernel
//             gathers with atomicMax on the bits of non-negative floats
//   h, S, P   fixed 16 (|h| <= 1, |S| <= N - 1, counts <= N): the predator-prey pattern (one-hot, counts, 1) is exact
//             in fp16 and needs no lo half; the traffic-junction route ratio is not, so its P is split as well.
// The weight-gradient row partition is that of the SIMT path (nb fixed blocks, rows in increasing order within a
// block, fp32 partials summed in float64 in block order by ic3_ff_grad_finish): bit-identical run to run.
#include <cstddef>
#include <cstring>

#include "ff_grad_tc.h"
#include "ic3_common.cuh"
#include "tc_common.cuh"

namespace {

constexpr int G_H = 128;
constexpr int G_HEADS = 8;                       // value + logits slots of dout (BP_HEADS of bptt_tc.cu)
constexpr int G_THREADS = 256;                   // two warpgroups
// dgrad: 128-row tiles (warpgroup w: rows 64 w ..), the dz image K-major, then the fp32 dS tile over it
constexpr int DG_TM = 128;
constexpr int DG_A_PART = DG_TM * G_H * 2;       // bytes of the hi (or lo) half of a tile's dz image
constexpr int DG_DS_LD = G_H + 8;                // fp32 dS rows, padded
constexpr int DG_A_BYTES = DG_TM * DG_DS_LD * 4;
static_assert(DG_A_BYTES >= 2 * DG_A_PART, "the dS tile overlays the dz image");
// wgrad: 32-row slabs, double-buffered: [A hi, A lo, B hi, B lo], each [16 column groups][4 row groups][8][8] halfs
constexpr int WS_ROWS = 32;
constexpr int WS_PART = WS_ROWS * G_H * 2;
constexpr int WS_STAGE = 4 * WS_PART;
constexpr int WS_SMEM = 2 * WS_STAGE;
constexpr float B_SCALE = SCALE_A;               // scale of the h / S / P operands (16)

struct FgtScalars {
  float wscale;                                  // scale of the weight images
  unsigned dzmax[IC3_MAX_PASSES];                // bits of max |dz| of the chunk, per pass
  unsigned dpmax;                                // bits of max |dpre| of the chunk
};
constexpr size_t TC_SC_BYTES = 256;              // the scale words, ahead of the images
static_assert(sizeof(FgtScalars) <= TC_SC_BYTES, "scale words");

template <bool COMM>
struct DgLayout {
  static constexpr int NOUT = COMM ? 2 * G_H : G_H;        // [dz F | dz C]
  static constexpr int W_PART = NOUT * G_H * 2;            // bytes of the hi (or lo) half of one pass's image
  static constexpr int W_BYTES = 2 * W_PART;
  static constexpr size_t SMEM = (size_t)W_BYTES + DG_A_BYTES + (G_HEADS * G_H + 2 * DG_TM + 8) * sizeof(float);
};

// 2^e with m * 2^e in [2^13, 2^14): hi below 2^14 in fp16, lo keeps 2^-35 of m; 1 for m = 0
__device__ __forceinline__ float pow2_scale(float m) {
  if (!(m > 0.f) || !isfinite(m)) return 1.f;
  int e;
  frexpf(m, &e);                                 // m = f 2^e, f in [0.5, 1)
  e = 14 - e;
  e = e > 100 ? 100 : (e < -100 ? -100 : e);
  return ldexpf(1.f, e);
}

__device__ __forceinline__ float max4(const float4& v) {
  return fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
}

// weight image of one pass and part, in halfs: element (output column n, contraction index k) -- K-major B operand
__host__ __device__ __forceinline__ size_t w_off(int nout, int n, int k) {
  return ((size_t)(k >> 3) * (nout / 8) + (n >> 3)) * 64 + (n & 7) * 8 + (k & 7);
}
// dz image of a dgrad tile, in halfs: row rl, float4 column q -- K-major A operand
__device__ __forceinline__ int dg_a_off(int rl, int q) {
  return ((q >> 1) * (DG_TM / 8) + (rl >> 3)) * 64 + (rl & 7) * 8 + (q & 1) * 4;
}
// one part of a wgrad slab, in halfs: slab row r, column c (MN-major: 8 consecutive columns are 16 contiguous bytes)
__device__ __forceinline__ int ws_off(int r, int c) { return (c >> 3) * 256 + (r >> 3) * 64 + (r & 7) * 8 + (c & 7); }

// ---------------------------------------------------------------------------------------------------------- weights
__global__ void __launch_bounds__(1024) fgt_wmax_kernel(const float* __restrict__ f, const float* __restrict__ c, int n,
                                                        FgtScalars* sc) {
  __shared__ float s_m[32];
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    m = fmaxf(m, fabsf(f[i]));
    if (c) m = fmaxf(m, fabsf(c[i]));
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(IC3_FULL_MASK, m, s));
  if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, s_m[w]);
    sc->wscale = pow2_scale(fmaxf(m, s_m[0]));
    for (int p = 0; p < IC3_MAX_PASSES; ++p) sc->dzmax[p] = 0u;
    sc->dpmax = 0u;
  }
}

// image of pass p: element (n, k) = F_p[k][n] = f_wT[p][n][k] for n < 128, C_p[k][n - 128] = c_wT[p][n - 128][k] above
__global__ void fgt_pack_kernel(const float* __restrict__ f_wT, const float* __restrict__ c_wT, int nout, int P,
                                __half* __restrict__ img, const FgtScalars* __restrict__ sc) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P * nout * G_H) return;
  const int p = idx / (nout * G_H), r = idx - p * nout * G_H, n = r >> 7, k = r & 127;
  const size_t HH = (size_t)G_H * G_H;
  const float v = n < G_H ? f_wT[p * HH + (size_t)n * G_H + k] : c_wT[p * HH + (size_t)(n - G_H) * G_H + k];
  __half hi, lo;
  split_f16(v, sc->wscale, hi, lo);
  __half* base = img + (size_t)p * 2 * nout * G_H;
  base[w_off(nout, n, k)] = hi;
  base[(size_t)nout * G_H + w_off(nout, n, k)] = lo;
}

// ---------------------------------------------------------------------------------------------------------- dgrad
struct DgradArgs {
  int N, Bk, epb, ntiles, last, first_acc, final_pass, hard_attn, comm_avg, nout, ps;
  const float* h_out;        // [R, H] h_{p+1}
  const float* xt;           // [R, H] tanh(x) (final pass)
  const float* dout; const float* head_w;
  const uint8_t* fresh; const uint8_t* comm_action; const uint8_t* alive; const uint8_t* valid;
  float* g; float* dx; float* dz;
  const __half* w_img;       // this pass's image
  FgtScalars* sc;
};

template <bool COMM>
__global__ void __launch_bounds__(G_THREADS, 1) fgt_dgrad_kernel(DgradArgs a) {
  using L = DgLayout<COMM>;
  extern __shared__ __align__(1024) unsigned char smem[];
  __half* s_a = reinterpret_cast<__half*>(smem + L::W_BYTES);
  float* s_ds = reinterpret_cast<float*>(smem + L::W_BYTES);
  float* s_hw = reinterpret_cast<float*>(smem + L::W_BYTES + DG_A_BYTES);    // head weights [8][H]
  float* s_gate = s_hw + G_HEADS * G_H;
  float* s_gs = s_gate + DG_TM;
  float* s_red = s_gs + DG_TM;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, w4 = warp & 3;
  const int N = a.N;
  for (int i = tid; i < L::W_BYTES / 16; i += G_THREADS)
    reinterpret_cast<uint4*>(smem)[i] = __ldg(reinterpret_cast<const uint4*>(a.w_img) + i);
  for (int i = tid; i < G_HEADS * G_H; i += G_THREADS) s_hw[i] = (i >> 7) < a.nout ? __ldg(a.head_w + i) : 0.f;
  __syncthreads();                 // the head weights are read by every thread of the first tile's dz stage
  const float wunscale = 1.f / a.sc->wscale;
  const uint32_t base = smem_u32(smem);
  // K-major, no swizzle: LBO = distance of K-adjacent core matrices, SBO = distance of 8-row groups
  const uint64_t dA = make_desc(base + L::W_BYTES + wg * 1024, (DG_TM / 8) * 128, 128);
  const uint64_t dB = make_desc(base, (L::NOUT / 8) * 128, 128);
  const int fr = lane >> 2, fc = 2 * (lane & 3);
  float dpmax = 0.f;

  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int e0 = tile * a.epb;
    const int nrows = min(a.epb, a.Bk - e0) * N;
    const size_t row0 = (size_t)e0 * N;
    if (COMM && tid < DG_TM) {                     // comm gate and mean factor, as policy_step_kernel stage A
      const int r = tid;
      float gt = 0.f, den = 1.f;
      if (r < nrows) {
        const int el = r / N, e = e0 + el, i = r - el * N;
        const bool fr0 = a.fresh && a.fresh[e];
        int n_alive = N, al = 1;
        if (a.alive && !fr0) {
          n_alive = 0;
          for (int j = 0; j < N; ++j) n_alive += a.alive[(size_t)e * N + j] != 0;
          al = a.alive[(size_t)e * N + i] != 0;
        }
        int cm = 1;
        if (a.hard_attn) cm = fr0 ? 0 : (a.comm_action[(size_t)e * N + i] != 0);
        gt = (float)(al * cm);
        if (a.comm_avg && n_alive > 1) den = (float)(n_alive - 1);
      }
      s_gate[r] = gt;
      s_gs[r] = gt / den;
    }
    // ---- dz = g (1 - h_{p+1}^2), dx (+)= dz; the tile's max |dz| ------------------------------------------------
    float4 v[DG_TM * G_H / 4 / G_THREADS];
    float m = 0.f;
#pragma unroll
    for (int k = 0; k < DG_TM * G_H / 4 / G_THREADS; ++k) {
      const int it = k * G_THREADS + tid, rl = it >> 5, q = it & 31;
      float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
      if (rl < nrows) {
        const size_t o = (row0 + rl) * G_H + 4 * q;
        if (!a.valid || a.valid[e0 + rl / N]) {
          float4 gin;
          if (a.last) {
            gin = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int k2 = 0; k2 < a.nout; ++k2) {
              const float dv = a.dout[(row0 + rl) * G_HEADS + k2];
              const float4 w = *reinterpret_cast<const float4*>(s_hw + k2 * G_H + 4 * q);
              gin.x = fmaf(dv, w.x, gin.x); gin.y = fmaf(dv, w.y, gin.y);
              gin.z = fmaf(dv, w.z, gin.z); gin.w = fmaf(dv, w.w, gin.w);
            }
          } else {
            gin = *reinterpret_cast<const float4*>(a.g + o);
          }
          const float4 h = __ldg(reinterpret_cast<const float4*>(a.h_out + o));
          d = make_float4(gin.x * (1.f - h.x * h.x), gin.y * (1.f - h.y * h.y), gin.z * (1.f - h.z * h.z),
                          gin.w * (1.f - h.w * h.w));
        }
        *reinterpret_cast<float4*>(a.dz + o) = d;
        float4 x = d;
        if (!a.first_acc) {
          const float4 p = *reinterpret_cast<const float4*>(a.dx + o);
          x = make_float4(p.x + d.x, p.y + d.y, p.z + d.z, p.w + d.w);
        }
        *reinterpret_cast<float4*>(a.dx + o) = x;
      }
      v[k] = d;
      m = fmaxf(m, max4(d));
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(IC3_FULL_MASK, m, s));
    if (lane == 0) s_red[warp] = m;
    __syncthreads();
    m = s_red[0];
#pragma unroll
    for (int w = 1; w < G_THREADS / 32; ++w) m = fmaxf(m, s_red[w]);
    if (tid == 0 && m > 0.f) atomicMax(&a.sc->dzmax[a.ps], __float_as_uint(m));
    const float sA = pow2_scale(m);
#pragma unroll
    for (int k = 0; k < DG_TM * G_H / 4 / G_THREADS; ++k) {
      const int it = k * G_THREADS + tid, rl = it >> 5, q = it & 31;
      store_split4(s_a, dg_a_off(rl, q), DG_A_PART / 2 + dg_a_off(rl, q), v[k], sA);
    }
    fence_proxy_async();           // the image (and, first tile, the weights) was written through the generic proxy
    __syncthreads();

    // ---- [dz F | dz C] = (sA dz) . (s_w [F | C]), fp32 accumulators -------------------------------------------------
    float d[L::NOUT / 2];
#pragma unroll
    for (int i = 0; i < L::NOUT / 2; ++i) d[i] = 0.f;
    wgmma_fence_regs(d);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < G_H / 16; ++ks) {
      const uint64_t da_hi = dA + ((ks * 2 * (DG_TM / 8) * 128) >> 4), da_lo = da_hi + (DG_A_PART >> 4);
      const uint64_t db_hi = dB + ((ks * 2 * (L::NOUT / 8) * 128) >> 4), db_lo = db_hi + (L::W_PART >> 4);
      if constexpr (COMM) {
        wgmma_m64n256_kk(d, da_hi, db_hi, ks != 0);
        wgmma_m64n256_kk(d, da_lo, db_hi, 1);
        wgmma_m64n256_kk(d, da_hi, db_lo, 1);
      } else {
        wgmma_m64n128_kk(d, da_hi, db_hi, ks != 0);
        wgmma_m64n128_kk(d, da_lo, db_hi, 1);
        wgmma_m64n128_kk(d, da_hi, db_lo, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    __syncthreads();               // every warp's MMAs have read the dz image: dS may overwrite it
    const float unscale = wunscale / sA;

    // ---- comm scatter: s_ds[row] = sum_{m != row, same env} gs_m dS_m ------------------------------------------------
    if constexpr (COMM) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int rl = 64 * wg + 16 * w4 + fr + 8 * i;
        const float f = unscale * s_gs[rl];
#pragma unroll
        for (int j = 16; j < 32; ++j)
          *reinterpret_cast<float2*>(s_ds + rl * DG_DS_LD + 8 * (j - 16) + fc) =
              make_float2(d[4 * j + 2 * i] * f, d[4 * j + 2 * i + 1] * f);
      }
      __syncthreads();
      const int nenv = nrows / N;
      for (int it = tid; it < nenv * (G_H / 4); it += G_THREADS) {
        const int rb = (it >> 5) * N, q = it & 31;
        float4 T = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < N; ++j) {
          const float4 x = *reinterpret_cast<const float4*>(s_ds + (rb + j) * DG_DS_LD + 4 * q);
          T.x += x.x; T.y += x.y; T.z += x.z; T.w += x.w;
        }
        for (int j = 0; j < N; ++j) {
          float4* p = reinterpret_cast<float4*>(s_ds + (rb + j) * DG_DS_LD + 4 * q);
          const float4 x = *p;
          *p = make_float4(T.x - x.x, T.y - x.y, T.z - x.z, T.w - x.w);
        }
      }
      __syncthreads();
    }

    // ---- g = dz F + scatter  (pass 0: dpre = (dx + g) (1 - tanh(x)^2)) ----------------------------------------------
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int rl = 64 * wg + 16 * w4 + fr + 8 * i;
      if (rl >= nrows) continue;
      const bool gated = COMM && s_gate[rl] != 0.f;
      const size_t rowo = (row0 + rl) * G_H;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = 8 * j + fc;
        float2 o = make_float2(d[4 * j + 2 * i] * unscale, d[4 * j + 2 * i + 1] * unscale);
        if (gated) {
          const float2 t = *reinterpret_cast<const float2*>(s_ds + rl * DG_DS_LD + col);
          o.x += t.x; o.y += t.y;
        }
        if (a.final_pass) {
          const float2 x = *reinterpret_cast<const float2*>(a.dx + rowo + col);
          const float2 xt = __ldg(reinterpret_cast<const float2*>(a.xt + rowo + col));
          o = make_float2((x.x + o.x) * (1.f - xt.x * xt.x), (x.y + o.y) * (1.f - xt.y * xt.y));
          dpmax = fmaxf(dpmax, fmaxf(fabsf(o.x), fabsf(o.y)));
        }
        *reinterpret_cast<float2*>(a.g + rowo + col) = o;
      }
    }
    __syncthreads();               // the next tile's image and gates replace this tile's
  }
  if (a.final_pass) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) dpmax = fmaxf(dpmax, __shfl_xor_sync(IC3_FULL_MASK, dpmax, s));
    if (lane == 0 && dpmax > 0.f) atomicMax(&a.sc->dpmax, __float_as_uint(dpmax));
  }
}

// ---------------------------------------------------------------------------------------------------------- wgrad
// part[blk][n][ld] (+)= sum over the rows of block blk of A[r][n] * B[r][c] (columns c of tile blockIdx.y).  PAT: B is
// the observation pattern (pos, ext); else B = b[blockIdx.y] dense [R, H] and (tile 0) bsum[blk][n] (+)= sum of A[r][n].
struct WgradArgs {
  int R, nb, ld, npos, ne, ps;     // ps: the dzmax word of A's scale; -1: dpmax
  const float* A;
  const float* b[2];
  float* part[2];
  size_t part_stride;              // floats per block
  const int32_t* pos; const float* ext;
  float* bsum;
  const FgtScalars* sc;
};

template <bool PAT, bool SPLIT>
__global__ void __launch_bounds__(G_THREADS, 2) fgt_wgrad_kernel(WgradArgs a) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ float s_bs[G_THREADS / 32][G_H];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, w4 = warp & 3;
  const int blk = blockIdx.x, y = blockIdx.y;
  const long r0 = (long)a.R * blk / a.nb, r1 = (long)a.R * (blk + 1) / a.nb;
  const float* B = PAT ? nullptr : (y == 0 ? a.b[0] : a.b[1]);     // (no dynamic index into the parameter)
  const int c0 = PAT ? y * G_H : 0;
  const float sA = pow2_scale(__uint_as_float(a.ps >= 0 ? a.sc->dzmax[a.ps] : a.sc->dpmax));
  const bool bias = !PAT && y == 0;
  const int q = tid & 31, rs = tid >> 5;           // staging: float4 column q of slab rows rs, rs + 8, rs + 16, rs + 24
  float bs[4] = {0.f, 0.f, 0.f, 0.f};
  float d[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  const uint32_t base = smem_u32(smem);
  const int nch = (int)((r1 - r0 + WS_ROWS - 1) / WS_ROWS);
  wgmma_fence_regs(d);
  for (int ch = 0; ch < nch; ++ch) {
    __half* st = reinterpret_cast<__half*>(smem + (ch & 1) * WS_STAGE);
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {             // two rows in flight per operand: 128 registers with the accumulators
      float4 va[2], vb[2];
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const long row = r0 + (long)ch * WS_ROWS + rs + 8 * (2 * h2 + k);
        va[k] = vb[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < r1) {
          va[k] = __ldg(reinterpret_cast<const float4*>(a.A + (size_t)row * G_H) + q);
          if (PAT) {
            const int p = a.pos[row];
            float w[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int c = c0 + 4 * q + j;
              w[j] = c < a.npos ? (c == p ? 1.f : 0.f) : (c - a.npos < a.ne ? a.ext[(size_t)row * a.ne + c - a.npos] : 0.f);
            }
            vb[k] = make_float4(w[0], w[1], w[2], w[3]);
          } else {
            vb[k] = __ldg(reinterpret_cast<const float4*>(B + (size_t)row * G_H) + q);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int r = rs + 8 * (2 * h2 + k);
        if (bias) { bs[0] += va[k].x; bs[1] += va[k].y; bs[2] += va[k].z; bs[3] += va[k].w; }
        store_split4(st, ws_off(r, 4 * q), WS_PART / 2 + ws_off(r, 4 * q), va[k], sA);
        store_split4(st, WS_PART + ws_off(r, 4 * q), 3 * WS_PART / 2 + ws_off(r, 4 * q), vb[k], B_SCALE);
      }
    }
    fence_proxy_async();
    __syncthreads();
    wgmma_fence();
    const uint32_t sb = base + (ch & 1) * WS_STAGE;
#pragma unroll
    for (int ks = 0; ks < WS_ROWS / 16; ++ks) {
      // MN-major no-swizzle: LBO = 128 B between the two 8-row (K) groups, SBO = 512 B between 8-column groups
      const uint64_t a_hi = make_desc(sb + wg * 8 * 512 + ks * 256, 128, 512), a_lo = a_hi + (WS_PART >> 4);
      const uint64_t b_hi = make_desc(sb + 2 * WS_PART + ks * 256, 128, 512), b_lo = b_hi + (WS_PART >> 4);
      wgmma_m64n128_mn(d, a_hi, b_hi, (ch | ks) != 0);
      wgmma_m64n128_mn(d, a_lo, b_hi, 1);
      if (SPLIT) wgmma_m64n128_mn(d, a_hi, b_lo, 1);
    }
    wgmma_commit();
    wgmma_wait<1>();               // the MMAs of slab ch - 1 have read their stage ...
    __syncthreads();               // ... in both warpgroups: slab ch + 1 may overwrite it
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  // flush: fragment (m, n) -> part[m][c0 + n]
  const float unscale = 1.f / (sA * B_SCALE);
  float* out = (PAT ? a.part[0] + c0 : (y == 0 ? a.part[0] : a.part[1])) + (size_t)blk * a.part_stride;
  const int fr = lane >> 2, fc = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int mrow = 64 * wg + 16 * w4 + fr + 8 * i;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) out[(size_t)mrow * a.ld + 8 * j + fc + c] += d[4 * j + 2 * i + c] * unscale;
  }
  if (bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j) s_bs[rs][4 * q + j] = bs[j];
    __syncthreads();
    if (tid < G_H) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < G_THREADS / 32; ++w) t += s_bs[w][tid];
      a.bsum[(size_t)blk * G_H + tid] += t;
    }
  }
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      n = 0;
  }
  return n;
}

template <bool COMM>
int dgrad_launch(const DgradArgs& a, cudaStream_t s) {
  static bool ready = false;
  const size_t smem = DgLayout<COMM>::SMEM;
  if (!ready) {
    cudaError_t e = cudaFuncSetAttribute(fgt_dgrad_kernel<COMM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    ready = true;
  }
  const int nsm = sm_count();
  if (nsm <= 0) return IC3_E_RANGE;
  fgt_dgrad_kernel<COMM><<<a.ntiles < nsm ? a.ntiles : nsm, G_THREADS, smem, s>>>(a);   // persistent: one CTA per SM
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

template <bool PAT, bool SPLIT>
int wgrad_launch(const WgradArgs& a, int ny, cudaStream_t s) {
  static bool ready = false;
  if (!ready) {
    cudaError_t e = cudaFuncSetAttribute(fgt_wgrad_kernel<PAT, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, WS_SMEM);
    if (e != cudaSuccess) return (int)e;
    ready = true;
  }
  fgt_wgrad_kernel<PAT, SPLIT><<<dim3(a.nb, ny), G_THREADS, WS_SMEM, s>>>(a);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

size_t img_bytes_per_pass(int comm) { return (size_t)2 * (comm ? 2 : 1) * G_H * G_H * 2; }

}  // namespace

uint64_t ic3_ff_grad_tc_bytes(int passes, int comm) {
  return (uint64_t)(TC_SC_BYTES + (size_t)passes * img_bytes_per_pass(comm));
}

int ic3_ff_grad_tc_pack(int passes, int comm, const float* f_wT, const float* c_wT, void* tc, cudaStream_t s) {
  FgtScalars* sc = reinterpret_cast<FgtScalars*>(tc);
  __half* img = reinterpret_cast<__half*>(reinterpret_cast<unsigned char*>(tc) + TC_SC_BYTES);
  const int n = passes * G_H * G_H, nout = comm ? 2 * G_H : G_H;
  fgt_wmax_kernel<<<1, 1024, 0, s>>>(f_wT, comm ? c_wT : nullptr, n, sc);
  IC3_LAUNCH_CHECK();
  const int items = passes * nout * G_H;
  fgt_pack_kernel<<<(items + 255) / 256, 256, 0, s>>>(f_wT, c_wT, nout, passes, img, sc);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

int ic3_ff_grad_tc_chunk(const FfGradTcChunk* c, cudaStream_t s) {
  FgtScalars* sc = reinterpret_cast<FgtScalars*>(c->tc);
  const unsigned char* img = reinterpret_cast<const unsigned char*>(c->tc) + TC_SC_BYTES;
  // the chunk's max |dz| / |dpre| words start from zero (the weight scale before them stays)
  cudaError_t e = cudaMemsetAsync(reinterpret_cast<unsigned char*>(c->tc) + offsetof(FgtScalars, dzmax), 0,
                                  sizeof(FgtScalars) - offsetof(FgtScalars, dzmax), s);
  if (e != cudaSuccess) return (int)e;
  const size_t RHs = (size_t)c->R * G_H, HH = (size_t)G_H * G_H;
  const int N = c->N;
  const int epb = DG_TM / N;
  int rc;
  for (int ps = c->P - 1; ps >= 0; --ps) {
    DgradArgs a;
    memset(&a, 0, sizeof(a));
    a.N = N; a.Bk = c->Bk; a.epb = epb; a.ntiles = (c->Bk + epb - 1) / epb;
    a.last = ps == c->P - 1; a.first_acc = ps == c->P - 1; a.final_pass = ps == 0;
    a.hard_attn = c->hard_attn; a.comm_avg = c->comm_avg; a.nout = c->nout; a.ps = ps;
    a.h_out = c->hs + (size_t)(ps + 1) * RHs; a.xt = c->hs;
    a.dout = c->dout; a.head_w = c->head_w;
    a.fresh = c->fresh; a.comm_action = c->comm_action; a.alive = c->alive; a.valid = c->valid;
    a.g = c->g; a.dx = c->dx; a.dz = c->dz;
    a.w_img = reinterpret_cast<const __half*>(img + (size_t)ps * img_bytes_per_pass(c->comm));
    a.sc = sc;
    rc = c->comm ? dgrad_launch<true>(a, s) : dgrad_launch<false>(a, s);
    if (rc) return rc;
    WgradArgs w;
    memset(&w, 0, sizeof(w));
    w.R = c->R; w.nb = c->nb; w.ld = G_H; w.ps = ps; w.A = c->dz;
    w.b[0] = c->hs + (size_t)ps * RHs;
    w.b[1] = c->comm ? c->ss + (size_t)ps * RHs : nullptr;
    w.part[0] = c->fpart + (size_t)ps * c->nb * HH;
    w.part[1] = c->comm ? c->cpart + (size_t)ps * c->nb * HH : nullptr;
    w.part_stride = HH;
    w.bsum = c->bpart + (size_t)ps * c->nb * G_H;
    w.sc = sc;
    rc = wgrad_launch<false, true>(w, c->comm ? 2 : 1, s);
    if (rc) return rc;
  }
  // encoder: Y += dpre^T P (dpre in g)
  WgradArgs w;
  memset(&w, 0, sizeof(w));
  w.R = c->R; w.nb = c->nb; w.ld = c->npad; w.npos = c->npos; w.ne = c->ne; w.ps = -1; w.A = c->g;
  w.part[0] = c->ypart;
  w.part_stride = (size_t)G_H * c->npad;
  w.pos = c->pos; w.ext = c->ext;
  w.sc = sc;
  return c->is_tj ? wgrad_launch<true, true>(w, c->npad / G_H, s) : wgrad_launch<true, false>(w, c->npad / G_H, s);
}
