// Per-row pieces of the encoder x = b + sum_f obs[f] * W_e[:, f] (comm.py:119), shared by the dense encoder
// (policy.cu), the index-form encoders (policy.cu) and the fused observation + encoder kernels (pp_env.cu,
// tj_env.cu).  One warp per agent row, lane = hidden units lane*CPT .. lane*CPT+CPT-1, wT = [O, H] (one H-row per
// feature, L2-resident).  Every form adds the non-zero features in increasing feature order, class terms and the
// other terms in two sums when the layout hint of ic3_policy_cfg is given (split), so all forms are bit-identical.
#pragma once
#include "ic3_common.cuh"

namespace {

template <int CPT>
__device__ __forceinline__ void axpy_row(float (&acc)[CPT], float v, const float* __restrict__ wrow, int lane) {
  if (CPT == 4) {
    const float4 wv = __ldg(reinterpret_cast<const float4*>(wrow) + lane);
    acc[0] = fmaf(v, wv.x, acc[0]); acc[1] = fmaf(v, wv.y, acc[1]);
    acc[2] = fmaf(v, wv.z, acc[2]); acc[3] = fmaf(v, wv.w, acc[3]);
  } else if (CPT == 2) {
    const float2 wv = __ldg(reinterpret_cast<const float2*>(wrow) + lane);
    acc[0] = fmaf(v, wv.x, acc[0]); acc[1] = fmaf(v, wv.y, acc[1]);
  } else {
    acc[0] = fmaf(v, __ldg(wrow + lane), acc[0]);
  }
}

template <int CPT>
__device__ __forceinline__ void store_x(const float (&acc)[CPT], float* __restrict__ xrow, int lane) {
  if (CPT == 4) reinterpret_cast<float4*>(xrow)[lane] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  else if (CPT == 2) reinterpret_cast<float2*>(xrow)[lane] = make_float2(acc[0], acc[1]);
  else xrow[lane] = acc[0];
}

template <int CPT>
__device__ __forceinline__ void store_x2(const float (&a)[CPT], const float (&b)[CPT], float* __restrict__ xrow, int lane) {
  float r[CPT];
#pragma unroll
  for (int c = 0; c < CPT; ++c) r[c] = a[c] + b[c];      // x = (bias + class terms) + (other terms)
  store_x<CPT>(r, xrow, lane);
}

// Predator-prey row: WW window cells of V = D*D + 4 features.  cell(w) returns the record of window cell w,
// cls | npred << 16 | nprey << 24 (pp_write_obs, pp_env.cu); cls is the position class or OUTSIDE = V - 3,
// the prey count is feature V - 2 and the predator count V - 1.  cell() is called by the whole warp.
template <int H, typename CellFn>
__device__ __forceinline__ void pp_encode_row(CellFn cell, int WW, int V, const float* __restrict__ wT,
                                              const float* __restrict__ bias, bool split, float* __restrict__ xrow,
                                              int lane) {
  constexpr int CPT = H / 32;
  float acc[CPT], acc2[CPT];
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
    acc[c] = __ldg(bias + lane * CPT + c);
    acc2[c] = 0.f;
  }
  for (int w = 0; w < WW; ++w) {
    const uint32_t info = cell(w);
    const int cls = (int)(info & 0xffffu), npred = (int)((info >> 16) & 0xffu), nprey = (int)(info >> 24);
    const float* wcell = wT + (size_t)w * V * H;
    axpy_row<CPT>(acc, 1.f, wcell + (size_t)cls * H, lane);
    if (split) {          // counts go to the second sum (ic3_policy_cfg.obs_vocab > 0)
      if (nprey) axpy_row<CPT>(acc2, (float)nprey, wcell + (size_t)(V - 2) * H, lane);
      if (npred) axpy_row<CPT>(acc2, (float)npred, wcell + (size_t)(V - 1) * H, lane);
    } else {
      if (nprey) axpy_row<CPT>(acc, (float)nprey, wcell + (size_t)(V - 2) * H, lane);
      if (npred) axpy_row<CPT>(acc, (float)npred, wcell + (size_t)(V - 1) * H, lane);
    }
  }
  store_x2<CPT>(acc, acc2, xrow, lane);
}

// Traffic-junction row: [last_act, route_id/(npath-1), WW cells x V classes], all zero for a dead car (x = b).
// cell(w) returns cls | count << 16 (tj_write_obs, tj_env.cu); the car count is feature car_cls > cls.
// SC (scalar vocabulary, never split: no layout hint): [last_act, route_id/(npath-1), pr, pc, WW cells x (ROAD, CAR)],
// cell column q is class q + 1, so OUTSIDE has no column and every in-map cell contributes at most its ROAD term.
template <int H, bool SC, typename CellFn>
__device__ __forceinline__ void tj_encode_row(bool alive, float la, float ri, float pr, float pc, CellFn cell, int WW,
                                              int V, int car_cls, const float* __restrict__ wT,
                                              const float* __restrict__ bias, bool split, float* __restrict__ xrow,
                                              int lane) {
  constexpr int CPT = H / 32;
  constexpr int S = SC ? 4 : 2, C0 = SC ? 1 : 0;   // scalar features; class of cell column 0
  float acc[CPT], acc2s[CPT];
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
    acc[c] = __ldg(bias + lane * CPT + c);
    acc2s[c] = 0.f;
  }
  // split (ic3_policy_cfg.obs_vocab > 0): scalars and car counts form the second sum
  if (alive) {
    if (split) {
      if (la != 0.f) axpy_row<CPT>(acc2s, la, wT, lane);
      if (ri != 0.f) axpy_row<CPT>(acc2s, ri, wT + H, lane);
    } else {
      if (la != 0.f) axpy_row<CPT>(acc, la, wT, lane);
      if (ri != 0.f) axpy_row<CPT>(acc, ri, wT + H, lane);
      if (SC && pr != 0.f) axpy_row<CPT>(acc, pr, wT + 2 * H, lane);
      if (SC && pc != 0.f) axpy_row<CPT>(acc, pc, wT + 3 * H, lane);
    }
    for (int w = 0; w < WW; ++w) {
      const uint32_t info = cell(w);
      const int cls = (int)(info & 0xffffu), cnt = (int)(info >> 16);
      const float* wcell = wT + (size_t)(S + w * V - C0) * H;     // row of class k: wcell + k * H
      // dense order: class index ascending; cls < car_cls always (BASE+2; scalar: ROAD 1 < CAR 2)
      if (!SC || cls >= C0) axpy_row<CPT>(acc, 1.f, wcell + (size_t)cls * H, lane);
      if (cnt) {
        if (split) axpy_row<CPT>(acc2s, (float)cnt, wcell + (size_t)car_cls * H, lane);
        else axpy_row<CPT>(acc, (float)cnt, wcell + (size_t)car_cls * H, lane);
      }
    }
  }
  store_x2<CPT>(acc, acc2s, xrow, lane);      // acc2s == 0 when not split: x = acc
}

}  // namespace
