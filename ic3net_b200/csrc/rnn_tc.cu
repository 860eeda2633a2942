// Policy step of the tanh RNN without communication (models.RNN with the vanilla recurrence: the IC and IRIC baselines,
// models.py:83-85) on the Hopper tensor cores, H = 128:
//   h' = tanh(x + W2 h + b2),  value / action heads, log-softmax, sampling.
//
// The only GEMM is h . W2^T (K = N = 128).  Its weight image -- the fp16 hi/lo split of 256 * W2 in the no-swizzle
// K-major core-matrix layout, 64 KB -- stays in shared memory for the whole launch; only activations stream.  Persistent
// CTAs of one warpgroup, two per SM, each looping over 64-row tiles:
//   A  x of the thread's accumulator fragment is requested from HBM (consumed in C, so its latency hides behind A and B)
//   A  h (zero for slots starting an episode) fp32 -> hi/lo fp16 (x 16) into the core-matrix layout in shared memory
//   B  8 k-steps x 3 wgmma m64n128k16 (hi.hi + lo.hi + hi.lo, tc_common.cuh) into 64 fp32 registers per thread
//   C  z = x + acc / 4096 + b2, h' = tanh(z) on the SFU, h' -> HBM and, as fp32, over the A image in shared memory
//   D  heads of the tile's rows from shared memory, one warp per row: the code of the SIMT kernel (policy_heads.cuh)
// No operand image goes through HBM and nothing is launched in front of the kernel but the encoder that writes x.
#include "ic3_common.cuh"
#include "policy_heads.cuh"
#include "policy_internal.h"
#include "tc_common.cuh"

namespace {

constexpr int RT_H = 128;
constexpr int RT_M = 64;                          // rows per tile: one warpgroup
constexpr int RT_THREADS = 128;
constexpr int RT_W_PART = RT_H * RT_H * 2;        // bytes of the hi (or lo) half of the weight image
constexpr int RT_A_PART = RT_M * RT_H * 2;        // bytes of the hi (or lo) half of a tile's h image
constexpr int RT_HP_LD = RT_H + 8;                // fp32 h' tile, rows padded: the fragment's float2 stores hit every bank once
constexpr int RT_AH_BYTES = RT_M * RT_HP_LD * 4;  // the h image (2 * RT_A_PART) and the h' tile share this region
constexpr size_t RT_SMEM_BYTES = 2 * RT_W_PART + RT_AH_BYTES + 2 * RT_H * sizeof(float);
static_assert(RT_AH_BYTES >= 2 * RT_A_PART, "the h' tile covers the h image");
static_assert(IC3_RNN_IMG_BYTES == 2 * RT_W_PART, "weight image size of the header");

// weight image, in halfs: [hi, lo][k >> 3][n >> 3][n & 7][k & 7]  (W2[n][k]: K-major B operand of h . W2^T)
__host__ __device__ __forceinline__ size_t rt_w_off(int n, int k, int part) {
  return (size_t)part * (RT_W_PART / 2) + ((size_t)(k >> 3) * (RT_H / 8) + (n >> 3)) * 64 + (n & 7) * 8 + (k & 7);
}

__global__ void rnn_tc_pack_kernel(const float* __restrict__ f_w, __half* __restrict__ img, int32_t* __restrict__ flags) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;      // (n, k)
  if (idx >= RT_H * RT_H) return;
  const int n = idx / RT_H, k = idx - n * RT_H;
  const float w = f_w[idx];
  __half hi, lo;
  split_f16(w, SCALE_B, hi, lo);
  if (flags && !(fabsf(w) * SCALE_B < 65504.f)) atomicOr(flags, IC3_ERR_FP16_RANGE);   // also catches NaN
  img[rt_w_off(n, k, 0)] = hi;
  img[rt_w_off(n, k, 1)] = lo;
}

struct RnnTcArgs {
  ic3_policy_cfg cfg;
  ic3_policy_io io;
  const __half* w_img;
  const float* f_b;
  const float* c_b;      // bias of the (zero) comm projection: x + C(0) = x + c_b, as the SIMT kernel adds it
  const float* head_w;
  const float* head_b;
  const int32_t* wflags;
  int ntiles;
};

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__global__ void __launch_bounds__(RT_THREADS, 2) rnn_tc_kernel(RnnTcArgs a) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __half* s_a = reinterpret_cast<__half*>(smem + 2 * RT_W_PART);
  float* s_hp = reinterpret_cast<float*>(smem + 2 * RT_W_PART);
  float* s_fb = reinterpret_cast<float*>(smem + 2 * RT_W_PART + RT_AH_BYTES);
  float* s_cb = s_fb + RT_H;
  const ic3_policy_cfg& cfg = a.cfg;
  const ic3_policy_io& io = a.io;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int N = cfg.N;
  const long R = (long)cfg.B * N;
  if (blockIdx.x == 0 && tid == 0 && a.wflags && io.err && *a.wflags) atomicOr(io.err, *a.wflags);
  for (int i = tid; i < 2 * RT_W_PART / 16; i += RT_THREADS)
    reinterpret_cast<uint4*>(smem)[i] = __ldg(reinterpret_cast<const uint4*>(a.w_img) + i);
  s_fb[tid] = __ldg(a.f_b + tid);
  s_cb[tid] = __ldg(a.c_b + tid);
  const uint32_t smem_base = smem_u32(smem);
  // K-major, no swizzle: LBO = distance of K-adjacent core matrices, SBO = distance of 8-row groups (tc_common.cuh)
  const uint64_t dA = make_desc(smem_base + 2 * RT_W_PART, (RT_M / 8) * 128, 128);
  const uint64_t dB = make_desc(smem_base, (RT_H / 8) * 128, 128);
  const int fr = lane >> 2, fc = 2 * (lane & 3);       // accumulator fragment: rows 16 warp + fr + 8 i, columns 8 j + fc + {0, 1}

  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const long row0 = (long)tile * RT_M;
    // ---- A: x of this thread's fragment; h -> operand image --------------------------------------
    float2 xv[32];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const long row = row0 + 16 * warp + fr + 8 * i;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        xv[16 * i + j] = row < R ? __ldg(reinterpret_cast<const float2*>(io.x + row * RT_H + 8 * j + fc)) : make_float2(0.f, 0.f);
    }
    // warp item = 8 rows x 4 float4 columns: every store instruction writes two whole 128-byte core matrices
#pragma unroll 4
    for (int item = warp; item < (RT_M / 8) * 8; item += RT_THREADS / 32) {
      const int rg = item & 7, qg = item >> 3;
      const int r8 = lane & 7, q = qg * 4 + (lane >> 3);
      const long row = row0 + rg * 8 + r8;
      float4 hv = make_float4(0.f, 0.f, 0.f, 0.f);
      // an episode start enters with h = 0 whatever io.h holds (trainer.py:50-51); h may alias h_out: plain loads
      if (row < R && !(io.fresh && io.fresh[row / N])) hv = *(reinterpret_cast<const float4*>(io.h + row * RT_H) + q);
      const float m = fmaxf(fmaxf(fabsf(hv.x), fabsf(hv.y)), fmaxf(fabsf(hv.z), fabsf(hv.w)));
      if (!(m * SCALE_A < 65504.f) && io.err) atomicOr(io.err, IC3_ERR_FP16_RANGE);
      const size_t off = (size_t)((q >> 1) * (RT_M / 8) + rg) * 64 + r8 * 8 + (q & 1) * 4;
      store_split4(s_a, off, off + RT_A_PART / 2, hv, SCALE_A);
    }
    fence_proxy_async();          // the image (and, first tile, the weights) was written through the generic proxy
    __syncthreads();

    // ---- B: acc = (16 h) . (256 W2)^T ------------------------------------------------------------
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    wgmma_fence_regs(d);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < RT_H / 16; ++ks) {
      const uint64_t da_hi = dA + ((ks * 2 * (RT_M / 8) * 128) >> 4), da_lo = da_hi + (RT_A_PART >> 4);
      const uint64_t db_hi = dB + ((ks * 2 * (RT_H / 8) * 128) >> 4), db_lo = db_hi + (RT_W_PART >> 4);
      wgmma_m64n128_kk(d, da_hi, db_hi, ks != 0);
      wgmma_m64n128_kk(d, da_lo, db_hi, 1);
      wgmma_m64n128_kk(d, da_hi, db_lo, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    __syncthreads();              // every warp's MMAs have read the h image: h' may overwrite it

    // ---- C: h' = tanh(x + h W2^T + b2) -----------------------------------------------------------
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
        if (row < R) *reinterpret_cast<float2*>(io.h_out + row * RT_H + col) = hn;
        *reinterpret_cast<float2*>(s_hp + rl * RT_HP_LD + col) = hn;
      }
    }
    __syncthreads();

    // ---- D: heads, log-softmax, sampling (comm.py:228-239, action_utils.py:32-36) ----------------
    const int nrows = (int)(R - row0 < RT_M ? R - row0 : RT_M);
    for (int rl = warp; rl < nrows; rl += RT_THREADS / 32) {
      float hv[RT_H / 32];
#pragma unroll
      for (int m = 0; m < RT_H / 32; ++m) hv[m] = s_hp[rl * RT_HP_LD + lane + 32 * m];
      const long row = row0 + rl;
      const int e = (int)(row / N), i = (int)(row - (long)e * N);
      heads_for_row<RT_H>(cfg, a.head_w, a.head_b, hv, (size_t)row, e, i, lane, io.tick, io.draws, io.value, io.logp,
                          io.action);
    }
    __syncthreads();              // the heads have read h' before the next tile's h image replaces it
  }
}

}  // namespace

bool ic3_rnn_tc_capable(const ic3_policy_cfg* cfg) {
  return cfg->cell == IC3_CELL_TANH && cfg->passes <= 1 && cfg->comm_mask_zero && !cfg->hard_attn && !cfg->x_tanh &&
         !cfg->h_from_x && cfg->H == RT_H;
}

int ic3_rnn_tc_pack(const ic3_policy_cfg* cfg, const ic3_policy_params* p, const ic3_policy_packed* out, cudaStream_t s) {
  if (!ic3_rnn_tc_capable(cfg)) return IC3_E_UNSUPPORTED;
  if (out->flags) {
    cudaError_t e = cudaMemsetAsync(out->flags, 0, sizeof(int32_t), s);
    if (e != cudaSuccess) return (int)e;
  }
  rnn_tc_pack_kernel<<<RT_H * RT_H / 256, 256, 0, s>>>(p->f_w_pass[0], reinterpret_cast<__half*>(out->rnn_img), out->flags);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

int ic3_rnn_tc_policy_step(const ic3_policy_cfg* cfg, const ic3_policy_packed* w, const ic3_policy_io* io, cudaStream_t s) {
  if (!ic3_rnn_tc_capable(cfg)) return IC3_E_UNSUPPORTED;
  if (!io->x || !w->rnn_img || !w->f_b) return IC3_E_NULL;
  static int max_ctas = 0;
  if (max_ctas == 0) {
    cudaError_t e = cudaFuncSetAttribute(rnn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RT_SMEM_BYTES);
    int per_sm = 0, dev = 0, nsm = 0;
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rnn_tc_kernel, RT_THREADS, RT_SMEM_BYTES);
    if (e == cudaSuccess) e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess || per_sm <= 0) return e != cudaSuccess ? (int)e : IC3_E_RANGE;
    max_ctas = per_sm * nsm;                                        // persistent grid: every CTA resident
  }
  const long R = (long)cfg->B * cfg->N;
  RnnTcArgs a{*cfg, *io, reinterpret_cast<const __half*>(w->rnn_img), w->f_b, w->c_b, w->head_w, w->head_b, w->flags,
              (int)((R + RT_M - 1) / RT_M)};
  ic3_prof_mark(0, s);
  ic3_prof_mark(1, s);
  rnn_tc_kernel<<<a.ntiles < max_ctas ? a.ntiles : max_ctas, RT_THREADS, RT_SMEM_BYTES, s>>>(a);
  IC3_LAUNCH_CHECK();
  ic3_prof_mark(2, s);
  ic3_prof_mark(3, s);
  return IC3_OK;
}
