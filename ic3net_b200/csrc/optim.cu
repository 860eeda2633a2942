// RMSprop update of the reference trainer over ONE flat fp32 buffer (all live parameters of the policy):
// torch.optim.RMSprop(lr, alpha=0.97, eps=1e-6), no momentum, not centered, no weight decay (reference
// trainer.py:21-22), preceded by the division of the summed gradient by the global number of env steps
// (trainer.py:251-253, multi_processing.py:95):
//   g  = grad / grad_div          (written back: p.grad holds the divided gradient afterwards, like the reference)
//   v  = alpha * v + (1 - alpha) * g * g
//   p -= lr * g / (sqrt(v) + eps)
// One pass, 12 bytes read + 12 bytes written per element (HBM-bound; 0.6 M elements at the BASELINE configs, i.e.
// launch-latency sized -- the point is that the update needs no per-tensor kernels and no gradient copies).
#include "ic3_common.cuh"

namespace {

// The update of elements i (float4 groups) and the < 4-element tail, shared by both entry points.
__device__ __forceinline__ void rmsprop_apply(long n, float lr, float alpha, float eps, float inv_div,
                                              float* __restrict__ grad, float* __restrict__ param, float* __restrict__ sq) {
  const long stride = (long)gridDim.x * blockDim.x;
  const long n4 = n >> 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 g4 = reinterpret_cast<const float4*>(grad)[i];
    float4 v = reinterpret_cast<float4*>(sq)[i];
    float4 p = reinterpret_cast<float4*>(param)[i];
    const float g[4] = {g4.x * inv_div, g4.y * inv_div, g4.z * inv_div, g4.w * inv_div};
    float* vv = &v.x;
    float* pp = &p.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      vv[k] = alpha * vv[k] + (1.f - alpha) * g[k] * g[k];
      pp[k] -= lr * g[k] / (sqrtf(vv[k]) + eps);
    }
    reinterpret_cast<float4*>(grad)[i] = make_float4(g[0], g[1], g[2], g[3]);
    reinterpret_cast<float4*>(sq)[i] = v;
    reinterpret_cast<float4*>(param)[i] = p;
  }
  for (long i = (n4 << 2) + (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {   // tail (< 4 elements)
    const float g = grad[i] * inv_div;
    const float v = alpha * sq[i] + (1.f - alpha) * g * g;
    grad[i] = g;
    sq[i] = v;
    param[i] -= lr * g / (sqrtf(v) + eps);
  }
}

__global__ void rmsprop_kernel(long n, float lr, float alpha, float eps, float inv_div, float* __restrict__ grad,
                               float* __restrict__ param, float* __restrict__ sq) {
  rmsprop_apply(n, lr, alpha, eps, inv_div, grad, param, sq);
}

// ic3_rmsprop_step_dev: the divisor is the step count of the statistics vector (stat[1]), read on the device.  A rollout
// that raised a device error flag (stat[3] != 0) updates nothing: the host raises on those flags, as before the update
// in the eager path.  A count that is not a positive finite number updates nothing and raises IC3_ERR_GRAD_DIV in err
// (the host form refuses it with IC3_E_RANGE; inside a CUDA graph nobody is there to see a return code).
__global__ void rmsprop_dev_kernel(long n, float lr, float alpha, float eps, const double* __restrict__ stat,
                                   float* __restrict__ grad, float* __restrict__ param, float* __restrict__ sq,
                                   int32_t* __restrict__ err) {
  if (stat[3] != 0.0) return;
  const float div = (float)stat[1];
  if (!(div > 0.f) || !isfinite(div)) {
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(err, IC3_ERR_GRAD_DIV);
    return;
  }
  rmsprop_apply(n, lr, alpha, eps, 1.f / div, grad, param, sq);
}

static int rmsprop_grid(int64_t n) {
  const int threads = 256;
  long blocks = ((n >> 2) + threads - 1) / threads;
  if (blocks < 1) blocks = 1;
  if (blocks > 132 * 8) blocks = 132 * 8;
  return (int)blocks;
}

}  // namespace

extern "C" int ic3_rmsprop_step(int64_t n, float lr, float alpha, float eps, float grad_div, float* grad, float* param,
                                float* square_avg, void* stream) {
  if (!grad || !param || !square_avg) return IC3_E_NULL;
  if (n <= 0 || !(grad_div > 0.f) || !(eps > 0.f)) return IC3_E_RANGE;
  if (((uintptr_t)grad | (uintptr_t)param | (uintptr_t)square_avg) & 15) return IC3_E_RANGE;   // float4 path
  rmsprop_kernel<<<rmsprop_grid(n), 256, 0, (cudaStream_t)stream>>>((long)n, lr, alpha, eps, 1.f / grad_div, grad, param,
                                                                   square_avg);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}

extern "C" int ic3_rmsprop_step_dev(int64_t n, float lr, float alpha, float eps, const double* stat, float* grad,
                                    float* param, float* square_avg, int32_t* err, void* stream) {
  if (!stat || !grad || !param || !square_avg || !err) return IC3_E_NULL;
  if (n <= 0 || !(eps > 0.f)) return IC3_E_RANGE;
  if (((uintptr_t)grad | (uintptr_t)param | (uintptr_t)square_avg) & 15) return IC3_E_RANGE;   // float4 path
  rmsprop_dev_kernel<<<rmsprop_grid(n), 256, 0, (cudaStream_t)stream>>>((long)n, lr, alpha, eps, stat, grad, param,
                                                                       square_avg, err);
  IC3_LAUNCH_CHECK();
  return IC3_OK;
}
