// Internal (non-ABI) entry points of the tensor-core policy path, called from policy.cu, and the policy argument
// checks shared with the fused observation + encoder entry points (pp_env.cu, tj_env.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/ic3net_b200.h"

uint64_t ic3_tc_workspace_bytes(const ic3_policy_cfg* cfg);
int ic3_tc_pack(const ic3_policy_cfg* cfg, const ic3_policy_params* p, const ic3_policy_packed* out, cudaStream_t s);
int ic3_tc_policy_step(const ic3_policy_cfg* cfg, const ic3_policy_packed* w, const ic3_policy_io* io, cudaStream_t s);
int ic3_tc_pass_states(const ic3_policy_cfg* cfg, const ic3_policy_packed* w, const ic3_policy_io* io, int npasses,
                       float* h_pass, float* c_pass, cudaStream_t s);
// tensor-core step of the non-recurrent tanh policies and of the one-pass tanh RNN without communication (ff_tc.cu):
// the configurations it covers, its scratch, its weight image (ic3_policy_packed.ff_img), the step and its pass-state
// form (non-recurrent only)
bool ic3_ff_tc_capable(const ic3_policy_cfg* cfg);
uint64_t ic3_ff_tc_workspace_bytes(const ic3_policy_cfg* cfg);
int ic3_ff_tc_pack(const ic3_policy_cfg* cfg, const ic3_policy_params* p, const ic3_policy_packed* out, cudaStream_t s);
int ic3_ff_tc_policy_step(const ic3_policy_cfg* cfg, const ic3_policy_packed* w, const ic3_policy_io* io, cudaStream_t s);
int ic3_ff_tc_states(const ic3_policy_cfg* cfg, const ic3_policy_packed* w, const ic3_policy_io* io, float* st_h,
                     float* st_s, cudaStream_t s);
// timing hook of ic3_policy_step_profile: records event i (0 .. 3) on s while a profiled step runs, else nothing
void ic3_prof_mark(int i, cudaStream_t s);
// grid of a persistent kernel `kern` (threads per CTA, dynamic shared memory smem) over nwork items that runs beside the
// tensor-core LSTM kernel: min(nwork, SMs x the CTAs of kern that fit on one SM next to a resident lstm_tc_kernel CTA --
// registers, shared memory, threads, CTA slots -- at least one per SM)
int ic3_grid_beside_lstm(const void* kern, int threads, size_t smem, int nwork, int* grid);
// grid of a persistent kernel `kern` (threads per CTA, dynamic shared memory smem, which it allows kern to use) over
// nwork items with every CTA resident: min(nwork, SMs x the CTAs of kern that fit on one SM)
int ic3_persistent_grid(const void* kern, int threads, size_t smem, int nwork, int* grid);
// return CALL with the compile-time hid_size HH = Hval (32 | 64 | 128)
#define IC3_DISPATCH_H(Hval, CALL)          \
  switch (Hval) {                           \
    case 32: { constexpr int HH = 32; return CALL; }   \
    case 64: { constexpr int HH = 64; return CALL; }   \
    case 128: { constexpr int HH = 128; return CALL; } \
    default: return IC3_E_UNSUPPORTED;      \
  }

// policy configuration and packed weights as every encoder entry point checks them
int ic3_encoder_check(const ic3_policy_cfg* cfg, const ic3_policy_packed* w);
// layout hint of ic3_policy_cfg vs the environment (IC3_OK when no hint is given)
int ic3_pp_layout_check(const ic3_pp_cfg* env, const ic3_policy_cfg* cfg);
int ic3_tj_layout_check(const ic3_tj_cfg* env, const ic3_policy_cfg* cfg);
