// Internal (non-ABI) interface of the tensor-core backward of the non-recurrent tanh policies (ff_grad_tc.cu), called
// from ic3_ff_grad_* (bptt_tc.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/ic3net_b200.h"

// workspace bytes of the pass weight images and the operand-scale words
uint64_t ic3_ff_grad_tc_bytes(int passes, int comm);

// Everything one chunk's backward reads and writes after the forward re-run and the heads (bptt_heads_kernel).  Blocks of
// [R, H] floats are the chunk's own rows, packed at the front of the workspace buffers.
struct FfGradTcChunk {
  int R, N, Bk, P, comm, hard_attn, comm_avg, nout;
  int npos, ne, npad, is_tj;
  const float* hs;             // [P + 1][R][H]: tanh(x), h_1 .. h_P
  const float* ss;             // [P][R][H]: S_0 .. S_{P-1}, or NULL without communication
  const float* dout;           // [R, 8] d loss / d (value, logits)
  const float* head_w;         // packed [1 + atot, H]
  const uint8_t* fresh; const uint8_t* comm_action; const uint8_t* alive; const uint8_t* valid;
  float* g; float* dx; float* dz;            // [R, H] scratch
  const int32_t* pos; const float* ext;      // observation pattern (ff_desc_kernel)
  float* fpart; float* cpart; float* bpart; float* ypart;   // the fixed row-block partials of ic3_ff_grad_finish
  int nb;                      // row blocks of those partials
  void* tc;                   // ic3_ff_grad_tc_bytes(P, comm) bytes: weight images + scale words
};

// once per ic3_ff_grad_begin: the dgrad weight images [F_p^T | C_p^T] of every pass from the SIMT-packed f_wT / c_wT
int ic3_ff_grad_tc_pack(int passes, int comm, const float* f_wT, const float* c_wT, void* tc, cudaStream_t s);
// one chunk: passes P-1 .. 0 (dgrad, weight gradient), then the encoder gradient
int ic3_ff_grad_tc_chunk(const FfGradTcChunk* c, cudaStream_t s);
