// The networks of the fp32 PPO minibatch (stx_mlp.cu), as the loss entries (stx_ppo_fp32.cu) use them: one network's forward /
// backward on a minibatch with the workspace carved as stx_ppo_workspace_bytes() sizes it.
#pragma once
#include "stx_common.cuh"

namespace stx {

struct SimtHeadBufs {
  float* head;            // (mb, head width) network output
  float* dhead;           // d(loss)/d(head), read by simt_net_backward
  double* loss_partials;  // [(mb + 255) / 256][6] per-block metric partials of a 256-thread loss kernel
  unsigned int* counter;  // last-block ticket, zero between calls
};

int simt_check_mlp(const StxMlp* m, const char* who);  // STX_OK or the STX_E_* of a malformed StxMlp (message set)
int simt_net_forward(const StxMlp* m, const float* x, int64_t ldx, const int32_t* idx, int64_t mb, void* workspace, SimtHeadBufs* out,
                     cudaStream_t st);
int simt_net_backward(const StxMlp* m, const float* x, int64_t ldx, const int32_t* idx, int64_t mb, void* workspace, float grad_weight,
                      float* net_grad, int overwrite, cudaStream_t st);

}  // namespace stx
