// The AC = 16 instantiations of the trust-region kernel (act_dim 9..16): spo_surrogate_grad, spo_fvp and
// spo_linesearch_eval reach them through spo_trust_launch_wide.  See spo_trust_kernel.cuh for why they have a file of their own.
#include "spo_trust_kernel.cuh"

int spo_trust_launch_wide(int mode, const void* args, cudaStream_t st) {
  const TrArgs& a = *static_cast<const TrArgs*>(args);
  switch (mode) {
    case MODE_GRAD: return launch_trust_ac<MODE_GRAD, 16>(a, st);
    case MODE_FVP: return launch_trust_ac<MODE_FVP, 16>(a, st);
    default: return launch_trust_ac<MODE_EVAL, 16>(a, st);
  }
}
