// The AC = 16 instantiation of the FFMA forward kernel: every forward call at act_dim 9..16 (the rollout step, the critic
// values, the actor means and KL passes) runs it.  See spo_ffma_forward.cuh for why it has a file of its own.
#include "spo_ffma_forward.cuh"

int spo_ffma_forward_launch_wide(const SpoFwdArgs& a, cudaStream_t stream) { return ffma_forward_launch<16>(a, stream); }
