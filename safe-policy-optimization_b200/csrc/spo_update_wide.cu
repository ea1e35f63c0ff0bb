// The AC = 16 instantiations of the minibatch update kernel (act_dim 9..16, single GPU): spo_pg_update reaches them through
// spo_update_launch_wide.  See spo_update_kernel.cuh for why they have a file of their own.  The clock64 phase timers
// (SPO_PHASE_TIMERS) cover the AC = 8 kernels only.
#undef SPO_PHASE_TIMERS
#include "spo_update_kernel.cuh"

int spo_update_launch_wide(int nt1, const void* args, cudaStream_t stream, bool pack_only) {
  const UpdArgs& a = *static_cast<const UpdArgs*>(args);
  if (pack_only) return nt1 == 1 ? launch_pack<1, 16>(a, stream) : launch_pack<2, 16>(a, stream);
  return nt1 == 1 ? launch_update<1, 16, false>(a, stream) : launch_update<2, 16, false>(a, stream);
}
