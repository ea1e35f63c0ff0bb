// Entry points of the minibatch update (spo_pg_update, spo_pg_update_dp) and the AC = 8 instantiations of its kernel; the
// kernel and its design notes are in spo_update_kernel.cuh.
#include <mutex>
#include "spo_update_kernel.cuh"

int spo_update_tile_pool(cudaMemPool_t* pool) {
  static std::mutex mu;
  static cudaMemPool_t pools[64] = {};
  int dev = 0;
  SPO_CUDA_TRY(cudaGetDevice(&dev));
  SPO_REQUIRE(dev >= 0 && dev < 64, SPO_ERR_UNSUPPORTED, "spo_pg_update: device %d", dev);
  std::lock_guard<std::mutex> lock(mu);
  if (!pools[dev]) {
    cudaMemPoolProps props{};
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    cudaMemPool_t p;
    SPO_CUDA_TRY(cudaMemPoolCreate(&p, &props));
    uint64_t keep = UINT64_MAX;   // never hand the blocks back to the driver between passes
    SPO_CUDA_TRY(cudaMemPoolSetAttribute(p, cudaMemPoolAttrReleaseThreshold, &keep));
    pools[dev] = p;
  }
  *pool = pools[dev];
  return SPO_OK;
}

#ifdef SPO_PHASE_TIMERS
extern "C" int spo_debug_phase_cycles(unsigned long long* out_16x24, int reset) {
  SPO_CUDA_TRY(cudaMemcpyFromSymbol(out_16x24, g_phase_cycles, sizeof(unsigned long long) * 16 * 24));
  if (reset) {
    unsigned long long z[16 * 24] = {0};
    SPO_CUDA_TRY(cudaMemcpyToSymbol(g_phase_cycles, z, sizeof(z)));
  }
  return SPO_OK;
}
#endif

extern "C" int spo_comm_slot_floats(const spo_dims* d, int* slot_floats) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(slot_floats, SPO_ERR_INVALID_ARG, "spo_comm_slot_floats: null output");
  // per net: four CTA slots of 8-byte {value, sequence} words
  const int nt1 = d->obs_dim <= 64 ? 1 : 2;
  *slot_floats = NQ * dp_slot_words(nt1) * 2;
  return SPO_OK;
}

extern "C" int spo_pg_update(const spo_dims* d, float* params, float* adam_m, float* adam_v, int* adam_t,
                             const spo_batch* data, const int64_t* perm, int64_t perm_len, int batch,
                             spo_loss_kind kind, const spo_hparams* hp, spo_update_ctrl* ctrl, void* stream) {
  return spo_pg_update_dp(d, params, adam_m, adam_v, adam_t, data, perm, perm_len, batch, kind, hp, ctrl, nullptr, stream);
}

extern "C" int spo_pg_update_dp(const spo_dims* d, float* params, float* adam_m, float* adam_v, int* adam_t,
                                const spo_batch* data, const int64_t* perm, int64_t perm_len, int batch,
                                spo_loss_kind kind, const spo_hparams* hp, spo_update_ctrl* ctrl,
                                const spo_comm* comm, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && adam_m && adam_v && adam_t && data && perm && hp && ctrl, SPO_ERR_INVALID_ARG, "spo_pg_update: null argument");
  SPO_REQUIRE(batch > 0 && perm_len > 0 && perm_len <= data->count && data->count <= 0x7fffffffLL, SPO_ERR_INVALID_ARG,
              "spo_pg_update: batch=%d perm_len=%lld count=%lld (count must be < 2^31)", batch, (long long)perm_len, (long long)data->count);
  SPO_REQUIRE(kind >= SPO_LOSS_PPO_CLIP && kind <= SPO_LOSS_CUP_PROJECTION, SPO_ERR_INVALID_ARG, "spo_pg_update: kind=%d", (int)kind);
  SPO_REQUIRE(data->obs && data->target_r && data->target_c, SPO_ERR_INVALID_ARG, "spo_pg_update: batch obs/targets null");
  if (kind != SPO_LOSS_CRITIC_ONLY)
    SPO_REQUIRE(data->act && data->logp && data->adv, SPO_ERR_INVALID_ARG, "spo_pg_update: actor loss needs act/logp/adv");
  if (kind == SPO_LOSS_FOCOPS || kind == SPO_LOSS_CUP_PROJECTION) {
    SPO_REQUIRE(data->old_mean && data->old_std, SPO_ERR_INVALID_ARG, "spo_pg_update: FOCOPS needs old_mean/old_std");
    SPO_REQUIRE(batch <= SPO_ROWS, SPO_ERR_UNSUPPORTED, "spo_pg_update: FOCOPS supports batch <= %d (got %d)", SPO_ROWS, batch);
  }
  UpdArgs a{};
  a.params = params; a.adam_m = adam_m; a.adam_v = adam_v; a.adam_t = adam_t;
  a.data = *data; a.perm = perm; a.perm_len = perm_len; a.batch = batch; a.kind = kind;
  a.D = d->obs_dim; a.A = d->act_dim; a.hp = *hp; a.ctrl = ctrl;
  if (kind == SPO_LOSS_CUP_PROJECTION) {
    // (c * ratio * adv [B] + kl [B,1]).mean() = mean(kl) + c * mean(ratio * adv): the FOCOPS loss
    // (kl - ratio * adv / lam) * 1(kl <= delta) with delta = inf (mask 1) and 1/lam = -c
    a.kind = SPO_LOSS_FOCOPS;
    a.actor_only = 1;
    a.hp.focops_kl = INFINITY;
    a.hp.focops_lam = -1.f / hp->focops_lam;   // c = 0 -> -inf -> 1/lam = -0
  }
  if (kind == SPO_LOSS_PG) {
    // the unclipped surrogate is the clipped one with an unbounded clip range: clamp(ratio) == ratio, the
    // min() keeps the first branch, value and gradient are those of pg.py:309 bit for bit
    a.kind = SPO_LOSS_PPO_CLIP;
    a.hp.clip_lo = -INFINITY;
    a.hp.clip_hi = INFINITY;
  }
  if (comm && comm->world > 1) {
    SPO_REQUIRE(comm->rank >= 0 && comm->rank < comm->world && comm->world <= 16 && comm->grad_bufs,
                SPO_ERR_INVALID_ARG, "spo_pg_update_dp: bad spo_comm (world=%d rank=%d)", comm->world, comm->rank);
    // the gradient slots of the in-kernel exchange carry one small parameter per thread: act_dim <= 8 (176 of them)
    SPO_REQUIRE(d->act_dim <= 8, SPO_ERR_UNSUPPORTED,
                "spo_pg_update_dp: act_dim=%d > 8 is single-GPU only (the cross-GPU update supports act_dim <= 8)", d->act_dim);
    a.comm = *comm;
  } else {
    a.comm.world = 1;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool dp = a.comm.world > 1;
  // action capacity: act_dim <= 8 runs the AC = 8 instantiations, 9..16 the AC = 16 ones (single GPU only)
  if (d->act_dim > 8) return spo_update_launch_wide(d->obs_dim <= 64 ? 1 : 2, &a, st, false);
  if (d->obs_dim <= 64) return dp ? launch_update<1, 8, true>(a, st) : launch_update<1, 8, false>(a, st);
  return dp ? launch_update<2, 8, true>(a, st) : launch_update<2, 8, false>(a, st);
}

// Test hook: the packed tiles of one pass (spo_pack_tiles, as spo_pg_update runs it for these dims / kind) into `out`,
// which holds ceil(perm_len / batch) * ceil(batch / 64) tiles of 64 * (ldx + 3 * AC + 4) floats.
extern "C" int spo_debug_pack_tiles(const spo_dims* d, const spo_batch* data, const int64_t* perm, int64_t perm_len, int batch,
                                    spo_loss_kind kind, spo_update_ctrl* ctrl, float* out, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(data && perm && ctrl && out && batch > 0 && perm_len > 0, SPO_ERR_INVALID_ARG, "spo_debug_pack_tiles: bad argument");
  UpdArgs a{};
  a.tiles = out; a.data = *data; a.perm = perm; a.perm_len = perm_len; a.batch = batch; a.kind = kind;
  a.D = d->obs_dim; a.A = d->act_dim; a.ctrl = ctrl;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nt1 = d->obs_dim <= 64 ? 1 : 2;
  if (d->act_dim > 8) return spo_update_launch_wide(nt1, &a, st, true);
  return nt1 == 1 ? launch_pack<1, 8>(a, st) : launch_pack<2, 8>(a, st);
}
