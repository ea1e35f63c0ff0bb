// Trust-region pieces of CPO / TRPO-Lag on the device.
//
// Reference: safepo/single_agent/cpo.py:70-157 (flat params, conjugate_gradients, fvp),
// :353-519 (losses, line search); trpo_lag.py:363-442.
//
//   spo_surrogate_grad   L = mean_i ratio_i * adv_i  and  dL/dtheta over the full batch
//   spo_fvp              (H + damping I) v,  H = Hessian of mean_{S*A} KL(old || new) at new = old.
//                        For a Gaussian with state-independent log_std this is
//                          [ 2 v_ls / A ;  J^T diag(sigma^-2) J v_mean / (S A) ]
//                        (SURVEY fact 7): one JVP and one VJP through the mean MLP, no
//                        autograd graph -- 8 tile GEMMs per 64 rows instead of ~12.
//   spo_linesearch_eval  mean(ratio*adv_a), mean(ratio*adv_b), mean_{S*A} KL(old||new)
//   spo_conjugate_gradient  cpo.py:81-106 with every dot / axpy / the residual test on device
//
// All three full-batch kernels share one persistent tile loop: one CTA per SM walk
// the [S,D] observations in 64-row tiles with the actor (and, for the FVP, the tangent
// vector reshaped as a second set of weights) resident in shared memory; parameter-shaped
// results are accumulated in registers across tiles and flushed once per CTA with atomics.
#include "spo_trust_kernel.cuh"

namespace {

// act_dim <= 8 runs the AC = 8 instantiations, 9..16 the AC = 16 ones
template <int MODE>
int launch_trust(const TrArgs& a, cudaStream_t st) {
  return a.A <= 8 ? launch_trust_ac<MODE, 8>(a, st) : spo_trust_launch_wide(MODE, &a, st);
}

// ---- conjugate gradient vector kernel (single CTA; P_a ~ 1e4) ---------------------------
// state: x (out), r, p, z in work[0..3P), scalars at work + 4P: [0] rdotr [1] done
__device__ float block_dot(const float* a, const float* b, int n, float* red) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s = fmaf(a[i], b[i], s);
  s = spo_warp_sum(s);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
  return t;
}

__global__ void __launch_bounds__(1024) spo_cg_init_kernel(const float* b, float* x, float* r, float* p, float* sc, int n) {
  __shared__ float red[32];
  for (int i = threadIdx.x; i < n; i += blockDim.x) { x[i] = 0.f; r[i] = b[i]; p[i] = b[i]; }   // fvp(0) == 0 exactly (cpo.py:91)
  __syncthreads();
  const float rr = block_dot(r, r, n, red);
  if (threadIdx.x == 0) { sc[0] = rr; sc[1] = 0.f; }
}

__global__ void __launch_bounds__(1024) spo_cg_step_kernel(float* x, float* r, float* p, const float* z, float* sc, int n,
                                                           float tol, float eps) {
  __shared__ float red[32];
  if (sc[1] != 0.f) return;   // residual test tripped earlier (cpo.py:101)
  const float rdotr = sc[0];
  const float pz = block_dot(p, z, n, red);
  const float alpha = rdotr / (pz + eps);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    x[i] = fmaf(alpha, p[i], x[i]);
    r[i] = fmaf(-alpha, z[i], r[i]);
  }
  __syncthreads();
  const float nrr = block_dot(r, r, n, red);
  if (sqrtf(nrr) < tol) {
    if (threadIdx.x == 0) sc[1] = 1.f;
    return;
  }
  const float mu = nrr / (rdotr + eps);
  for (int i = threadIdx.x; i < n; i += blockDim.x) p[i] = fmaf(mu, p[i], r[i]);
  if (threadIdx.x == 0) sc[0] = nrr;
}

int check_trust_args(const spo_dims* d, const float* params, const float* obs, int64_t count, const char* who) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(params && obs && count > 0, SPO_ERR_INVALID_ARG, "%s: null params/obs or count<=0", who);
  SPO_REQUIRE(spo_obs_aligned(obs, d->obs_dim), SPO_ERR_INVALID_ARG,
              "%s: obs must be 16-byte aligned when obs_dim %% 4 == 0 (obs_dim=%d)", who, d->obs_dim);
  return SPO_OK;
}

}  // namespace

extern "C" {

int spo_surrogate_grad(const spo_dims* d, const float* params, const float* obs, const float* act,
                       const float* logp_old, const float* adv, int64_t count,
                       float* out_loss, float* grad, void* stream) {
  int rc = check_trust_args(d, params, obs, count, "spo_surrogate_grad");
  if (rc) return rc;
  SPO_REQUIRE(act && logp_old && adv && out_loss && grad, SPO_ERR_INVALID_ARG, "spo_surrogate_grad: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const SpoNetOff off = spo_net_off(d->obs_dim, d->act_dim, 0);
  SPO_CUDA_TRY(cudaMemsetAsync(grad, 0, sizeof(float) * off.count, st));
  SPO_CUDA_TRY(cudaMemsetAsync(out_loss, 0, sizeof(float), st));
  TrArgs a{};
  a.params = params; a.obs = obs; a.act = act; a.logp_old = logp_old; a.adv_a = adv; a.out = grad; a.out_loss = out_loss;
  a.count = count; a.D = d->obs_dim; a.A = d->act_dim;
  return launch_trust<MODE_GRAD>(a, st);
}

int spo_fvp(const spo_dims* d, const float* params, const float* obs, int64_t count,
            const float* v, float damping, float* out, void* stream) {
  int rc = check_trust_args(d, params, obs, count, "spo_fvp");
  if (rc) return rc;
  SPO_REQUIRE(v && out && v != out, SPO_ERR_INVALID_ARG, "spo_fvp: null or aliased v/out");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const SpoNetOff off = spo_net_off(d->obs_dim, d->act_dim, 0);
  SPO_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * off.count, st));
  TrArgs a{};
  a.params = params; a.obs = obs; a.v = v; a.out = out; a.count = count; a.D = d->obs_dim; a.A = d->act_dim;
  rc = launch_trust<MODE_FVP>(a, st);
  if (rc) return rc;
  spo_fvp_finalize_kernel<<<(off.count + 255) / 256, 256, 0, st>>>(out, v, off.count, d->act_dim, damping);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_linesearch_eval(const spo_dims* d, const float* params, const float* obs, const float* act,
                        const float* logp_old, const float* adv_a, const float* adv_b,
                        const float* old_mean, const float* old_log_std, int64_t count,
                        float* out3, void* stream) {
  int rc = check_trust_args(d, params, obs, count, "spo_linesearch_eval");
  if (rc) return rc;
  SPO_REQUIRE(act && logp_old && adv_a && old_mean && old_log_std && out3, SPO_ERR_INVALID_ARG, "spo_linesearch_eval: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SPO_CUDA_TRY(cudaMemsetAsync(out3, 0, 3 * sizeof(float), st));
  TrArgs a{};
  a.params = params; a.obs = obs; a.act = act; a.logp_old = logp_old; a.adv_a = adv_a; a.adv_b = adv_b;
  a.old_mean = old_mean; a.old_log_std = old_log_std; a.out = out3; a.count = count; a.D = d->obs_dim; a.A = d->act_dim;
  return launch_trust<MODE_EVAL>(a, st);
}

// Data-parallel ranks cannot use the monolithic solver below: every Fisher-vector product has to be averaged across the
// ranks before the step that consumes it (SURVEY section 8e, exchange 3').  The same two vector kernels, one call each:
//   spo_cg_begin   x = 0, r = p = b, rdotr = r.r                (work: r | p | z | - | scalars, like spo_conjugate_gradient)
//   (host)         spo_fvp(p = work + P  ->  z = work + 2P), all-reduce z, ...
//   spo_cg_update  one iteration of cpo.py:92-105 with the z it finds in work + 2P
int spo_cg_begin(const spo_dims* d, const float* b, float* x, float* work, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(b && x && work, SPO_ERR_INVALID_ARG, "spo_cg_begin: null argument");
  const int P = spo_net_off(d->obs_dim, d->act_dim, 0).count;
  spo_cg_init_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(b, x, work, work + P, work + 4 * P, P);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_cg_update(const spo_dims* d, float* x, float* work, float residual_tol, float eps, void* stream) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(x && work, SPO_ERR_INVALID_ARG, "spo_cg_update: null argument");
  const int P = spo_net_off(d->obs_dim, d->act_dim, 0).count;
  spo_cg_step_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(x, work, work + P, work + 2 * P, work + 4 * P, P, residual_tol, eps);
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_conjugate_gradient(const spo_dims* d, const float* params, const float* obs, int64_t count,
                           const float* b, int iters, float damping, float residual_tol, float eps,
                           float* x, float* work, void* stream) {
  int rc = check_trust_args(d, params, obs, count, "spo_conjugate_gradient");
  if (rc) return rc;
  SPO_REQUIRE(b && x && work && iters >= 0, SPO_ERR_INVALID_ARG, "spo_conjugate_gradient: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int P = spo_net_off(d->obs_dim, d->act_dim, 0).count;
  float *r = work, *p = work + P, *z = work + 2 * P, *sc = work + 4 * P;
  spo_cg_init_kernel<<<1, 1024, 0, st>>>(b, x, r, p, sc, P);
  SPO_CUDA_TRY(cudaGetLastError());
  for (int it = 0; it < iters; ++it) {
    rc = spo_fvp(d, params, obs, count, p, damping, z, stream);
    if (rc) return rc;
    spo_cg_step_kernel<<<1, 1024, 0, st>>>(x, r, p, z, sc, P, residual_tol, eps);
    SPO_CUDA_TRY(cudaGetLastError());
  }
  return SPO_OK;
}

}  // extern "C"
