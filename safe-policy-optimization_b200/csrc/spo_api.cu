// libspo: version, error reporting, parameter layout queries.
#include <stdarg.h>
#include <string.h>
#include "spo_common.cuh"

static thread_local char g_err[512] = "";

void spo_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int spo_check_dims(const spo_dims* d) {
  SPO_REQUIRE(d != nullptr, SPO_ERR_INVALID_ARG, "spo_dims is NULL");
  SPO_REQUIRE(d->hidden == SPO_HID, SPO_ERR_UNSUPPORTED, "hidden=%d unsupported (only two tanh layers of 64)", d->hidden);
  SPO_REQUIRE(d->obs_dim >= 1 && d->obs_dim <= SPO_MAX_OBS, SPO_ERR_UNSUPPORTED, "obs_dim=%d outside [1,%d]", d->obs_dim, SPO_MAX_OBS);
  SPO_REQUIRE(d->act_dim >= 1 && d->act_dim <= SPO_MAX_ACT_WIDE, SPO_ERR_UNSUPPORTED, "act_dim=%d outside [1,%d]", d->act_dim, SPO_MAX_ACT_WIDE);
  return SPO_OK;
}

int spo_sm_count() {
  static int n = 0;   // per process: one process drives one GPU
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      (void)cudaGetLastError();
      n = 132;   // H100 SXM
    }
  }
  return n;
}

extern "C" {

int spo_version(void) { return SPO_VERSION; }

const char* spo_last_error(void) { return g_err; }

int spo_sync_check(void* stream) {
  SPO_CUDA_TRY(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  SPO_CUDA_TRY(cudaGetLastError());
  return SPO_OK;
}

int spo_param_count(const spo_dims* d, int* actor, int* critic, int* total) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SpoNetOff a = spo_net_off(d->obs_dim, d->act_dim, 0), c = spo_net_off(d->obs_dim, d->act_dim, 1);
  if (actor) *actor = a.count;
  if (critic) *critic = c.count;
  if (total) *total = a.count + 2 * c.count;
  return SPO_OK;
}

int spo_param_offsets(const spo_dims* d, int net, int* log_std, int* w1, int* b1, int* w2, int* b2, int* w3, int* b3) {
  int rc = spo_check_dims(d);
  if (rc) return rc;
  SPO_REQUIRE(net >= 0 && net <= 2, SPO_ERR_INVALID_ARG, "net=%d outside [0,2]", net);
  SpoNetOff o = spo_net_off(d->obs_dim, d->act_dim, net);
  if (log_std) *log_std = o.log_std;
  if (w1) *w1 = o.w1;
  if (b1) *b1 = o.b1;
  if (w2) *w2 = o.w2;
  if (b2) *b2 = o.b2;
  if (w3) *w3 = o.w3;
  if (b3) *b3 = o.b3;
  return SPO_OK;
}

int spo_comm_alloc(size_t bytes, void** ptr) {
  SPO_REQUIRE(ptr && bytes > 0, SPO_ERR_INVALID_ARG, "spo_comm_alloc: null output or zero size");
  SPO_CUDA_TRY(cudaMalloc(ptr, bytes));
  SPO_CUDA_TRY(cudaMemset(*ptr, 0, bytes));
  SPO_CUDA_TRY(cudaDeviceSynchronize());
  return SPO_OK;
}

int spo_comm_free(void* ptr) {
  SPO_CUDA_TRY(cudaFree(ptr));
  return SPO_OK;
}

int spo_comm_export(void* ptr, unsigned char* handle64) {
  SPO_REQUIRE(ptr && handle64, SPO_ERR_INVALID_ARG, "spo_comm_export: null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle is 64 bytes");
  cudaIpcMemHandle_t h;
  SPO_CUDA_TRY(cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle64, &h, 64);
  return SPO_OK;
}

int spo_comm_import(const unsigned char* handle64, void** ptr) {
  SPO_REQUIRE(ptr && handle64, SPO_ERR_INVALID_ARG, "spo_comm_import: null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  SPO_CUDA_TRY(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return SPO_OK;
}

int spo_comm_close(void* imported_ptr) {
  SPO_CUDA_TRY(cudaIpcCloseMemHandle(imported_ptr));
  return SPO_OK;
}

}  // extern "C"
