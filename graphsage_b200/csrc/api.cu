// Library-wide plumbing: version, thread-local error string, tuning knobs, host helpers.
#include <stdarg.h>

#include <map>
#include <set>
#include <utility>
#include <mutex>
#include <string>

#include "common.cuh"

namespace gs {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int32_t cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return GS_ERR_CUDA;
}

static std::mutex g_mu;
static std::map<std::string, int32_t>& knobs() {
  static std::map<std::string, int32_t> m;
  return m;
}

int32_t tuning(const char* key, int32_t dflt) {
  std::lock_guard<std::mutex> l(g_mu);
  auto it = knobs().find(key);
  return it == knobs().end() ? dflt : it->second;
}

int sm_count() {
  static int n[64] = {0};                        // per device ordinal
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (n[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[dev] = v;
  }
  return n[dev];
}

int32_t ensure_dyn_smem(const void* kernel, int bytes) {
  // the attribute belongs to the kernel in the CURRENT device's context, so remember it per (device, kernel)
  static std::mutex mu;
  static std::set<std::pair<int, const void*>> done;
  int dev = 0;
  GS_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> l(mu);
  if (done.count(std::make_pair(dev, kernel))) return GS_OK;
  GS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.insert(std::make_pair(dev, kernel));
  return GS_OK;
}

}  // namespace gs

extern "C" {

int32_t gs_version(void) { return GS_ABI_VERSION; }

const char* gs_last_error_string(void) { return gs::g_err; }

int32_t gs_set_tuning(const char* key, int32_t value) {
  if (!key) return 0;
  std::lock_guard<std::mutex> l(gs::g_mu);
  int32_t prev = 0;
  auto it = gs::knobs().find(key);
  if (it != gs::knobs().end()) prev = it->second;
  gs::knobs()[key] = value;
  return prev;
}

int32_t gs_perm_prefix_host(uint64_t seed, uint64_t counter, int32_t max_deg, int32_t k, int32_t* out_host) {
  GS_REQUIRE(out_host != nullptr || k == 0, "gs_perm_prefix_host: out_host is NULL");
  GS_REQUIRE(max_deg > 0 && k >= 0 && k <= max_deg, "gs_perm_prefix_host: need 0 <= k <= max_deg (k=%d, max_deg=%d)", k,
             max_deg);
  std::string buf((size_t)max_deg * sizeof(int32_t), '\0');
  int32_t* p = (int32_t*)&buf[0];
  for (int i = 0; i < max_deg; ++i) p[i] = i;
  for (int i = 0; i < k; ++i) {
    uint32_t r = gs::philox_draw(seed, counter, 0u, gs::kStreamPadded, i);
    int j = i + (int)gs::mulhi32(r, (uint32_t)(max_deg - i));
    int32_t t = p[i];
    p[i] = p[j];
    p[j] = t;
  }
  for (int i = 0; i < k; ++i) out_host[i] = p[i];
  return GS_OK;
}

int32_t gs_pipeline_step(const void* ids_host, void* ids_dev, int64_t ids_bytes, void* const* graph_execs_host,
                         int32_t n_graphs, const void* out_dev, void* out_host, int64_t out_bytes, void* h2d_stream,
                         void* compute_stream, void* copy_stream, void* ev_ids, void* ev_done, void* ev_drained) {
  GS_REQUIRE(ids_host && ids_dev && graph_execs_host && out_dev && out_host && ev_ids && ev_done && ev_drained &&
                 n_graphs >= 1,
             "gs_pipeline_step: NULL argument");
  cudaStream_t hs = (cudaStream_t)h2d_stream, cs = (cudaStream_t)compute_stream, ps = (cudaStream_t)copy_stream;
  GS_CUDA(cudaStreamWaitEvent(hs, (cudaEvent_t)ev_done, 0));
  GS_CUDA(cudaMemcpyAsync(ids_dev, ids_host, (size_t)ids_bytes, cudaMemcpyHostToDevice, hs));
  GS_CUDA(cudaEventRecord((cudaEvent_t)ev_ids, hs));
  GS_CUDA(cudaStreamWaitEvent(cs, (cudaEvent_t)ev_ids, 0));
  GS_CUDA(cudaStreamWaitEvent(cs, (cudaEvent_t)ev_drained, 0));
  for (int i = 0; i < n_graphs; ++i) GS_CUDA(cudaGraphLaunch((cudaGraphExec_t)graph_execs_host[i], cs));
  GS_CUDA(cudaEventRecord((cudaEvent_t)ev_done, cs));
  GS_CUDA(cudaStreamWaitEvent(ps, (cudaEvent_t)ev_done, 0));
  GS_CUDA(cudaMemcpyAsync(out_host, out_dev, (size_t)out_bytes, cudaMemcpyDeviceToHost, ps));
  GS_CUDA(cudaEventRecord((cudaEvent_t)ev_drained, ps));
  return GS_OK;
}

}  // extern "C"
