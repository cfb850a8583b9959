// Error plumbing and device queries of the C ABI.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "common.cuh"

namespace yb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
  return YB_ERR_CUDA;
}

int num_sms() {                       // of the CURRENT device (cached per device ordinal)
  static int sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  int& s = sms[dev & 63];
  if (s == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    s = v;
  }
  return s;
}

// Opt in to > 48 KB dynamic shared memory once per (kernel, device).
static std::mutex g_attr_mutex;
int ensure_smem_attr(DeviceOnce& once, const void* kernel, int bytes) {
  int dev = 0;
  YB_CUDA(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  std::lock_guard<std::mutex> lock(g_attr_mutex);
  if (once.mask & bit) return YB_OK;
  YB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  once.mask |= bit;
  return YB_OK;
}

// ---- runtime switches (A/B experiments and tests only; DESIGN.md 5b).  Seeded ONCE from the YB_* environment
// ---- variables, changed afterwards only through yb_set_option(): no getenv() on any call path.
struct Opt { const char* key; char val[32]; };
static Opt g_opts[] = {{"YB_CONV_MODE", ""}, {"YB_CONV_MC", ""}, {"YB_CONV_MCAST", ""}, {"YB_CONV_RES", ""}, {"YB_CONV_EPI", ""}, {"YB_CONV_EG", ""}, {"YB_CONV_PP", ""}, {"YB_CONV_CTAS", ""}, {"YB_THIN", ""}, {"YB_STEM_DBG", ""},
                       {"YB_STEM_WGRAD", ""}, {"YB_WGRAD_TP", ""}, {"YB_DGRAD_S2", ""},
                       {"YB_HALO", ""}, {"YB_STEM_FUSE", ""},
                       {"YB_BN_CPT", ""}, {"YB_BN_FIN", ""}, {"YB_PACK_MT", ""}, {"YB_WGRAD_EPI", ""}, {"YB_WGRAD_SPLITS", ""}, {"YB_STEM_TRAIN", ""}, {"YB_WGRAD_STREAM", ""}, {"YB_STEM_SPLIT", ""}, {"YB_HEAD_STREAM", ""},
                       {"YB_JPEG_SUBSEQ_BITS", ""}};
static std::once_flag g_opt_once;
static void seed_opts() {
  for (auto& o : g_opts) {
    const char* e = getenv(o.key);
    if (e) { strncpy(o.val, e, sizeof(o.val) - 1); o.val[sizeof(o.val) - 1] = 0; }
  }
}
const char* opt(const char* key) {
  std::call_once(g_opt_once, seed_opts);
  for (auto& o : g_opts) if (strcmp(o.key, key) == 0) return o.val;
  return "";
}
int opt_int(const char* key, int dflt) {
  const char* v = opt(key);
  return v[0] ? atoi(v) : dflt;
}

}  // namespace yb

extern "C" int yb_version(void) { return 200; }

extern "C" int yb_set_option(const char* key, const char* value) {
  YB_REQUIRE(key, "set_option: null key");
  std::call_once(yb::g_opt_once, yb::seed_opts);
  for (auto& o : yb::g_opts) {
    if (strcmp(o.key, key) == 0) {
      const char* v = value ? value : "";
      YB_REQUIRE(strlen(v) < sizeof(o.val), "set_option: value too long");
      strcpy(o.val, v);
      return YB_OK;
    }
  }
  yb::set_error("set_option: unknown option '%s'", key);
  return YB_ERR_INVALID_ARGUMENT;
}

extern "C" const char* yb_get_option(const char* key) { return key ? yb::opt(key) : ""; }

extern "C" const char* yb_last_error_string(void) { return yb::g_err; }

extern "C" int yb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  YB_CUDA(cudaGetDevice(&dev));
  if (sm_count) YB_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
  if (cc_major) YB_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
  if (cc_minor) YB_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
  return YB_OK;
}
