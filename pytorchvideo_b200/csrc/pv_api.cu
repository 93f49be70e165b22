// Library-level C ABI: error reporting, device info, launch accounting, conv dispatch.
#include "pv_common.cuh"

#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <string.h>

namespace pv {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};
// per-kernel-instance launch counts, keyed by the address of the launch site's name literal (one hash update per
// eager launch; graph replays do not come through here)
static std::mutex g_kernel_mu;
static std::unordered_map<const char*, long long> g_kernel_counts;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(const char* name) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  std::lock_guard<std::mutex> lock(g_kernel_mu);
  ++g_kernel_counts[name];
}

int conv3d_check(const pv_conv3d_desc* d);
int conv3d_direct_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, const void* residual, void* y, cudaStream_t s);
int conv3d_tcgen05_supported(const pv_conv3d_desc* d, char* why, size_t why_len);
int conv3d_group_span(const pv_conv3d_desc* d, int* span_groups, int* span_k, int* span_n);   // pv_igemm.cu
int conv3d_tcgen05_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                          const float* bias, const void* residual, void* y, cudaStream_t s);
int conv3d_gather_supported(const pv_conv3d_desc* d);
int conv3d_gather_launch(const pv_conv3d_desc* d, const void* x, const void* w, const float* scale,
                         const float* bias, const void* residual, void* y, cudaStream_t s);
// narrow inputs (C_in < 64, weights packed with the un-padded per-tap K extent) take the gather-fed
// variant, everything else the TMA-fed one
bool conv3d_tma_narrow(const pv_conv3d_desc* d);   // pv_igemm.cu: C_in = 16 / 32 go through TMA boxes of 32 / 64 bytes
static bool wants_gather(const pv_conv3d_desc* d) { return d->Ci < 64 && d->ci_pad64 == d->Ci && !conv3d_tma_narrow(d); }

}  // namespace pv

extern "C" int pv_abi_version(void) { return PV_ABI_VERSION; }
extern "C" const char* pv_last_error(void) { return pv::g_err; }
extern "C" long long pv_launch_count(void) { return pv::g_launches.load(); }

extern "C" int pv_kernel_counts(char* buf, int len) {
  std::map<std::string, long long> by_name;   // the same name may be spelled at several sites: merge, sort
  {
    std::lock_guard<std::mutex> lock(pv::g_kernel_mu);
    for (const auto& kv : pv::g_kernel_counts) by_name[kv.first] += kv.second;
  }
  std::string out;
  for (const auto& kv : by_name) out += kv.first + " " + std::to_string(kv.second) + "\n";
  if (buf && len > (int)out.size()) memcpy(buf, out.c_str(), out.size() + 1);
  else if (buf && len > 0) buf[0] = '\0';
  return (int)out.size();
}

extern "C" int pv_device_info(int* sm_count, int* cc) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    (void)cudaGetLastError();
    pv::set_error("no CUDA device visible");
    return PV_ERR_NO_DEVICE;
  }
  int dev = 0, sms = 0, major = 0, minor = 0;
  PV_CUDA_OK(cudaGetDevice(&dev));
  PV_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  PV_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  PV_CUDA_OK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (sm_count) *sm_count = sms;
  if (cc) *cc = major * 10 + minor;
  if (major != 9 || minor != 0) {
    pv::set_error("device is sm_%d%d; this library contains sm_90a code only", major, minor);
    return PV_ERR_NO_DEVICE;
  }
  return PV_OK;
}

extern "C" int pv_conv3d_tcgen05_supported(const pv_conv3d_desc* d) {
  if (!d || !pv::act_known(d->act) || pv::conv3d_has_prologue(d)) return 0;
  if (pv::wants_gather(d)) return pv::conv3d_gather_supported(d);
  return pv::conv3d_tcgen05_supported(d, nullptr, 0);
}

extern "C" int pv_conv3d_group_span(const pv_conv3d_desc* d, int* span_groups, int* span_k, int* span_n) {
  int sg = 0, sk = 0, sn = 0;
  const bool known = d && d->groups > 1 && pv::conv3d_group_span(d, &sg, &sk, &sn);
  if (span_groups) *span_groups = sg;
  if (span_k) *span_k = sk;
  if (span_n) *span_n = sn;
  if (!known || !pv::act_known(d->act)) return 0;
  pv_conv3d_desc q = *d;
  q.ci_pad64 = sk;             // grouped mode packs the weights at the span width
  return pv::conv3d_tcgen05_supported(&q, nullptr, 0);
}

extern "C" int pv_conv3d_fwd(const pv_conv3d_desc* d, int algo, const void* x, const void* w,
                             const float* scale, const float* bias, const void* residual, void* y,
                             void* stream) {
  int rc = pv::conv3d_check(d);
  if (rc != PV_OK) return rc;
  if (pv::conv3d_has_prologue(d)) {
    pv::set_error("pv_conv3d_fwd takes no pre-activation prologue (pv_dwconv3d_fwd / pv_dwplane_fwd do)");
    return PV_ERR_UNSUPPORTED;
  }
  PV_CHECK_ARG(x && w && scale && bias && y, "null pointer");
  PV_CHECK_ARG(!d->has_residual || residual, "has_residual set but residual is null");
  cudaStream_t s = (cudaStream_t)stream;
  if (algo == PV_ALGO_AUTO)   // dense or grouped mode on the tensor cores when they take it; depthwise never does
    algo = pv_conv3d_tcgen05_supported(d) ? PV_ALGO_TCGEN05 : PV_ALGO_DIRECT;
  if (algo == PV_ALGO_TCGEN05) {
    if (pv::wants_gather(d)) return pv::conv3d_gather_launch(d, x, w, scale, bias, residual, y, s);
    return pv::conv3d_tcgen05_launch(d, x, w, scale, bias, residual, y, s);
  }
  if (algo == PV_ALGO_DIRECT) return pv::conv3d_direct_launch(d, x, w, scale, bias, residual, y, s);
  pv::set_error("unknown algo %d", algo);
  return PV_ERR_INVALID;
}
