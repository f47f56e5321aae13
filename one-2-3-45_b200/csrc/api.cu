// Library-wide plumbing of libo2345_sm90.so: error string, device query.
#include <stdarg.h>

#include <stdlib.h>

#include "common.cuh"

namespace o2345 {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("O2345_PDL");
    on = (e && e[0] == '0') ? 0 : 1;
  }
  return on == 1;
}

int sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;
  }
  return sms;
}

}  // namespace o2345

extern "C" int o2345_abi_version(void) { return O2345_ABI_VERSION; }

extern "C" int o2345_last_error(char* buf, size_t n) {
  if (!buf || n == 0) return O2345_EINVAL;
  strncpy(buf, o2345::g_err, n - 1);
  buf[n - 1] = 0;
  return O2345_OK;
}

extern "C" int o2345_device_info(int* major, int* minor, int* sms) {
  int dev = 0, ma = 0, mi = 0, n = 0;
  O2345_CUDA(cudaGetDevice(&dev));
  O2345_CUDA(cudaDeviceGetAttribute(&ma, cudaDevAttrComputeCapabilityMajor, dev));
  O2345_CUDA(cudaDeviceGetAttribute(&mi, cudaDevAttrComputeCapabilityMinor, dev));
  O2345_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  if (major) *major = ma;
  if (minor) *minor = mi;
  if (sms) *sms = n;
  if (ma != 9 || mi != 0) {
    o2345::set_error("o2345_device_info: device is sm_%d%d, this library is built for sm_90a only", ma, mi);
    return O2345_EUNSUPPORTED;
  }
  return O2345_OK;
}
