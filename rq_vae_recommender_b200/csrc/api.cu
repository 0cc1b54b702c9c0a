// C-ABI plumbing shared by every entry point of librqb200: version, thread-local error text.
#include "common.cuh"
#include <cstring>

static thread_local char g_err[512] = "";

void rqb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* rqb200_last_error(void) { return g_err; }
extern "C" int rqb200_version(void) { return 101; }

// number of SMs / compute capability of the current device (host logic sizes persistent grids with it)
extern "C" int rqb200_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  RQB_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  RQB_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return RQB_OK;
}
