// Library probes and process-wide state of libdisvae_b200.so.
#include "dv_common.cuh"

namespace dv {
thread_local int g_last_cuda_error = 0;
long long g_launches = 0;
}

extern "C" {

int dv_version(void) { return 100; }            // 0.1.0
int dv_built_arch(void) { return 90; }

const char* dv_status_string(int status) {
  switch (status) {
    case DV_OK: return "ok";
    case DV_ERR_BAD_SHAPE: return "unsupported shape";
    case DV_ERR_BAD_ARG: return "bad argument";
    case DV_ERR_WORKSPACE: return "workspace too small";
    case DV_ERR_CUDA: return "CUDA runtime error";
    case DV_ERR_ARCH: return "device is not sm_90";
    default: return "unknown status";
  }
}

int dv_last_cuda_error(void) { return dv::g_last_cuda_error; }

int dv_device_check(void) {
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    dv::g_last_cuda_error = (int)cudaGetLastError();
    return DV_ERR_CUDA;
  }
  return (prop.major == 9 && prop.minor == 0) ? DV_OK : DV_ERR_ARCH;
}

long long dv_launch_count(void) { return dv::g_launches; }

}  // extern "C"
