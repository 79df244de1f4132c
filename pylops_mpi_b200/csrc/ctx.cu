// Context handle + error strings for libb200lops.
#include <stdio.h>
#include <string.h>
#include "common.cuh"

extern "C" int b2_version(void) { return B2_VERSION; }

extern "C" const char* b2_strerror(int code) {
  static thread_local char buf[128];
  if (code == 0) return "ok";
  if (code >= 2000) {
    switch (code) {
      case B2_ERR_DTYPE: return "b200lops: unsupported dtype for this entry point";
      case B2_ERR_ARG: return "b200lops: invalid argument";
      case B2_ERR_HALO: return "b200lops: halo rows missing for a stencil that reaches a neighbour rank";
      case B2_ERR_WORKSPACE: return "b200lops: internal workspace too small";
      case B2_ERR_UNSUPPORTED: return "b200lops: unsupported kind/order";
      case B2_ERR_ALIGN: return "b200lops: pointer alignment requirement not met";
      case B2_ERR_CONVERGE: return "b200lops: iteration did not reach its fixed point within max_iter";
      default: return "b200lops: unknown library error";
    }
  }
  if (code >= 1000) {
    snprintf(buf, sizeof buf, "NCCL error %d", code - 1000);
    return buf;
  }
  return cudaGetErrorString((cudaError_t)code);
}

extern "C" int b2_ctx_create(int device, b2_ctx** out) {
  if (!out) return B2_ERR_ARG;
  B2_CUDA(cudaSetDevice(device));
  b2_ctx* c = new b2_ctx();
  memset(c, 0, sizeof(*c));
  c->device = device;
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) { delete c; return (int)e; }
  c->sm_count = prop.multiProcessorCount;
  e = cudaMalloc((void**)&c->red_partials, sizeof(double) * B2_RED_MAX_BLOCKS * B2_RED_MAX_OUT);
  if (e != cudaSuccess) { delete c; return (int)e; }
  e = cudaMalloc((void**)&c->tickets, sizeof(unsigned int) * B2_TICKETS);
  if (e != cudaSuccess) { cudaFree(c->red_partials); delete c; return (int)e; }
  e = cudaMemset(c->tickets, 0, sizeof(unsigned int) * B2_TICKETS);
  if (e != cudaSuccess) { cudaFree(c->red_partials); cudaFree(c->tickets); delete c; return (int)e; }
  *out = c;
  return B2_OK;
}

extern "C" int b2_ctx_destroy(b2_ctx* c) {
  if (!c) return B2_OK;
  cudaSetDevice(c->device);
  if (c->red_partials) cudaFree(c->red_partials);
  if (c->tickets) cudaFree(c->tickets);
  if (c->gemv_partials) cudaFree(c->gemv_partials);
  for (int i = 0; i < c->gemv_retired_n; ++i) cudaFree(c->gemv_retired[i]);
  for (int s = 0; s < 3; ++s) {
    for (int k = 0; k < 2; ++k)
      if (c->pipe_buf[s][k]) cudaFree(c->pipe_buf[s][k]);
    if (c->pipe_stream[s]) cudaStreamDestroy(c->pipe_stream[s]);
    for (int k = 0; k < 3; ++k)
      if (c->pipe_ev[s][k]) cudaEventDestroy(c->pipe_ev[s][k]);
  }
  delete c;
  return B2_OK;
}

extern "C" int b2_ctx_sm_count(const b2_ctx* c, int* out) {
  if (!c || !out) return B2_ERR_ARG;
  *out = c->sm_count;
  return B2_OK;
}
