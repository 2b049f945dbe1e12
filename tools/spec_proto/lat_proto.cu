// lat_proto.cu -- stand-alone timing of the low-latency specialised kernel (wavenet_lat.cuh): one stream, 64-frame calls.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "spec_model.h"

#include "../../neuralampmodelercore_b200/csrc/wavenet_spec.cuh"
#include "../../neuralampmodelercore_b200/csrc/wavenet_lat.cuh"

#define CK(x)                                                                                                        \
  do                                                                                                                 \
  {                                                                                                                  \
    cudaError_t e = (x);                                                                                             \
    if (e != cudaSuccess)                                                                                            \
    {                                                                                                                \
      fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e));                                                        \
      exit(1);                                                                                                       \
    }                                                                                                                \
  } while (0)

int main(int argc, char** argv)
{
  const int batch = argc > 1 ? atoi(argv[1]) : 1, n = argc > 2 ? atoi(argv[2]) : 64, calls = argc > 3 ? atoi(argv[3]) : 1500;
  constexpr int FW = NAMB200_LAT_FW, F = 32 * FW;
  const size_t smem = (size_t)namb200_lat::Plan<F>::total_float4() * 16;
  CK(cudaFuncSetAttribute(wavenet_lat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, wavenet_lat_kernel));
  float *state, *in, *out;
  CK(cudaMalloc(&state, (size_t)batch * spec::state_floats * 4));
  CK(cudaMemset(state, 0, (size_t)batch * spec::state_floats * 4));
  CK(cudaMalloc(&in, (size_t)batch * n * 4));
  CK(cudaMalloc(&out, (size_t)batch * n * 4));
  std::vector<float> h((size_t)batch * n);
  for (size_t i = 0; i < h.size(); i++)
    h[i] = 0.3f * sinf(0.01f * (float)(i % 100003));
  CK(cudaMemcpy(in, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  namb200::LatParams p{{state, spec::state_floats, in, out, n, n, batch, n, 0u, nullptr}, nullptr, 0u};
  {
    // correctness: the same calls through the throughput kernel (wavenet_spec.cuh) on a second copy of the state
    float *state2, *out2;
    CK(cudaMalloc(&state2, (size_t)batch * spec::state_floats * 4));
    CK(cudaMemset(state2, 0, (size_t)batch * spec::state_floats * 4));
    CK(cudaMalloc(&out2, (size_t)batch * n * 4));
    int pmax = 0;
    for (int a = 0; a < spec::NA; a++)
      pmax = spec::A[a].C / 4 > pmax ? spec::A[a].C / 4 : pmax;
    const size_t smem2 = (size_t)pmax * (spec::LS + NAMB200_SPEC_NT) * 16;
    CK(cudaFuncSetAttribute(wavenet_spec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    namb200::JitParams q{state2, spec::state_floats, in, out2, n, n, batch, n, 0u, nullptr};
    std::vector<float> a(h.size()), b(h.size());
    double worst = 0;
    for (int call = 0; call < 40; call++)
    {
      wavenet_lat_kernel<<<batch, 128 * FW, smem>>>(p);
      wavenet_spec_kernel<<<batch, NAMB200_SPEC_NT, smem2>>>(q);
      CK(cudaDeviceSynchronize());
      CK(cudaMemcpy(a.data(), out, a.size() * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(b.data(), out2, b.size() * 4, cudaMemcpyDeviceToHost));
      double e = 0;
      for (size_t i = 0; i < a.size(); i++)
        e = fmax(e, fabs((double)a[i] - b[i]));
      if (call < 4 || e > worst)
        printf("call %d: max |lat - spec| = %.3e (first values %.6f %.6f)\n", call, e, a[0], b[0]);
      worst = fmax(worst, e);
      p.t_base += (unsigned)n;
      q.t_base += (unsigned)n;
    }
    printf("worst %.3e\n", worst);
  }
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int i = 0; i < 20; i++)
  {
    wavenet_lat_kernel<<<batch, 128 * FW, smem>>>(p);
    p.t_base += (unsigned)n;
  }
  CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(e0));
  for (int i = 0; i < calls; i++)
  {
    wavenet_lat_kernel<<<batch, 128 * FW, smem>>>(p);
    p.t_base += (unsigned)n;
  }
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  CK(cudaGetLastError());
  float ms;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  CK(cudaMemcpy(h.data(), out, h.size() * 4, cudaMemcpyDeviceToHost));
  double cs = 0;
  for (size_t i = 0; i < h.size(); i++)
    cs += h[i];
  printf("{\"test\": \"lat_proto\", \"FW\": %d, \"regs\": %d, \"smem\": %zu, \"batch\": %d, \"n\": %d, \"calls\": %d, "
         "\"us_per_call_back_to_back\": %.2f, \"checksum\": %.6g}\n",
         FW, fa.numRegs, smem, batch, n, calls, ms * 1e3 / calls, cs);
  return 0;
}
