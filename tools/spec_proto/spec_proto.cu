// spec_proto.cu -- stand-alone timing of the model-specialised kernel (wavenet_spec.cuh) on a generated model header.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -I<dir of spec_model.h> -o spec_proto spec_proto.cu
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "spec_model.h"

#include "../../neuralampmodelercore_b200/csrc/wavenet_spec.cuh"

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
  const int batch = argc > 1 ? atoi(argv[1]) : 4096, n = argc > 2 ? atoi(argv[2]) : 4096, reps = argc > 3 ? atoi(argv[3]) : 5;
  constexpr int NT = NAMB200_SPEC_NT, S = NAMB200_SPEC_S, MINB = NAMB200_SPEC_MINB;
  int pmax = 0;
  for (int a = 0; a < spec::NA; a++)
    pmax = spec::A[a].C / 4 > pmax ? spec::A[a].C / 4 : pmax;
  const size_t smem = (size_t)pmax * S * (spec::LS + NT) * 16; // S = 2: twice the (sub-)planes
  CK(cudaFuncSetAttribute(wavenet_spec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, wavenet_spec_kernel, NT, smem));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, wavenet_spec_kernel));
  const int grid = occ * prop.multiProcessorCount < batch ? occ * prop.multiProcessorCount : batch;
  float *state, *in, *out;
  CK(cudaMalloc(&state, (size_t)batch * spec::state_floats * 4));
  CK(cudaMemset(state, 0, (size_t)batch * spec::state_floats * 4));
  CK(cudaMalloc(&in, (size_t)batch * n * 4));
  CK(cudaMalloc(&out, (size_t)batch * n * 4));
  std::vector<float> h((size_t)batch * n);
  for (size_t i = 0; i < h.size(); i++)
    h[i] = 0.3f * sinf(0.01f * (float)(i % 100003));
  CK(cudaMemcpy(in, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  float* scratch = nullptr;
  if (S == 2)
    CK(cudaMalloc(&scratch, (size_t)grid * 2 * spec::state_floats * 4));
  namb200_spec::SpecParams p{state, spec::state_floats, in, out, n, n, batch, n, 0u, scratch, 2 * spec::state_floats};
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  double best = 1e30;
  for (int r = 0; r < reps + 2; r++)
  {
    CK(cudaEventRecord(e0));
    wavenet_spec_kernel<<<grid, NT, smem>>>(p);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (r >= 2 && ms < best)
      best = ms;
    p.t_base += (unsigned)n;
  }
  CK(cudaMemcpy(h.data(), out, h.size() * 4, cudaMemcpyDeviceToHost));
  double cs = 0;
  for (size_t i = 0; i < h.size(); i += 997)
    cs += h[i];
  printf("{\"test\": \"spec_proto\", \"NT\": %d, \"S\": %d, \"minb\": %d, \"regs\": %d, \"ctas_per_sm\": %d, \"smem\": %zu, \"batch\": %d, "
         "\"n\": %d, \"ms\": %.3f, \"msamples_per_s\": %.1f, \"checksum\": %.6g}\n",
         NT, S, MINB, fa.numRegs, occ, smem, batch, n, best, (double)batch * n / best / 1e3, cs);
  return 0;
}
