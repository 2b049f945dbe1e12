// spec_proto.cu -- stand-alone timing of the model-specialised kernel (wavenet_spec.cuh) on a generated model header.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -I<dir of spec_model.h> -o spec_proto spec_proto.cu
//   -DNAMB200_SPEC_NT=512 -DNAMB200_SPEC_MINB=2: the two-CTA geometry;  -DNAMB200_SPEC_PROBE: after the timed launches, one
//   more launch with the kernel's attribution probe, printed as a table of cycles per layer (wavenet_spec.cuh, spec_probe)
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <string>
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
  constexpr int NT = NAMB200_SPEC_NT, MINB = NAMB200_SPEC_MINB;
  int pmax = 0;
  for (int a = 0; a < spec::NA; a++)
    pmax = spec::A[a].C / 4 > pmax ? spec::A[a].C / 4 : pmax;
  const size_t smem = (size_t)pmax * (spec::LS + NT) * 16;
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
  namb200::JitParams p{state, spec::state_floats, in, out, n, n, batch, n, 0u, nullptr};
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
  unsigned long long hash = 1469598103934665603ull; // FNV-1a of every output bit: variants must agree exactly
  const unsigned char* hb = reinterpret_cast<const unsigned char*>(h.data());
  for (size_t i = 0; i < h.size() * 4; i++)
    hash = (hash ^ hb[i]) * 1099511628211ull;
  printf("{\"test\": \"spec_proto\", \"NT\": %d, \"minb\": %d, \"regs\": %d, \"ctas_per_sm\": %d, \"smem\": %zu, \"batch\": %d, "
         "\"n\": %d, \"ms\": %.3f, \"msamples_per_s\": %.1f, \"checksum\": %.6g, \"hash\": \"%016llx\"}\n",
         NT, MINB, fa.numRegs, occ, smem, batch, n, best, (double)batch * n / best / 1e3, cs, hash);
#ifdef NAMB200_SPEC_PROBE
  // per unit (layer, or an array's convolutional head): clock64 cycles of its history wait, its B0 and its B1, per warp and
  // tile, and their share of all warp cycles spent in tiles; then how many cycles later than the CTA's median warp warp 0
  // arrives at B0 and at B1, per CTA and tile
  constexpr int NS = 5 * (spec::NL + 2) + 2;
  std::vector<unsigned long long> pr(NS, 0ull);
  CK(cudaMemcpyToSymbol(namb200_spec::spec_probe, pr.data(), NS * 8));
  wavenet_spec_kernel<<<grid, NT, smem>>>(p);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpyFromSymbol(pr.data(), namb200_spec::spec_probe, NS * 8));
  const double wt = (double)pr[NS - 1], tile = (double)pr[NS - 2], ct = wt / (NT / 32);
  printf("probe NT=%d minb=%d: %.0f warp-tiles, %.0f cycles per tile, %.1f cycles per frame per SM\n", NT, MINB, wt, tile / wt,
         tile / wt / ((double)NT * occ));
  printf("%-6s %10s %10s %10s %8s %8s %8s %10s %10s\n", "unit", "wait", "B0", "B1", "wait%", "B0%", "B1%", "w0late B0",
         "w0late B1");
  double sum[5] = {0, 0, 0, 0, 0};
  for (int u = 0; u < spec::NL + 2; u++)
  {
    double v[5];
    for (int k = 0; k < 5; k++)
      v[k] = (double)(long long)pr[5 * u + k];
    if (v[0] + v[1] + v[2] == 0.0)
      continue;
    for (int k = 0; k < 5; k++)
      sum[k] += v[k];
    printf("%-6s %10.0f %10.0f %10.0f %7.2f%% %7.2f%% %7.2f%% %10.0f %10.0f\n",
           u < spec::NL ? std::to_string(u).c_str() : ("head" + std::to_string(u - spec::NL)).c_str(), v[0] / wt, v[1] / wt,
           v[2] / wt, 100 * v[0] / tile, 100 * v[1] / tile, 100 * v[2] / tile, v[3] / ct, v[4] / ct);
  }
  printf("%-6s %10.0f %10.0f %10.0f %7.2f%% %7.2f%% %7.2f%% %10.0f %10.0f\n", "all", sum[0] / wt, sum[1] / wt, sum[2] / wt,
         100 * sum[0] / tile, 100 * sum[1] / tile, 100 * sum[2] / tile, sum[3] / ct, sum[4] / ct);
#endif
  return 0;
}
