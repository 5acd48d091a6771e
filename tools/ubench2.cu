// tools/ubench2.cu — compute-only ceilings of the two halves of the fused kernel (no memory traffic):
//   HH: HighwayHash half-state updates per clock,  GF: (12 -> 4) packed GF(2^8) products per clock.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I minio_b200/csrc [-DMEC_XTIME=n] -o ubench2 tools/ubench2.cu
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "ec_device.cuh"
using namespace mec;

#define ITERS 2048

__global__ void __launch_bounds__(1024, 1) k_hh(uint64_t* out, long long* cyc, uint64_t seed, uint32_t one) {
  HHHalf s;
  const uint64_t key[4] = {seed, seed * 3, seed * 5, seed * 7};
  hh_init(s, key, threadIdx.x & 1);
  uint64_t a0 = seed + threadIdx.x, a1 = seed * 11 + blockIdx.x;
  __syncthreads();
  long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < ITERS; i += 8) {
#pragma unroll
    for (int j = 0; j < 8; j++) { hh_update(s, a0, a1, one); a0 += 0x9e3779b97f4a7c15ull; a1 ^= a0; }
  }
  long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = s.v0[0] ^ s.v0[1] ^ s.v1[0] ^ s.v1[1] ^ s.m0[0] ^ s.m0[1] ^ s.m1[0] ^ s.m1[1];
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int K, int M>
__global__ void __launch_bounds__(1024, 1) k_gf(uint32_t* out, long long* cyc, uint32_t seed) {
  uint32_t in[K];
  for (int t = 0; t < K; t++) in[t] = seed * (t + 3) + threadIdx.x * 2654435761u + blockIdx.x;
  uint32_t acc = 0;
  __syncthreads();
  long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < ITERS / 8; i++) {
    uint32_t o[M];
    GfStaticApply<EncodeMatrix<K, M>>::run(in, o);
#pragma unroll
    for (int j = 0; j < M; j++) acc ^= o[j];
#pragma unroll
    for (int t = 0; t < K; t++) in[t] += acc + t;   // keeps the inputs live and changing (K extra adds)
  }
  long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

static double avg_cycles(long long* d, int n) {
  std::vector<long long> h(n);
  cudaMemcpy(h.data(), d, n * sizeof(long long), cudaMemcpyDeviceToHost);
  double a = 0; for (auto v : h) a += v; return a / n;
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  const int sms = p.multiProcessorCount;
  uint64_t* o64; uint32_t* o32; long long* cyc;
  cudaMalloc(&o64, (size_t)sms * 1024 * 8); cudaMalloc(&o32, (size_t)sms * 1024 * 4); cudaMalloc(&cyc, sms * 8);
  for (int thr : {768}) {
    for (int rep = 0; rep < 2; rep++) k_hh<<<sms, thr>>>(o64, cyc, 12345, 1u);
    cudaDeviceSynchronize();
    double c = avg_cycles(cyc, sms);
    // one hh_update = one half packet = 16 hashed bytes = 4 hashed words per thread
    double upd = (double)ITERS * thr / c;  // half-updates per clk per SM
    printf("HH  thr/SM=%4d: %.3f half-updates/clk/SM = %.2f hashed B/clk/SM  (%.1f cyc per warp-update per SMSP)\n", thr, upd, upd * 16,
           4.0 * 32 / upd);
    for (int rep = 0; rep < 2; rep++) k_gf<12, 4><<<sms, thr>>>(o32, cyc, 777);
    cudaDeviceSynchronize();
    c = avg_cycles(cyc, sms);
    double cols = (double)(ITERS / 8) * thr / c;  // word-columns (12 data words -> 4 parity words) per clk per SM
    printf("GF  thr/SM=%4d: %.3f word-columns/clk/SM = %.2f data B/clk/SM  (%.1f cyc per warp-column per SMSP)\n", thr, cols, cols * 48,
           4.0 * 32 / cols);
    double hh_B = upd * 16, gf_B = cols * 48;
    // fused ceiling: per data byte, GF handles 1 byte and HH hashes 16/12 bytes
    double fused = 1.0 / (1.0 / gf_B + (16.0 / 12.0) / hh_B);
    printf("    => compute-only fused ceiling %.2f data B/clk/SM = %.0f GB/s object at 1.9 GHz x %d SMs\n", fused, fused * 1.9 * sms, sms);
  }
  return 0;
}
