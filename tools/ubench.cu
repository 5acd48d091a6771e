// tools/ubench.cu — integer-pipe throughput microbenchmarks for sm_90a (H100).
// Reports warp-instructions issued per clock per SM for the op classes the fused kernel is made of,
// to decide how to balance GF(2^8)/HighwayHash work between the ALU pipe (LOP3/PRMT/IADD3/SHF) and
// the FMA pipe (IMAD*).  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o ubench ubench.cu
#include <cstdio>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

#define ITERS 4096
#define CHAINS 8

template <int OP>
__device__ __forceinline__ void op(uint32_t& a, uint32_t& b, uint32_t c) {
  if constexpr (OP == 0) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(b), "r"(c));
  if constexpr (OP == 1) asm volatile("prmt.b32 %0, %0, %1, %2;" : "+r"(a) : "r"(b), "r"(c));
  if constexpr (OP == 2) asm volatile("add.u32 %0, %0, %1;" : "+r"(a) : "r"(b));
  if constexpr (OP == 3) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(b), "r"(c));
  if constexpr (OP == 4) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(a) : "r"(b));
  if constexpr (OP == 5) {
    uint64_t w;
    asm volatile("mad.wide.u32 %0, %1, %2, %3;" : "=l"(w) : "r"(a), "r"(b), "l"((uint64_t)c));
    a = (uint32_t)w ^ (uint32_t)(w >> 32);
  }
  if constexpr (OP == 6) asm volatile("shf.l.wrap.b32 %0, %0, %1, %2;" : "+r"(a) : "r"(b), "r"(c));
  if constexpr (OP == 7) {  // LOP3 + IMAD alternating (1:1)
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(b), "r"(c));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(b) : "r"(a), "r"(c));
  }
  if constexpr (OP == 8) {  // LOP3 x2 + IMAD x1
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(b), "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(b) : "r"(a), "r"(c));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(b), "r"(c));
  }
  if constexpr (OP == 9) {  // PRMT + LOP3 (same pipe?)
    asm volatile("prmt.b32 %0, %0, %1, %2;" : "+r"(a) : "r"(b), "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(b) : "r"(a), "r"(c));
  }
  if constexpr (OP == 10) {  // 64-bit add (IADD3 + IADD3.X)
    uint64_t x = ((uint64_t)a << 32) | b;
    asm volatile("add.u64 %0, %0, %1;" : "+l"(x) : "l"((uint64_t)c * 0x100000001ull));
    a = (uint32_t)(x >> 32); b = (uint32_t)x;
  }
  if constexpr (OP == 11) {  // mul.hi + lop3
    asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(a) : "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(b) : "r"(a), "r"(c));
  }
  if constexpr (OP == 12) {  // LOP3 with immediate + IMAD with immediate (fewer register reads)
    asm volatile("lop3.b32 %0, %0, %1, 0x1d1d1d1d, 0x96;" : "+r"(a) : "r"(b));
    asm volatile("mad.lo.u32 %0, %0, 3, %1;" : "+r"(b) : "r"(a));
  }
  if constexpr (OP == 13) {  // LOP3 : PRMT : IMAD 1:1:1
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(b), "r"(c));
    asm volatile("prmt.b32 %0, %0, %1, 0x5140;" : "+r"(b) : "r"(a));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a) : "r"(b), "r"(c));
  }
  if constexpr (OP == 14) {  // 2-register LOP3 (and) + 2-register add
    asm volatile("and.b32 %0, %0, %1;" : "+r"(a) : "r"(b));
    asm volatile("mad.lo.u32 %0, %0, 5, %1;" : "+r"(b) : "r"(a));
  }
  if constexpr (OP == 15) {  // LOP3 x3 + IMAD x1
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(b), "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(b) : "r"(a), "r"(c));
    asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a) : "r"(b), "r"(c));
    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(b) : "r"(a), "r"(c));
  }
}
template <int OP> constexpr int ops_per_call() { return (OP == 7 || OP == 9 || OP == 11 || OP == 12 || OP == 14) ? 2 : ((OP == 8 || OP == 13) ? 3 : (OP == 15 ? 4 : (OP == 5 ? 2 : (OP == 10 ? 2 : 1)))); }

template <int OP>
__global__ void bench(uint32_t* out, long long* cycles, uint32_t seed) {
  uint32_t a[CHAINS], b[CHAINS];
  for (int i = 0; i < CHAINS; i++) { a[i] = seed + threadIdx.x * 7 + i; b[i] = seed * 3 + i * 11 + blockIdx.x; }
  const uint32_t c = seed | 0x3210;
  __syncthreads();
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int i = 0; i < CHAINS; i++) op<OP>(a[i], b[i], c);
  }
  long long t1 = clock64();
  uint32_t acc = 0;
  for (int i = 0; i < CHAINS; i++) acc ^= a[i] ^ b[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int OP>
void run(const char* name, int sms, int threads, int blocks_per_sm) {
  int blocks = sms * blocks_per_sm;
  uint32_t* out; long long* cyc;
  cudaMalloc(&out, (size_t)blocks * threads * 4);
  cudaMalloc(&cyc, blocks * sizeof(long long));
  bench<OP><<<blocks, threads>>>(out, cyc, 12345);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  bench<OP><<<blocks, threads>>>(out, cyc, 12345);
  cudaEventRecord(e1);
  cudaDeviceSynchronize();
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  std::vector<long long> h(blocks);
  cudaMemcpy(h.data(), cyc, blocks * sizeof(long long), cudaMemcpyDeviceToHost);
  double avg = 0; for (auto v : h) avg += v; avg /= blocks;
  double warp_instr_per_sm = (double)ITERS * CHAINS * ops_per_call<OP>() * (threads / 32) * blocks_per_sm;
  printf("%-28s thr/SM=%4d  warp-instr/clk/SM = %6.3f   (lanes/clk/SM = %6.1f)  eff.clk = %.0f MHz\n", name,
         threads * blocks_per_sm, warp_instr_per_sm / avg, 32.0 * warp_instr_per_sm / avg, avg / (ms * 1e3));
  cudaFree(out); cudaFree(cyc);
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  int sms = p.multiProcessorCount;
  printf("device %s, %d SMs\n", p.name, sms);
  for (int tpb : {1024, 512}) {
    int bps = 1;
    run<0>("LOP3", sms, tpb, bps);
    run<1>("PRMT", sms, tpb, bps);
    run<2>("IADD", sms, tpb, bps);
    run<6>("SHF", sms, tpb, bps);
    run<3>("IMAD.LO", sms, tpb, bps);
    run<4>("IMAD.HI (mul.hi)", sms, tpb, bps);
    run<5>("IMAD.WIDE (+xor)", sms, tpb, bps);
    run<10>("ADD.U64", sms, tpb, bps);
    run<7>("LOP3:IMAD 1:1", sms, tpb, bps);
    run<8>("LOP3:IMAD 2:1", sms, tpb, bps);
    run<9>("PRMT:LOP3 1:1", sms, tpb, bps);
    run<11>("MULHI:LOP3 1:1", sms, tpb, bps);
    run<12>("LOP3imm:IMADimm 1:1", sms, tpb, bps);
    run<13>("LOP3:PRMT:IMAD 1:1:1", sms, tpb, bps);
    run<14>("AND2:IMADimm 1:1", sms, tpb, bps);
    run<15>("LOP3:IMAD 3:1", sms, tpb, bps);
    printf("\n");
  }
  return 0;
}
