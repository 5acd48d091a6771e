// copy_probe: what the copy engine sustains for a train of small pinned H2D copies (the coalescer's staging pattern), alone and
// with a D2H train on another stream.  nvcc -O2 -arch=sm_90a -o copy_probe copy_probe.cu
#include <cuda_runtime.h>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <vector>
int main() {
  const size_t total = 512ull << 20;
  char *h = nullptr, *h2 = nullptr, *d = nullptr, *d2 = nullptr;
  cudaHostAlloc(&h, total, cudaHostAllocPortable);
  cudaHostAlloc(&h2, total, cudaHostAllocPortable);
  cudaMalloc(&d, total);
  cudaMalloc(&d2, total);
  cudaStream_t s1, s2, s3;
  cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&s3, cudaStreamNonBlocking);
  for (size_t piece : {64u << 10, 256u << 10, 1u << 20, 4u << 20, 16u << 20, 512u << 20}) {
    for (int mode = 0; mode < 5; mode++) {  // 0: H2D alone, 1: H2D + D2H (1/3 of the bytes), 2: H2D split over two streams, 3/4: cudaMemcpyBatchAsync (40 per call) alone / with D2H
      const size_t n = total / piece;
      double best = 0, best_issue = 0;
      for (int rep = 0; rep < 3; rep++) {
        cudaDeviceSynchronize();
        auto t0 = std::chrono::steady_clock::now();
        if (mode >= 3) {
          std::vector<void*> dsts(n), srcs(n);
          std::vector<size_t> sizes(n, piece);
          for (size_t i = 0; i < n; i++) { dsts[i] = d + i * piece; srcs[i] = h + ((i * 7) % n) * piece; }
          cudaMemcpyAttributes at = {};
          at.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
          size_t idx0 = 0, fail = 0;
          for (size_t i = 0; i < n; i += 40) {
            const size_t cnt = n - i < 40 ? n - i : 40;
            cudaError_t e = cudaMemcpyBatchAsync(dsts.data() + i, srcs.data() + i, sizes.data() + i, cnt, &at, &idx0, 1, &fail, s1);
            if (e != cudaSuccess) { printf("batch copy: %s\n", cudaGetErrorString(e)); return 1; }
            if (mode == 4)
              for (size_t j = i; j < i + cnt; j += 3) cudaMemcpyAsync(h2 + j * piece, d2 + j * piece, piece, cudaMemcpyDeviceToHost, s2);
          }
        } else
        for (size_t i = 0; i < n; i++) {
          cudaMemcpyAsync(d + i * piece, h + ((i * 7) % n) * piece, piece, cudaMemcpyHostToDevice, (mode == 2 && (i & 1)) ? s3 : s1);
          if (mode == 1 && i % 3 == 0) cudaMemcpyAsync(h2 + i * piece, d2 + i * piece, piece, cudaMemcpyDeviceToHost, s2);
        }
        auto t1 = std::chrono::steady_clock::now();
        cudaStreamSynchronize(s1);
        cudaStreamSynchronize(s3);
        auto t2 = std::chrono::steady_clock::now();
        cudaStreamSynchronize(s2);
        const double sec = std::chrono::duration<double>(t2 - t0).count(), issue = std::chrono::duration<double>(t1 - t0).count();
        if (total / sec > best) { best = total / sec; best_issue = issue / n * 1e6; }
      }
      printf("{\"piece_KiB\": %zu, \"mode\": \"%s\", \"h2d_GBps\": %.1f, \"issue_us_per_copy\": %.2f}\n", piece >> 10,
             mode == 0 ? "h2d" : mode == 1 ? "h2d+d2h/3" : mode == 2 ? "h2d 2 streams" : mode == 3 ? "batch40" : "batch40+d2h/3", best / 1e9, best_issue);
    }
  }
  // the GetObject staging pattern: rows of 32 + S bytes (a bitrot frame) from k part files into an arena with a 16-byte-aligned row pitch,
  // and rows of S bytes back out into the object at pitch block_size: one 2-D copy per file vs one batched call of 1-D rows
  {
    const size_t S = 87382, F = 32 + S, P = (F + 15) / 16 * 16, rows = 256, k = 12, bs = 1 << 20;
    for (int mode = 0; mode < 6; mode++) {  // 4: 2-D H2D + ONE contiguous D2H of the same bytes, 5: contiguous both ways; 0: 2-D H2D, 1: batched rows H2D, 2: 2-D both directions, 3: batched rows both directions
      double best = 0;
      for (int rep = 0; rep < 3; rep++) {
        cudaDeviceSynchronize();
        auto t0 = std::chrono::steady_clock::now();
        for (int it = 0; it < 4; it++) {
          if (mode == 4 || mode == 5) {
            if (mode == 4) for (size_t t = 0; t < k; t++) cudaMemcpy2DAsync(d + t * rows * P, P, h + t * rows * F, F, F, rows, cudaMemcpyHostToDevice, s1);
            else cudaMemcpyAsync(d, h, k * rows * F, cudaMemcpyHostToDevice, s1);
            cudaMemcpyAsync(h2, d2, k * rows * S, cudaMemcpyDeviceToHost, s2);
          } else if (mode == 0 || mode == 2) {
            for (size_t t = 0; t < k; t++) cudaMemcpy2DAsync(d + t * rows * P, P, h + t * rows * F, F, F, rows, cudaMemcpyHostToDevice, s1);
            if (mode == 2)
              for (size_t t = 0; t < k; t++) cudaMemcpy2DAsync(h2 + t * S, bs, d2 + t * rows * P + 32, P, S, rows, cudaMemcpyDeviceToHost, s2);
          } else {
            std::vector<void*> dsts, srcs;
            std::vector<size_t> sizes;
            for (size_t t = 0; t < k; t++)
              for (size_t r = 0; r < rows; r++) { dsts.push_back(d + (t * rows + r) * P); srcs.push_back(h + (t * rows + r) * F); sizes.push_back(F); }
            cudaMemcpyAttributes at = {};
            at.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
            size_t idx0 = 0, fail = 0;
            cudaMemcpyBatchAsync(dsts.data(), srcs.data(), sizes.data(), dsts.size(), &at, &idx0, 1, &fail, s1);
            if (mode == 3) {
              dsts.clear(); srcs.clear(); sizes.clear();
              for (size_t t = 0; t < k; t++)
                for (size_t r = 0; r < rows; r++) { dsts.push_back(h2 + r * bs + t * S); srcs.push_back(d2 + (t * rows + r) * P + 32); sizes.push_back(S); }
              cudaMemcpyBatchAsync(dsts.data(), srcs.data(), sizes.data(), dsts.size(), &at, &idx0, 1, &fail, s2);
            }
          }
        }
        cudaStreamSynchronize(s1);
        cudaStreamSynchronize(s2);
        const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        const double gb = 4.0 * k * rows * F / sec / 1e9;
        if (gb > best) best = gb;
      }
      printf("{\"pattern\": \"getobject rows\", \"mode\": \"%s\", \"h2d_GBps\": %.1f}\n",
             mode == 0 ? "2-D h2d" : mode == 1 ? "batched rows h2d" : mode == 2 ? "2-D h2d + 2-D d2h" : mode == 3 ? "batched rows both ways" : mode == 4 ? "2-D h2d + contiguous d2h" : "contiguous both ways", best);
    }
  }
  return 0;
}
