// Microbenchmark: the instruction caches one warp sees.  One warp of one CTA runs a loop whose body is S KB of
// straight-line integer instructions (64 instructions of 16 B = 1 KB per step), eight independent chains
// that depend on a kernel argument so that nothing folds.  Cycles per instruction against S, read with clock64 around
// the loop after one warm pass, step up where the body stops fitting a cache level; the step times 8 (instructions per
// 128-byte line) is the cost of a line fetched from the next level.  The second table runs two different bodies of S
// KB each, one after the other in every iteration: code of two event types that take turns.  Only a timing; it
// changes no state of the device.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o icache_footprint icache_footprint.cu
#include <cstdio>
#include <cuda_runtime.h>

// 8 instructions: each chain x_i <- x_i * x_{i+1} + c (IMAD with two register sources: no algebra folds a run of them)
#define STEP8(c)                                                                                                       \
  x0 = x0 * x1 + (c); x1 = x1 * x2 + (c); x2 = x2 * x3 + (c); x3 = x3 * x4 + (c);                                    \
  x4 = x4 * x5 + (c); x5 = x5 * x6 + (c); x6 = x6 * x7 + (c); x7 = x7 * x0 + (c);
#define STEP64(c) STEP8(c) STEP8(c) STEP8(c) STEP8(c) STEP8(c) STEP8(c) STEP8(c) STEP8(c)

#define STEP1K(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c) \
                  STEP64(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c) STEP64(c)

// KB KB of straight-line code: blocks of 16 KB and 1 KB expanded by recursion
template <int KB, int SALT>
__device__ __forceinline__ void body(unsigned& x0, unsigned& x1, unsigned& x2, unsigned& x3, unsigned& x4, unsigned& x5,
                                     unsigned& x6, unsigned& x7, unsigned c) {
  if constexpr (KB >= 16) {
    STEP1K(c + SALT)
    body<KB - 16, SALT>(x0, x1, x2, x3, x4, x5, x6, x7, c);
  } else if constexpr (KB >= 1) {
    STEP64(c + SALT)
    body<KB - 1, SALT>(x0, x1, x2, x3, x4, x5, x6, x7, c);
  }
}

// TWO == 0: one body of KB; TWO == 1: bodies A and B of KB each, alternately
template <int KB, int TWO>
__global__ void run(unsigned a, int iters, long long* cycles, unsigned* sink) {
  unsigned x0 = a, x1 = a + 1, x2 = a + 2, x3 = a + 3, x4 = a + 4, x5 = a + 5, x6 = a + 6, x7 = a + 7;
  long long t0 = 0;
  for (int it = -1; it < iters; it++) {  // iteration -1 is the warm pass
    if (it == 0) t0 = clock64();
    body<KB, 1>(x0, x1, x2, x3, x4, x5, x6, x7, a);
    if (TWO) body<KB, 3>(x0, x1, x2, x3, x4, x5, x6, x7, a);
  }
  const long long t1 = clock64();
  if (threadIdx.x == 0) cycles[0] = t1 - t0;
  sink[threadIdx.x] = x0 ^ x1 ^ x2 ^ x3 ^ x4 ^ x5 ^ x6 ^ x7;
}

#define CK(x)                                                                                                          \
  do {                                                                                                                 \
    cudaError_t e_ = (x);                                                                                              \
    if (e_ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); return 1; }      \
  } while (0)

template <int KB, int TWO>
int measure(long long* dCyc, unsigned* dSink) {
  const long long instr = 64ll * KB * (TWO ? 2 : 1);
  const int iters = (int)(4000000 / instr) < 8 ? 8 : (int)(4000000 / instr);
  double best = 1e30;
  for (int rep = 0; rep < 3; rep++) {  // the least of three launches
    run<KB, TWO><<<1, 32>>>(12345u + rep, iters, dCyc, dSink);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    long long cyc = 0;
    CK(cudaMemcpy(&cyc, dCyc, sizeof(cyc), cudaMemcpyDeviceToHost));
    const double cpi = (double)cyc / ((double)iters * instr);
    if (cpi < best) best = cpi;
  }
  printf("| %4d KB | %s | %6.1f KB | %8d | %6.3f |\n", KB * (TWO ? 2 : 1), TWO ? "2 x " : "1 x ",
         (double)KB, iters, best);
  return 0;
}

int main() {
  cudaDeviceProp p;
  CK(cudaGetDeviceProperties(&p, 0));
  int clk = 0;
  CK(cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0));
  printf("# instruction-cache footprint: %s, %d SMs, max SM clock %d MHz\n\n", p.name, p.multiProcessorCount, clk / 1000);
  long long* dCyc;
  unsigned* dSink;
  CK(cudaMalloc(&dCyc, sizeof(long long)));
  CK(cudaMalloc(&dSink, 32 * sizeof(unsigned)));
  printf("| code run per iteration | bodies | KB per body | iterations | cycles / instruction |\n|---|---|---|---|---|\n");
  int rc = 0;
  rc |= measure<4, 0>(dCyc, dSink);   rc |= measure<8, 0>(dCyc, dSink);   rc |= measure<16, 0>(dCyc, dSink);
  rc |= measure<24, 0>(dCyc, dSink);  rc |= measure<32, 0>(dCyc, dSink);  rc |= measure<48, 0>(dCyc, dSink);
  rc |= measure<64, 0>(dCyc, dSink);  rc |= measure<96, 0>(dCyc, dSink);  rc |= measure<128, 0>(dCyc, dSink);
  rc |= measure<160, 0>(dCyc, dSink); rc |= measure<192, 0>(dCyc, dSink); rc |= measure<256, 0>(dCyc, dSink);
  rc |= measure<384, 0>(dCyc, dSink); rc |= measure<512, 0>(dCyc, dSink);
  rc |= measure<8, 1>(dCyc, dSink);   rc |= measure<16, 1>(dCyc, dSink);  rc |= measure<32, 1>(dCyc, dSink);
  rc |= measure<48, 1>(dCyc, dSink);  rc |= measure<64, 1>(dCyc, dSink);  rc |= measure<96, 1>(dCyc, dSink);
  rc |= measure<128, 1>(dCyc, dSink); rc |= measure<256, 1>(dCyc, dSink);
  CK(cudaFree(dCyc));
  CK(cudaFree(dSink));
  return rc;
}
