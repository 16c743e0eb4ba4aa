// Microbenchmark: does a global store leave the line in L1 for a later load by the same SM?
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o l1_store_load l1_store_load.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(int* buf, long long* out) {
  // single thread; buf is large; use distinct lines per experiment
  volatile int sink = 0;
  int* a = buf;
  long long t0, t1;
  // (1) cold load (L2 or DRAM)
  t0 = clock64(); int v = a[0]; sink += v; t1 = clock64(); out[0] = t1 - t0;
  // (2) warm load same line (L1 hit)
  t0 = clock64(); v = a[1]; sink += v; t1 = clock64(); out[1] = t1 - t0;
  // (3) store to a line never loaded, then load it
  a[1024] = 7; 
  t0 = clock64(); v = a[1024]; sink += v; t1 = clock64(); out[2] = t1 - t0;
  // (3b) load again
  t0 = clock64(); v = a[1025]; sink += v; t1 = clock64(); out[3] = t1 - t0;
  // (4) load a line (L1 resident), store to it, load again
  v = a[2048]; sink += v;
  a[2048] = v + 1;
  t0 = clock64(); v = a[2048]; sink += v; t1 = clock64(); out[4] = t1 - t0;
  // (4b) different word of the same line after the store
  t0 = clock64(); v = a[2049]; sink += v; t1 = clock64(); out[5] = t1 - t0;
  // (5) store then load with several hundred cycles in between
  a[4096] = 3;
  for (int i = 0; i < 200; i++) sink += i;
  t0 = clock64(); v = a[4096]; sink += v; t1 = clock64(); out[6] = t1 - t0;
  // (6) shared memory round trip for reference
  __shared__ int s[32];
  s[0] = 5;
  t0 = clock64(); v = ((volatile int*)s)[0]; sink += v; t1 = clock64(); out[7] = t1 - t0;
  out[8] = sink;
}
int main() {
  int* buf; long long* out;
  cudaMalloc(&buf, 1 << 24); cudaMemset(buf, 0, 1 << 24);
  cudaMalloc(&out, 128);
  for (int rep = 0; rep < 3; rep++) {
    k<<<1, 1>>>(buf, out);
    long long h[9];
    cudaMemcpy(h, out, sizeof h, cudaMemcpyDeviceToHost);
    printf("cold %lld | warm(L1) %lld | store->load(new line) %lld, again %lld | load,store,load %lld, other word %lld | store..load later %lld | smem %lld\n",
           h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7]);
  }
  return 0;
}
