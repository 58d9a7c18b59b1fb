// Measures the machine's rate for scattered (one distinct address per lane) global-memory operations:
// the ceiling for an open-addressed hash aggregate whose table lives in L2 / HBM.  No input stream is
// read (addresses come from a hash of the row number), so the result is the pure LSU / L2-atomic rate.
//   build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o profiles/bin/scatter_peak profiles/src/scatter_peak.cu
//   usage: scatter_peak [rows=1e8]
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}

// MODE 0: 1 RED.f64   1: RED.f64 + RED.u64   2: LDG(key) + RED.f64 + RED.u64   3: LDG only
template <int MODE>
__global__ void __launch_bounds__(256) k_scatter(unsigned long long* keys, double* sums, unsigned long long* counts, long long n,
                                                  unsigned long long mask, unsigned long long* sink) {
  unsigned long long acc = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned long long h = mix64((unsigned long long)i) & mask;
    if (MODE >= 2) acc += __ldcg(&keys[h]);
    if (MODE <= 2) atomicAdd(&sums[h], 1.0);
    if (MODE == 1 || MODE == 2) atomicAdd(&counts[h], 1ull);
  }
  if (acc == 0x1234567ull) *sink = acc;
}

template <int MODE>
static void run(const char* what, int ops, long long n, long long slots, unsigned long long* keys, double* sums, unsigned long long* counts,
                unsigned long long* sink, int sms) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int it = 0; it < 4; it++) {
    cudaEventRecord(e0);
    k_scatter<MODE><<<sms * 8, 256>>>(keys, sums, counts, n, (unsigned long long)slots - 1, sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (it && ms < best) best = ms;
  }
  printf("slots=%-10lld %-28s %8.3f ms  %7.1f Gops/s  %6.3f cyc/lane/SM @1.9GHz\n", slots, what, best, ops * double(n) / best / 1e6,
         best * 1e-3 * 1.9e9 * sms / (ops * double(n)));
}

int main(int argc, char** argv) {
  const long long n = argc > 1 ? (long long)atof(argv[1]) : 100000000ll;
  cudaDeviceProp pr; cudaGetDeviceProperties(&pr, 0);
  const int sms = pr.multiProcessorCount;
  for (long long slots : {1ll << 18, 1ll << 21, 1ll << 25}) {
    unsigned long long *keys, *counts, *sink; double* sums;
    cudaMalloc(&keys, slots * 8); cudaMalloc(&sums, slots * 8); cudaMalloc(&counts, slots * 8); cudaMalloc(&sink, 8);
    cudaMemset(keys, 0, slots * 8); cudaMemset(sums, 0, slots * 8); cudaMemset(counts, 0, slots * 8);
    run<0>("1x RED.f64", 1, n, slots, keys, sums, counts, sink, sms);
    run<1>("RED.f64 + RED.u64", 2, n, slots, keys, sums, counts, sink, sms);
    run<2>("LDG + RED.f64 + RED.u64", 3, n, slots, keys, sums, counts, sink, sms);
    run<3>("1x LDG", 1, n, slots, keys, sums, counts, sink, sms);
    cudaFree(keys); cudaFree(sums); cudaFree(counts); cudaFree(sink);
  }
  return 0;
}
