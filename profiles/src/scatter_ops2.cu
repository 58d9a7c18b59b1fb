// Round-2 microbenchmark: can the GROUP BY update use fewer / cheaper scattered operations per row than
// "key LDG + one RED per aggregate"?  Every variant touches one pseudo-random 32-byte slot per row of an
// L2-resident table (no input stream), like profiles/src/scatter_peak.cu.
//   M0  LDG + RED.f64 + RED.u64, SoA arrays (the round-1 pattern)
//   M1  LDG + RED.f64 + RED.u64, AoS 32-byte slot (all three in one sector)
//   M2  ATOMG.ADD.u64 (returning) + RED.f64, AoS      (probe and COUNT folded into one returning atomic)
//   M3  ATOMG.ADD.u64 only
//   M4  LDG + one 16-byte TMA reduction  cp.reduce.async.bulk .add.f64 {v, 1.0}  (SUM and COUNT in one op)
//   M5  the 16-byte TMA reduction only
//   M6  RED.v2.f32 only (vector reduction, for the rate of a 2-element RED)
//   M7  LDG.128 only (probe of a 16-byte {key, aux})
//   M8  2 x LDG.128 of a 32-byte line {key, min, max, -} + RED.f64 on a separate array (the hybrid layout's row)
//   M9  2 x LDG.128 only         M10  RED.u32 only          M11  LDG + RED.f64 + RED.u32 (32-bit COUNT)
//   build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o profiles/bin/scatter_ops2 profiles/src/scatter_ops2.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

template <int MODE>
__global__ void __launch_bounds__(256) k_ops(unsigned long long* tab, unsigned long long* soa1, unsigned long long* soa2, long long n,
                                              unsigned long long mask, unsigned long long* sink) {
  __shared__ __align__(16) double s_src[2][256][2];
  unsigned long long acc = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  int buf = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned long long h = mix64((unsigned long long)i) & mask;
    if (MODE == 0) {
      acc += __ldcg(&tab[h]);
      atomicAdd((double*)&soa1[h], 1.0);
      atomicAdd(&soa2[h], 1ull);
    } else if (MODE == 1) {
      acc += __ldcg(&tab[h * 4]);
      atomicAdd((double*)&tab[h * 4 + 1], 1.0);
      atomicAdd(&tab[h * 4 + 2], 1ull);
    } else if (MODE == 2) {
      acc += atomicAdd(&tab[h * 4], 1ull);
      atomicAdd((double*)&tab[h * 4 + 1], 1.0);
    } else if (MODE == 3) {
      acc += atomicAdd(&tab[h * 4], 1ull);
    } else if (MODE == 4 || MODE == 5) {
      if (MODE == 4) acc += __ldcg(&tab[h * 4]);
      // the source cell of the previous-but-one iteration must have been read by the TMA engine
      asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      s_src[buf][threadIdx.x][0] = 1.0;
      s_src[buf][threadIdx.x][1] = 1.0;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f64 [%0], [%1], 16;" ::"l"(&tab[h * 4 + 2]),
                   "r"(smem_u32(&s_src[buf][threadIdx.x][0]))
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      buf ^= 1;
    } else if (MODE == 6) {
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(&tab[h * 4 + 2]), "f"(1.0f), "f"(1.0f) : "memory");
    } else if (MODE == 7) {
      const ulonglong2 v = __ldcg((const ulonglong2*)&tab[h * 4]);
      acc += v.x + v.y;
    } else if (MODE == 8 || MODE == 9) {
      unsigned long long a, b, c, d;
      asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(&tab[h * 4]));
      asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(c), "=l"(d) : "l"(&tab[h * 4 + 2]));
      acc += a + b + c + d;
      if (MODE == 8) atomicAdd((double*)&soa1[h], 1.0);
    } else if (MODE == 10) {
      atomicAdd((unsigned*)&soa2[h], 1u);
    } else if (MODE == 11) {
      acc += __ldcg(&tab[h]);
      atomicAdd((double*)&soa1[h], 1.0);
      atomicAdd((unsigned*)&soa2[h], 1u);
    }
  }
  if (MODE == 4 || MODE == 5) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  if (acc == 0x1234567ull) *sink = acc;
}

template <int MODE>
static void run(const char* what, int ops, long long n, long long slots, unsigned long long* tab, unsigned long long* s1, unsigned long long* s2,
                unsigned long long* sink, int sms) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int it = 0; it < 4; it++) {
    cudaEventRecord(e0);
    k_ops<MODE><<<sms * 8, 256>>>(tab, s1, s2, n, (unsigned long long)slots - 1, sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (it && ms < best) best = ms;
  }
  cudaError_t e = cudaGetLastError();
  printf("slots=%-9lld %-44s %8.3f ms  %7.1f Gops/s  %6.3f cyc/row/SM @1.9GHz %s\n", slots, what, best, ops * double(n) / best / 1e6,
         best * 1e-3 * 1.9e9 * sms / double(n), e == cudaSuccess ? "" : cudaGetErrorString(e));
}

int main(int argc, char** argv) {
  const long long n = argc > 1 ? (long long)atof(argv[1]) : 100000000ll;
  cudaDeviceProp pr; cudaGetDeviceProperties(&pr, 0);
  const int sms = pr.multiProcessorCount;
  for (long long slots : {1ll << 18, 1ll << 21}) {
    unsigned long long *tab, *s1, *s2, *sink;
    cudaMalloc(&tab, slots * 32); cudaMalloc(&s1, slots * 8); cudaMalloc(&s2, slots * 8); cudaMalloc(&sink, 8);
    cudaMemset(tab, 0, slots * 32); cudaMemset(s1, 0, slots * 8); cudaMemset(s2, 0, slots * 8);
    run<0>("M0 LDG + RED.f64 + RED.u64 (SoA)", 3, n, slots, tab, s1, s2, sink, sms);
    run<1>("M1 LDG + RED.f64 + RED.u64 (AoS, one sector)", 3, n, slots, tab, s1, s2, sink, sms);
    run<2>("M2 ATOMG.ADD(ret) + RED.f64 (AoS)", 2, n, slots, tab, s1, s2, sink, sms);
    run<3>("M3 ATOMG.ADD(ret)", 1, n, slots, tab, s1, s2, sink, sms);
    run<4>("M4 LDG + TMA reduce 16B add.f64", 2, n, slots, tab, s1, s2, sink, sms);
    run<5>("M5 TMA reduce 16B add.f64", 1, n, slots, tab, s1, s2, sink, sms);
    run<6>("M6 RED.v2.f32", 1, n, slots, tab, s1, s2, sink, sms);
    run<7>("M7 LDG.128", 1, n, slots, tab, s1, s2, sink, sms);
    run<8>("M8 2xLDG.128 (AoS line) + RED.f64 (array)", 2, n, slots, tab, s1, s2, sink, sms);
    run<9>("M9 2xLDG.128", 1, n, slots, tab, s1, s2, sink, sms);
    run<10>("M10 RED.u32", 1, n, slots, tab, s1, s2, sink, sms);
    run<11>("M11 LDG + RED.f64 + RED.u32 (SoA)", 3, n, slots, tab, s1, s2, sink, sms);
    cudaFree(tab); cudaFree(s1); cudaFree(s2); cudaFree(sink);
  }
  return 0;
}
