// Round-2 prototype (compiled, NOT yet run on a GPU): is hash-partitioning worth it for GROUP BY tables
// that do not fit L2?  Same SUM+COUNT update as k_hash_agg on synthetic (key, value) rows, two ways:
//   A  direct     : one pass, open-addressed AoS table (32-byte slots) in HBM, slot = low bits of the hash
//   B  partitioned: histogram + scatter of the rows into 256 partitions by the TOP 8 bits of the hash,
//                   then the same update with slot = HIGH bits of the hash, so that the rows of one
//                   partition touch one contiguous 1/256th of the table (L2 resident while it is hot)
// Prints the time of every pass and checks that A and B produce the same table contents.
//   build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o profiles/bin/partition_agg profiles/src/partition_agg.cu
//   usage: partition_agg [rows=1e8] [groups=1e7]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}
constexpr unsigned long long EMPTY = ~0ull;
constexpr int P = 256;          // partitions
constexpr int CHUNK = 1 << 16;  // rows per partitioning work item (one CTA at a time)

__global__ void k_gen(unsigned long long* keys, double* vals, long long n, unsigned long long groups) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned long long r = mix64((unsigned long long)i * 0x9e3779b97f4a7c15ull + 12345);
    keys[i] = mix64(r % groups + 1);  // scrambled, never the EMPTY marker in practice
    vals[i] = double(r >> 11) * (1.0 / 9007199254740992.0);
  }
}

__global__ void k_init(unsigned long long* table, long long words) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += stride) table[i] = (i & 3) == 0 ? EMPTY : 0ull;
}

// slot layout: [key, sum(f64 bits), count, pad] = 32 bytes
template <bool HIGH_BITS>
__global__ void __launch_bounds__(256) k_agg(const unsigned long long* __restrict__ keys, const double* __restrict__ vals, long long n,
                                              unsigned long long* table, int log2cap, unsigned long long* failed) {
  const unsigned long long mask = (1ull << log2cap) - 1ull;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned long long key = __ldg(&keys[i]);
    const double v = __ldg(&vals[i]);
    const unsigned long long hsh = mix64(key);
    unsigned long long h = HIGH_BITS ? (hsh >> (64 - log2cap)) : (hsh & mask);
    bool done = false;
    for (int probe = 0; probe < 256 && !done; probe++) {
      unsigned long long cur = __ldcg(&table[h * 4]);
      if (cur == EMPTY) cur = atomicCAS(&table[h * 4], EMPTY, key), cur = cur == EMPTY ? key : cur;
      if (cur == key) {
        atomicAdd((double*)&table[h * 4 + 1], v);
        atomicAdd(&table[h * 4 + 2], 1ull);
        done = true;
      } else {
        h = (h + 1) & mask;
      }
    }
    if (!done) atomicAdd(failed, 1ull);
  }
}

// pass 1: per-chunk histogram of the partition ids (top 8 bits of the hash)
__global__ void __launch_bounds__(256) k_hist(const unsigned long long* __restrict__ keys, long long n, unsigned* hist /*[nchunks][P]*/) {
  __shared__ unsigned s_h[P];
  for (long long chunk = blockIdx.x; chunk * CHUNK < n; chunk += gridDim.x) {
    s_h[threadIdx.x] = 0;
    __syncthreads();
    const long long b = chunk * CHUNK, e = b + CHUNK < n ? b + CHUNK : n;
    for (long long i = b + threadIdx.x; i < e; i += 256) atomicAdd(&s_h[mix64(__ldg(&keys[i])) >> 56], 1u);
    __syncthreads();
    hist[chunk * P + threadIdx.x] = s_h[threadIdx.x];
    __syncthreads();
  }
}

// exclusive scan of hist in (partition-major, chunk-minor) order -> start offset of every (chunk, partition)
__global__ void __launch_bounds__(256) k_scan(const unsigned* hist, long long nchunks, long long* offs /*[nchunks][P]*/, long long* part_begin /*[P+1]*/) {
  __shared__ long long s_tot[P];
  const int p = threadIdx.x;  // one thread per partition: sequential over chunks (nchunks ~ 1.5e3)
  long long run = 0;
  for (long long c = 0; c < nchunks; c++) run += hist[c * P + p];
  s_tot[p] = run;
  __syncthreads();
  if (p == 0) {
    long long acc = 0;
    for (int q = 0; q < P; q++) { const long long t = s_tot[q]; s_tot[q] = acc; part_begin[q] = acc; acc += t; }
    part_begin[P] = acc;
  }
  __syncthreads();
  run = s_tot[p];
  for (long long c = 0; c < nchunks; c++) { offs[c * P + p] = run; run += hist[c * P + p]; }
}

// pass 2: scatter (key, value) to the partitioned arrays; cursors of the chunk live in shared memory
__global__ void __launch_bounds__(256) k_scatter(const unsigned long long* __restrict__ keys, const double* __restrict__ vals, long long n,
                                                  const long long* __restrict__ offs, unsigned long long* out_keys, double* out_vals) {
  __shared__ unsigned long long s_cur[P];
  for (long long chunk = blockIdx.x; chunk * CHUNK < n; chunk += gridDim.x) {
    s_cur[threadIdx.x] = (unsigned long long)offs[chunk * P + threadIdx.x];
    __syncthreads();
    const long long b = chunk * CHUNK, e = b + CHUNK < n ? b + CHUNK : n;
    for (long long i = b + threadIdx.x; i < e; i += 256) {
      const unsigned long long key = __ldg(&keys[i]);
      const unsigned long long at = atomicAdd(&s_cur[mix64(key) >> 56], 1ull);
      out_keys[at] = key;
      out_vals[at] = __ldg(&vals[i]);
    }
    __syncthreads();
  }
}

// order-independent digest of a table: sum over occupied slots of mix(key) * count, plus the value sums
__global__ void k_digest(const unsigned long long* table, long long slots, unsigned long long* dig /*[3]*/) {
  unsigned long long a = 0, c = 0;
  double s = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < slots; i += stride) {
    const unsigned long long k = table[i * 4];
    if (k == EMPTY) continue;
    a += mix64(k) * table[i * 4 + 2];
    c += 1;
    s += __longlong_as_double((long long)table[i * 4 + 1]);
  }
  atomicAdd(&dig[0], a);
  atomicAdd(&dig[1], c);
  atomicAdd((double*)&dig[2], s);
}

static float timed(cudaEvent_t e0, cudaEvent_t e1) { float ms; CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1)); return ms; }

int main(int argc, char** argv) {
  const long long n = argc > 1 ? (long long)atof(argv[1]) : 100000000ll;
  const unsigned long long groups = argc > 2 ? (unsigned long long)atof(argv[2]) : 10000000ull;
  cudaDeviceProp pr; CK(cudaGetDeviceProperties(&pr, 0));
  const int sms = pr.multiProcessorCount, grid = sms * 8;
  int log2cap = 1; while ((1ull << log2cap) < groups * 2) log2cap++;
  const long long slots = 1ll << log2cap, nchunks = (n + CHUNK - 1) / CHUNK;
  printf("rows=%lld groups=%llu table=%lld slots (%.0f MB) chunks=%lld\n", n, groups, slots, slots * 32 / 1e6, nchunks);
  unsigned long long *keys, *pkeys, *tabA, *tabB, *misc; double *vals, *pvals; unsigned* hist; long long *offs, *pbegin;
  CK(cudaMalloc(&keys, n * 8)); CK(cudaMalloc(&vals, n * 8)); CK(cudaMalloc(&pkeys, n * 8)); CK(cudaMalloc(&pvals, n * 8));
  CK(cudaMalloc(&tabA, slots * 32)); CK(cudaMalloc(&tabB, slots * 32)); CK(cudaMalloc(&misc, 64));
  CK(cudaMalloc(&hist, nchunks * P * 4)); CK(cudaMalloc(&offs, nchunks * P * 8)); CK(cudaMalloc(&pbegin, (P + 1) * 8));
  k_gen<<<grid, 256>>>(keys, vals, n, groups);
  cudaEvent_t e[8]; for (auto& x : e) CK(cudaEventCreate(&x));
  for (int rep = 0; rep < 3; rep++) {
    CK(cudaMemset(misc, 0, 64));
    k_init<<<grid, 256>>>(tabA, slots * 4);
    k_init<<<grid, 256>>>(tabB, slots * 4);
    CK(cudaEventRecord(e[0]));
    k_agg<false><<<grid, 256>>>(keys, vals, n, tabA, log2cap, misc);
    CK(cudaEventRecord(e[1]));
    k_hist<<<grid, 256>>>(keys, n, hist);
    CK(cudaEventRecord(e[2]));
    k_scan<<<1, 256>>>(hist, nchunks, offs, pbegin);
    CK(cudaEventRecord(e[3]));
    k_scatter<<<grid, 256>>>(keys, vals, n, offs, pkeys, pvals);
    CK(cudaEventRecord(e[4]));
    k_agg<true><<<grid, 256>>>(pkeys, pvals, n, tabB, log2cap, misc + 1);
    CK(cudaEventRecord(e[5]));
    k_digest<<<grid, 256>>>(tabA, slots, misc + 2);
    k_digest<<<grid, 256>>>(tabB, slots, misc + 5);
    CK(cudaGetLastError());
    unsigned long long h[8];
    CK(cudaMemcpy(h, misc, 64, cudaMemcpyDeviceToHost));
    const float a = timed(e[0], e[1]), hi = timed(e[1], e[2]), sc = timed(e[2], e[3]), st = timed(e[3], e[4]), b = timed(e[4], e[5]);
    double sa, sb; memcpy(&sa, &h[4], 8); memcpy(&sb, &h[7], 8);
    printf("rep %d  A direct %.3f ms | B hist %.3f + scan %.3f + scatter %.3f + agg %.3f = %.3f ms | groups A %llu B %llu, digests %s, sums %.6f / %.6f, failed %llu/%llu\n",
           rep, a, hi, sc, st, b, hi + sc + st + b, h[3], h[6], (h[2] == h[5] && h[3] == h[6]) ? "equal" : "DIFFERENT", sa, sb, h[0], h[1]);
  }
  return 0;
}
