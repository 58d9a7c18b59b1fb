// join.cu — inner equi-join on integer and Utf8 keys: a hash table built over the build (right) input, a two-pass probe of each
// probe (left) batch, and a gather of the output columns by row index.  The reference has no join (its ROADMAP.md
// lists "JOIN support (hash join ...)" for 0.7.0); include/dfgpu.h documents the semantics.
//
// Build (dfgpu_join_build), for n build rows:
//   k_join_build    one thread per row packs the key, claims the key's slot (atomicCAS on the key word, the key equal
//                   to EMPTY_KEY takes slot cap) and records the row's slot; each warp counts its rows per slot with one
//                   atomic per distinct slot
//   scan            the counts of the cap + 1 slots become each slot's start (scan_exclusive, scan.cuh)
//   k_join_scatter  every row writes its row number into its slot's range: the build rows of one key are contiguous
// Probe (dfgpu_join_probe), for n probe rows:
//   k_join_count    per row: the number of build rows with its key (0 for a null key or a miss) and their start
//   scan            64-bit offsets of each row's output range; the total is the output row count
//   k_join_emit     per OUTPUT position: the probe row owning it (a search of the offsets restricted to the rows of the
//                   CTA's tile) and its build row.  The work is spread by output, so a probe row with millions of
//                   matches is written by as many threads as rows with one match each.
//   gathers         gather_column (gather.cuh)
//
// Semi / anti join (dfgpu_join_semi), on the same build:
//   k_join_mark     per probe row: one pass bit (match for semi, no match for anti), written as 32-bit words with
//                   __ballot_sync, and each tile's pass count (k_join_utf8_mark for a key with Utf8 parts)
//   scan            the tile counts become each tile's output offset; the total is the output row count
//   k_join_select   per tile: the passing row numbers in row order (select_rows, gather.cuh)
//   gathers         as above, for the probe columns only
//
// A key with Utf8 parts takes its own build and count kernels; the scan, k_join_scatter, k_join_emit and the gathers
// are shared.  Each row has a 64-bit tag (the packed integer parts and the hash of each Utf8 part), and a slot holds
// one distinct KEY, not one tag: its tag, its integer word and a representative build row, the smallest with the key.
//   k_join_utf8_place   one round over the rows not yet placed: a row stops at the first slot of this round with its
//                       tag, or claims an empty one (atomicCAS on the tag), and atomicMin's its row into the slot's
//                       representative
//   k_join_utf8_verify  after the round: a row whose key equals its slot's representative is placed and counted (one
//                       atomic per warp and slot); any other row goes to the next round, which starts past the slots
//                       sealed here.  With 64-bit tags there is one round unless two keys collide.
//   k_join_utf8_count   the probe: at a slot with the row's tag, the key is confirmed against the representative
//                       (integer word, then each Utf8 part's length and bytes) before the slot counts as a match
#include <memory>

#include "gather.cuh"
#include "hash_table.cuh"
#include "scan.cuh"
#include "utf8_words.cuh"

namespace dfgpu {

constexpr int kMaxJoinKeys = 4;
constexpr long long JN_MIN_CAP = 1024;  // the build table never grows: no floor beyond a small minimum
constexpr int JN_THREADS = SEL_THREADS;
constexpr int EMIT_TILE = 2048;  // output positions per CTA tile of k_join_emit

// The key columns of one input: each part is read as its raw integer, sign- or zero-extended to 64 bits, masked to its
// width and shifted into place (the aggregate's packing: the last key in the low bits, a single key keeps its 64-bit
// value).  A row with a null part has no key.
struct JoinKeys {
  const void* vals[kMaxJoinKeys];
  const unsigned char* valid[kMaxJoinKeys];  // null: no nulls
  unsigned long long mask[kMaxJoinKeys];
  int width[kMaxJoinKeys];
  int is_signed[kMaxJoinKeys];
  int shift[kMaxJoinKeys];
  int nkeys;
};

__device__ __forceinline__ bool join_key(const JoinKeys& k, long long r, unsigned long long* out) {
  unsigned long long key = 0;
#pragma unroll
  for (int i = 0; i < kMaxJoinKeys; i++) {
    if (i >= k.nkeys) break;
    if (k.valid[i] && !((k.valid[i][r >> 3] >> (r & 7)) & 1)) return false;
    unsigned long long v;
    switch (k.width[i]) {
      case 1: v = k.is_signed[i] ? (unsigned long long)(long long)((const signed char*)k.vals[i])[r] : (unsigned long long)((const unsigned char*)k.vals[i])[r]; break;
      case 2: v = k.is_signed[i] ? (unsigned long long)(long long)((const short*)k.vals[i])[r] : (unsigned long long)((const unsigned short*)k.vals[i])[r]; break;
      case 4: v = k.is_signed[i] ? (unsigned long long)(long long)((const int*)k.vals[i])[r] : (unsigned long long)((const unsigned*)k.vals[i])[r]; break;
      default: v = ((const unsigned long long*)k.vals[i])[r]; break;
    }
    key |= (v & k.mask[i]) << k.shift[i];
  }
  *out = key;
  return true;
}

// ---- build -------------------------------------------------------------------------------------------------------
// Both build kernels walk the rows a warp at a time (all lanes together, so that the warp can combine its rows) and
// aggregate the slot counters per warp: the lanes whose rows share a slot (__match_any_sync) make ONE atomic, so a key
// repeated millions of times costs one atomic per 32 rows instead of one per row.
constexpr unsigned long long NO_SLOT = ~0ull;

__global__ void __launch_bounds__(JN_THREADS) k_join_build(JoinKeys k, long long n, ProbeRule t, unsigned long long* __restrict__ keys,
                                                          unsigned* __restrict__ counts, unsigned long long* __restrict__ row_slot) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
    const long long r = base + lane;
    unsigned long long key, h = NO_SLOT;
    if (r < n && join_key(k, r, &key)) {
      h = (unsigned long long)t.cap;  // the key that equals the empty marker
      if (key != EMPTY_KEY) {
        h = t.home(mix64(key));
        for (;;) {  // at most n distinct keys in at least 2n slots: an empty slot is always found
          unsigned long long cur = __ldcg(keys + h);
          if (cur == EMPTY_KEY) cur = atomicCAS(keys + h, EMPTY_KEY, key);
          if (cur == EMPTY_KEY || cur == key) break;
          h = t.next(h);
        }
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, h);
    if (h != NO_SLOT && lane == __ffs(peers) - 1) atomicAdd(counts + h, (unsigned)__popc(peers));
    if (r < n) row_slot[r] = h;
  }
}

// counts[s] still holds the slot's row count: the rows of a slot take its places from the end of its range, a warp's
// rows of one slot with one atomic
__global__ void __launch_bounds__(JN_THREADS) k_join_scatter(const unsigned long long* __restrict__ row_slot, long long n,
                                                            const unsigned long long* __restrict__ start, unsigned* __restrict__ counts,
                                                            unsigned* __restrict__ rows) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
    const long long r = base + lane;
    const unsigned long long s = r < n ? row_slot[r] : NO_SLOT;
    const unsigned peers = __match_any_sync(0xffffffffu, s);
    const int leader = __ffs(peers) - 1;
    unsigned end = 0;
    if (s != NO_SLOT && lane == leader) end = atomicSub(counts + s, (unsigned)__popc(peers));
    end = __shfl_sync(0xffffffffu, end, leader);
    if (s == NO_SLOT) continue;
    const unsigned k = end - (unsigned)__popc(peers) + (unsigned)__popc(peers & ((1u << lane) - 1u));
    rows[start[s] + k] = (unsigned)r;
  }
}

// ---- Utf8 keys ---------------------------------------------------------------------------------------------------
// The Utf8 parts of a key, in key order.  The integer parts stay in a JoinKeys, packed as above (with no integer part
// the word is 0).  Byte buffers are 16-byte aligned and allocated in whole 16-byte words, so that load16 may read the
// aligned word that holds a string's last byte.
struct Utf8Keys {
  const int* off[kMaxJoinKeys];
  const unsigned char* bytes[kMaxJoinKeys];
  const unsigned char* valid[kMaxJoinKeys];  // null: no nulls
  int n;
};

// A row's integer word and tag: mix64 over the word and each Utf8 part's utf8_hash_bytes, cut to the tag width (its
// top bits, which home() reads) and never EMPTY_KEY.  False for a row with a null part.
__device__ __forceinline__ bool utf8_tag(const JoinKeys& k, const Utf8Keys& u, unsigned long long tag_mask, long long r, unsigned long long* word,
                                         unsigned long long* tag) {
  if (!join_key(k, r, word)) return false;
  unsigned long long h = mix64(*word);
  for (int i = 0; i < kMaxJoinKeys; i++) {
    if (i >= u.n) break;
    if (u.valid[i] && !((u.valid[i][r >> 3] >> (r & 7)) & 1)) return false;
    h = mix64(h ^ utf8_hash_bytes(u.bytes[i], __ldg(u.off[i] + r), __ldg(u.off[i] + r + 1)));
  }
  h &= tag_mask;
  *tag = h == EMPTY_KEY ? EMPTY_KEY - 1ull : h;
  return true;
}

// the low k bytes of a 32-bit word (k <= 0: none)
__device__ __forceinline__ unsigned low_bytes(int k) { return k >= 4 ? ~0u : (k <= 0 ? 0u : (1u << (8 * k)) - 1u); }

// bytes [a0, a0 + len) of a equal bytes [b0, b0 + len) of b, compared one 16-byte word of each side per step
__device__ __forceinline__ bool bytes_equal(const unsigned char* a, long long a0, const unsigned char* b, long long b0, int len) {
  for (int i = 0; i < len; i += 16) {
    const uint4 x = load16(a, a0 + i, len - i), y = load16(b, b0 + i, len - i);
    const int k = len - i;
    if (((x.x ^ y.x) & low_bytes(k)) | ((x.y ^ y.y) & low_bytes(k - 4)) | ((x.z ^ y.z) & low_bytes(k - 8)) | ((x.w ^ y.w) & low_bytes(k - 12)))
      return false;
  }
  return true;
}

// every Utf8 part of row ra of a equals that of row rb of b: the lengths, then the bytes
__device__ __forceinline__ bool utf8_parts_equal(const Utf8Keys& a, long long ra, const Utf8Keys& b, long long rb) {
  for (int i = 0; i < kMaxJoinKeys; i++) {
    if (i >= a.n) break;
    const int a0 = __ldg(a.off[i] + ra), la = __ldg(a.off[i] + ra + 1) - a0;
    const int b0 = __ldg(b.off[i] + rb), lb = __ldg(b.off[i] + rb + 1) - b0;
    if (la != lb || !bytes_equal(a.bytes[i], a0, b.bytes[i], b0, la)) return false;
  }
  return true;
}

// One build round over the rows of `list` (null: rows 0..n).  A slot sealed in an earlier round is passed over: every
// row of one key stops at the same slot in a round (the first of that round with its tag, or the empty one they all
// race for), so a key still unplaced has no sealed slot.  The row's slot goes to row_slot, NO_SLOT for a null key.
__global__ void __launch_bounds__(JN_THREADS) k_join_utf8_place(JoinKeys k, Utf8Keys u, unsigned long long tag_mask, const unsigned* __restrict__ list,
                                                               long long n, ProbeRule t, unsigned long long* __restrict__ tags,
                                                               const unsigned char* __restrict__ sealed, unsigned* __restrict__ rep,
                                                               unsigned long long* __restrict__ row_slot) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = list ? (long long)list[i] : i;
    unsigned long long word, tag, h = NO_SLOT;
    if (utf8_tag(k, u, tag_mask, r, &word, &tag)) {
      h = t.home(tag);
      for (;;) {  // at most n distinct keys in at least 2n slots, one key per slot: an empty slot is always found
        unsigned long long cur = __ldcg(tags + h);
        if (cur == EMPTY_KEY) cur = atomicCAS(tags + h, EMPTY_KEY, tag);
        if ((cur == EMPTY_KEY || cur == tag) && !sealed[h]) break;
        h = t.next(h);
      }
      atomicMin(rep + h, (unsigned)r);
    }
    row_slot[r] = h;
  }
}

// After a round, when every representative is final: a row equal to its slot's representative is placed and counted,
// a warp's rows of one slot with one atomic; any other row is appended to `next`.  The representative seals its slot
// and records the slot's integer word.
__global__ void __launch_bounds__(JN_THREADS) k_join_utf8_verify(JoinKeys k, Utf8Keys u, const unsigned* __restrict__ list, long long n,
                                                                const unsigned* __restrict__ rep, unsigned char* __restrict__ sealed,
                                                                unsigned long long* __restrict__ words, const unsigned long long* __restrict__ row_slot,
                                                                unsigned* __restrict__ counts, unsigned* __restrict__ next,
                                                                unsigned long long* __restrict__ n_next) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
    const long long i = base + lane;
    long long r = 0;
    unsigned long long h = NO_SLOT;
    bool retry = false;
    if (i < n) {
      r = list ? (long long)list[i] : i;
      h = row_slot[r];
      if (h != NO_SLOT) {
        const unsigned q = rep[h];
        unsigned long long w, wq;
        join_key(k, r, &w);
        if (q == (unsigned)r) {
          sealed[h] = 1;
          words[h] = w;
        } else if (!join_key(k, q, &wq) || w != wq || !utf8_parts_equal(u, r, u, q)) {
          retry = true;
          h = NO_SLOT;
        }
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, h);
    if (h != NO_SLOT && lane == __ffs(peers) - 1) atomicAdd(counts + h, (unsigned)__popc(peers));
    const unsigned again = __ballot_sync(0xffffffffu, retry);
    if (again) {
      const int leader = __ffs(again) - 1;
      unsigned long long at = 0;
      if (lane == leader) at = atomicAdd(n_next, (unsigned long long)__popc(again));
      at = __shfl_sync(0xffffffffu, at, leader);
      if (retry) next[at + (unsigned)__popc(again & ((1u << lane) - 1u))] = (unsigned)r;
    }
  }
}

// ---- probe -----------------------------------------------------------------------------------------------------------
// The slot of a packed integer key: slot cap for the key equal to EMPTY_KEY, -1 when the key is not in the table.
__device__ __forceinline__ long long find_slot(const ProbeRule& t, const unsigned long long* __restrict__ keys, unsigned long long key) {
  long long s = -1;
  if (key == EMPTY_KEY) {
    s = t.cap;
  } else {
    unsigned long long h = t.home(mix64(key));
    for (long long probes = 0; probes < t.cap; probes++) {
      const unsigned long long cur = keys[h];
      if (cur == key) { s = (long long)h; break; }
      if (cur == EMPTY_KEY) break;
      h = t.next(h);
    }
  }
  return s;
}

__global__ void __launch_bounds__(JN_THREADS) k_join_count(JoinKeys k, long long n, ProbeRule t, const unsigned long long* __restrict__ keys,
                                                          const unsigned long long* __restrict__ start, unsigned* __restrict__ cnt,
                                                          unsigned* __restrict__ bpos) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    unsigned long long key;
    unsigned c = 0, b = 0;
    if (join_key(k, r, &key)) {
      const long long s = find_slot(t, keys, key);
      if (s >= 0) {
        const unsigned long long s0 = start[s];
        c = (unsigned)(start[s + 1] - s0);
        b = (unsigned)s0;
      }
    }
    cnt[r] = c;
    bpos[r] = b;
  }
}

// The slot of a key with Utf8 parts (probe row r of `u`, its integer word and tag) in *slot: at a slot with the row's
// tag, the key is confirmed against the slot's integer word and its representative's Utf8 parts (`b`: the join's copy of
// the build key columns) before it counts as a match; two keys with one tag never match.  False when the key is not in
// the table.
__device__ __forceinline__ bool find_utf8_slot(const ProbeRule& t, const unsigned long long* __restrict__ tags,
                                               const unsigned long long* __restrict__ words, const unsigned* __restrict__ rep,
                                               const Utf8Keys& u, long long r, const Utf8Keys& b, unsigned long long word,
                                               unsigned long long tag, unsigned long long* slot) {
  unsigned long long h = t.home(tag);
  for (long long probes = 0; probes < t.cap; probes++) {
    const unsigned long long cur = tags[h];
    if (cur == EMPTY_KEY) break;
    if (cur == tag && words[h] == word && utf8_parts_equal(u, r, b, rep[h])) {
      *slot = h;
      return true;
    }
    h = t.next(h);
  }
  return false;
}

__global__ void __launch_bounds__(JN_THREADS) k_join_utf8_count(JoinKeys k, Utf8Keys u, unsigned long long tag_mask, long long n, ProbeRule t,
                                                               const unsigned long long* __restrict__ tags, const unsigned long long* __restrict__ words,
                                                               const unsigned* __restrict__ rep, Utf8Keys b, const unsigned long long* __restrict__ start,
                                                               unsigned* __restrict__ cnt, unsigned* __restrict__ bpos) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    unsigned long long word, tag, h;
    unsigned c = 0, bp = 0;
    if (utf8_tag(k, u, tag_mask, r, &word, &tag) && find_utf8_slot(t, tags, words, rep, u, r, b, word, tag, &h)) {
      const unsigned long long s0 = start[h];
      c = (unsigned)(start[h + 1] - s0);
      bp = (unsigned)s0;
    }
    cnt[r] = c;
    bpos[r] = bp;
  }
}

// ---- semi / anti join: one pass bit per probe row, then an order-preserving compaction ---------------------------------
// A probe row passes when it has a match (semi) or has none (anti); a row with a null key part passes when `null_pass`
// is set (anti; null-aware anti only over an empty build side).  The rows are cut into tiles of MARK_TILE: k_join_mark
// writes the tile's MARK_TILE / 32 mask words (warp w of the CTA writes words i * 8 + w, one __ballot_sync each) and
// its pass count; the counts are scanned into tile offsets; k_join_select writes the passing row numbers of each tile,
// in row order, at its offset (mark_tiles and select_rows: gather.cuh).
__global__ void __launch_bounds__(JN_THREADS) k_join_mark(JoinKeys k, long long n, ProbeRule t, const unsigned long long* __restrict__ keys,
                                                         const unsigned long long* __restrict__ start, int anti, int null_pass,
                                                         unsigned* __restrict__ mask, unsigned* __restrict__ tile_cnt) {
  mark_tiles(n, mask, tile_cnt, [&](long long r) {
    unsigned long long key;
    if (!join_key(k, r, &key)) return null_pass != 0;
    const long long s = find_slot(t, keys, key);
    const bool hit = s >= 0 && (s < t.cap || start[s + 1] != start[s]);  // slot cap holds rows only if the key occurs
    return hit != (anti != 0);
  });
}

__global__ void __launch_bounds__(JN_THREADS) k_join_utf8_mark(JoinKeys k, Utf8Keys u, unsigned long long tag_mask, long long n, ProbeRule t,
                                                              const unsigned long long* __restrict__ tags, const unsigned long long* __restrict__ words,
                                                              const unsigned* __restrict__ rep, Utf8Keys b, int anti, int null_pass,
                                                              unsigned* __restrict__ mask, unsigned* __restrict__ tile_cnt) {
  mark_tiles(n, mask, tile_cnt, [&](long long r) {
    unsigned long long word, tag, h;
    if (!utf8_tag(k, u, tag_mask, r, &word, &tag)) return null_pass != 0;
    return find_utf8_slot(t, tags, words, rep, u, r, b, word, tag, &h) != (anti != 0);
  });
}

// the last row p in [lo, hi] with off[p] <= o: the probe row whose output range holds position o
__device__ __forceinline__ long long owner_row(const unsigned long long* __restrict__ off, unsigned long long o, long long lo, long long hi) {
  while (lo < hi) {
    const long long mid = lo + (hi - lo + 1) / 2;
    if (off[mid] <= o) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(JN_THREADS) k_join_emit(const unsigned long long* __restrict__ off, long long n, const unsigned* __restrict__ bpos,
                                                         const unsigned* __restrict__ rows, unsigned long long total,
                                                         unsigned* __restrict__ out_probe, unsigned* __restrict__ out_build) {
  __shared__ long long s_range[2];
  for (unsigned long long o0 = (unsigned long long)blockIdx.x * EMIT_TILE; o0 < total; o0 += (unsigned long long)gridDim.x * EMIT_TILE) {
    const unsigned long long o1 = min(total, o0 + EMIT_TILE) - 1ull;
    if (threadIdx.x == 0) s_range[0] = owner_row(off, o0, 0, n - 1);
    if (threadIdx.x == 32) s_range[1] = owner_row(off, o1, 0, n - 1);
    __syncthreads();
    const long long lo = s_range[0], hi = s_range[1];
    for (unsigned long long o = o0 + threadIdx.x; o <= o1; o += JN_THREADS) {
      const long long p = owner_row(off, o, lo, hi);
      out_probe[o] = (unsigned)p;
      out_build[o] = rows[bpos[p] + (unsigned)(o - off[p])];
    }
    __syncthreads();
  }
}

// ---- host side ---------------------------------------------------------------------------------------------------------
namespace {

// The key columns of one batch.  A key program that is a plain column is read in place; any other program is
// evaluated by the projection operator (no predicate), so its values are exactly the expression VM's.  The integer
// parts go to `k`, the Utf8 parts to `u` (with their columns in `ucols`), each in key order.
struct KeyColumns {
  JoinKeys k{};
  Utf8Keys u{};
  const DevColumn* ucols[kMaxJoinKeys] = {};
  int dtypes[kMaxJoinKeys] = {};
  std::vector<std::unique_ptr<dfgpu_result, int (*)(dfgpu_result*)>> evaluated;
};

void key_columns(dfgpu_ctx* ctx, const dfgpu_batch* b, const dfgpu_insn* const* keys, const int* key_len, int nkeys, KeyColumns* out) {
  if (nkeys < 1 || !keys || !key_len) fail(DFGPU_ERR_GENERAL, "JOIN needs at least one key");
  if (nkeys > kMaxJoinKeys) fail(DFGPU_ERR_NOT_IMPLEMENTED, "JOIN on more than " + std::to_string(kMaxJoinKeys) + " keys");
  std::vector<int32_t> col_dtypes;
  for (const DevColumn& c : b->cols) col_dtypes.push_back(c.dtype);
  int bits = 0;
  std::string widths;
  for (int i = 0; i < nkeys; i++) {
    int32_t dt = 0;
    const int rc = dfgpu_check_program(col_dtypes.empty() ? nullptr : col_dtypes.data(), int(col_dtypes.size()), keys[i], key_len[i], &dt);
    if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
    if (!is_int(dt) && dt != DFGPU_UTF8)
      fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("JOIN keys of type ") + dtype_name(dt) + " are not supported (integer keys only)");
    out->dtypes[i] = dt;
    if (dt == DFGPU_UTF8) continue;  // Utf8 parts are hashed, not packed: they do not count toward the 64 bits
    bits += dtype_width(dt) * 8;
    widths += (widths.empty() ? "" : " + ") + std::string(dtype_name(dt));
  }
  if (bits > 64) fail(DFGPU_ERR_NOT_IMPLEMENTED, "JOIN keys wider than 64 bits (" + widths + ")");
  // the integer parts, in key order; with no Utf8 part they are the key
  std::vector<int> ints;
  for (int i = 0; i < nkeys; i++)
    if (out->dtypes[i] != DFGPU_UTF8) ints.push_back(i);
  const int nints = int(ints.size());
  JoinKeys& k = out->k;
  k.nkeys = nints;
  int shift = 0;
  for (int i = nints - 1; i >= 0; i--) {
    const int w = dtype_width(out->dtypes[ints[size_t(i)]]);
    k.width[i] = w;
    k.is_signed[i] = is_signed_int(out->dtypes[ints[size_t(i)]]) ? 1 : 0;
    k.shift[i] = shift;
    k.mask[i] = w == 8 ? ~0ull : ((1ull << (8 * w)) - 1ull);
    shift += 8 * w;
  }
  if (nints == 1) k.mask[0] = ~0ull;  // a single key keeps its sign- or zero-extended 64-bit value
  for (int i = 0; i < nkeys; i++) {
    const DevColumn* c = nullptr;
    if (key_len[i] == 1 && keys[i][0].op == DFGPU_OP_COL) {
      c = &b->cols[size_t(keys[i][0].col)];
    } else {
      dfgpu_result* r = nullptr;
      const int rc = dfgpu_filter_project(ctx, b, nullptr, 0, &keys[i], &key_len[i], 1, &r);
      if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
      out->evaluated.emplace_back(r, dfgpu_result_free);
      c = &r->cols[0];
    }
    const unsigned char* valid = c->null_count > 0 ? c->validity : nullptr;
    if (out->dtypes[i] == DFGPU_UTF8) {
      // every Utf8 buffer of the engine is allocated in whole 16-byte words: uploads, gathers and function outputs
      Utf8Keys& u = out->u;
      out->ucols[u.n] = c;
      u.off[u.n] = c->offsets;
      u.bytes[u.n] = (const unsigned char*)c->values;
      u.valid[u.n] = valid;
      u.n++;
    } else {
      const int p = int(std::find(ints.begin(), ints.end(), i) - ints.begin());
      k.vals[p] = c->values;
      k.valid[p] = valid;
    }
  }
}

// DFGPU_JOIN_TAG_BITS=n (1..64, default 64): keep only the top n bits of a Utf8 key's tag, so that distinct keys share
// tags and the confirmation is exercised
unsigned long long join_tag_mask() {
  const char* e = getenv("DFGPU_JOIN_TAG_BITS");
  if (!e || !*e) return ~0ull;
  char* end = nullptr;
  const long bits = strtol(e, &end, 10);
  if (*end || bits < 1 || bits > 64) fail(DFGPU_ERR_GENERAL, std::string("DFGPU_JOIN_TAG_BITS must be 1 to 64, not '") + e + "'");
  return ~0ull << (64 - bits);
}

// The join's own device copy of one build column of n rows (Utf8 bytes in whole 16-byte words, as in the source)
DevColumn copy_column(dfgpu_ctx* ctx, const DevColumn& s, long long n) {
  DevColumn d;
  d.dtype = s.dtype;
  d.values_bytes = s.values_bytes;
  d.null_count = s.null_count;
  const size_t vb = s.dtype == DFGPU_UTF8 ? (s.values_bytes + 15) & ~size_t(15) : s.values_bytes;
  d.values = ctx->alloc(vb);
  if (vb) DF_CUDA(cudaMemcpyAsync(d.values, s.values, vb, cudaMemcpyDeviceToDevice, ctx->stream));
  if (s.validity && s.null_count > 0) {
    d.validity = (uint8_t*)ctx->alloc(size_t(n + 7) / 8);
    DF_CUDA(cudaMemcpyAsync(d.validity, s.validity, size_t(n + 7) / 8, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  if (s.offsets) {
    d.offsets = (int32_t*)ctx->alloc(size_t(n + 1) * 4);
    DF_CUDA(cudaMemcpyAsync(d.offsets, s.offsets, size_t(n + 1) * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  return d;
}

}  // namespace
}  // namespace dfgpu

using namespace dfgpu;

struct dfgpu_join {
  dfgpu_ctx* ctx = nullptr;
  int nkeys = 0;
  int key_dtypes[kMaxJoinKeys] = {};
  ProbeRule t{};
  unsigned long long* keys = nullptr;   // cap + 1 key words, EMPTY_KEY when free; slot cap is the key EMPTY_KEY
  unsigned long long* start = nullptr;  // cap + 2: the first entry of each slot's rows, then the number of rows with a key
  unsigned* rows = nullptr;             // build row numbers, grouped by slot
  long long nrows = 0;
  long long null_rows = 0;         // build rows with a null key part (null-aware anti join)
  std::vector<int> keep;           // build column numbers kept
  std::vector<DevColumn> cols;     // their device copies, in the order of `keep`
  // a key with Utf8 parts: `keys` holds each slot's tag, and a slot one distinct key
  unsigned long long tag_mask = ~0ull;  // DFGPU_JOIN_TAG_BITS at build time
  unsigned long long* words = nullptr;  // cap: each slot's packed integer word
  unsigned* rep = nullptr;              // cap: each slot's representative build row
  std::vector<DevColumn> ukeys;         // device copies of the build side's Utf8 key columns, in key order
  ~dfgpu_join() {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    ctx->free(keys);
    ctx->free(start);
    ctx->free(rows);
    ctx->free(words);
    ctx->free(rep);
    for (auto& c : ukeys) free_column(ctx, c);
    for (auto& c : cols) free_column(ctx, c);
  }
};

// The table of a key with Utf8 parts: rounds of k_join_utf8_place and k_join_utf8_verify until every row with a key is
// placed, leaving each slot's row count in `counts` and each row's slot in `row_slot`, as k_join_build does.  Each
// round seals at least one slot, the one of its smallest pending row.  Keeps a copy of the Utf8 key columns for the
// probe's confirmation.
static void build_utf8(dfgpu_ctx* ctx, const KeyColumns& kc, long long n, dfgpu_join* j, DevBufs& scratch, unsigned* counts,
                       unsigned long long* row_slot) {
  const long long cap = j->t.cap;
  j->words = (unsigned long long*)ctx->alloc(size_t(cap) * 8);
  j->rep = (unsigned*)ctx->alloc(size_t(cap) * 4);
  for (int i = 0; i < kc.u.n; i++) j->ukeys.push_back(copy_column(ctx, *kc.ucols[i], n));
  DF_CUDA(cudaMemsetAsync(j->rep, 0xff, size_t(cap) * 4, ctx->stream));
  if (n == 0) return;
  unsigned char* sealed = scratch.alloc<unsigned char>(size_t(cap));
  unsigned long long* d_next = scratch.alloc<unsigned long long>(sizeof(unsigned long long));
  unsigned* lists[2] = {scratch.alloc<unsigned>(size_t(n) * sizeof(unsigned)), nullptr};
  DF_CUDA(cudaMemsetAsync(sealed, 0, size_t(cap), ctx->stream));
  const unsigned* list = nullptr;  // the first round takes every row
  long long pending = n;
  for (int round = 0;; round++) {
    unsigned* next = lists[round & 1];
    if (!next) next = lists[1] = scratch.alloc<unsigned>(size_t(n) * sizeof(unsigned));
    DF_CUDA(cudaMemsetAsync(d_next, 0, 8, ctx->stream));
    launch(ctx, "k_join_utf8_place", k_join_utf8_place, grid_for(ctx, pending, JN_THREADS, 16), JN_THREADS, PROFILED, kc.k, kc.u, j->tag_mask, list, pending, (ProbeRule)j->t,
           j->keys, (const unsigned char*)sealed, j->rep, row_slot);
    launch(ctx, "k_join_utf8_verify", k_join_utf8_verify, grid_for(ctx, pending, JN_THREADS, 16), JN_THREADS, PROFILED, kc.k, kc.u, list, pending, (const unsigned*)j->rep,
           sealed, j->words, (const unsigned long long*)row_slot, counts, next, d_next);
    const long long left = (long long)read_word(ctx, d_next);
    if (left == 0) return;
    if (left >= pending) fail(DFGPU_ERR_INTERNAL, "JOIN build: a Utf8 key round placed no row");
    list = next;
    pending = left;
  }
}

extern "C" int dfgpu_join_build(dfgpu_ctx* ctx, const dfgpu_batch* build, const dfgpu_insn* const* keys, const int* key_len, int nkeys,
                                const int* keep_cols, int n_keep, dfgpu_join** out) {
  return guarded([&] {
    if (!ctx || !build || !out || (n_keep > 0 && !keep_cols) || n_keep < 0) fail(DFGPU_ERR_GENERAL, "dfgpu_join_build: null argument");
    ctx->use();
    const long long n = build->nrows;
    if (n >= (1ll << 32)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "JOIN build side of 2^32 rows or more");
    for (int i = 0; i < n_keep; i++)
      if (keep_cols[i] < 0 || size_t(keep_cols[i]) >= build->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "keep column " + std::to_string(keep_cols[i]) + " out of range");
    KeyColumns kc;
    key_columns(ctx, build, keys, key_len, nkeys, &kc);
    auto j = std::make_unique<dfgpu_join>();
    j->ctx = ctx;
    j->nkeys = nkeys;
    for (int i = 0; i < nkeys; i++) j->key_dtypes[i] = kc.dtypes[i];
    j->nrows = n;
    j->t.set_cap(table_cap(n, JN_MIN_CAP));
    const long long cap = j->t.cap;
    j->keys = (unsigned long long*)ctx->alloc(size_t(cap + 1) * 8);
    j->start = (unsigned long long*)ctx->alloc(size_t(cap + 2) * 8);
    j->rows = (unsigned*)ctx->alloc(size_t(std::max(1ll, n)) * 4);
    DevBufs scratch(ctx);
    unsigned* counts = scratch.alloc<unsigned>(size_t(cap + 1) * sizeof(unsigned));
    unsigned long long* row_slot = scratch.alloc<unsigned long long>(size_t(std::max(1ll, n)) * sizeof(unsigned long long));
    DF_CUDA(cudaMemsetAsync(j->keys, 0xff, size_t(cap + 1) * 8, ctx->stream));
    DF_CUDA(cudaMemsetAsync(counts, 0, size_t(cap + 1) * 4, ctx->stream));
    if (kc.u.n == 0) {
      if (n > 0) launch(ctx, "k_join_build", k_join_build, grid_for(ctx, n, JN_THREADS, 16), JN_THREADS, PROFILED, kc.k, n, (ProbeRule)j->t, j->keys, counts, row_slot);
    } else {
      j->tag_mask = join_tag_mask();
      build_utf8(ctx, kc, n, j.get(), scratch, counts, row_slot);
    }
    j->null_rows = n - (long long)scan_exclusive<unsigned, unsigned long long>(ctx, counts, j->start, cap + 1, true);  // start[cap + 1]: the rows with a key
    if (n > 0)
      launch(ctx, "k_join_scatter", k_join_scatter, grid_for(ctx, n, JN_THREADS, 16), JN_THREADS, PROFILED, (const unsigned long long*)row_slot, n,
             (const unsigned long long*)j->start, counts, j->rows);
    // the join's own copy of the kept columns: the caller may free the batch
    for (int i = 0; i < n_keep; i++) {
      j->keep.push_back(keep_cols[i]);
      j->cols.push_back(copy_column(ctx, build->cols[size_t(keep_cols[i])], n));
    }
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    *out = j.release();
  });
}

extern "C" int dfgpu_join_probe(dfgpu_join* j, const dfgpu_batch* probe, const dfgpu_insn* const* keys, const int* key_len, int nkeys,
                                const int* probe_cols, int n_probe_cols, const int* build_cols, int n_build_cols, dfgpu_result** out) {
  return guarded([&] {
    if (!j || !probe || !out || (n_probe_cols > 0 && !probe_cols) || (n_build_cols > 0 && !build_cols) || n_probe_cols < 0 || n_build_cols < 0)
      fail(DFGPU_ERR_GENERAL, "dfgpu_join_probe: null argument");
    dfgpu_ctx* ctx = j->ctx;
    ctx->use();
    const long long n = probe->nrows;
    if (n >= (1ll << 32)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "JOIN probe batch of 2^32 rows or more");
    for (int i = 0; i < n_probe_cols; i++)
      if (probe_cols[i] < 0 || size_t(probe_cols[i]) >= probe->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "probe column " + std::to_string(probe_cols[i]) + " out of range");
    std::vector<const DevColumn*> bsrc;
    for (int i = 0; i < n_build_cols; i++) {
      auto it = std::find(j->keep.begin(), j->keep.end(), build_cols[i]);
      if (it == j->keep.end()) fail(DFGPU_ERR_GENERAL, "build column " + std::to_string(build_cols[i]) + " was not kept by dfgpu_join_build");
      bsrc.push_back(&j->cols[size_t(it - j->keep.begin())]);
    }
    if (nkeys != j->nkeys) fail(DFGPU_ERR_GENERAL, "JOIN probe has " + std::to_string(nkeys) + " keys, the build side " + std::to_string(j->nkeys));
    KeyColumns kc;
    key_columns(ctx, probe, keys, key_len, nkeys, &kc);
    for (int i = 0; i < nkeys; i++)
      if (kc.dtypes[i] != j->key_dtypes[i])
        fail(DFGPU_ERR_EXECUTION, std::string("JOIN key types differ: ") + dtype_name(kc.dtypes[i]) + " and " + dtype_name(j->key_dtypes[i]));
    DevBufs scratch(ctx);
    unsigned* cnt = scratch.alloc<unsigned>(size_t(std::max(1ll, n)) * sizeof(unsigned));
    unsigned* bpos = scratch.alloc<unsigned>(size_t(std::max(1ll, n)) * sizeof(unsigned));
    unsigned long long* off = scratch.alloc<unsigned long long>(size_t(n + 1) * sizeof(unsigned long long));
    if (n > 0 && kc.u.n == 0)
      launch(ctx, "k_join_count", k_join_count, grid_for(ctx, n, JN_THREADS, 16), JN_THREADS, PROFILED, kc.k, n, (ProbeRule)j->t, (const unsigned long long*)j->keys,
             (const unsigned long long*)j->start, cnt, bpos);
    if (n > 0 && kc.u.n > 0) {
      Utf8Keys b{};
      for (const DevColumn& c : j->ukeys) {
        b.off[b.n] = c.offsets;
        b.bytes[b.n] = (const unsigned char*)c.values;
        b.n++;
      }
      launch(ctx, "k_join_utf8_count", k_join_utf8_count, grid_for(ctx, n, JN_THREADS, 16), JN_THREADS, PROFILED, kc.k, kc.u, j->tag_mask, n, (ProbeRule)j->t,
             (const unsigned long long*)j->keys, (const unsigned long long*)j->words, (const unsigned*)j->rep, b, (const unsigned long long*)j->start,
             cnt, bpos);
    }
    const unsigned long long total = n > 0 ? scan_exclusive<unsigned, unsigned long long>(ctx, cnt, off, n, true) : 0ull;
    if (total >= (1ull << 32)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "JOIN probe batch producing 2^32 or more output rows");
    const long long m = (long long)total;
    unsigned* pidx = scratch.alloc<unsigned>(size_t(std::max(1ll, m)) * sizeof(unsigned));
    unsigned* bidx = scratch.alloc<unsigned>(size_t(std::max(1ll, m)) * sizeof(unsigned));
    if (m > 0) {
      const int grid = grid_for(ctx, m, EMIT_TILE, 8);
      launch(ctx, "k_join_emit", k_join_emit, grid, JN_THREADS, PROFILED, (const unsigned long long*)off, n, (const unsigned*)bpos, (const unsigned*)j->rows,
             total, pidx, bidx);
    }
    auto res = std::make_unique<dfgpu_result>();
    res->ctx = ctx;
    res->nrows = m;
    unsigned long long* d_nulls = scratch.alloc<unsigned long long>(sizeof(unsigned long long));
    unsigned long long *p64 = nullptr, *b64 = nullptr;
    for (int i = 0; i < n_probe_cols; i++) {
      res->cols.emplace_back();
      gather_column(ctx, probe->cols[size_t(probe_cols[i])], pidx, m, scratch, p64, d_nulls, &res->cols.back());
    }
    for (int i = 0; i < n_build_cols; i++) {
      res->cols.emplace_back();
      gather_column(ctx, *bsrc[size_t(i)], bidx, m, scratch, b64, d_nulls, &res->cols.back());
    }
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    *out = res.release();
  });
}

extern "C" int dfgpu_join_semi(dfgpu_join* j, const dfgpu_batch* probe, const dfgpu_insn* const* keys, const int* key_len, int nkeys, int kind,
                               const int* probe_cols, int n_probe_cols, dfgpu_result** out) {
  return guarded([&] {
    if (!j || !probe || !out || (n_probe_cols > 0 && !probe_cols) || n_probe_cols < 0) fail(DFGPU_ERR_GENERAL, "dfgpu_join_semi: null argument");
    if (kind != DFGPU_JOIN_SEMI && kind != DFGPU_JOIN_ANTI && kind != DFGPU_JOIN_ANTI_NULL_AWARE)
      fail(DFGPU_ERR_GENERAL, "dfgpu_join_semi: unknown kind " + std::to_string(kind));
    if (kind == DFGPU_JOIN_ANTI_NULL_AWARE && nkeys != 1) fail(DFGPU_ERR_GENERAL, "a null-aware anti join takes exactly one key");
    dfgpu_ctx* ctx = j->ctx;
    ctx->use();
    const long long n = probe->nrows;
    if (n >= (1ll << 32)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "JOIN probe batch of 2^32 rows or more");
    for (int i = 0; i < n_probe_cols; i++)
      if (probe_cols[i] < 0 || size_t(probe_cols[i]) >= probe->cols.size()) fail(DFGPU_ERR_INVALID_COLUMN, "probe column " + std::to_string(probe_cols[i]) + " out of range");
    if (nkeys != j->nkeys) fail(DFGPU_ERR_GENERAL, "JOIN probe has " + std::to_string(nkeys) + " keys, the build side " + std::to_string(j->nkeys));
    KeyColumns kc;
    key_columns(ctx, probe, keys, key_len, nkeys, &kc);
    for (int i = 0; i < nkeys; i++)
      if (kc.dtypes[i] != j->key_dtypes[i])
        fail(DFGPU_ERR_EXECUTION, std::string("JOIN key types differ: ") + dtype_name(kc.dtypes[i]) + " and " + dtype_name(j->key_dtypes[i]));
    // NOT IN over a set holding a null is never true: no row passes, and nothing is launched
    const bool none = kind == DFGPU_JOIN_ANTI_NULL_AWARE && j->null_rows > 0;
    const int anti = kind != DFGPU_JOIN_SEMI;
    const int null_pass = kind == DFGPU_JOIN_ANTI || (kind == DFGPU_JOIN_ANTI_NULL_AWARE && j->nrows == 0);
    DevBufs scratch(ctx);
    const long long ntiles = (n + MARK_TILE - 1) / MARK_TILE;
    long long m = 0;
    unsigned* idx = nullptr;
    if (n > 0 && !none) {
      unsigned* mask = scratch.alloc<unsigned>(size_t(ntiles) * MARK_WORDS * sizeof(unsigned));
      unsigned* tile_cnt = scratch.alloc<unsigned>(size_t(ntiles) * sizeof(unsigned));
      unsigned long long* tile_off = scratch.alloc<unsigned long long>(size_t(ntiles + 1) * sizeof(unsigned long long));
      const int grid = grid_for(ctx, n, MARK_TILE, 8);
      if (kc.u.n == 0) {
        launch(ctx, "k_join_mark", k_join_mark, grid, JN_THREADS, PROFILED, kc.k, n, (ProbeRule)j->t, (const unsigned long long*)j->keys,
               (const unsigned long long*)j->start, anti, null_pass, mask, tile_cnt);
      } else {
        Utf8Keys b{};
        for (const DevColumn& c : j->ukeys) {
          b.off[b.n] = c.offsets;
          b.bytes[b.n] = (const unsigned char*)c.values;
          b.n++;
        }
        launch(ctx, "k_join_utf8_mark", k_join_utf8_mark, grid, JN_THREADS, PROFILED, kc.k, kc.u, j->tag_mask, n, (ProbeRule)j->t,
               (const unsigned long long*)j->keys, (const unsigned long long*)j->words, (const unsigned*)j->rep, b, anti, null_pass, mask, tile_cnt);
      }
      m = (long long)scan_exclusive<unsigned, unsigned long long>(ctx, tile_cnt, tile_off, ntiles, true);
      idx = scratch.alloc<unsigned>(size_t(std::max(1ll, m)) * sizeof(unsigned));
      if (m > 0)
        select_rows(ctx, grid, mask, ntiles, tile_off, idx);
    }
    auto res = std::make_unique<dfgpu_result>();
    res->ctx = ctx;
    res->nrows = m;
    unsigned long long* d_nulls = scratch.alloc<unsigned long long>(sizeof(unsigned long long));
    unsigned long long* idx64 = nullptr;
    for (int i = 0; i < n_probe_cols; i++) {
      res->cols.emplace_back();
      gather_column(ctx, probe->cols[size_t(probe_cols[i])], idx, m, scratch, idx64, d_nulls, &res->cols.back());
    }
    DF_CUDA(cudaStreamSynchronize(ctx->stream));
    *out = res.release();
  });
}

extern "C" int dfgpu_join_free(dfgpu_join* j) {
  return guarded([&] { delete j; });
}
