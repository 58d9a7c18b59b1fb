"""Mirrors of the device hash formulas (numpy only) and keys crafted to collide in the GPU hash tables.

Every open-addressed table of the project follows csrc/hash_table.cuh: a 64-bit hash, a power-of-two capacity, the home
slot is the hash's top log2(cap) bits, and probing steps linearly and wraps from slot cap - 1 to slot 0.  mix64 is a
bijection (each xor-shift by 33 is its own inverse, and its multipliers are odd, so invertible mod 2^64), so a key can be
built for any chosen hash with unmix64.  Two facts make crafted keys adversarial at every capacity:
* hashes whose top 40 bits are equal share one home slot at every capacity up to 2^40, and one front-table slot
  ((h >> 40) & (FS - 1)) as well;
* top 40 bits all ones put the home at cap - 1 for every capacity, so the cluster wraps to slot 0; top bits all zeros put
  it at slot 0, where the wrapped cluster runs into it.

tests/test_hash_ref_cpu.py pins every formula here to the CUDA source text, so an edit on either side fails on a CPU
before it silently disarms the GPU tests.  Arrays are uint64 unless stated otherwise."""
import numpy as np

M64 = (1 << 64) - 1
EMPTY_KEY = M64                 # hash_table.cuh: the empty-slot marker; the key equal to it lives in slot cap
C1, C2 = 0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53
C1_INV, C2_INV = pow(C1, -1, 1 << 64), pow(C2, -1, 1 << 64)
GOLDEN = 0x9e3779b97f4a7c15     # seed and part multiplier of the wide-key hash (aggregate.cu k_hash_agg_wide)
FNV_OFFSET, FNV_PRIME = 0xcbf29ce484222325, 0x100000001b3
UTF8_MIX = 0xd6e8feb86659fd93   # the finaliser multiplier of utf8_hash_bytes (utf8_words.cuh)

AG_MAX_PROBE = 1 << 14          # aggregate.cu: a new key is refused after this many probes
AG_MIN_CAP = 1 << 22            # the group table's smallest capacity
AG_SET_MIN_CAP = 1 << 20        # the COUNT(DISTINCT) pair sets' smallest capacity
AG_FRONT_SLOTS = 2048           # the per-CTA shared-memory front table
AG_FRONT_PROBES = 8             # probes in the front table before a row goes to the global table
AG_THREADS = 256
JN_MIN_CAP = 1024               # join.cu: the build table's smallest capacity

TOP = 40                        # hashes equal in their top TOP bits share a home at every capacity up to 2^TOP
LOW = 64 - TOP

_S33 = np.uint64(33)


def u64(x):
    """x as a uint64 array; Python ints and signed arrays are taken mod 2^64."""
    if isinstance(x, int):
        return np.array([x & M64], dtype=np.uint64)
    a = np.asarray(x)
    if a.dtype == np.uint64:
        return a.copy()
    if a.dtype.kind in "iu":
        return a.astype(np.int64).view(np.uint64) if a.dtype.kind == "i" else a.astype(np.uint64)
    return np.array([int(v) & M64 for v in a.ravel()], dtype=np.uint64).reshape(a.shape)


def mix64(x):
    """hash_table.cuh mix64 (the murmur3 finaliser)."""
    x = u64(x)
    with np.errstate(over="ignore"):
        x ^= x >> _S33
        x *= np.uint64(C1)
        x ^= x >> _S33
        x *= np.uint64(C2)
        x ^= x >> _S33
    return x


def unmix64(h):
    """The inverse of mix64: unmix64(mix64(x)) == x."""
    x = u64(h)
    with np.errstate(over="ignore"):
        x ^= x >> _S33
        x *= np.uint64(C2_INV)
        x ^= x >> _S33
        x *= np.uint64(C1_INV)
        x ^= x >> _S33
    return x


def log2_cap(cap):
    assert cap > 0 and cap & (cap - 1) == 0, cap
    return cap.bit_length() - 1


def home(h, cap):
    """ProbeRule::home: the top log2(cap) bits of the hash."""
    shift = 64 - log2_cap(cap)
    h = u64(h)
    return np.zeros_like(h) if shift >= 64 else h >> np.uint64(shift)


def next_slot(slot, cap):
    """ProbeRule::next: one slot on, wrapping at cap."""
    return (u64(slot) + np.uint64(1)) & np.uint64(cap - 1)


def table_cap(n, min_cap):
    """hash_table.cuh table_cap: at least min_cap and twice n, a power of two."""
    p = 1
    while p < 2 * n:
        p <<= 1
    return max(min_cap, p)


def front_slot(h, fs=AG_FRONT_SLOTS):
    """The front table's first slot of a key with hash h (aggregate.cu hash_agg_body)."""
    return (u64(h) >> np.uint64(40)) & np.uint64(fs - 1)


def agg_key_hash(keys):
    """The hash of a packed (or single, sign-extended) GROUP BY key word."""
    return mix64(keys)


def pack_i32_pair(a, b):
    """The packed key word of an (Int32, Int32) GROUP BY key: the last key in the low bits."""
    return (u64(np.asarray(a, np.int32).astype(np.uint32)) << np.uint64(32)) | u64(np.asarray(b, np.int32).astype(np.uint32))


def split_i32_pair(w):
    """The (Int32, Int32) parts of packed key words (the inverse of pack_i32_pair)."""
    w = u64(w)
    return (w >> np.uint64(32)).astype(np.uint32).view(np.int32), (w & np.uint64(0xffffffff)).astype(np.uint32).view(np.int32)


def utf8_hash_bytes(s):
    """utf8_words.cuh utf8_hash_bytes: FNV-1a-64 over the UTF-8 bytes, then a 64-bit mixer.  s: str or bytes."""
    h = FNV_OFFSET
    for c in (s.encode() if isinstance(s, str) else bytes(s)):
        h = ((h ^ c) * FNV_PRIME) & M64
    h ^= h >> 32
    h = (h * UTF8_MIX) & M64
    h ^= h >> 32
    return h


def utf8_hashes(strings):
    return np.array([utf8_hash_bytes(s) for s in strings], dtype=np.uint64)


def _part_term(v, k):
    with np.errstate(over="ignore"):
        return u64(v) + np.uint64((GOLDEN * (k + 1)) & M64)


def wide_hash(parts):
    """The wide-key hash of k_hash_agg_wide over the key parts, in key order: each part's 64-bit value (a fixed-width
    part sign- or zero-extended, a Utf8 part its utf8_hash_bytes)."""
    h = np.full(len(parts[0]), GOLDEN, dtype=np.uint64)
    for k, v in enumerate(parts):
        h = mix64(h ^ _part_term(v, k))
    return h


def wide_tag(h):
    """aggregate.cu wide_tag: the ready tag of a wide hash, low bit set and never EMPTY_KEY."""
    t = u64(h) | np.uint64(1)
    t[t == np.uint64(EMPTY_KEY)] ^= np.uint64(2)
    return t


def join_utf8_tag(word, utf8_part_hashes):
    """join.cu utf8_tag at the full 64-bit width: mix64 over the packed integer word (0 when there is no integer part),
    then h = mix64(h ^ H(s)) per Utf8 part; a tag equal to EMPTY_KEY becomes EMPTY_KEY - 1."""
    h = mix64(word)
    for hs in utf8_part_hashes:
        h = mix64(h ^ u64(hs))
    h[h == np.uint64(EMPTY_KEY)] = np.uint64(EMPTY_KEY - 1)
    return h


def distinct_norm(v):
    """aggregate.cu distinct_norm on the widened 64-bit argument words: +-0.0 are one value, every NaN is one value.
    v: a numeric array; returns the words the pair set stores."""
    v = np.asarray(v)
    if v.dtype == np.float64:
        w = v.view(np.uint64).copy()
        w[v == 0] = 0
        w[np.isnan(v)] = np.uint64(0x7ff8000000000000)
        return w
    if v.dtype == np.float32:
        w = v.view(np.uint32).astype(np.uint64)
        w[v == 0] = 0
        w[np.isnan(v)] = np.uint64(0x7fc00000)
        return w
    return u64(v)


def pair_hash(key, val):
    """set_insert's hash of a (packed group key, normalised value) pair: mix64(val ^ mix64(key)).  key is 0 without
    GROUP BY."""
    return mix64(u64(val) ^ mix64(key))


def owner_of(keys, world):
    """aggregate.cu owner_of: the rank that merges a packed group key across ranks; the key equal to EMPTY_KEY belongs
    to rank 0."""
    k = u64(keys)
    own = ((mix64(k) & np.uint64(0xffffffff)) % np.uint64(world)).astype(np.int64)
    own[k == np.uint64(EMPTY_KEY)] = 0
    return own


# ---- crafting ------------------------------------------------------------------------------------------------------
def keys_for_hashes(h):
    """The 64-bit key words whose mix64 is h."""
    return unmix64(h)


def cluster_hashes(rng, m, top="ones", exclude=()):
    """m distinct hashes with equal top TOP bits: all ones (home cap - 1 at every capacity, the cluster wraps) or all
    zeros (home 0).  Hashes in `exclude` are left out."""
    hi = ((1 << TOP) - 1) << LOW if top == "ones" else 0
    ex = set(int(x) for x in u64(np.asarray(list(exclude), dtype=np.uint64))) if len(exclude) else set()
    out = []
    while len(out) < m:
        low = rng.choice(1 << LOW, size=m + len(ex) + 8, replace=False).astype(np.uint64)
        cand = [int(x) | hi for x in low]
        out = [c for c in dict.fromkeys(cand) if c not in ex][:m]
    return np.array(out, dtype=np.uint64)


def cluster_keys(rng, m, top="ones"):
    """m distinct key words whose hashes share their top TOP bits (see cluster_hashes); never the EMPTY_KEY word, which
    has its own slot."""
    return keys_for_hashes(cluster_hashes(rng, m, top, exclude=mix64(EMPTY_KEY)))


def wide_last_part(prefix_parts, target):
    """The last part that gives the key parts `prefix_parts` + [it] the wide hash `target` (both arrays of equal length).
    prefix_parts: the 64-bit values of the parts before the last."""
    n = len(target)
    h = np.full(n, GOLDEN, dtype=np.uint64)
    for k, v in enumerate(prefix_parts):
        h = mix64(h ^ _part_term(v, k))
    k = len(prefix_parts)
    with np.errstate(over="ignore"):
        return (unmix64(target) ^ h) - np.uint64((GOLDEN * (k + 1)) & M64)


def alias_hashes(h):
    """For each hash, another hash with the same wide tag: they differ only in bit 0, except that EMPTY_KEY pairs with
    EMPTY_KEY - 3 (both tag to EMPTY_KEY ^ 2)."""
    h = u64(h)
    a = h ^ np.uint64(1)
    a[h == np.uint64(EMPTY_KEY)] = np.uint64(EMPTY_KEY - 3)
    a[h == np.uint64(EMPTY_KEY - 3)] = np.uint64(EMPTY_KEY)
    return a


def join_word_for_tag(strings, target):
    """The packed integer word that gives a (Utf8, integer) join key with Utf8 part strings[i] the 64-bit tag target[i]:
    unmix64(unmix64(target) ^ H(s))."""
    return unmix64(unmix64(target) ^ utf8_hashes(strings))


def distinct_values_for(key, target):
    """The argument words v whose pair (key, v) has the set hash `target`.  key: the packed group key word (0 without
    GROUP BY), one or one per target."""
    return unmix64(target) ^ mix64(np.broadcast_to(u64(key), np.shape(target)))


def distinct_keys_for(val, target):
    """The packed group key words k whose pair (k, val) has the set hash `target`."""
    return unmix64(unmix64(target) ^ np.broadcast_to(u64(val), np.shape(target)))


def background_hashes(rng, m):
    """m distinct random hashes whose top two bits are 01 or 10: they home in the middle half of a table of any capacity,
    away from the crafted clusters at both ends."""
    out = np.zeros(0, dtype=np.uint64)
    while len(out) < m:
        h = rng.integers(0, 1 << 62, size=2 * m + 8, dtype=np.uint64) | np.uint64(1 << 62)
        h[: len(h) // 2] ^= np.uint64(3 << 62)  # 01 -> 10 for half of them
        out = np.unique(np.concatenate([out, h]))
    return rng.permutation(out)[:m]


def background_keys(rng, m):
    """m distinct key words with background_hashes, never EMPTY_KEY (which has its own slot)."""
    k = keys_for_hashes(background_hashes(rng, m + 1))
    return k[k != np.uint64(EMPTY_KEY)][:m]


def probe_chain(hashes, cap):
    """Insert keys with these (distinct) hashes in order into an empty table of cap slots under the probe rule; returns
    each key's number of probes (1 = its home).  For checking that a crafted set forms one cluster."""
    used = np.zeros(cap, dtype=bool)
    probes = []
    for s0 in home(hashes, cap):
        s, n = int(s0), 1
        while used[s]:
            s, n = (s + 1) & (cap - 1), n + 1
        used[s] = True
        probes.append(n)
    return np.array(probes)
