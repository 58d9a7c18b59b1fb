"""tests/hash_ref.py on a CPU: the inverse of mix64, the crafted keys landing where each helper says under the mirror,
the mirror pinned to the CUDA source text, and parallel.owner_of agreeing with the device formula."""
import os
import re

import numpy as np
import pytest

import hash_ref as H
from datafusion_archive_b200 import parallel

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "datafusion_archive_b200", "csrc")
EDGES = [0, 1, 2, 3, H.EMPTY_KEY, H.EMPTY_KEY - 1, H.EMPTY_KEY - 3, 1 << 63, (1 << 63) - 1, 1 << 32, (1 << 32) - 1,
         H.GOLDEN, H.C1, H.C2, 0x5555555555555555, 0xaaaaaaaaaaaaaaaa]


def mix64_int(x):
    """mix64 on one Python int, written out independently of the numpy mirror."""
    x ^= x >> 33
    x = (x * H.C1) & H.M64
    x ^= x >> 33
    x = (x * H.C2) & H.M64
    x ^= x >> 33
    return x


def test_unmix64_inverts_mix64():
    rng = np.random.default_rng(1)
    x = np.concatenate([np.array(EDGES, dtype=np.uint64), rng.integers(0, 2 ** 64, 100_000, dtype=np.uint64, endpoint=False)])
    assert np.array_equal(H.unmix64(H.mix64(x)), x)
    assert np.array_equal(H.mix64(H.unmix64(x)), x)
    assert [int(v) for v in H.mix64(np.array(EDGES, dtype=np.uint64))] == [mix64_int(e) for e in EDGES]
    assert int(H.mix64(0)[0]) == 0  # the packed word 0 hashes to 0: Utf8 join keys without an integer part start there


def test_home_and_wrap():
    for lg in range(0, 41, 5):
        cap = 1 << lg
        assert int(H.home(H.EMPTY_KEY, cap)[0]) == cap - 1
        assert int(H.next_slot(cap - 1, cap)[0]) == 0
        assert int(H.home((1 << 64) - (1 << H.LOW), cap)[0]) == cap - 1
    assert int(H.home(H.EMPTY_KEY, 1)[0]) == 0
    assert H.table_cap(0, H.AG_MIN_CAP) == H.AG_MIN_CAP and H.table_cap(3_000_000, H.AG_MIN_CAP) == 1 << 23
    assert H.table_cap(600, H.JN_MIN_CAP) == 2048 and H.table_cap(512, H.JN_MIN_CAP) == 1024


@pytest.mark.parametrize("top,where", [("ones", "end"), ("zeros", "start")])
def test_cluster_keys_share_one_home_and_front_slot(top, where):
    rng = np.random.default_rng(2)
    k = H.cluster_keys(rng, 3000, top)
    assert len(np.unique(k)) == 3000 and not np.any(k == np.uint64(H.EMPTY_KEY))
    h = H.mix64(k)
    for cap in (1 << 10, 1 << 20, 1 << 22, 1 << 26, 1 << 40):
        assert np.all(H.home(h, cap) == np.uint64(cap - 1 if where == "end" else 0)), cap
    assert len(np.unique(H.front_slot(h))) == 1
    assert int(H.front_slot(h)[0]) == (H.AG_FRONT_SLOTS - 1 if top == "ones" else 0)
    # inserted into one table, they form one run of probes 1, 2, ..., m: the cluster at cap - 1 wraps to slot 0
    assert np.array_equal(np.sort(H.probe_chain(h, 1 << 12)), np.arange(1, 3001))


def test_background_keys_stay_away_from_the_ends():
    rng = np.random.default_rng(3)
    k = H.background_keys(rng, 5000)
    assert len(np.unique(k)) == 5000 and not np.any(k == np.uint64(H.EMPTY_KEY))
    top2 = H.mix64(k) >> np.uint64(62)
    assert set(top2.tolist()) <= {1, 2}


def test_packed_i32_pair_round_trip():
    rng = np.random.default_rng(4)
    w = H.cluster_keys(rng, 1000)
    a, b = H.split_i32_pair(w)
    assert a.dtype == np.int32 and np.array_equal(H.pack_i32_pair(a, b), w)


def test_wide_keys_with_one_exact_hash():
    rng = np.random.default_rng(5)
    target = np.full(500, 0xfffffffffe123457, dtype=np.uint64)
    first = rng.permutation(10_000)[:500].astype(np.int64)
    last = H.wide_last_part([first], target)
    assert np.all(H.wide_hash([first, last]) == target)
    assert len(np.unique(np.stack([first.view(np.uint64), last]), axis=1)[0]) == 500  # distinct keys
    strings = ["s%d" % i for i in range(300)]
    hs = H.utf8_hashes(strings)
    last = H.wide_last_part([hs], target[:300])
    assert np.all(H.wide_hash([hs, last]) == target[:300])


def test_tag_aliases():
    h = np.array([H.EMPTY_KEY, H.EMPTY_KEY - 3, 0x123456789abcdef0, 0xfffffffffe000002], dtype=np.uint64)
    a = H.alias_hashes(h)
    assert np.all(a != h) and np.array_equal(H.wide_tag(a), H.wide_tag(h))
    assert int(H.wide_tag(H.EMPTY_KEY)[0]) == H.EMPTY_KEY ^ 2
    assert not np.any(H.wide_tag(np.concatenate([h, a])) == np.uint64(H.EMPTY_KEY))


def test_utf8_hash_bytes_known_values():
    # FNV-1a-64 of "" is its offset basis; the mixer then runs over it
    h = H.FNV_OFFSET
    h ^= h >> 32
    h = (h * H.UTF8_MIX) & H.M64
    h ^= h >> 32
    assert H.utf8_hash_bytes("") == h
    assert H.utf8_hash_bytes("é") == H.utf8_hash_bytes(b"\xc3\xa9") != H.utf8_hash_bytes("e")


def test_join_keys_with_one_exact_tag():
    strings = ["k%d" % i for i in range(200)] + ["", "x" * 40]
    target = np.full(len(strings), 0xffffffffff0000aa, dtype=np.uint64)
    word = H.join_word_for_tag(strings, target)
    assert np.all(H.join_utf8_tag(word, [H.utf8_hashes(strings)]) == target)
    # tags that would be EMPTY_KEY become EMPTY_KEY - 1, the tag of the second pair as well
    t = np.array([H.EMPTY_KEY, H.EMPTY_KEY - 1], dtype=np.uint64)
    w = H.join_word_for_tag(["a", "b"], t)
    assert np.all(H.join_utf8_tag(w, [H.utf8_hashes(["a", "b"])]) == np.uint64(H.EMPTY_KEY - 1))


def test_distinct_pairs_with_chosen_hashes():
    rng = np.random.default_rng(6)
    target = H.cluster_hashes(rng, 400)
    for key in (0, 12345, H.EMPTY_KEY):
        v = H.distinct_values_for(key, target)
        assert np.all(H.pair_hash(np.uint64(key), v) == target)
    k = H.distinct_keys_for(H.EMPTY_KEY, target)
    assert np.all(H.pair_hash(k, np.uint64(H.EMPTY_KEY)) == target)
    assert np.array_equal(H.distinct_norm(np.array([-0.0, 0.0, np.nan, -np.nan, 1.5])),
                          np.array([0, 0, 0x7ff8000000000000, 0x7ff8000000000000, np.float64(1.5).view(np.uint64)], dtype=np.uint64))


@pytest.mark.parametrize("world", [1, 2, 3, 7, 64])
def test_parallel_owner_of_matches_the_device_formula(world):
    rng = np.random.default_rng(world)
    k = np.concatenate([np.array(EDGES, dtype=np.uint64), rng.integers(0, 2 ** 64, 20_000, dtype=np.uint64, endpoint=False)])
    exp = np.array([0 if int(x) == H.EMPTY_KEY else (mix64_int(int(x)) & 0xffffffff) % world for x in k], dtype=np.int64)
    assert np.array_equal(H.owner_of(k, world), exp)
    assert np.array_equal(parallel.owner_of(k, world), exp)
    assert np.array_equal(parallel.owner_of(k.view(np.int64), world), exp)
    assert np.array_equal(parallel.mix64(k), H.mix64(k))


# ---- the mirror pinned to the CUDA source ----------------------------------------------------------------------------
def source(name):
    with open(os.path.join(CSRC, name)) as f:
        return re.sub(r"\s+", "", f.read())


def pinned():
    """(file, code that must occur in it, whitespace removed), built from the mirror's constants."""
    return [
        ("hash_table.cuh", "constexprunsignedlonglongEMPTY_KEY=~0ull;"),
        ("hash_table.cuh", "x^=x>>33;x*=0x%xull;x^=x>>33;x*=0x%xull;x^=x>>33;returnx;" % (H.C1, H.C2)),
        ("hash_table.cuh", "hshift=64-lg;"),
        ("hash_table.cuh", "returnhshift>=64?0ull:hash>>hshift;"),
        ("hash_table.cuh", "return(slot+1ull)&((unsignedlonglong)cap-1ull);"),
        ("hash_table.cuh", "returnstd::max(min_cap,next_pow2(2*n));"),
        ("utf8_words.cuh", "unsignedlonglongh=0x%xull;for(;b<e;b++){h^=bytes[b];h*=0x%xull;}h^=h>>32;h*=0x%xull;h^=h>>32;returnh;"
         % (H.FNV_OFFSET, H.FNV_PRIME, H.UTF8_MIX)),
        ("aggregate.cu", "constexprintAG_MAX_PROBE=1<<%d;" % (H.AG_MAX_PROBE.bit_length() - 1)),
        ("aggregate.cu", "constexprlonglongAG_MIN_CAP=1ll<<%d;" % (H.AG_MIN_CAP.bit_length() - 1)),
        ("aggregate.cu", "constexprlonglongAG_SET_MIN_CAP=1ll<<%d;" % (H.AG_SET_MIN_CAP.bit_length() - 1)),
        ("aggregate.cu", "constexprintAG_FRONT_SLOTS=%d;" % H.AG_FRONT_SLOTS),
        ("aggregate.cu", "constexprintAG_FRONT_PROBES=%d;" % H.AG_FRONT_PROBES),
        ("aggregate.cu", "constexprintAG_THREADS=%d;" % H.AG_THREADS),
        # the front slot and its probe step
        ("aggregate.cu", "unsignedfh=(unsigned)(mix64(key[r])>>40)&(unsigned)(FS-1);"),
        ("aggregate.cu", "fh=(fh+1)&(unsigned)(FS-1);"),
        # the scans' home of a packed key
        ("aggregate.cu", "constunsignedlonglonghs=mix64(key[r]);h[r]=p.t.home(hs);"),
        ("aggregate.cu", "slot[r]=p.t.home(mix64(k[r]));"),
        ("aggregate.cu", "unsignedlonglongh=home(mix64(k));"),
        ("aggregate.cu", "unsignedlonglongh=p.t.home(mix64(key));"),
        # the wide hash and its tag
        ("aggregate.cu", "hsh[r]=0x%xull;" % H.GOLDEN),
        ("aggregate.cu", "hsh[r]=mix64(hsh[r]^(v[r]+0x%xull*(unsignedlonglong)(k+1)));" % H.GOLDEN),
        ("aggregate.cu", "unsignedlonglongt=h|1ull;if(t==EMPTY_KEY)t^=2ull;returnt;"),
        ("aggregate.cu", "unsignedlonglongh=p.t.home(hsh[r]);"),
        ("aggregate.cu", "unsignedlonglongh=p.to.home(tag&~1ull);"),
        # the pair sets
        ("aggregate.cu", "unsignedlonglongh=set.home(mix64(val^mix64(key)));"),
        ("aggregate.cu", "returnd!=d?0x7ff8000000000000ull:(d==0.0?0ull:v);"),
        ("aggregate.cu", "returnf!=f?0x7fc00000ull:(f==0.0f?0ull:(v&0xffffffffull));"),
        # the owner of a key across ranks
        ("aggregate.cu", "returnkey==EMPTY_KEY?0:(int)((mix64(key)&0xffffffffull)%(unsignedlonglong)world);"),
        # the join's build table and Utf8 tags
        ("join.cu", "constexprlonglongJN_MIN_CAP=%d;" % H.JN_MIN_CAP),
        ("join.cu", "h=t.home(mix64(key));"),
        ("join.cu", "unsignedlonglongh=t.home(mix64(key));"),
        ("join.cu", "unsignedlonglongh=mix64(*word);"),
        ("join.cu", "h=mix64(h^utf8_hash_bytes(u.bytes[i],__ldg(u.off[i]+r),__ldg(u.off[i]+r+1)));"),
        ("join.cu", "*tag=h==EMPTY_KEY?EMPTY_KEY-1ull:h;"),
        ("join.cu", "h=t.home(tag);"),
        ("join.cu", "unsignedlonglongh=t.home(tag);"),
    ]


@pytest.mark.parametrize("i", range(len(pinned())))
def test_mirror_is_pinned_to_the_cuda_source(i):
    name, code = pinned()[i]
    assert code in source(name), "%s no longer contains %s: update tests/hash_ref.py with it" % (name, code)


def test_pins_cover_every_hash_and_home():
    # every line of the table code that calls mix64 or home() is pinned: a new hash or home rule needs a mirror here
    pins = {}
    for name, code in pinned():
        pins.setdefault(name, []).append(code)
    for name in ("aggregate.cu", "join.cu"):
        with open(os.path.join(CSRC, name)) as f:
            lines = f.read().splitlines()
        calls = 0
        for line in lines:
            code = re.sub(r"\s+", "", line.split("//")[0])
            if "mix64(" not in code and "home(" not in code:
                continue
            calls += 1
            assert any(code in p or p in code for p in pins[name]), (name, line.strip())
        assert calls >= 5, name
