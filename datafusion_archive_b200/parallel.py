"""Multi-GPU host logic (SURVEY.md §8e): one process per GPU, contiguous row-range partitioning,
no collective for filter/project (outputs concatenate in rank order), one owner-partitioned
partial-aggregate merge for aggregates.

This module is a numpy MODEL of that protocol (row ranges, owner function, per-owner merge, gather) so
that the world_size>1 host logic can be exercised on CPU over gloo.  It is not the product's merge: on
GPUs the exchange runs inside libdfgpu.so (aggregate.cu agg_exchange_groups: k_owner_count /
k_owner_scatter -> grouped ncclSend/ncclRecv -> k_merge -> k_compact -> grouped ncclBroadcast), which is
tested under NCCL on two GPUs (tests/test_multiprocess.py) and checked against numpy inside bench.py at
every N."""
import numpy as np

from . import _abi as A


def row_range(rank, world, nrows):
    """GPU g of G owns rows [g*ceil(N/G), min(N, (g+1)*ceil(N/G)))."""
    per = -(-nrows // world)
    lo = min(nrows, rank * per)
    return lo, min(nrows, lo + per)


def shard(arrays, rank, world):
    lo, hi = row_range(rank, world, len(arrays[0]))
    return [a[lo:hi] for a in arrays]


def merge_partials(partials, funcs):
    """partials: list (one per rank) of [key_col, agg_col...] with unique keys per rank;
    funcs: DFGPU_AGG_* per aggregate column.  Returns merged [keys, aggs...] sorted by key."""
    keys = np.concatenate([p[0] for p in partials])
    uk, inv = np.unique(keys, return_inverse=True)
    out = [uk]
    for j, f in enumerate(funcs):
        vals = np.concatenate([p[1 + j] for p in partials])
        if f in (A.AGG_SUM, A.AGG_COUNT):
            acc = np.zeros(len(uk), dtype=vals.dtype)
            np.add.at(acc, inv, vals)
        elif f == A.AGG_MIN:
            acc = np.full(len(uk), np.inf if vals.dtype.kind == "f" else np.iinfo(vals.dtype).max, dtype=vals.dtype)
            np.minimum.at(acc, inv, vals)
        else:
            acc = np.full(len(uk), -np.inf if vals.dtype.kind == "f" else np.iinfo(vals.dtype).min, dtype=vals.dtype)
            np.maximum.at(acc, inv, vals)
        out.append(acc)
    return out


def concat_in_rank_order(parts):
    """filter/project: rank-ordered concatenation preserves global row order."""
    return [np.concatenate([p[i] for p in parts]) for i in range(len(parts[0]))]


_M1, _M2 = np.uint64(0xff51afd7ed558ccd), np.uint64(0xc4ceb9fe1a85ec53)


def mix64(x):
    """The table / owner hash of csrc/aggregate.cu (murmur3 finaliser) on uint64 arrays."""
    x = np.asarray(x).astype(np.uint64, copy=True)
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(33)
        x *= _M1
        x ^= x >> np.uint64(33)
        x *= _M2
        x ^= x >> np.uint64(33)
    return x


def owner_of(keys, world):
    """Owner rank of every packed 64-bit group key, as aggregate.cu owner_of computes it: the low 32 bits of
    mix64(key), which a table of up to 2^32 slots does not use for the home slot, modulo the world size; the key that
    equals the empty marker belongs to rank 0."""
    k = np.asarray(keys).view(np.uint64) if np.asarray(keys).dtype.itemsize == 8 else np.asarray(keys).astype(np.int64).view(np.uint64)
    own = ((mix64(k) & np.uint64(0xffffffff)) % np.uint64(world)).astype(np.int64)
    own[k == np.uint64(0xFFFFFFFFFFFFFFFF)] = 0
    return own


def partition_by_owner(partial, world):
    """Split one rank's partial aggregate [keys, aggs...] into per-owner segments."""
    own = owner_of(partial[0], world)
    return [[c[own == r] for c in partial] for r in range(world)]
