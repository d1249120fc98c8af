"""Checker for the damage locator (swec_locate_ec_damage / swec_locate_damage_device), sharing nothing with its method.

The syndrome of every byte column is computed from oracle.rs_numpy's matrix.  It is then looked up in a table of the
syndromes of EVERY error pattern within the radius: every single shard and, at radius 2, every pair of shards, each
with every non-zero error value.  A column whose syndrome is not in the table is uncorrectable.  The report and the
page ranges are built the way include/swec.h describes them.
"""
from __future__ import annotations

import functools

import numpy as np

from oracle import rs_numpy as rn

PAGE = 4096


def parity_check(k: int, m: int) -> np.ndarray:
    """H = [P | I], m x (k+m): H·c = 0 for every codeword column c."""
    p = rn.build_matrix(k, k + m)[k:]
    return np.concatenate([p, np.eye(m, dtype=np.uint8)], axis=1)


def gf_rank(a: np.ndarray) -> int:
    a = a.copy()
    rank = 0
    for c in range(a.shape[1]):
        piv = next((r for r in range(rank, a.shape[0]) if a[r, c]), None)
        if piv is None:
            continue
        a[[rank, piv]] = a[[piv, rank]]
        a[rank] = rn.MUL[rn.gf_div(1, int(a[rank, c])), a[rank]]
        for r in range(a.shape[0]):
            if r != rank and a[r, c]:
                a[r] ^= rn.MUL[int(a[r, c]), a[rank]]
        rank += 1
    return rank


def _keys(s: np.ndarray) -> np.ndarray:
    key = np.zeros(s.shape[:-1], dtype=np.uint64)
    for i in range(s.shape[-1]):
        key |= s[..., i].astype(np.uint64) << np.uint64(8 * i)
    return key


@functools.lru_cache(maxsize=None)
def syndrome_table(k: int, m: int, radius: int):
    """Sorted syndrome keys of every pattern of 1..radius wrong shards with every non-zero value, and its shards."""
    h = parity_check(k, m)
    n = k + m
    e = np.arange(1, 256, dtype=np.uint8)
    cols = [rn.MUL[e[:, None], h[:, j][None, :]] for j in range(n)]  # (255, m): e·h_j
    keys, a, b = [], [], []
    for j in range(n):
        keys.append(_keys(cols[j]))
        a.append(np.full(255, j, dtype=np.int8))
        b.append(np.full(255, -1, dtype=np.int8))
    if radius >= 2:
        for x in range(n):
            for y in range(x + 1, n):
                keys.append(_keys(cols[x][:, None, :] ^ cols[y][None, :, :]).ravel())
                a.append(np.full(255 * 255, x, dtype=np.int8))
                b.append(np.full(255 * 255, y, dtype=np.int8))
    keys, a, b = np.concatenate(keys), np.concatenate(a), np.concatenate(b)
    order = np.argsort(keys, kind="stable")
    keys, a, b = keys[order], a[order], b[order]
    assert (np.diff(keys) != 0).all(), "two patterns within the radius share a syndrome: the code is not MDS"
    return keys, a, b


def syndromes(shards: list[np.ndarray], k: int, m: int) -> np.ndarray:
    """(columns, m): parity recomputed from the data shards XOR the stored parity."""
    comp = rn.apply_rows(rn.build_matrix(k, k + m)[k:], list(shards[:k]))
    return np.stack([c ^ s for c, s in zip(comp, shards[k:])], axis=1)


def locate_columns(shards: list[np.ndarray], k: int, m: int, radius: int = 1):
    """Damaged column offsets and the one or two shards each is blamed on (-1: none; both -1: uncorrectable)."""
    s = syndromes(shards, k, m)
    cols = np.flatnonzero(s.any(axis=1))
    keys, a, b = syndrome_table(k, m, radius)
    q = _keys(s[cols])
    pos = np.minimum(np.searchsorted(keys, q), len(keys) - 1)
    found = keys[pos] == q
    return cols, np.where(found, a[pos], -1).astype(np.int64), np.where(found, b[pos], -1).astype(np.int64)


def _page_runs(cols: np.ndarray, length: int, shard_id: int) -> list[tuple[int, int, int]]:
    pages = np.unique(cols // PAGE)
    if not len(pages):
        return []
    cuts = np.flatnonzero(np.diff(pages) != 1) + 1
    out = []
    for run in np.split(pages, cuts):
        off = int(run[0]) * PAGE
        out.append((shard_id, off, min((int(run[-1]) + 1) * PAGE, length) - off))
    return out


def report(length: int, n: int, cols: np.ndarray, a: np.ndarray, b: np.ndarray) -> dict:
    """The report and ranges of include/swec.h from per-column blame, with "ok" as the file-level call returns it."""
    per = {sid: cols[(a == sid) | (b == sid)] for sid in range(n)}
    per = {sid: c for sid, c in per.items() if len(c)}
    unc = cols[(a < 0) & (b < 0)]
    ranges = []
    for sid, c in sorted(per.items()):
        ranges += _page_runs(c, length, sid)
    ranges += _page_runs(unc, length, -1)
    return {"ok": len(cols) == 0, "columns": length, "damaged_columns": len(cols), "uncorrectable_columns": len(unc),
            "first_uncorrectable": int(unc[0]) if len(unc) else -1,
            "last_uncorrectable": int(unc[-1]) if len(unc) else -1,
            "shards": {sid: (len(c), int(c[0]), int(c[-1])) for sid, c in per.items()},
            "ranges": ranges, "n_ranges": len(ranges)}


def locate(shards: list[np.ndarray], k: int, m: int, radius: int = 1) -> dict:
    return report(len(shards[0]), k + m, *locate_columns(shards, k, m, radius))
