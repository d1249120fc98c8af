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


# ---------------------------------------------------------------------------------------------- any m (up to 31)
# The functions above pack a syndrome into one uint64 and so stop at m = 8.  These key a syndrome by its m bytes,
# compared as a fixed-width string, decode the punctured code of a presence mask as well as the full code, and build the
# report from per-column blame with whole-array operations, so that it also serves 2^28-column shard sets on the GPU.


def byte_keys(s: np.ndarray) -> np.ndarray:
    """One key per row of s (..., c) uint8: its c bytes as a fixed-width string (any c)."""
    s = np.ascontiguousarray(s, dtype=np.uint8).reshape(-1, s.shape[-1])
    return s.view(np.dtype((np.void, s.shape[-1]))).ravel()


@functools.lru_cache(maxsize=None)
def punctured_rows(k: int, m: int, present: tuple | None = None):
    """(info ids, check ids, lost ids, P' = G[C]·G[I]^-1, R = G[lost]·G[I]^-1) for a presence mask: I the first k present
    shards, C the other present ones.  present None: the full code, P' = P."""
    g = rn.build_matrix(k, k + m)
    present = present or (True,) * (k + m)
    ids = [i for i in range(k + m) if present[i]]
    info, checks = ids[:k], ids[k:]
    lost = [i for i in range(k + m) if not present[i]]
    ginv = rn.mat_inv(g[info])
    pc = rn.mat_mul(g[checks], ginv) if checks else np.zeros((0, k), dtype=np.uint8)
    r = rn.mat_mul(g[lost], ginv) if lost else np.zeros((0, k), dtype=np.uint8)
    return info, checks, lost, pc, r


@functools.lru_cache(maxsize=None)
def error_table(k: int, m: int, radius: int, present: tuple | None = None):
    """Every pattern of 1..radius wrong positions of the (punctured) code with every non-zero value, sorted by byte key:
    (keys, syndromes (N, c), positions a < b (-1: none), values va, vb).  Positions [0, k) are the information set,
    [k, k+c) the check shards.  Asserts that no two patterns share a syndrome (the code is MDS within the radius)."""
    pc = punctured_rows(k, m, present)[3]
    c = pc.shape[0]
    h = np.concatenate([pc, np.eye(c, dtype=np.uint8)], axis=1)
    n = k + c
    e = np.arange(1, 256, dtype=np.uint8)
    cols = [rn.MUL[e[:, None], h[:, j][None, :]] for j in range(n)]  # (255, c): e·h_j
    syn, a, b, va, vb = [np.zeros((0, c), dtype=np.uint8)], [], [], [], []
    if radius >= 1:
        for j in range(n):
            syn.append(cols[j])
            a.append(np.full(255, j, dtype=np.int16))
            b.append(np.full(255, -1, dtype=np.int16))
            va.append(e)
            vb.append(np.zeros(255, dtype=np.uint8))
    if radius >= 2:
        for x in range(n):
            for y in range(x + 1, n):
                syn.append((cols[x][:, None, :] ^ cols[y][None, :, :]).reshape(-1, c))
                a.append(np.full(255 * 255, x, dtype=np.int16))
                b.append(np.full(255 * 255, y, dtype=np.int16))
                va.append(np.repeat(e, 255))
                vb.append(np.tile(e, 255))
    syn = np.concatenate(syn)
    a, b, va, vb = (np.concatenate(v) if v else np.zeros(0, dtype=t) for v, t in
                    ((a, np.int16), (b, np.int16), (va, np.uint8), (vb, np.uint8)))
    keys = byte_keys(syn)
    order = np.argsort(keys, kind="stable")
    keys, syn = keys[order], syn[order]
    assert not (keys[1:] == keys[:-1]).any(), "two patterns within the radius share a syndrome: the code is not MDS"
    return keys, syn, a[order], b[order], va[order], vb[order]


def decode_columns(shards: list, k: int, m: int, radius: int, present: tuple | None = None):
    """Damaged columns of a shard set (lost shards may be None) and what decoding within the radius finds in each:
    (cols, positions a, b (-1: none; both -1: uncorrectable), values va, vb, position -> shard id)."""
    info, checks, _, pc, _ = punctured_rows(k, m, present)
    comp = rn.apply_rows(pc, [shards[i] for i in info])
    s = np.stack([x ^ shards[i] for x, i in zip(comp, checks)], axis=1)
    cols = np.flatnonzero(s.any(axis=1))
    keys, _, a, b, va, vb = error_table(k, m, radius, present)
    q = byte_keys(s[cols])
    pos = np.minimum(np.searchsorted(keys, q), max(len(keys) - 1, 0))
    found = (keys[pos] == q) if len(keys) else np.zeros(len(cols), dtype=bool)
    pick = [np.where(found, v[pos] if len(v) else fill, fill) for v, fill in ((a, -1), (b, -1), (va, 0), (vb, 0))]
    return cols, pick[0].astype(np.int64), pick[1].astype(np.int64), pick[2].astype(np.uint8), \
        pick[3].astype(np.uint8), np.array(info + checks, dtype=np.int64)


def _runs(flags: np.ndarray, length: int, shard_id: int) -> list[tuple[int, int, int]]:
    """(shard id, offset, length) of every maximal run of flagged pages."""
    pages = np.flatnonzero(flags)
    if not len(pages):
        return []
    cut = np.flatnonzero(np.diff(pages) != 1) + 1
    starts, ends = pages[np.r_[0, cut]], pages[np.r_[cut - 1, len(pages) - 1]] + 1
    return [(shard_id, int(s) * PAGE, min(int(e) * PAGE, length) - int(s) * PAGE) for s, e in zip(starts, ends)]


def dense_report(a, b, damaged, n: int) -> dict:
    """damage_oracle.report from per-column blame: torch tensors over every column (on any device) of the shard ids a
    and b each column is blamed on (-1: none) and whether it is damaged.  One pass over the columns per shard, no Python
    loop per column, so it takes the 2^28 columns of a device call."""
    import torch
    length = damaged.numel()
    whole = length // PAGE * PAGE

    def summary(mask):
        cnt = int(mask.sum())
        if not cnt:
            return 0, -1, -1, np.zeros(0, dtype=bool)
        first = int(mask.to(torch.uint8).argmax())
        last = length - 1 - int(mask.flip(0).to(torch.uint8).argmax())
        flags = mask[:whole].view(-1, PAGE).any(1)
        if whole < length:
            flags = torch.cat([flags, mask[whole:].any().view(1)])
        return cnt, first, last, flags.cpu().numpy()

    shards, ranges = {}, []
    for sid in range(n):
        cnt, first, last, flags = summary((a == sid) | (b == sid))
        if cnt:
            shards[sid] = (cnt, first, last)
            ranges += _runs(flags, length, sid)
    unc, first_u, last_u, flags = summary(damaged & (a < 0) & (b < 0))
    ranges += _runs(flags, length, -1)
    n_damaged = int(damaged.sum())
    return {"ok": n_damaged == 0, "columns": length, "damaged_columns": n_damaged, "uncorrectable_columns": unc,
            "first_uncorrectable": first_u, "last_uncorrectable": last_u, "shards": shards, "ranges": ranges,
            "n_ranges": len(ranges)}
