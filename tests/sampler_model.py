"""Exact model of the device triple sampler (mmssl_b200/csrc/sampler.cu) in plain numpy: the same counter RNG, the same claim
rounds and select keys, the same positive / negative draws, so that a batch of the kernels can be compared with it bit for bit.

  rnd32(seed, step, t, draw)   splitmix64(splitmix64(seed ^ (step << 32 | t)) + draw) >> 32
  below(r, n)                  (r * n) >> 32 (multiply-shift range reduction)
  slot_key(seed, step, s)      hash32(seed ^ KEY_STREAM ^ (step << 32 | s)) << 32 | s

One CTA (batch <= 1024, ``one_cta``): without replacement, rounds of "every pending thread draws a candidate slot; of the
threads that drew a free slot the smallest id wins it"; a thread's draw counter advances only in the rounds it takes part in.
Threads still pending after ROUNDS rounds are served by the claim finish: the free slots in cyclic order from a start drawn
from the finish stream, handed out in thread order.  Any batch (``multi``): the slots of the `batch` smallest keys, in key
order.  With replacement (batch > n_exist) both paths draw one uniform slot per thread, so its triple's draws start at 1.

A triple (``draw_triple``): positive = row[below(rnd, deg)]; negative = below(rnd, n_items) rejected while it is in the row,
at most NEG_TRIES times, then the j-th item missing from the row, j = below(rnd, n_items - deg).

``info`` of every call reports which rare branches the batch took: ``finish`` (threads served by the claim finish) and
``fallback`` (triples whose negative came from the complement draw); ``slots`` are the triples' slots (for ``owned``)."""
from __future__ import annotations

import numpy as np

KEY_STREAM = 0x6A09E667F3BCC908
FINISH_STREAM = 0xBB67AE8584CAA73B
ROUNDS = 64
NEG_TRIES = 4096
ONE_CTA_MAX = 1024


def splitmix64(x):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def _u64(v):
    return np.uint64(int(v) & 0xFFFFFFFFFFFFFFFF)


def rnd32(seed, step, t, draw):
    """uint32 draw number `draw` of thread `t` (arrays broadcast)."""
    t = np.asarray(t, dtype=np.uint64)
    draw = np.asarray(draw, dtype=np.uint64)
    base = splitmix64(_u64(seed) ^ ((_u64(step) << np.uint64(32)) | t))
    with np.errstate(over="ignore"):
        return (splitmix64(base + draw) >> np.uint64(32)).astype(np.uint64)


def below(r, n):
    """uint32 r -> [0, n): (r * n) >> 32, n < 2^32."""
    return ((np.asarray(r, dtype=np.uint64) * np.asarray(n, dtype=np.uint64)) >> np.uint64(32)).astype(np.int64)


def slot_key(seed, step, s):
    s = np.asarray(s, dtype=np.uint64)
    h = splitmix64(splitmix64(_u64(seed) ^ np.uint64(KEY_STREAM) ^ ((_u64(step) << np.uint64(32)) | s))) >> np.uint64(32)
    return (h << np.uint64(32)) | s


def finish_start(seed, step, n_exist):
    """First slot of the claim finish's cyclic sweep."""
    return int(below(rnd32(_u64(seed) ^ np.uint64(FINISH_STREAM), step, 0, 0), n_exist))


def slot_bits(n_exist):
    b = 1
    while (1 << b) < n_exist:
        b += 1
    return b


# ------------------------------------------------------------------------------------------------------------ slot choice
def claim_slots(seed, step, n_exist, batch):
    """One-CTA slots of threads 0..batch-1 and each thread's next unused draw number; info["finish"] = threads the finish
    served."""
    t_all = np.arange(batch, dtype=np.int64)
    if batch > n_exist:
        return below(rnd32(seed, step, t_all, 0), n_exist), np.ones(batch, np.int64), {"finish": 0}
    slots = np.full(batch, -1, np.int64)
    draws = np.zeros(batch, np.int64)
    taken = np.zeros(n_exist, bool)
    pending = t_all
    for _ in range(ROUNDS):
        cand = below(rnd32(seed, step, pending, draws[pending]), n_exist)
        draws[pending] += 1
        free = ~taken[cand]
        # pending is ascending: the first occurrence of a candidate is its smallest contender
        fc, ft = cand[free], pending[free]
        _, first = np.unique(fc, return_index=True)
        win_t, win_s = ft[first], fc[first]
        slots[win_t] = win_s
        taken[win_s] = True
        won = np.zeros(batch, bool)
        won[win_t] = True
        pending = pending[~won[pending]]
        if len(pending) == 0:
            break
    n_fin = len(pending)
    if n_fin:
        start = finish_start(seed, step, n_exist)
        order = (start + np.arange(n_exist)) % n_exist
        free_slots = order[~taken[order]]
        slots[pending] = free_slots[:n_fin]
    return slots, draws, {"finish": n_fin}


def select_slots(seed, step, n_exist, batch):
    """Multi-CTA slots: the `batch` smallest keys in key order (distinct), or with replacement above n_exist."""
    if batch > n_exist:
        return below(rnd32(seed, step, np.arange(batch), 0), n_exist), np.ones(batch, np.int64)
    keys = slot_key(seed, step, np.arange(n_exist, dtype=np.uint64))
    if batch < n_exist:
        part = np.argpartition(keys, batch - 1)[:batch]
        sel = part[np.argsort(keys[part])]
    else:
        sel = np.argsort(keys)
    return sel.astype(np.int64), np.zeros(batch, np.int64)


# ------------------------------------------------------------------------------------------------------------ the triples
class Rows:
    """The training matrix as the kernels see it: sorted CSR rows and the slots (rows with >= 1 item, ascending)."""

    def __init__(self, csr):
        csr = csr.tocsr()
        csr.sort_indices()
        self.indptr = np.asarray(csr.indptr, np.int64)
        self.indices = np.asarray(csr.indices, np.int64)
        self.n_users, self.n_items = csr.shape
        self.exist = np.nonzero(np.diff(self.indptr) > 0)[0].astype(np.int64)
        self._pairs()

    def _pairs(self):
        """row * n_items + item of every entry: ascending, as the rows are sorted."""
        self.pairs = np.repeat(np.arange(self.n_users, dtype=np.int64), np.diff(self.indptr)) * self.n_items + self.indices

    @classmethod
    def from_arrays(cls, indptr, indices, n_items):
        self = cls.__new__(cls)
        self.indptr = np.asarray(indptr, np.int64)
        self.indices = np.asarray(indices, np.int64)
        self.n_users, self.n_items = len(self.indptr) - 1, int(n_items)
        self.exist = np.nonzero(np.diff(self.indptr) > 0)[0].astype(np.int64)
        self._pairs()
        return self

    @property
    def n_exist(self):
        return len(self.exist)


def draw_triples(rows, slots, draws, seed, step):
    """[3, B] int64 (users, pos, neg) of threads 0..B-1 with their slots and next draw numbers; and the number of triples whose
    negative came from the complement fallback."""
    B = len(slots)
    t = np.arange(B, dtype=np.int64)
    r = rows.exist[slots]
    b, e = rows.indptr[r], rows.indptr[r + 1]
    deg = e - b
    d = draws.copy()
    pos = rows.indices[b + below(rnd32(seed, step, t, d), deg)]
    d += 1
    n_items = rows.n_items
    neg = np.zeros(B, np.int64)
    left = np.arange(B)
    for _ in range(NEG_TRIES):
        ng = below(rnd32(seed, step, t[left], d[left]), n_items)
        d[left] += 1
        neg[left] = ng
        # the binary search of the kernel: the first entry of the row >= ng (rows are sorted runs of `pairs`)
        key = r[left] * n_items + ng
        j = np.minimum(np.searchsorted(rows.pairs, key, side="left"), len(rows.pairs) - 1)
        left = left[rows.pairs[j] == key]
        if len(left) == 0:
            break
    for i in left:              # the complement draw: the j-th item missing from the sorted row
        row = rows.indices[b[i]:e[i]]
        if len(row) >= n_items:
            continue            # a full row has no negative (refused by the sampler classes)
        j = int(below(rnd32(seed, step, t[i], d[i]), n_items - len(row)))
        m = int(np.searchsorted(row - np.arange(len(row)), j, side="right"))
        neg[i] = j + m
    return np.stack([r, pos, neg]), len(left)


def one_cta(rows, batch, seed, step):
    """The batch of ``mmssl_sample_triples`` (batch <= 1024) and info {"finish", "fallback", "slots"}."""
    assert 1 <= batch <= ONE_CTA_MAX
    slots, draws, info = claim_slots(seed, step, rows.n_exist, batch)
    out, info["fallback"] = draw_triples(rows, slots, draws, seed, step)
    info["slots"] = slots
    return out, info


def multi(rows, batch, seed, step):
    """The batch of ``mmssl_sample_triples_multi`` (any batch) and info {"finish": 0, "fallback", "slots"}."""
    slots, draws = select_slots(seed, step, rows.n_exist, batch)
    out, fb = draw_triples(rows, slots, draws, seed, step)
    return out, {"finish": 0, "fallback": fb, "slots": slots}


def sample(rows, batch, seed, step):
    """``DeviceTripleSampler.sample_into``: one CTA up to 1024 triples, the select above."""
    return one_cta(rows, batch, seed, step) if batch <= ONE_CTA_MAX else multi(rows, batch, seed, step)


def owned(out, slots, slot_lo, slot_hi):
    """The owned (row-sharded) form of a batch `out` whose triples have slots `slots`: entries whose slot lies outside
    [slot_lo, slot_hi) are zero (the kernels add row0 to the local row, which gives the global user again)."""
    keep = (slots >= slot_lo) & (slots < slot_hi)
    return np.where(keep[None, :], out, 0)
