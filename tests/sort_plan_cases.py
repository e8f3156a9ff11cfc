"""Consolidation's sort plans (csrc/sort.cu, csrc/consolidate.cu) at the sizes where they change, with the plan each
call ran as a witness.

`KeyPlan` and `expected_plan` mirror the plan table of sort.cu's header comment and the bit packing of
consolidate.cu: from the rows alone they say how many `radix_sort`, `chunk_sort`, `pack_keys` and `seg_reduce`
profile scopes a consolidation records, and how many bytes the two sort scopes account (the splitter plan's bytes
depend on its bucket count, so they show `nb`).  `check_plan` compares that with `Backend.profile_read()` and fails
with "plan X expected, Y ran".  The generators fix the key widths through the lanes' ranges; the expected rows come
from numpy (`exact_model.consolidate_np`), never from the oracle."""
import numpy as np

from dbsp_b200 import Proj, Schema, col, fanout_index, key, lval, rval, val
from exact_model import flips

# sort.cu
CS_HALF = 3072
SPLITTER_MODE_MIN_ROWS = 262_144
MAX_BUCKETS = 32_768
OVERSAMPLE = 8
LSD_MAX_ROWS = MAX_BUCKETS * 768   # 25 165 824: above, plain LSD


def n_buckets(n):
    """splitter mode's bucket count: 256, doubled while nb * 768 < n, at most MAX_BUCKETS"""
    nb = 256
    while nb * 768 < n and nb < MAX_BUCKETS:
        nb *= 2
    return nb


def sample_positions(n):
    """The rows k_sample reads (sort.cu): sample j of m = nb * OVERSAMPLE takes row lo + hash(j) % (hi - lo) of its
    stride [j n / m, (j + 1) n / m).  Mirrors sort.cu; a drift shows as a plan the witness did not expect."""
    m = n_buckets(n) * OVERSAMPLE
    j = np.arange(m, dtype=np.uint64)
    lo, hi = j * np.uint64(n) // np.uint64(m), (j + np.uint64(1)) * np.uint64(n) // np.uint64(m)
    x = j * np.uint64(0x9E3779B97F4A7C15)   # wraps mod 2^64, like the kernel
    x ^= x >> np.uint64(29)
    span = hi - lo
    return (lo + np.where(span > 0, x % np.maximum(span, np.uint64(1)), np.uint64(0))).astype(np.int64)


class KeyPlan:
    """What consolidate.cu's census makes of the rows: per-lane bits (0 for a lane that equals an earlier lane in
    every row), the key words' widths, W, whether lane 0 arrives ordered, whether the rows are ordered already."""

    def __init__(self, schema, cols, weights):
        raw = [np.asarray(c).view(np.uint64) for c in cols]
        keyed = [c ^ f for c, f in zip(raw, flips(schema))]
        L = len(keyed)
        # k_props compares the lanes' raw bits
        alias = [next((j for j in range(l) if np.array_equal(raw[l], raw[j])), -1) if l else -1 for l in range(L)]
        self.bits = [0 if alias[l] >= 0 else int(keyed[l].max() - keyed[l].min()).bit_length() for l in range(L)]
        total = sum(self.bits)
        if total <= 128:
            self.W, self.B = (1 if total <= 64 else 2), total
        else:   # whole lanes per word, last lane first
            words, used = [0], 0
            for b in reversed(self.bits):
                if used + b > 64:
                    words.append(0)
                    used = 0
                used += b
                words[-1] = used
            self.W, self.B = len(words), words
        # the census: inversions (row i-1 > row i), adjacent duplicates, zero weights
        gt, eq = np.zeros(len(keyed[0]) - 1, bool), np.ones(len(keyed[0]) - 1, bool)
        for c in keyed:
            gt |= eq & (c[:-1] > c[1:])
            eq &= c[:-1] == c[1:]
        self.ordered = not gt.any()
        self.presorted = self.W <= 2 and not self.ordered and self.bits[0] > 0 and bool(np.all(keyed[0][1:] >= keyed[0][:-1]))
        self.adoptable = self.ordered and not eq.any() and not np.any(np.asarray(weights) == 0)


class Plan:
    def __init__(self, name, counts):
        self.name, self.counts = name, counts


def _one_sort(n, b, ws, presorted, force_lsd):
    """(name, radix launches, radix bytes, chunk launches, chunk bytes) of one radix_sort_pairs call over n pairs of
    `ws` key words holding b bits (sort_impl)."""
    pair = 8 * ws + 4

    def lsd(m):
        p = min(-(-b // 8), 16)
        return 1 + p, m * 8 * ws + p * m * 2 * pair

    if n <= 1 or b <= 0:
        return "nothing to sort", 0, 0, 0, 0
    if force_lsd:
        return ("lsd",) + lsd(n) + (0, 0)
    if n <= CS_HALF:
        return "one chunk", 0, 0, 1, n * 2 * pair
    if presorted:
        return "chunks", 0, 0, 1, n * 2 * pair
    if n > LSD_MAX_ROWS:
        return ("lsd",) + lsd(n) + (0, 0)
    if n < SPLITTER_MODE_MIN_ROWS:
        if b <= 16:
            return ("lsd",) + lsd(n) + (0, 0)
        return "top digit", 2, n * 8 * ws + n * 2 * pair, 1, n * 2 * pair
    nb = n_buckets(n)
    sl, sb = lsd(nb * OVERSAMPLE)
    radix = sl + 1 + 3, sb + n * (8 * ws + 2) + n * 2 + 2 * n * 2 * (pair + 2)
    return (f"splitters({nb})",) + radix + (1, n * (2 * pair + 2))


def expected_plan(n, B, W, presorted=False, fallback=False, ordered=False, adopted=False):
    """The profile of one consolidation of n unordered rows whose key is W words: B bits (W <= 2, one sort over the
    whole key) or the list of the words' widths (W >= 3, one sort per word, least significant word first).
    presorted: lane 0 arrives ordered.  fallback: a bucket overflowed a chunk, every word is sorted again by LSD.
    ordered: the rows arrive ordered (no pack, no sort); adopted: ... and the input buffer becomes the batch."""
    if ordered:
        return Plan("adopted" if adopted else "ordered",
                    {"radix_sort": (0, 0), "chunk_sort": (0, 0), "pack_keys": 0, "seg_reduce": 0 if adopted else 1})
    words = [(B, W)] if W <= 2 else [(b, 1) for b in B]
    names, rl, rb, cl, cb = [], 0, 0, 0, 0
    for attempt in ((False, True) if fallback else (False,)):
        for b, ws in words:
            name, a, x, c, y = _one_sort(n, b, ws, presorted and W <= 2, attempt)
            names.append(name)
            rl, rb, cl, cb = rl + a, rb + x, cl + c, cb + y
    packs = (1 if W <= 2 else W) * (2 if fallback else 1)
    name = names[0] + (" -> lsd fallback" if fallback else "")
    if W > 2:
        name = f"{W} words, {name}"
    return Plan(name, {"radix_sort": (rl, rb), "chunk_sort": (cl, cb), "pack_keys": packs, "seg_reduce": 2 if fallback else 1})


def observed(prof):
    g = lambda k, f: prof.get(k, {}).get(f, 0)
    return {"radix_sort": (g("radix_sort", "launches"), g("radix_sort", "alg_bytes")),
            "chunk_sort": (g("chunk_sort", "launches"), g("chunk_sort", "alg_bytes")),
            "pack_keys": g("pack_keys", "launches"), "seg_reduce": g("seg_reduce", "launches")}


def check_plan(prof, n, kp, want, what):
    """The consolidation profiled in `prof` ran the plan `want` names (e.g. "splitters(32768) -> lsd fallback"),
    which is what the rows' key plan `kp` implies at n rows."""
    fallback = want.endswith("-> lsd fallback")
    exp = expected_plan(n, kp.B, kp.W, kp.presorted, fallback, kp.ordered, kp.adoptable)
    assert exp.name == want or exp.name.endswith(", " + want), f"{what}: the rows make plan {exp.name}, the case means {want}"
    got = observed(prof)
    if got != exp.counts:
        ran = [p.name for p in (expected_plan(n, kp.B, kp.W, ps, fb, kp.ordered, kp.adoptable)
                                for ps in (False, True) for fb in (False, True)) if p.counts == got]
        raise AssertionError(f"{what}: plan {exp.name} expected, {ran[0] if ran else got} ran (expected {exp.counts})")


# ---- generators: (schema, cols, weights); the leading lanes' ranges fix the key widths --------------------------
def u(a):
    return np.asarray(a).astype(np.uint64)


def one_word(n, seed):
    """(a): Schema("u","u"), 20 + 18 = 38 key bits"""
    rng = np.random.default_rng(seed)
    c0, c1 = u(rng.integers(0, 1 << 20, n)), u(rng.integers(0, 1 << 18, n))
    c0[:2], c1[:2] = (0, (1 << 20) - 1), (0, (1 << 18) - 1)
    return Schema("u", "u"), [c0, c1], rng.integers(-2, 3, n)


DISTS = ["uniform", "loguniform", "hitters", "fewvalues", "descending", "cancelling"]


def distribution(n, dist, seed):
    """(b): Schema("u","uu") with the key lane drawn from `dist` (the shapes of test_sort_splitter_mode, plus
    distinct keys in descending order, and rows whose weights cancel)"""
    rng = np.random.default_rng(seed)
    if dist == "uniform":
        k = rng.integers(0, 1 << 40, n)
    elif dist == "loguniform":   # prices: a quarter of the rows under one top-bits prefix
        k = np.ceil(np.power(10.0, rng.random(n) * 6.0) * 100.0).astype(np.int64)
    elif dist == "hitters":
        hot = rng.random(n) < 0.6
        k = np.where(hot, rng.choice(np.array([5, 77, 1 << 33]), n), rng.integers(0, 1 << 35, n))
    elif dist == "fewvalues":
        k = rng.integers(0, 7, n)
    elif dist == "descending":
        k = np.arange(n, 0, -1)
    else:
        k = rng.integers(0, 1 << 22, n)
    cols = [u(k), u(rng.integers(0, 1 << 18, n)), u(rng.integers(0, 50, n))]
    if dist == "hitters":   # whole rows repeat (equal packed keys): three rows hold 60 % of the input, odd buckets
        cols[1][hot], cols[2][hot] = 1000, 7
    w = rng.integers(-1, 3, n)
    if dist == "cancelling":   # the second half repeats rows of the first half with the weight negated
        h = n // 2
        pick = rng.integers(0, h, n - h)
        for c in cols:
            c[h:] = c[pick]
        w[h:] = -w[pick]
    return Schema("u", "uu"), cols, w


def ordered_rows(n, dups, seed):
    """(c): rows already in order.  dups=False: distinct rows, non-zero weights (the input buffer becomes the
    batch); dups=True: groups of four rows holding two distinct rows, weights in -1..1 (the identity-order
    epilogue sums them and drops zero sums)"""
    rng = np.random.default_rng(seed)
    if not dups:
        c0 = np.cumsum(rng.integers(1, 4, n)).astype(np.uint64)
        return Schema("u", "u"), [c0, u(rng.integers(0, 1 << 30, n))], rng.integers(1, 4, n) * rng.choice([-1, 1], n)
    i = np.arange(n)
    return Schema("u", "u"), [u(i // 4 * 3), u((i % 4) // 2)], rng.integers(-1, 2, n)


Q7 = Schema("u", "uuuuu")   # q7's bids_by_price: (price, auction, bidder, price, date_time, extra)


def q7_rows(n, seed, run=0):
    """(d): the q7 row shape, lane 3 always equal to lane 0 (left out of the key), more than 64 key bits.  run > 0:
    lane 0 is a time that arrives ordered, in runs of `run` equal values (bids_by_time); else a log-uniform price,
    with exact duplicates and rows that cancel"""
    rng = np.random.default_rng(seed)
    if run:
        lead = np.uint64(1436918400000) + u(np.arange(n) // run)
    else:
        lead = u(np.ceil(np.power(10.0, rng.random(n) * 6.0) * 100.0))
    cols = [lead, u(rng.integers(1000, 300_000, n)), u(rng.integers(1000, 100_000, n)), lead,
            np.uint64(1436918400000) + u(rng.integers(0, 10_000, n)), u(rng.integers(0, 1 << 32, n))]
    w = rng.integers(-1, 2, n)
    if not run:
        t = n // 10
        for c in cols:
            c[:t] = c[t:2 * t]
    return Q7, cols, w


def sample_defeating(n, seed, two_words=False):
    """(e): the smallest row at every row the splitter sample reads, distinct rows everywhere else: every splitter
    equals the smallest key and one even bucket holds almost every row, so a chunk overflows and the sort falls
    back to LSD.  two_words: the q7 row shape (two key words)."""
    rng = np.random.default_rng(seed)
    dense = u(rng.permutation(n) + 1)   # distinct, never the minimum
    pos = sample_positions(n)
    if two_words:
        schema, cols, w = q7_rows(n, seed)
        cols[0], cols[3] = dense, dense.copy()
        for c in cols:   # each lane's own minimum keeps the lanes' widths (and two key words)
            c[pos] = 0 if c is cols[0] or c is cols[3] else c.min()
    else:
        schema, cols, w = Schema("u", "u"), [dense, u(rng.integers(0, 1 << 12, n))], rng.integers(-2, 3, n)
        cols[1][pos] = 0
        cols[0][pos] = 0
    return schema, cols, w


HANDFUL = np.array([3, 1 << 21, (1 << 40) + 5, (1 << 61) + 17, (1 << 62) - 1], np.uint64)


def wide_rows(n, seed, defeat_word0=False):
    """(f): rows wider than 128 key bits, sorted word by word (consolidate.cu): lanes 0 and 1 take a handful of
    values spread over 62 bits each (a word of their own), lane 2 is random.  Rows equal in lanes 0 and 1 come out
    in lane 2 order only if every word's sort is stable.  defeat_word0: lane 2 (word 0) is the sample-defeating
    construction of `sample_defeating`, so word 0's sort falls back while words 1 and 2 still run their plan."""
    rng = np.random.default_rng(seed)
    if defeat_word0:
        c2 = u(rng.permutation(n) + 1)
        c2[sample_positions(n)] = 0
    else:
        c2 = u(rng.integers(0, 1 << 40, n))
    cols = [rng.choice(HANDFUL, n), rng.choice(HANDFUL, n), c2]
    return Schema("u", "uu"), cols, rng.integers(-1, 3, n)


def cancelling_runs(n, run, seed):
    """(g): n rows of two lanes: two rows repeated `run` times each, spread over the input, whose weights sum to 0
    (the row vanishes) and to i64::MIN (mod 2^64); every other row random"""
    rng = np.random.default_rng(seed)
    cols = [u(rng.integers(0, 1 << 20, n)), u(rng.integers(0, 1 << 17, n))]
    w = rng.integers(-3, 4, n)
    stride = n // (2 * run)
    for r, (row, target) in enumerate((((7, 9), 0), ((1 << 19, 3), -(1 << 63)))):
        at = np.arange(run) * stride * 2 + r * stride
        cols[0][at], cols[1][at] = row
        ws = rng.integers(-(1 << 63), (1 << 63) - 1, run, dtype=np.int64)
        last = (target - int(ws[:-1].view(np.uint64).sum())) & ((1 << 64) - 1)   # the sum wraps mod 2^64
        ws[-1] = last - (1 << 64) if last >> 63 else last
        w[at] = ws
    return Schema("u", "u"), cols, w


# ---- how users get there: closures whose model is one numpy line ---------------------------------------------
HOP = 2000


def fanout_table(n, seed, n_out=64):
    """(h) batch_from_table with the fan-out (col(0), col(1) - j * 2000): the shape of q5's hopping windows.
    Returns (table cols, weights, proj, model schema, model cols, model weights)."""
    rng = np.random.default_rng(seed)
    cols = [u(rng.integers(0, 1 << 20, n)), u(rng.integers(0, 1 << 16, n)) + np.uint64(HOP * n_out)]
    w = rng.integers(-2, 3, n)
    proj = Proj(Schema("u", "u"), [col(0), col(1) - fanout_index() * HOP], fanout=n_out)
    j = np.arange(n_out, dtype=np.uint64) * np.uint64(HOP)
    out = [np.repeat(cols[0], n_out), np.repeat(cols[1], n_out) - np.tile(j, n)]
    return cols, w, proj, proj.schema, out, np.repeat(w, n_out)


def fanout_map(rows, n_out=32):
    """(h) map_index with the fan-out (val(0), key(0) + j * 1000) over the consolidated rows (cols, weights) of a
    Schema("u","u") batch"""
    (k, v), w = rows
    proj = Proj(Schema("u", "u"), [val(0), key(0) + fanout_index() * 1000], fanout=n_out)
    j = np.arange(n_out, dtype=np.uint64) * np.uint64(1000)
    n = len(w)
    return proj, [np.repeat(v, n_out), np.repeat(k, n_out) + np.tile(j, n)], np.repeat(w, n_out)


def join_sides(n_keys, n_left, n_right, seed):
    """(h) join_batches inputs: every key holds n_left left values and n_right right values (14 bits each, distinct
    per key), so the join has n_keys * n_left * n_right rows; the projection (rval, lval) drops the key and
    equal pairs of different keys sum.  Returns (left cols, left w, right cols, right w, proj, model)."""
    rng = np.random.default_rng(seed)
    k = np.arange(n_keys, dtype=np.uint64)[:, None]
    lv = (u(rng.integers(0, 1 << 14, (n_keys, 1))) + np.arange(n_left, dtype=np.uint64) * np.uint64(97)) & np.uint64((1 << 14) - 1)
    rv = (u(rng.integers(0, 1 << 14, (n_keys, 1))) + np.arange(n_right, dtype=np.uint64) * np.uint64(151)) & np.uint64((1 << 14) - 1)
    lw = rng.choice(np.array([-2, -1, 1, 2]), (n_keys, n_left))
    rw = rng.choice(np.array([-2, -1, 1, 3]), (n_keys, n_right))
    left = [np.broadcast_to(k, lv.shape).ravel(), lv.ravel()]
    right = [np.broadcast_to(k, rv.shape).ravel(), rv.ravel()]
    proj = Proj(Schema("u", "u"), [rval(0), lval(0)])
    shape = (n_keys, n_left, n_right)
    model = [np.broadcast_to(rv[:, None, :], shape).ravel(), np.broadcast_to(lv[:, :, None], shape).ravel()]
    return left, lw.ravel(), right, rw.ravel(), proj, (model, (lw[:, :, None] * rw[:, None, :]).ravel())
