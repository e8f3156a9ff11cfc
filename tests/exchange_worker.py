"""The in-library exchange (csrc/comm.cu) on ONE GPU: P contexts of this process, one worker thread per rank, the
model the reference's runtime uses (one thread per worker) and the same-process branch of dbsp_comm_connect (peers
reached through their raw pointers).  Every kernel of comm.cu and the whole round protocol run here; only the CUDA
IPC mapping between processes and the NVLink transport do not (tests/test_multigpu.py covers those on >= 2 GPUs).

    python tests/exchange_worker.py <scenario> <P>      prints EXCHANGE_OK on success

Run by tests/test_gpu_exchange.py in a subprocess with CUDA_DEVICE_MAX_CONNECTIONS=32 (no peer's signal kernel
queued behind a spinning wait kernel in a shared hardware queue), a bounded DBSP_COMM_TIMEOUT_S (a protocol bug
ends as an error status, not a long wait), DBSP_POOL_SLAB_MB (P pools on one card) and CUDA_MODULE_LOADING=EAGER
(ranks on one device share one CUDA context; under lazy loading a rank's first launch of a kernel would wait for a
peer's spinning wait kernel, so dbsp_comm_connect refuses that setup).

Rules of the harness:
  * every rank thread issues the same sequence of exchange calls (SPMD); ranks start, and enter rounds, at
    slightly different times so that the order in which they arrive varies;
  * no assertion between exchange calls: a rank that stopped early would leave its peers waiting for its flag.
    A rank thread only downloads its outputs to numpy; all comparisons with the model (tests/exchange_model.py)
    happen after every thread has joined;
  * every library object stays in the thread that made it (a context's pool is not thread-safe, so a batch must
    not be freed by another thread): rank threads return numpy data only."""
import os
import sys
import threading
import time
import traceback

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import numpy as np

import edge_cases as ec
import exact_model as em
import exchange_model as xm
from dbsp_b200 import Schema
from dbsp_b200._capi import DbspError
from exact_model import MAX, MIN, UMAX

CONCAT_SORT_MAX_ROWS = 1 << 20   # comm.cu: above this many received rows the receiver merges by a tree
SIZES = [0, 1, 31, 32, 33, 2047, 2048, 2049, 3 * 2048 + 1, 5 * 2048]   # PT_TILE = 2048, lane stride padding 32


def seg_bytes(n, L):
    """Bytes of one received segment of n rows and L lanes (lane stride = n rounded up past n to 32 rows)."""
    return ((n + 32) & ~31) * 8 * (L + 1)


def slot_for(*segs):
    """slot_bytes holding the given (rows, lanes) segments of one round, each starting 256-byte aligned."""
    return sum((seg_bytes(n, L) + 255) & ~255 for n, L in segs) + 4096


class Group:
    """P contexts on device 0 connected as one exchange group through the same-process branch of comm_connect."""

    def __init__(self, P, slot_bytes, make_backend=None):
        if make_backend is None:
            from dbsp_b200.runtime import Runtime

            make_backend = lambda: Runtime(0)
        self.P, self.calls = P, 0
        self.bes = [make_backend() for _ in range(P)]
        blobs = b"".join(be.comm_create(r, P, slot_bytes) for r, be in enumerate(self.bes))
        for be in self.bes:   # every context maps every region before any rank starts
            be.comm_connect(blobs)

    def run(self, fn):
        """fn(rank, backend) on P threads; returns the P results after all have joined."""
        P = self.P
        self.calls += 1
        out, err = [None] * P, [None] * P

        def body(r):
            time.sleep(0.002 * ((3 * r + self.calls) % 5))
            try:
                out[r] = fn(r, self.bes[r])
            except BaseException:
                err[r] = traceback.format_exc()

        ts = [threading.Thread(target=body, args=(r,)) for r in range(P)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        bad = [f"rank {r}:\n{e}" for r, e in enumerate(err) if e]
        if bad:
            raise RuntimeError("\n".join(bad))
        return out

    def close(self):
        for be in self.bes:
            be.comm_destroy()
            be.close()


def jitter(r, k):
    """A rank- and round-dependent pause before a round: the arrival order of the ranks changes every round."""
    time.sleep(1e-4 * ((5 * r + 3 * k) % 7))


def sent(be):
    return be.comm_info()[2]


# ---- inputs ------------------------------------------------------------------------
def full_rows(rng, schema, n):
    """n rows of full-range lanes with extremes, repeated rows and edge weights (numpy uint64 columns, int64 weights)."""
    return ec.with_duplicates(rng, [ec.full_lane(rng, t, n) for t in schema.lanes], ec.edge_weights(rng, n))


def cat(schema, *parts):
    parts = [p for p in parts if len(p[1])]
    if not parts:
        return [np.zeros(0, np.uint64) for _ in range(schema.nl)], np.zeros(0, np.int64)
    return [np.concatenate([p[0][l] for p in parts]) for l in range(schema.nl)], np.concatenate([p[1] for p in parts])


def rows_to(rng, schema, counts, pools):
    """Distinct rows, counts[p] of them owned by rank p (keys drawn without repeats from pools[p], values full-range)."""
    parts = []
    for p, c in enumerate(counts):
        if c == 0:
            continue
        idx = rng.choice(len(pools[p][0]), c, replace=False)
        keys = [k[idx] for k in pools[p]]
        vals = [ec.full_lane(rng, t, c) for t in schema.val]
        parts.append((keys + vals, ec.edge_weights(rng, c)))
    return cat(schema, *parts)


def upload(be, schema, inp):
    return be.batch_from_columns(schema, inp[0], inp[1])


# ---- checks (main thread, after the join) ------------------------------------------
def check(schema, got, expect, what):
    em.assert_download_is(schema, got, expect, what)


def check_empty(got, what):
    assert len(got["diffs"]) == 0, f"{what}: {len(got['diffs'])} tuples, expected none"


def same(a, b, what):
    """Two downloads are bit for bit the same batch."""
    assert len(a["diffs"]) == len(b["diffs"]), f"{what}: {len(a['diffs'])} vs {len(b['diffs'])} tuples"
    for part in ("keys", "vals"):
        for i, (x, y) in enumerate(zip(a[part], b[part])):
            assert np.array_equal(x, y), f"{what}: {part} lane {i} differs"
    if a["offs"] is not None:
        assert np.array_equal(a["offs"], b["offs"]), f"{what}: offs differ"
    assert np.array_equal(a["diffs"], b["diffs"]), f"{what}: weights differ"


def check_bytes(schema_rounds, P, got_bytes, what):
    """got_bytes[r] = bytes rank r's dbsp_comm_info count grew by; schema_rounds = [(schema, inputs, root)]."""
    for r in range(P):
        want = sum(xm.bytes_sent(s, inputs[r], r, P, root) for s, inputs, root in schema_rounds)
        assert got_bytes[r] == want, f"{what}: rank {r} counted {got_bytes[r]} bytes sent, model {want}"


# ---- scenarios ---------------------------------------------------------------------
ALLREDUCE_TOPS = [[1 << 63, (1 << 63) - 1, 0], [UMAX, (1 << 63) - 1, 1 << 63, 0], [(1 << 63) - 1, 0, 3],
                  [UMAX - 1, 1 << 63, (1 << 63) - 1, 0], [(1 << 63) + 1, 1 << 63, (1 << 63) - 1, 0], [UMAX, 0, 1],
                  [1 << 62, 0, 5]]


def allreduce_values(P, k):
    """P distinct values of round k, the maximum first in the list, on rank (3k + 1) % P; every round's maximum
    differs from the two rounds before it, so a value read from the other parity's slot (or a stale one) shows."""
    vals = (ALLREDUCE_TOPS[k % len(ALLREDUCE_TOPS)] + [1000 + j for j in range(P)])[:P]
    m = (3 * k + 1) % P
    return [vals[(r - m) % P] for r in range(P)]


def scenario_allreduce(P):
    rounds = 2 * len(ALLREDUCE_TOPS)
    s = Schema("u", "i")
    rng = np.random.default_rng(100 + P)
    shard_in = {k: [full_rows(rng, s, 20 + 13 * r) for r in range(P)] for k in range(1, rounds, 2)}
    g = Group(P, slot_for((20 + 13 * P, 2)))

    def rank(r, be):
        red, shards = [], {}
        for k in range(rounds):
            jitter(r, k)
            red.append(be.allreduce_max(allreduce_values(P, k)[r]))
            if k in shard_in:   # the exchange rounds' sequence numbers run apart from the reductions'
                shards[k] = be.shard(upload(be, s, shard_in[k][r])).download()
        return red, shards

    out = g.run(rank)
    g.close()
    for k in range(rounds):
        want = xm.allreduce_max(allreduce_values(P, k))
        for r in range(P):
            assert out[r][0][k] == want, f"allreduce round {k} rank {r}: {out[r][0][k]:#x}, model {want:#x}"
    for k, inputs in shard_in.items():
        model = xm.shard(s, inputs, P)
        for r in range(P):
            check(s, out[r][1][k], model[r], f"shard between reductions, round {k} rank {r}")


def scenario_shard_model(P):
    small = P > 8
    sizes = [0, 1, 5, 40, 200] if small else [0, 3, 300, 2500, 9000]
    cases = []
    rng = np.random.default_rng(200 + P)
    for i, s in enumerate(ec.SCHEMAS):
        shared = full_rows(rng, s, 64)   # the same rows on several ranks: equal rows from several sources meet
        inputs = []
        for r in range(P):
            own = full_rows(rng, s, sizes[(i + r) % len(sizes)])
            pick = rng.random(64) < 0.5
            inputs.append(cat(s, own, ([c[pick] for c in shared[0]], ec.edge_weights(rng, int(pick.sum())))))
        cases.append((s, inputs))
    g = Group(P, slot_for((max(sizes) + 64, 8)))

    def rank(r, be):
        res = []
        b0 = sent(be)
        for k, (s, inputs) in enumerate(cases):
            jitter(r, k)
            got = be.shard(upload(be, s, inputs[r])).download()
            union = be.batch_from_columns(s, *cat(s, *inputs))
            part = be.shard_partition(union, P)[r].download()   # k_shard_flags: the other CUDA hash
            res.append((got, part))
        return res, sent(be) - b0

    out = g.run(rank)
    g.close()
    for k, (s, inputs) in enumerate(cases):
        model = xm.shard(s, inputs, P)
        owners = {}
        for r in range(P):
            got, part = out[r][0][k]
            check(s, got, model[r], f"shard {ec.sid(s)} rank {r}")
            check(s, part, model[r], f"shard_partition(union) {ec.sid(s)} part {r}")
            for key in zip(*[x.tolist() for x in got["keys"]]):
                assert owners.setdefault(key, r) == r, f"{ec.sid(s)}: key {key} on ranks {owners[key]} and {r}"
    check_bytes([(s, inputs, None) for s, inputs in cases], P, [o[1] for o in out], "shard_model")


def scenario_sizes(P):
    n = len(SIZES)
    rng = np.random.default_rng(300 + P)
    su, si = Schema("u", "u"), Schema("i", "iu")
    pools = xm.keys_with_dest(rng, si.nk, P, max(SIZES))
    rounds = []
    for j in range(n):   # per-rank input sizes around the tile (k_shard_hist, k_shard_scatter2)
        rounds.append((su, [full_rows(rng, su, SIZES[(j + r) % n]) for r in range(P)]))
    for j in range(n):   # per-destination segment sizes around the 32-row padding and the tile
        rounds.append((si, [rows_to(rng, si, [SIZES[(j + 3 * r + p) % n] for p in range(P)], pools) for r in range(P)]))
    g = Group(P, slot_for((max(SIZES), 3)))

    def rank(r, be):
        b0, res = sent(be), []
        for k, (s, inputs) in enumerate(rounds):
            jitter(r, k)
            res.append(be.shard(upload(be, s, inputs[r])).download())
        return res, sent(be) - b0

    out = g.run(rank)
    g.close()
    for k, (s, inputs) in enumerate(rounds):
        model = xm.shard(s, inputs, P)
        for r in range(P):
            check(s, out[r][0][k], model[r], f"sizes round {k} rank {r}")
    check_bytes([(s, inputs, None) for s, inputs in rounds], P, [o[1] for o in out], "sizes")


def path_round(rng, s, P, totals, pool):
    """Inputs whose segments to rank p add up to exactly totals[p] rows, every sender non-empty towards every p
    with totals[p] >= P.  Senders overlap in keys (values follow the key), so equal rows meet from several sources."""
    inputs = [[] for _ in range(P)]
    for p, t in enumerate(totals):
        if t == 0:
            continue
        per = [t // P + (1 if r < t % P else 0) for r in range(P)]
        step = max(1, (len(pool[p][0]) - max(per)) // max(P - 1, 1))
        for r, c in enumerate(per):
            keys = [k[r * step: r * step + c] for k in pool[p]]
            vals = [(keys[0] * np.uint64(3 + l)) ^ (em.SIGN if t_ == "i" else np.uint64(0)) for l, t_ in enumerate(s.val)]
            inputs[r].append((keys + vals, ec.edge_weights(rng, c)))
    return [cat(s, *parts) for parts in inputs]


def scenario_receiver_paths(P):
    """P >= 3: exactly 2^20 received rows (one rank-merge launch, k_pway_rank + seg_reduce) and 2^20 + 1 (the merge
    tree, merge_tiles), told apart by the kernels' profiler names on the receiving context; P = 2: the tree."""
    s = Schema("i", "u")
    rng = np.random.default_rng(400 + P)
    T = CONCAT_SORT_MAX_ROWS
    totals = [T, T + 1] + [50 * P + r for r in range(2, P)] if P >= 3 else [T, 3000]
    per_max = T // P + 1
    pool = xm.keys_with_dest(rng, 1, P, [int(per_max * 1.6) + 64 if t >= P else t + 64 for t in totals])
    inputs = path_round(rng, s, P, totals, pool)
    g = Group(P, slot_for((per_max, 2)))

    def rank(r, be):
        b = upload(be, s, inputs[r])
        be.sync()
        be.profile(True)
        got = be.shard(b)
        prof = sorted(be.profile_read())
        be.profile(False)
        return got.download(), prof

    out = g.run(rank)
    g.close()
    model = xm.shard(s, inputs, P)
    for r in range(P):
        check(s, out[r][0], model[r], f"receiver rank {r} ({totals[r]} rows received)")
    for r in range(P):
        prof = out[r][1]
        if P >= 3 and totals[r] <= T:
            assert "merge_tiles" not in prof and "seg_reduce" in prof, (f"rank {r}, {totals[r]} rows from {P} sources: "
                                                                     f"not the rank merge: {prof}")
        else:
            assert "merge_tiles" in prof, f"rank {r}, {totals[r]} rows: not the merge tree: {prof}"


def cancel_round(rng, s, P, d, pool, m, pure):
    """Every row owned by rank d.  A: m rows on rank 0, the same rows on rank 1 with the negated weights (mod 2^64:
    MIN stays MIN); S: fresh rows on ranks >= 2 that survive.  `pure`: nothing else, so that the segments of ranks 0
    and 1 cancel completely and the merge of what is left starts from an empty batch.  Otherwise also X: one row on
    ranks 0 and 1 with weight MIN each; Y: one row whose weights on up to four ranks sum to 0 only mod 2^64; Z: one
    row on every rank that survives."""
    keys = pool[d]
    ka = [k[:m] for k in keys]
    wa = ec.edge_weights(rng, m)
    va = [ec.full_lane(rng, t, m) for t in s.val]
    kx, ky, kz = ([k[m + i: m + i + 1] for k in keys] for i in range(3))
    val1 = [np.array([em.u64(MAX if t == "i" else UMAX)], np.uint64) for t in s.val]
    yw = {2: [-(1 << 62), 1 << 62], 3: [1 << 62, 1 << 62, MIN]}.get(P, [1 << 62] * 4)
    inputs = []
    for r in range(P):
        parts = []
        if r == 0:
            parts.append((ka + va, wa))
        if r == 1:
            parts.append((ka + va, (np.uint64(0) - wa.view(np.uint64)).view(np.int64)))
        if r < 2 and not pure:
            parts.append((kx + val1, np.array([MIN], np.int64)))
        if r < len(yw) and not pure:
            parts.append((ky + val1, np.array([yw[r]], np.int64)))
        if not pure:
            parts.append((kz + val1, np.array([ec.W_POOL[r % len(ec.W_POOL)]], np.int64)))
        if r >= 2:
            c = 40 + 5 * r
            off = m + 3 + 200 * r
            parts.append(([k[off: off + c] for k in keys] + [ec.full_lane(rng, t, c) for t in s.val], ec.edge_weights(rng, c)))
        inputs.append(cat(s, *parts))
    gone = [] if pure else [tuple(int(k[0]) for k in kx), tuple(int(k[0]) for k in ky)]
    return inputs, gone


def scenario_cancel_across_ranks(P):
    s = Schema("i", "u")
    rng = np.random.default_rng(500 + P)
    big = CONCAT_SORT_MAX_ROWS // 2 + 1000   # rank 0 + rank 1 > 2^20 rows: the tree; small: the rank merge
    pool = xm.keys_with_dest(rng, 1, P, big + 3 + 200 * P + 64)
    rounds = []
    for m, d, pure in ((3000, 0, False), (big, 1 % P, True), (big, P - 1, False), (2000, P // 2, True)):
        inputs, gone = cancel_round(rng, s, P, d, pool, m, pure)
        rounds.append((d, m, pure, inputs, gone))
    g = Group(P, slot_for((big + 8, 2)))

    def rank(r, be):
        res = []
        for k, (d, m, pure, inputs, gone) in enumerate(rounds):
            jitter(r, k)
            res.append(be.shard(upload(be, s, inputs[r])).download())
        return res

    out = g.run(rank)
    g.close()
    for k, (d, m, pure, inputs, gone) in enumerate(rounds):
        model = xm.shard(s, inputs, P)
        keys = set(model[d][0][0].tolist())
        assert not any(key[0] in keys for key in gone), "the model keeps a row whose weights sum to 0 mod 2^64"
        assert len(model[d][1]) == (sum(40 + 5 * r for r in range(2, P)) + (0 if pure else 1))   # S (+ Z) survive
        for r in range(P):
            check(s, out[r][k], model[r], f"cancel round {k} ({m} cancelling rows{', nothing else' if pure else ''}, "
                                          f"owner {d}) rank {r}")


def scenario_gather(P):
    s = Schema("uu", "i")
    rng = np.random.default_rng(600 + P)
    rounds = []
    for root in range(P):
        shared = full_rows(rng, s, 16)
        rounds.append((root, [cat(s, full_rows(rng, s, 30 + 7 * r), shared) for r in range(P)]))
        lone = (root + 1) % P if root % 2 == 0 else root   # a lone segment from a peer, or the root's own
        rounds.append((root, [full_rows(rng, s, 500) if r == lone else full_rows(rng, s, 0) for r in range(P)]))
        rounds.append((root, [full_rows(rng, s, 0) for r in range(P)]))
    g = Group(P, slot_for((500 + 16, 3)))

    def rank(r, be):
        b0, res = sent(be), []
        for k, (root, inputs) in enumerate(rounds):
            jitter(r, k)
            res.append(be.gather(upload(be, s, inputs[r]), root).download())
        return res, sent(be) - b0

    out = g.run(rank)
    g.close()
    for k, (root, inputs) in enumerate(rounds):
        model = xm.gather(s, inputs, root, P)
        for r in range(P):
            check(s, out[r][0][k], model[r], f"gather round {k} to root {root}, rank {r}")
    check_bytes([(s, inputs, root) for root, inputs in rounds], P, [o[1] for o in out], "gather")


def scenario_shard2(P):
    sa, sb = Schema("u", "uu"), Schema("i", "i")
    rng = np.random.default_rng(700 + P)
    near = [31, 32, 33, 63, 64, 65, 0, 1]   # the first stream's segment ends just below / at / above a 32-row stride
    pools = xm.keys_with_dest(rng, sa.nk, P, max(near))
    rounds = [
        ([full_rows(rng, sa, 0 if r % 2 == 0 else 300 + r) for r in range(P)],
         [full_rows(rng, sb, 0 if r % 3 == 0 else 200 + 3 * r) for r in range(P)]),
        ([rows_to(rng, sa, [near[(r + p) % len(near)] for p in range(P)], pools) for r in range(P)],
         [full_rows(rng, sb, 100 + r) for r in range(P)]),
        ([full_rows(rng, sa, 0) for r in range(P)], [full_rows(rng, sb, 150) for r in range(P)]),
        ([full_rows(rng, sa, 150) for r in range(P)], [full_rows(rng, sb, 0) for r in range(P)]),
    ]
    g = Group(P, slot_for((300 + P, 3), (200 + 3 * P, 2)))

    def rank(r, be):
        b0, res = sent(be), []
        for k, (ia, ib) in enumerate(rounds):
            jitter(r, k)
            a, b = upload(be, sa, ia[r]), upload(be, sb, ib[r])
            oa, ob = be.shard2(a, b)
            res.append((oa.download(), ob.download(), be.shard(a).download(), be.shard(b).download()))
        return res, sent(be) - b0

    out = g.run(rank)
    g.close()
    for k, (ia, ib) in enumerate(rounds):
        ma, mb = xm.shard(sa, ia, P), xm.shard(sb, ib, P)
        for r in range(P):
            oa, ob, a1, b1 = out[r][0][k]
            check(sa, oa, ma[r], f"shard2 round {k} stream 0 rank {r}")
            check(sb, ob, mb[r], f"shard2 round {k} stream 1 rank {r}")
            same(oa, a1, f"shard2 round {k} stream 0 vs shard, rank {r}")
            same(ob, b1, f"shard2 round {k} stream 1 vs shard, rank {r}")
    rounds_b = [(sa, ia, None) for ia, _ in rounds] + [(sb, ib, None) for _, ib in rounds]
    check_bytes(rounds_b + rounds_b, P, [o[1] for o in out], "shard2")


def scenario_retention(P):
    """Outputs of every round stay alive; after later rounds rewrote both parities' slots, they are read again."""
    s = Schema("i", "u")
    rng = np.random.default_rng(800 + P)
    rounds = []
    for k in range(8):
        if k % 2 == 0:   # one source only: every receiver's output is a lone segment (a copy of its slot)
            src = (k // 2) % P
            rounds.append([full_rows(rng, s, 40 * P) if r == src else full_rows(rng, s, 0) for r in range(P)])
        else:
            rounds.append([full_rows(rng, s, 40 * P + 7 * r) for r in range(P)])
    g = Group(P, slot_for((40 * P + 7 * P, 2)))

    def rank(r, be):
        keep, first = [], []
        for k, inputs in enumerate(rounds):
            jitter(r, k)
            o = be.shard(upload(be, s, inputs[r]))
            keep.append(o)
            first.append(o.download())
        return first, [o.download() for o in keep]

    out = g.run(rank)
    g.close()
    for k, inputs in enumerate(rounds):
        model = xm.shard(s, inputs, P)
        for r in range(P):
            check(s, out[r][0][k], model[r], f"retention round {k} rank {r}, read at once")
            check(s, out[r][1][k], model[r], f"retention round {k} rank {r}, read after round {len(rounds) - 1}")


def scenario_slot_overflow(P):
    s = Schema("u", "u")
    rng = np.random.default_rng(900 + P)
    slot = 64 << 10
    over = 4000   # one segment of 4000 rows x 3 words > 64 KiB
    assert seg_bytes(over, 2) > slot
    pools = xm.keys_with_dest(rng, s.nk, P, over)
    bad = [rows_to(rng, s, [0] * (P - 1) + [over], pools) if r == 0 else full_rows(rng, s, 10) for r in range(P)]
    good = [[full_rows(rng, s, 60 + r) for r in range(P)] for _ in range(2)]
    g = Group(P, slot)

    def rank(r, be):
        try:
            be.shard(upload(be, s, bad[r]))
            err = None
        except DbspError as e:
            err = str(e)
        after = []
        for k, inputs in enumerate(good):
            jitter(r, k)
            after.append(be.shard(upload(be, s, inputs[r])).download())
        return err, after

    out = g.run(rank)
    g.close()
    for r in range(P):
        err = out[r][0]
        assert err is not None and "UNSUPPORTED" in err and "receive slot is too small" in err, f"rank {r}: {err}"
    for k, inputs in enumerate(good):
        model = xm.shard(s, inputs, P)
        for r in range(P):
            check(s, out[r][1][k], model[r], f"round {k} after the refused round, rank {r}")


class ThreadComm:
    """What RootCircuit needs of a communicator, over the context's in-library exchange (parallel.Comm needs
    torch.distributed, whose process groups have one rank per process)."""

    def __init__(self, be, P):
        self.native, self.world_size = be, P

    def shard(self, be, b):
        return be.shard(b)

    def shard_many(self, be, bs):
        return list(be.shard2(*bs))

    def gather(self, be, b, root=0):
        return be.gather(b, root)

    def allreduce_max(self, x):
        return self.native.allreduce_max(x)


def scenario_circuits(P):
    """The sharded q3 / q4 / q7 (inputs col[rank::P], output gathered to rank 0) == one context fed the union, bit for
    bit, every step: shard_with (shard2) in the joins, the watermark's allreduce_max, q7's local Min."""
    from dbsp_b200 import RootCircuit
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.nexmark import queries as nq
    from dbsp_b200.runtime import Runtime
    from parity_util import build_query, feed

    for query in ("q3", "q4", "q7"):
        rate = 100_000 if query == "q7" else 0
        n_events, step = (400_000, 100_000) if query != "q7" else (2_400_000, 300_000)
        gen = NexmarkGenerator(first_event_rate=rate)
        tables = [gen.tables(s0, step) for s0 in range(0, n_events, step)]
        g = Group(P, 64 << 20)

        def rank(r, be):
            c = RootCircuit(be, ThreadComm(be, P))
            inp, handles = nq.add_nexmark_input(c)
            out = nq.QUERIES[query](inp).gather(0).output()
            got = []
            for i, t in enumerate(tables):
                jitter(r, i)
                feed(handles, {k: [col[r::P].copy() for col in v] for k, v in t.items()})
                c.step()
                got.append(out.value.download())
            return got

        out = g.run(rank)
        g.close()
        single = Runtime(0)
        c1, h1, o1 = build_query(single, query)
        total = 0
        for i, t in enumerate(tables):
            feed(h1, t)
            c1.step()
            want = o1.value.download()
            same(out[0][i], want, f"{query} at {P} ranks: gathered != single context at step {i}")
            for r in range(1, P):
                check_empty(out[r][i], f"{query} step {i}: gather output on rank {r}")
            total += len(want["diffs"])
        assert total > 0, query
        del c1, h1, o1
        single.close()


SCENARIOS = {
    "allreduce": scenario_allreduce,
    "shard_model": scenario_shard_model,
    "sizes": scenario_sizes,
    "receiver_paths": scenario_receiver_paths,
    "cancel_across_ranks": scenario_cancel_across_ranks,
    "gather": scenario_gather,
    "shard2": scenario_shard2,
    "retention": scenario_retention,
    "slot_overflow": scenario_slot_overflow,
    "circuits": scenario_circuits,
}


def main():
    name, P = sys.argv[1], int(sys.argv[2])
    t0 = time.time()
    SCENARIOS[name](P)
    print(f"EXCHANGE_OK {name} P={P} {time.time() - t0:.1f}s")


if __name__ == "__main__":
    main()
