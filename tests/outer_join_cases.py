"""dbsp_antijoin_delta, Stream.antijoin on it, and the outer joins (operator/join.rs:294-386) against non-incremental
numpy models.

For a key k let N(k) be the number of distinct (k, v2) rows of the other side's integral (those of positive weight).
The antijoin gives a row (k, v1, w) the weight w·(1 − N(k)), wrapping: negative once N(k) >= 2, as in the
reference.  outer_join(f, fl, fr) = join(f) + antijoin(a, b).map(fl) + antijoin(b, a).map(fr).  A circuit's output
at a step is model(t) − model(t−1).  Each case takes the backend under test and optionally a second one (`ref`),
whose outputs must then be equal bit for bit.
"""
import numpy as np
import pytest

import exact_model as em
import horizon_cases as hc
from dbsp_b200 import Max, Min, Proj, RootCircuit, Schema, Spine, capi, col, const, key, lval, rval
from dbsp_b200._capi import DbspError
from dbsp_b200.zset import Fn
from edge_cases import edge_weights, full_lane
from parity_util import assert_batches_equal
from refusal_cases import INVALID, out, refused


# ---- the model --------------------------------------------------------------------------------------------------------
def cat(s, *zs):
    return [np.concatenate([z[0][l] for z in zs]) if zs else np.zeros(0, np.uint64) for l in range(s.nl)], \
        np.concatenate([z[1] for z in zs]) if zs else np.zeros(0, np.int64)


def counts_at(kq, kt, wt):
    """The weight of each query key in a consolidated key table (keys kt, weights wt), 0 where it is absent."""
    u, inv = np.unique(np.concatenate([kt, kq]), return_inverse=True)
    acc = np.zeros(len(u), np.uint64)
    acc[inv[: len(kt)]] = np.asarray(wt, np.int64).view(np.uint64)
    return acc[inv[len(kt):]]


def m_antijoin_delta(s, D, T, KD, KT):
    """delta·(1 − key_trace(k)) − trace ⋉ key_delta; T and KT are lists of batches (cols, weights)."""
    nk, ks = s.nk, Schema(s.key)
    kt = em.consolidate_np(ks, *cat(ks, *KT))
    kd = em.consolidate_np(ks, *KD)
    t = cat(s, *T)
    n = counts_at(hc.keyv(D[0], nk), hc.keyv(kt[0], nk), kt[1])
    w1 = D[1].view(np.uint64) * (np.uint64(1) - n)
    dn = counts_at(hc.keyv(t[0], nk), hc.keyv(kd[0], nk), kd[1])
    w2 = np.uint64(0) - dn * t[1].view(np.uint64)
    return em.consolidate_np(s, [np.concatenate([a, b]) for a, b in zip(D[0], t[0])],
                             np.concatenate([w1, w2]).view(np.int64))


def m_antijoin(s, L, R, nk):
    """Rows of L weighted w·(1 − N(k)), N(k) the number of rows of distinct(R) on k."""
    rk = hc.keyv(hc.f_distinct(R)[0], nk)
    kl = hc.keyv(L[0], nk)
    u, inv = np.unique(np.concatenate([kl, rk]), return_inverse=True)
    m = np.bincount(inv[len(kl):], minlength=len(u)).astype(np.uint64)[inv[: len(kl)]]
    return em.consolidate_np(s, L[0], (L[1].view(np.uint64) * (np.uint64(1) - m)).view(np.int64))


def m_outer(pair, L, R):
    """join(f) + antijoin(L, R).map(fl) + antijoin(R, L).map(fr), with f = pair.proj and fl / fr = f with the other
    side's value lanes read as 0."""
    nk = pair.sl.nk
    J = hc.f_join(pair, L, R)
    AL, AR = m_antijoin(pair.sl, L, R, nk), m_antijoin(pair.sr, R, L, nk)
    zl, zr = np.zeros(len(AL[1]), np.uint64), np.zeros(len(AR[1]), np.uint64)
    cols = []
    for j, (p, i) in enumerate(pair.lanes):
        left = AL[0][i] if p == "k" else AL[0][nk + i] if p == "l" else zl
        right = AR[0][i] if p == "k" else AR[0][nk + i] if p == "r" else zr
        cols.append(np.concatenate([J[0][j], left, right]))
    return em.consolidate_np(pair.out, cols, np.concatenate([J[1], AL[1], AR[1]]))


def check(got, schema, expect, what, other=None):
    em.assert_download_is(schema, got.download(), expect, what)
    if other is not None:
        assert_batches_equal(got, other, f"{what}: vs the oracle")


def upload(be, s, z):
    return be.batch_from_columns(s, z[0], z[1]) if len(z[1]) else be.batch_empty(s)


# ---- dbsp_antijoin_delta called directly ----------------------------------------------------------------------------
DIRECT_SCHEMAS = [Schema("i", "u"), Schema("uu", "i"), Schema("u"), Schema("iu", "iuu")]
COUNTS = (0, 1, 2, 5)


def key_table(rng, s, n_keys):
    """n_keys distinct full-range keys (cols)."""
    cols = [full_lane(rng, t, n_keys * 2) for t in s.key]
    kv = hc.keyv(cols, s.nk)
    _, first = np.unique(kv, return_index=True)
    first = np.sort(first)[:n_keys]
    return [c[first] for c in cols]


def rows_on(rng, s, keys, n, weights=None):
    pick = rng.integers(0, len(keys[0]), n)
    cols = [k[pick] for k in keys] + [full_lane(rng, t, n) for t in s.val]
    return em.consolidate_np(s, cols, edge_weights(rng, n) if weights is None else weights)


def filler_keys(s, n, base):
    """n distinct keys base + j on key lane 0 (other key lanes 0): apart from key_table's random ones."""
    j = np.arange(n, dtype=np.uint64) + np.uint64(base)
    return [j] + [np.zeros(n, np.uint64) for _ in s.key[1:]]


def direct_inputs(s, seed, n_kt_batches=18):
    """Keys with N(k) of 0, 1, 2 and 5 in a key trace of n_kt_batches batches, whose rows cancel across batches;
    count changes that take keys from 0 to 1 and from 1 to 0 (and by more); a delta on those keys and on keys the
    counts never saw, and a trace of four batches.  Key-trace batch i is filled up to 2^(n−1−i) rows with keys
    counted once, so that no two batches merge and the spine holds more than MAX_REFS of them."""
    rng = np.random.default_rng(seed)
    ks = Schema(s.key)
    keys = key_table(rng, s, 48)
    n = np.array([COUNTS[i % 4] for i in range(48)], np.int64)
    # each key's count spread over the ten largest batches as +1 rows, plus +1 / −1 pairs in different batches
    kt_rows = [[] for _ in range(n_kt_batches)]
    for i in range(48):
        for _ in range(int(n[i])):
            kt_rows[rng.integers(0, 10)].append((i, 1))
        for _ in range(int(rng.integers(0, 3))):
            a, b = rng.choice(10, 2, replace=False)
            kt_rows[a].append((i, 1))
            kt_rows[b].append((i, -1))
    KT, base = [], 0x5555_0000_0000_0000
    for b, r in enumerate(kt_rows):
        z = em.consolidate_np(ks, [k[[i for i, _ in r]] for k in keys], np.array([w for _, w in r], np.int64))
        pad = (1 << (n_kt_batches - 1 - b)) - len(z[1])
        KT.append(cat(ks, z, (filler_keys(s, pad, base), np.ones(pad, np.int64))))
        base += pad
    # ΔN with N_{t−1} = N_t − ΔN >= 0: 1 -> 0 (ΔN = −1 at N = 0), 0 -> 1 (ΔN = 1 at N = 1), 2 -> 5, 5 -> 2 ...
    dn = np.array([[-1, 0][rng.integers(0, 2)] if n[i] == 0 else
                   [1, -1, 0][rng.integers(0, 3)] if n[i] == 1 else
                   [3, -3, 2, 0][rng.integers(0, 4)] for i in range(48)], np.int64)
    m = dn != 0
    KD = em.consolidate_np(ks, [k[m] for k in keys], dn[m])
    strangers = key_table(np.random.default_rng(seed + 1), s, 8)
    counted_once = filler_keys(s, 16, 0x5555_0000_0000_0000)
    D = em.consolidate_np(s, *cat(s, rows_on(rng, s, keys, 300), rows_on(rng, s, strangers, 40),
                                  rows_on(rng, s, counted_once, 40)))
    T = [rows_on(rng, s, keys, 200) for _ in range(3)] + [rows_on(rng, s, strangers, 30)]
    return D, T, KD, KT


def call_direct(be, s, D, T, KD, KT):
    tr, kt = Spine(be, s), Spine(be, Schema(s.key))
    for z in T:
        tr.insert(upload(be, s, z))
    for z in KT:
        kt.insert(upload(be, Schema(s.key), z))
    if len(KT) > hc.MAX_REFS:
        assert kt.stats()[1] > hc.MAX_REFS, f"the key trace must span more than one lookup chunk: {kt.stats()}"
    return be.antijoin_delta(upload(be, s, D), tr, upload(be, Schema(s.key), KD), kt)


def run_direct(be, ref, s, seed=7):
    D, T, KD, KT = direct_inputs(s, seed)
    e, ke = hc.empty(s), hc.empty(Schema(s.key))
    cases = {"full": (D, T, KD, KT), "empty delta": (e, T, KD, KT), "empty key_delta": (D, T, ke, KT),
             "empty trace": (D, [], KD, KT), "empty key_trace": (D, T, KD, []), "all empty": (e, [], ke, [])}
    for name, args in cases.items():
        what = f"antijoin_delta {s} {name}"
        got = call_direct(be, s, *args)
        check(got, s, m_antijoin_delta(s, *args), what, call_direct(ref, s, *args) if ref is not None else None)


# ---- refusals -----------------------------------------------------------------------------------------------------------
def run_refusals(be):
    s, ks = Schema("i", "u"), Schema("i")
    d, kd = be.batch_empty(s), be.batch_empty(ks)
    tr, kt = Spine(be, s), Spine(be, ks)
    call = "antijoin_delta"
    o = out()
    for i, name in enumerate(("ctx", "delta", "trace", "key_delta", "key_trace", "out")):
        args = [be.ctx, d.h, tr.h, kd.h, kt.h, C_ref(o)]
        args[i] = None
        refused(be, call, *args, names=f"{name} is NULL", outs=[o])
    bad = [("delta and trace differ in schema", Spine(be, Schema("i", "i")), None, None, None),
           ("no key lanes", None, None, None, None),
           ("key_delta must have exactly", None, None, be.batch_empty(Schema("u")), None),
           ("key_delta must have exactly", None, None, be.batch_empty(Schema("i", "u")), None),
           ("key_trace must have exactly", None, None, None, Spine(be, Schema("iu"))),
           ("key_trace must have exactly", None, None, None, Spine(be, Schema("i", "i")))]
    for text, t2, _, kd2, kt2 in bad:
        if text == "no key lanes":
            s0 = Schema("", "u")
            d0, t0 = be.batch_empty(s0), Spine(be, s0)
            args = (be.ctx, d0.h, t0.h, kd.h, kt.h, C_ref(o))
        else:
            args = (be.ctx, d.h, (t2 or tr).h, (kd if kd2 is None else kd2).h, (kt2 or kt).h, C_ref(o))
        refused(be, call, *args, names=text, status=INVALID, outs=[o])


def C_ref(o):
    import ctypes

    return ctypes.byref(o)


def run_python_refusals(be):
    """outer_join refuses what it cannot run before any step: fan-out closures, output schemas that differ, and a
    key-less stream."""
    pair = hc.PAIRS["i_i"]
    c = RootCircuit(be)
    a, _ = c.add_input_zset(pair.sl)
    b, _ = c.add_input_zset(pair.sr)
    f = pair.proj
    fl, fr = zeroed(pair, "r"), zeroed(pair, "l")
    fan = Proj(pair.out, [key(0), lval(0), rval(0)], fanout=2)
    for args in ((fan, fl, fr), (f, fan, fr), (f, fl, fan)):
        with pytest.raises(ValueError, match="fan-out"):
            a.outer_join(b, *args)
    with pytest.raises(ValueError, match="fan-out"):
        a.outer_join_default(b, fan)
    other = Proj(Schema("i", "u"), [key(0), lval(0)])
    with pytest.raises(ValueError, match="one out_schema"):
        a.outer_join(b, f, other, fr)
    s0 = Schema("", "u")
    a0, _ = c.add_input_zset(s0)
    b0, _ = c.add_input_zset(s0)
    with pytest.raises(ValueError, match="key-less"):
        a0.outer_join(b0, Proj(Schema("", "uu"), [lval(0), rval(0)]), Proj(Schema("", "uu"), [lval(0), const(0)]),
                      Proj(Schema("", "uu"), [const(0), rval(0)]))


# ---- circuits ------------------------------------------------------------------------------------------------------------
def zeroed(pair, side):
    """pair.proj with the `side` ("l" / "r") value lanes read as 0: the fl / fr of outer_join_default, written out."""
    src = {"k": key, "l": lval, "r": rval}
    return Proj(pair.out, [const(0) if p == side else src[p](i) for p, i in pair.lanes])


def as_tree(pair):
    """pair.proj as a row function: every lane a tree (x + 0), which no dbsp_proj holds."""
    src = {"k": key, "l": lval, "r": rval}
    return Proj(pair.out, [Fn(capi.FN_ADD, src[p](i), const(0)) for p, i in pair.lanes])


def run_circuit(be, ref, regime, pair_name, seed=3, scale=0.1):
    """A regime of horizon_cases through a RootCircuit: both antijoins, outer_join with a dbsp_proj closure and fl / fr
    written out, and outer_join_default with a row-function closure, every step against the model."""
    pair = hc.PAIRS[pair_name]
    sl, sr = pair.sl, pair.sr
    reg = hc.REGIMES[regime](pair, seed, scale)
    bes = [be] + ([ref] if ref is not None else [])
    cur = [{} for _ in bes]
    outs = []
    for b, st in zip(bes, cur):
        c = RootCircuit(b)
        a = c.add_source(lambda st=st: st["a"], sl)
        r = c.add_source(lambda st=st: st["b"], sr)
        o = {"anti_ab": a.antijoin(r), "anti_ba": r.antijoin(a),
             "outer": a.outer_join(r, pair.proj, zeroed(pair, "r"), zeroed(pair, "l")),
             "outer_default_fn": a.outer_join_default(r, as_tree(pair))}
        outs.append((c, {k: v.output() for k, v in o.items()}))
    L, R = hc.empty(sl), hc.empty(sr)
    nk = sl.nk
    for t in range(reg.n):
        dl, dr = reg.deltas(t, L, R)
        for b, st in zip(bes, cur):
            st.update(a=upload(b, sl, dl), b=upload(b, sr, dr))
        for c, _ in outs:
            c.step()
        L1, R1 = hc.plus(sl, L, dl), hc.plus(sr, R, dr)
        kv = np.union1d(hc.keyv(dl[0], nk), hc.keyv(dr[0], nk))
        Lk, Rk, L1k, R1k = (hc.restrict(s, z, kv) for s, z in ((sl, L), (sr, R), (sl, L1), (sr, R1)))
        outer = hc.plus(pair.out, m_outer(pair, L1k, R1k), m_outer(pair, Lk, Rk), -1)
        want = {"anti_ab": (sl, hc.plus(sl, m_antijoin(sl, L1k, R1k, nk), m_antijoin(sl, Lk, Rk, nk), -1)),
                "anti_ba": (sr, hc.plus(sr, m_antijoin(sr, R1k, L1k, nk), m_antijoin(sr, Rk, Lk, nk), -1)),
                "outer": (pair.out, outer), "outer_default_fn": (pair.out, outer)}
        for name, (schema, expect) in want.items():
            check(outs[0][1][name].value, schema, expect, f"{regime}/{pair_name} step {t} {name}",
                  outs[1][1][name].value if ref else None)
        L, R = L1, R1


# ---- a skewed key ------------------------------------------------------------------------------------------------------
SKEW = 70_000


def skew_circuit(be):
    s = Schema("u", "u")
    c = RootCircuit(be)
    st = {}
    a = c.add_source(lambda: st["a"], s)
    b = c.add_source(lambda: st["b"], s)
    return c, st, a, b


def run_skew(be, ref=None):
    """One key with 70 000 rows on each side: 4.9·10^9 matches for self − self ⋈ distinct(other), which the join
    refuses; the antijoin gives each row w·(1 − 70 000), then +1 when one value of the other side is retracted."""
    s = Schema("u", "u")
    outs = []
    for b in [be] + ([ref] if ref is not None else []):
        c, st, a, r = skew_circuit(b)
        o = a.antijoin(r).output()
        vals = np.arange(SKEW, dtype=np.uint64)
        k = np.full(SKEW, 7, np.uint64)
        w = np.where(np.arange(SKEW) % 3 == 0, 2, 1).astype(np.int64)
        st.update(a=b.batch_from_columns(s, [k, vals], w), b=b.batch_from_columns(s, [k, vals * 5], None))
        c.step()
        got1 = o.value
        check(got1, s, ([k, vals], (w.view(np.uint64) * np.uint64(1 - SKEW & ((1 << 64) - 1))).view(np.int64)),
              "skewed key, step 1")
        st.update(a=b.batch_empty(s), b=b.batch_from_columns(s, [k[:1], vals[:1] * 5], np.array([-1], np.int64)))
        c.step()
        check(o.value, s, ([k, vals], w), "skewed key, step 2: one value of the other side retracted")
        outs.append((got1, o.value))
    if ref is not None:
        assert_batches_equal(outs[0][0], outs[1][0], "skewed key step 1 vs the oracle")
        assert_batches_equal(outs[0][1], outs[1][1], "skewed key step 2 vs the oracle")


def run_skew_composition_refused(be):
    """The composition the antijoin replaced refuses the skewed key: 2^32−1 or more matches in one step."""
    s = Schema("u", "u")
    c, st, a, r = skew_circuit(be)
    a._antijoin_composed(r)
    vals = np.arange(SKEW, dtype=np.uint64)
    k = np.full(SKEW, 7, np.uint64)
    st.update(a=be.batch_from_columns(s, [k, vals]), b=be.batch_from_columns(s, [k, vals * 5]))
    with pytest.raises(DbspError, match="UNSUPPORTED"):
        c.step()


# ---- the first five outer joins of Nexmark q17 ----------------------------------------------------------------------
DAY_MS = 86_400_000
RANK1, RANK2 = 10_000, 1_000_000


def q17_first5(inp):
    """q17.rs:76-161 up to its fifth outer join: per (auction, day = date_time / 86 400 000), the total bid count, the
    counts of prices below 10 000, in [10 000, 1 000 000) and from 1 000 000 up, and the minimum and maximum price,
    put side by side by five outer_join_default calls, each followed by .index(2).  Out: (auction, day) -> (total,
    rank1, rank2, rank3, min, max), 8 lanes.  (The sixth join, sum and average, needs 10 lanes.)"""
    bids = inp.bid.flat_map_index(Proj(Schema("uu", "u"), [col(0), col(3).divu(DAY_MS), col(2)]))   # q17.rs:76-86
    price = lval(0)
    total = bids.aggregate_linear(const(1))
    rank1 = bids.filter(price.lt(RANK1)).aggregate_linear(const(1))
    rank2 = bids.filter(price.ge(RANK1), price.lt(RANK2)).aggregate_linear(const(1))
    rank3 = bids.filter(price.ge(RANK2)).aggregate_linear(const(1))
    acc = total
    for other in (rank1, rank2, rank3, bids.aggregate(Min), bids.aggregate(Max)):
        nv = acc.schema.nv
        f = Proj(Schema("uu" + acc.schema.val + other.schema.val), [key(0), key(1)] + [lval(j) for j in range(nv)] + [rval(0)])
        acc = acc.outer_join_default(other, f).index(2)
    return acc


def m_q17_first5(bids):
    """GROUP BY (auction, day) over the live bids {(auction, bidder, price, date_time, extra): weight}."""
    groups = {}
    for (auction, _, price, dt, _), w in bids.items():
        if w == 0:
            continue
        g = groups.setdefault((auction, dt // DAY_MS), [0, 0, 0, 0, None, None])
        g[0] += w
        g[1 if price < RANK1 else 2 if price < RANK2 else 3] += w
        g[4] = price if g[4] is None else min(g[4], price)
        g[5] = price if g[5] is None else max(g[5], price)
    return {k + tuple(v): 1 for k, v in groups.items()}


def bid(auction, bidder, price, date_time):
    return (auction, bidder, price, date_time, 0)


# (bid, weight) per step: ranks 1 to 3 on one day, a second day, a count that falls back to 0, a group that vanishes
Q17_STEPS = [
    [(bid(1, 1, 100, 5), 1), (bid(1, 2, 20_000, 6), 1), (bid(1, 3, 2_000_000, 7), 1), (bid(2, 1, 5, 8), 1),
     (bid(1, 4, 50_000, DAY_MS + 5), 1)],
    [(bid(2, 2, 1_500_000, 9), 1), (bid(1, 5, 9_999, 10), 2), (bid(3, 1, 10_000, 2 * DAY_MS), 1)],
    [(bid(2, 1, 5, 8), -1), (bid(3, 1, 10_000, 2 * DAY_MS), -1), (bid(1, 6, 999_999, DAY_MS + 6), 1),
     (bid(1, 2, 20_000, 6), -1)],
    [],
    [(bid(2, 3, 1, 11), 1), (bid(1, 1, 100, 5), -1), (bid(4, 1, RANK2, 3 * DAY_MS - 1), 3)],
]


def run_q17_bids(be):
    """q17_first5 on hand-written bids, its integral against the GROUP BY model after every step."""
    from dbsp_b200.nexmark import queries as nq

    c = RootCircuit(be)
    inp, handles = nq.add_nexmark_input(c)
    q = q17_first5(inp)
    assert q.schema == Schema("uu", "iiiiuu"), q.schema
    integral = q.integrate().output()
    live = {}
    for t, step in enumerate(Q17_STEPS):
        for k in ("person", "auction"):
            handles[k].set([np.zeros(0, np.uint64)] * 5)
        rows = [b for b, _ in step]
        handles["bid"].set([np.array(x, np.uint64) for x in zip(*rows)] if rows else [np.zeros(0, np.uint64)] * 5,
                           np.array([w for _, w in step], np.int64))
        c.step()
        for b, w in step:
            live[b] = live.get(b, 0) + w
        got = {r[:-1]: r[-1] for r in integral.value.rows()}
        assert got == m_q17_first5(live), (t, got, m_q17_first5(live))


def run_q17_generated(be, n_events=40_000, steps=3):
    """q17_first5 on generated events (bids from several days' auctions), its integral against the GROUP BY model."""
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.nexmark import queries as nq

    gen = NexmarkGenerator(0x7FC359184519C0AA, first_event_rate=1)   # one event per second: the bids span two days
    c = RootCircuit(be)
    inp, handles = nq.add_nexmark_input(c)
    integral = q17_first5(inp).integrate().output()
    live = {}
    for s in range(steps):
        t = gen.tables(s * n_events, n_events)
        for k in ("person", "auction", "bid"):
            handles[k].set(t[k])
        c.step()
        for b in zip(*[x.tolist() for x in t["bid"]]):
            live[b] = live.get(b, 0) + 1
    want = m_q17_first5(live)
    assert len({k[1] for k in want}) > 1, "the bids must span more than one day"
    assert {r[:-1]: r[-1] for r in integral.value.rows()} == want


def run_q17_nexmark(be, ref, n_events=5_000_000, steps=5):
    """q17_first5 on `steps` steps of `n_events` generated events, every step's output equal on both backends."""
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.nexmark import queries as nq

    gen = NexmarkGenerator(0x7FC359184519C0AA)
    runs = []
    for b in (be, ref):
        c = RootCircuit(b)
        inp, handles = nq.add_nexmark_input(c)
        runs.append((c, handles, q17_first5(inp).output()))
    total = 0
    for s in range(steps):
        t = gen.tables(s * n_events, n_events)
        for c, handles, _ in runs:
            for k in ("person", "auction", "bid"):
                handles[k].set(t[k])
            c.step()
        assert_batches_equal(runs[0][2].value, runs[1][2].value, f"q17 first five joins, step {s}")
        total += len(runs[0][2].value)
    assert total > 0
    return total


ALL_CASES = {f"direct_{s.key}_{s.val}": (lambda be, ref=None, s=s: run_direct(be, ref, s)) for s in DIRECT_SCHEMAS}
ALL_CASES["skew"] = run_skew
ALL_CASES["q17_bids"] = lambda be, ref=None: run_q17_bids(be)
ALL_CASES["q17_generated"] = lambda be, ref=None: run_q17_generated(be)
for _p in hc.PAIRS:
    for _r in ("growth", "churn", "hot"):
        ALL_CASES[f"circuit_{_r}_{_p}"] = lambda be, ref=None, r=_r, p=_p: run_circuit(be, ref, r, p)


def run_profile_class(be):
    s = Schema("i", "u")
    D, T, KD, KT = direct_inputs(s, 11)
    be.profile(True)
    call_direct(be, s, D, T, KD, KT)
    prof = be.profile_read()
    be.profile(False)
    assert prof["antijoin_scale"]["launches"] == 1, prof
    assert prof["antijoin_scale"]["alg_bytes"] == 28 * len(D[1]), prof
