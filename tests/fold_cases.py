"""dbsp_aggregate_fold and Stream.aggregate(Fold) (operator/aggregate/fold.rs) against a non-incremental Python model,
and Nexmark q18 / q6, which the reference writes with Fold.

The model integrates the input, groups it by key and folds each key's consolidated values in value order: `step`
runs on every value (its weight is never 0 in a consolidated Z-set) and replaces the accumulator when its keep flag
is non-zero; a key with values gets (key, output(acc)) unless output's keep flag is 0.  The programs run on
rowfn_cases.run_code, the tests' own stack machine, over the instruction arrays the libraries get.  A circuit's
output at step t must be model(t) − model(t−1).  Each case takes the backend under test and optionally a second one
(`ref`), whose outputs must then be equal bit for bit.
"""
import json
import os

import numpy as np
import pytest

import exact_model as em
import horizon_cases as hc
from dbsp_b200 import Fold, FoldCount, FoldSum, Max, Min, Proj, RootCircuit, Schema, Spine, acc, capi, const, key, lval, weight
from dbsp_b200._capi import CFold, DbspError
from edge_cases import edge_weights, full_lane
from exact_model import u64, w64
from parity_util import assert_batches_equal
from refusal_cases import INVALID, out, refused
from rowfn_cases import run_code

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fold_nexmark.json")


# ---- the model --------------------------------------------------------------------------------------------------------
class _Weight:
    """env[SRC_WEIGHT]: the value's weight whatever idx a PUSH names"""

    def __init__(self, w):
        self.w = u64(w)

    def __getitem__(self, _):
        return self.w


def codes(fold):
    f = fold._c
    step = [(i.op, i.kind, i.idx, i.cst) for i in f.step[: f.n_step]]
    output = [(i.op, i.kind, i.idx, i.cst) for i in f.output.code[: f.output.n_insn]]
    return step, output, [int(x) for x in f.init[: f.n_acc]]


def m_fold_groups(out_schema, fold, groups):
    """{key: [(value, weight)..]} (value order, weights != 0) -> Z of (key, output) rows, weight 1."""
    step, output, init = codes(fold)
    n = len(init)
    res = em.Z(out_schema)
    for k, vs in groups.items():
        a = list(init)
        ku = tuple(u64(x) for x in k)
        for v, w in vs:
            vu = tuple(u64(x) for x in v)
            st = run_code(step, (ku, vu, vu, None, None, a, _Weight(w)))
            assert len(st) == n + 1
            if st[n]:
                a = st[:n]
        if not vs:
            continue
        st = run_code(output, (ku, (), (), None, None, a, _Weight(0)))
        if st[-1]:
            res.add([k + tuple(st[:-1]) + (1,)])
    return res


def m_fold(out_schema, fold, z):
    """the fold of a Z-set (exact_model.Z), every key"""
    return m_fold_groups(out_schema, fold, z.groups())


def out_schema_of(s, fold):
    return Schema(s.key, fold.output.schema.val)


def z_of(s, cols, w):
    return em.Z(s, [tuple(int(c[i]) for c in cols) + (int(w[i]),) for i in range(len(w))])


def upload(be, s, z):
    return be.batch_from_columns(s, z[0], z[1]) if len(z[1]) else be.batch_empty(s)


# ---- folds ----------------------------------------------------------------------------------------------------------
def f_sum_weighted():
    """n_acc 2: sum of value·weight, and the number of values"""
    return Fold([0, 0], [acc(0) + lval(0) * weight(), acc(1) + 1],
                output=Proj(Schema("", "iu"), [acc(0), acc(1)]))


def f_acc15():
    """n_acc 15: a shift register of the last 14 values' lane 0 and a running xor of the weights; the output mixes
    every word into 4 lanes"""
    step = [acc(i + 1) for i in range(13)] + [lval(0), acc(14) ^ weight()]
    mix = [sum((acc(i) for i in range(j, 15, 4)), const(j)) for j in range(4)]
    return Fold([i * 7 for i in range(15)], step, output=Proj(Schema("", "uuui"), mix))


def f_keep_step():
    """the step keeps only values whose lane 0 is odd (a Fold with a filter)"""
    return Fold([5], [acc(0) * 3 + lval(0)], where=lval(0).remu(2).eq(1))


def f_keep_output():
    """the output drops keys whose count is even"""
    return Fold([0], [acc(0) + 1], output=Proj(Schema("", "u"), [acc(0)], where=[acc(0).remu(2).eq(1)]))


def f_keep_both():
    """the step keeps values with a positive weight; the output drops keys where none was kept"""
    return Fold([0, 0], [acc(0) + lval(0), const(1)], where=weight().gt(0).signed(),
                output=Proj(Schema("", "u"), [acc(0)], where=[acc(1).eq(1)]))


def f_weight():
    """the weight itself, wrapping: w·v summed, the product of the weights, and the minimum weight"""
    return Fold([0, 1, (1 << 63) - 1], [acc(0) + weight() * lval(0), acc(1) * weight(), acc(2).min(weight()).signed()],
                output=Proj(Schema("", "uii"), [acc(0), acc(1), acc(2)]))


def f_copy_last(s):
    """the last value in value order (what Max picks), as its own lanes"""
    nv = s.nv
    return Fold([0] * nv, [lval(i) for i in range(nv)], output=Proj(Schema("", s.val), [acc(i) for i in range(nv)]))


def f_copy_first(s):
    """the first value (what Min picks): a word marks that one was seen"""
    nv = s.nv
    return Fold([0] * (nv + 1), [lval(i) for i in range(nv)] + [const(1)], where=acc(nv).eq(0),
                output=Proj(Schema("", s.val), [acc(i) for i in range(nv)]))


def f_count():
    return Fold([0], [acc(0) + 1])


def f_sum():
    return Fold([0], [acc(0) + lval(0)])


FOLDS = {"sum_weighted": f_sum_weighted, "acc15": f_acc15, "keep_step": f_keep_step, "keep_output": f_keep_output,
         "keep_both": f_keep_both, "weight": f_weight, "n_acc1": f_sum}


# ---- random programs ------------------------------------------------------------------------------------------------
_BINOPS = [capi.FN_ADD, capi.FN_SUB, capi.FN_MUL, capi.FN_DIV, capi.FN_REMU, capi.FN_XOR, capi.FN_MINU, capi.FN_MAX,
           capi.FN_SHR, capi.FN_LT, capi.FN_GEU, capi.FN_AND]


def random_code(rng, nk, nv, n_acc, n_out, kinds):
    """a valid postfix program leaving n_out values then a keep flag, pushing from `kinds`"""
    code, depth = [], 0

    def push():
        k = kinds[rng.integers(0, len(kinds))]
        idx = {capi.SRC_KEY: nk, capi.SRC_LVAL: nv, capi.SRC_ACC: n_acc}.get(k, 256)   # WEIGHT / CONST: idx ignored
        cst = int(rng.choice([0, 1, 3, -1, 1 << 63, 12345]))
        code.append((capi.FN_PUSH, k, int(rng.integers(0, max(idx, 1))), cst))

    for _ in range(n_out + 1):
        push()
        depth += 1
        for _ in range(int(rng.integers(0, 3))):
            push()
            code.append((int(rng.choice(_BINOPS)), 0, 0, 0))
        if rng.random() < 0.2:
            code.append((capi.FN_LNOT, 0, 0, 0) if rng.random() < 0.5 else (capi.FN_ABS, 0, 0, 0))
    return code


class RawFold(Fold):
    """A Fold-shaped wrapper of raw programs: the backends get the CFold, the model its codes."""

    def __init__(self, init, step, output, out_val):
        f = CFold()
        f.n_acc, f.n_step = len(init), len(step)
        for i, x in enumerate(init):
            f.init[i] = u64(x)
        for i, (op, kind, idx, cst) in enumerate(step):
            f.step[i].op, f.step[i].kind, f.step[i].idx, f.step[i].cst = op, kind, idx, w64(cst)
        f.output.out_schema = Schema("", out_val).c()
        f.output.n_insn = len(output)
        for i, (op, kind, idx, cst) in enumerate(output):
            f.output.code[i].op, f.output.code[i].kind, f.output.code[i].idx, f.output.code[i].cst = op, kind, idx, w64(cst)
        self._c = f
        self.output = Proj(Schema("", out_val), [const(0)] * len(out_val))   # its schema only


def random_fold(seed, s):
    rng = np.random.default_rng(seed)
    n_acc = int(rng.integers(1, 6))
    n_out = int(rng.integers(1, 9 - s.nk))
    out_val = "".join(rng.choice(["u", "i"], n_out))
    step = random_code(rng, s.nk, s.nv, n_acc, n_acc, [capi.SRC_KEY, capi.SRC_LVAL, capi.SRC_ACC, capi.SRC_WEIGHT,
                                                       capi.SRC_CONST])
    output = random_code(rng, s.nk, 0, n_acc, n_out, [capi.SRC_KEY, capi.SRC_ACC, capi.SRC_CONST])
    return RawFold([int(x) for x in rng.integers(-5, 5, n_acc)], step, output, out_val)


# ---- direct calls ---------------------------------------------------------------------------------------------------
def call_direct(be, s, fold, D, T, O):
    """dbsp_aggregate_fold(D, spine of T's batches, spine of O's batches)"""
    os_ = out_schema_of(s, fold)
    tr, ot = Spine(be, s), Spine(be, os_)
    for z in T:
        tr.insert(upload(be, s, z))
    for z in O:
        ot.insert(upload(be, os_, z))
    return be.aggregate_fold(upload(be, s, D), tr, ot, fold), tr


def m_direct(s, fold, D, T, O):
    """−old +new for D's keys, T and O being lists of batches"""
    os_ = out_schema_of(s, fold)
    tz, oz = em.Z(s), em.Z(os_)
    for z in T:
        tz.add(z_of(s, *z).rows())
    for z in O:
        oz.add(z_of(os_, *z).rows())
    keys = set(z_of(s, *D).groups())
    new = m_fold_groups(os_, fold, {k: v for k, v in tz.groups().items() if k in keys})
    old = em.Z(os_, [r for r in oz.rows() if r[: s.nk] in keys])
    return new.add(old.rows(), -1)


def check(got, schema, expect, what, other=None):
    em.assert_batch_is(got, expect, what)
    if other is not None:
        assert_batches_equal(got, other, f"{what}: vs the oracle")


def direct(be, ref, s, fold, D, T, O, what, min_batches=0):
    got, tr = call_direct(be, s, fold, D, T, O)
    if min_batches:
        assert tr.stats()[1] >= min_batches, f"{what}: the trace must hold {min_batches} batches: {tr.stats()}"
    check(got, out_schema_of(s, fold), m_direct(s, fold, D, T, O), what,
          call_direct(ref, s, fold, D, T, O)[0] if ref is not None else None)


def rows_full(rng, s, n, n_keys, weights=None):
    """full-range lanes on n_keys keys, weights from the edge pool unless given"""
    keys = [full_lane(rng, t, n_keys) for t in s.key]
    pick = rng.integers(0, n_keys, n)
    cols = [k[pick] for k in keys] + [full_lane(rng, t, n) for t in s.val]
    return em.consolidate_np(s, cols, edge_weights(rng, n) if weights is None else weights)


def run_direct(be, ref, s, fold_name, seed=5):
    """full-range lanes and weights over a three-batch trace, with an output trace holding old values for some keys"""
    rng = np.random.default_rng(seed)
    fold = FOLDS[fold_name]() if isinstance(fold_name, str) else fold_name
    T = [rows_full(rng, s, 600, 40) for _ in range(3)]
    D = T[2]
    os_ = out_schema_of(s, fold)
    # old output rows on 20 of delta's keys (some of them equal to the new ones after the call) and on other keys
    old = rows_full(rng, os_, 40, 40, np.ones(40, np.int64))
    m = min(20, len(old[1]) // 2)
    O = [em.consolidate_np(os_, [np.concatenate([D[0][l][:m], old[0][l][:m]]) for l in range(s.nk)] +
                           [np.concatenate([c[:m], c[m:2 * m]]) for c in old[0][s.nk:]], np.ones(2 * m, np.int64))]
    direct(be, ref, s, fold, D, T, O, f"aggregate_fold {s} {fold_name}")
    direct(be, ref, s, fold, hc.empty(s), T, O, f"aggregate_fold {s} {fold_name}: empty delta")


def run_cancel_across_batches(be, ref=None):
    """(k, v) at +1 in one trace batch and at −1 in another sums to 0 and is skipped; a key whose only value cancels
    has no new row, so its old one is retracted (−old only)"""
    s = Schema("u", "u")
    fold = f_sum_weighted()
    big = em.consolidate_np(s, [np.arange(4096, dtype=np.uint64) + np.uint64(100), np.arange(4096, dtype=np.uint64)],
                            np.ones(4096, np.int64))
    a = em.consolidate_np(s, [np.array([1, 1, 2], np.uint64), np.array([10, 11, 20], np.uint64)], np.array([1, 3, 1], np.int64))
    b = em.consolidate_np(s, [np.array([1, 2], np.uint64), np.array([10, 20], np.uint64)], np.array([-1, -1], np.int64))
    T = [hc.plus(s, big, a), b]
    O = [em.consolidate_np(out_schema_of(s, fold), [np.array([1, 2], np.uint64), np.array([13, 20], np.uint64),
                                                    np.array([2, 1], np.uint64)], np.ones(2, np.int64))]
    direct(be, ref, s, fold, b, T, O, "values cancelling across batches", min_batches=2)


def run_many_batches(be, ref=None, n_batches=18):
    """a trace of more than MAX_REFS (16) batches: batch i holds 2^(n−1−i) rows, so that no two merge"""
    s = Schema("iu", "iu")
    rng = np.random.default_rng(9)
    T, base = [], 0
    for b in range(n_batches):
        n = 1 << (n_batches - 1 - b)
        k0 = np.concatenate([np.arange(base, base + n - 8, dtype=np.int64), rng.integers(0, 8, min(8, n))]).view(np.uint64)
        cols = [k0, np.zeros(len(k0), np.uint64)] + [full_lane(rng, t, len(k0)) for t in s.val]
        T.append(em.consolidate_np(s, cols, edge_weights(rng, len(k0))))
        base += n
    D = em.consolidate_np(s, [np.arange(12, dtype=np.uint64), np.zeros(12, np.uint64), np.zeros(12, np.uint64),
                              np.zeros(12, np.uint64)], np.ones(12, np.int64))
    direct(be, ref, s, f_weight(), D, T, [], "a trace of 18 batches", min_batches=hc.MAX_REFS + 1)


def run_keyless(be, ref=None):
    """no key lanes: the whole input is one group"""
    s = Schema("", "iu")
    rng = np.random.default_rng(3)
    T = [rows_full(rng, s, 300, 1), rows_full(rng, s, 100, 1)]
    fold = Fold([0, 0], [acc(0) + lval(0), acc(1) ^ lval(1)], output=Proj(Schema("", "iu"), [acc(0), acc(1)]))
    direct(be, ref, s, fold, T[1], T, [], "key-less input")
    run_circuit_random(be, ref, s, fold, steps=4, seed=4, n=200, n_keys=1, what="key-less circuit")


# ---- circuits ---------------------------------------------------------------------------------------------------------
def fold_circuit(b, s, fold, stream=False):
    c = RootCircuit(b)
    st = {}
    src = c.add_source(lambda: st["d"], s)
    o = (src.stream_aggregate(fold) if stream else src.aggregate(fold)).output()
    return c, st, o


def run_circuit_deltas(be, ref, s, fold, deltas, what):
    """aggregate(fold) over the deltas: every step's output is model(I_t) − model(I_{t−1}) on the touched keys, and
    (given ref) bit for bit the oracle's"""
    os_ = out_schema_of(s, fold)
    runs = [fold_circuit(b, s, fold) for b in [be] + ([ref] if ref is not None else [])]
    integral = hc.empty(s)
    for t, d in enumerate(deltas):
        for (c, st, _), b in zip(runs, [be, ref]):
            st["d"] = upload(b, s, d)
            c.step()
        new = hc.plus(s, integral, d)
        kv = hc.keyv(d[0], s.nk) if s.nk else None
        part = (lambda z: hc.restrict(s, z, kv)) if s.nk else (lambda z: z)
        want = m_fold(os_, fold, z_of(s, *part(new))).add(m_fold(os_, fold, z_of(s, *part(integral))).rows(), -1)
        check(runs[0][2].value, os_, want, f"{what} step {t}", runs[1][2].value if ref is not None else None)
        integral = new


def run_circuit_random(be, ref, s, fold, steps=6, seed=1, n=400, n_keys=30, what="circuit"):
    """random deltas that insert and retract: keys lose their last value (−old only) and come back"""
    rng = np.random.default_rng(seed)
    deltas, live = [], hc.empty(s)
    for t in range(steps):
        d = rows_full(rng, s, n, n_keys, hc.weights(rng, n))
        if len(live[1]):
            take = rng.random(len(live[1])) < 0.5
            d = hc.plus(s, d, (([c[take] for c in live[0]]), hc.negw(live[1][take])))
        deltas.append(d)
        live = hc.plus(s, live, d)
    # a step that retracts everything: every key's new row is gone
    deltas.append(em.consolidate_np(s, live[0], hc.negw(live[1])))
    run_circuit_deltas(be, ref, s, fold, deltas, what)


def run_regime(be, ref, regime, pair_name, seed=3, scale=0.1):
    """a horizon_cases regime's left deltas through aggregate(Fold) (growth / churn / hot)"""
    pair = hc.PAIRS[pair_name]
    s = pair.sl
    reg = hc.REGIMES[regime](pair, seed, scale)
    fold = f_weight() if pair_name == "i_i" else f_copy_first(s)
    L, R, deltas = hc.empty(s), hc.empty(pair.sr), []
    for t in range(reg.n):
        dl, dr = reg.deltas(t, L, R)
        deltas.append(dl)
        L, R = hc.plus(s, L, dl), hc.plus(pair.sr, R, dr)
    run_circuit_deltas(be, ref, s, fold, deltas, f"{regime}/{pair_name}")


SKEW = 70_000


def run_hot_key(be, ref=None):
    """one key of 70 000 values, walked by one thread; then a value in the middle is retracted"""
    s = Schema("u", "i")
    v = np.arange(SKEW, dtype=np.int64) - SKEW // 2
    d1 = em.consolidate_np(s, [np.full(SKEW, 7, np.uint64), v.view(np.uint64)], np.where(v % 3 == 0, 2, 1).astype(np.int64))
    d2 = em.consolidate_np(s, [np.array([7, 8], np.uint64), np.array([5, 1], np.int64).view(np.uint64)], np.array([-2, 1], np.int64))
    for name, fold in (("weighted sum", f_sum_weighted()), ("shift register", f_acc15())):
        run_circuit_deltas(be, ref, s, fold, [d1, d2], f"hot key, {name}")


def run_builtin_equivalents(be, ref=None):
    """Fold programs equal to FoldCount, FoldSum, Max and Min give the built-in kinds' batches bit for bit"""
    for s in (Schema("i", "iu"), Schema("iu", "u")):
        rng = np.random.default_rng(11)
        deltas, live = [], hc.empty(s)
        for t in range(5):
            d = em.consolidate_np(s, *hc.gen_rows(rng, s, hc.PAIRS["i_i" if s.nk == 1 else "iu_uiu"],
                                                   rng.integers(-40, 40, 500)))
            if len(live[1]):
                take = rng.random(len(live[1])) < 0.3
                d = hc.plus(s, d, ([c[take] for c in live[0]], hc.negw(live[1][take])))
            deltas.append(d)
            live = hc.plus(s, live, d)
        pairs = [(FoldCount, f_count()), (FoldSum, f_sum()), (Max, f_copy_last(s)), (Min, f_copy_first(s))]
        for b in [be] + ([ref] if ref is not None else []):
            for builtin, fold in pairs:
                c = RootCircuit(b)
                st = {}
                src = c.add_source(lambda: st["d"], s)
                o1, o2 = src.aggregate(builtin).output(), src.aggregate(fold).output()
                o3, o4 = src.stream_aggregate(builtin).output(), src.stream_aggregate(fold).output()
                for t, d in enumerate(deltas):
                    st["d"] = upload(b, s, d)
                    c.step()
                    assert_batches_equal(o1.value, o2.value, f"{builtin.__name__} as a Fold, {s} step {t}")
                    assert_batches_equal(o3.value, o4.value, f"stream_aggregate {builtin.__name__} as a Fold, {s} step {t}")


def run_stream_aggregate(be, ref=None):
    """stream_aggregate(Fold): the fold of each step's batch alone"""
    s = Schema("u", "iu")
    rng = np.random.default_rng(2)
    fold = f_weight()
    os_ = out_schema_of(s, fold)
    runs = [fold_circuit(b, s, fold, stream=True) for b in [be] + ([ref] if ref is not None else [])]
    for t in range(3):
        d = rows_full(rng, s, 300, 20)
        for (c, st, _), b in zip(runs, [be, ref]):
            st["d"] = upload(b, s, d)
            c.step()
        check(runs[0][2].value, os_, m_fold(os_, fold, z_of(s, *d)), f"stream_aggregate step {t}",
              runs[1][2].value if ref is not None else None)


# ---- refusals -----------------------------------------------------------------------------------------------------------
def _ref(o):
    import ctypes

    return ctypes.byref(o)


def run_refusals(be):
    """one refusal per rule of valid_fold, made on the host before anything runs"""
    import ctypes

    s = Schema("i", "uu")
    d = be.batch_empty(s)
    tr, ot = Spine(be, s), Spine(be, Schema("i", "u"))
    good = f_sum()
    call = "aggregate_fold"
    o = out()
    for i, name in enumerate(("ctx", "delta", "in_trace", "out_trace", "fold", "out")):
        args = [be.ctx, d.h, tr.h, ot.h, _ref(good._c), _ref(o)]
        args[i] = None
        refused(be, call, *args, names=f"{name} is NULL", outs=[o])

    def bad(text, mutate=None, delta=None, in_tr=None, out_tr=None):
        f = CFold.from_buffer_copy(good._c)
        if mutate:
            mutate(f)
        args = (be.ctx, (delta or d).h, (in_tr or tr).h, (out_tr or ot).h, _ref(f), _ref(o))
        refused(be, call, *args, names=text, status=INVALID, outs=[o])

    def push(f, where, i, kind, idx=0):
        code = f.step if where == "step" else f.output.code
        code[i].op, code[i].kind, code[i].idx = capi.FN_PUSH, kind, idx

    bad("fold.n_acc = 0", lambda f: setattr(f, "n_acc", 0))
    bad("fold.n_acc = 16", lambda f: setattr(f, "n_acc", 16))
    bad("fold.n_step = 65", lambda f: setattr(f, "n_step", 65))
    bad("fold.step.code[0].idx = 1: SRC_KEY has 1 lanes", lambda f: push(f, "step", 0, capi.SRC_KEY, 1))
    bad("fold.step.code[0].idx = 2: SRC_LVAL has 2 lanes", lambda f: push(f, "step", 0, capi.SRC_LVAL, 2))
    bad("fold.step.code[0].idx = 2: SRC_RVAL has 2 lanes", lambda f: push(f, "step", 0, capi.SRC_RVAL, 2))
    bad("fold.step.code[0].idx = 1: SRC_ACC has 1 words", lambda f: push(f, "step", 0, capi.SRC_ACC, 1))
    bad("fold.step.code[0].kind = 4 is not a source kind", lambda f: push(f, "step", 0, capi.SRC_FANOUT))
    bad("fold.step.code[0].kind = 7 is not a source kind", lambda f: push(f, "step", 0, 7))
    bad("fold.step ends with stack depth 3, needs 2 (the accumulator words, then the keep flag)",
        lambda f: (setattr(f, "n_step", f.n_step + 1), push(f, "step", f.n_step - 1, capi.SRC_CONST)))
    bad("fold.step.code[0]: stack underflow", lambda f: setattr(f.step[0], "op", capi.FN_ADD))
    bad("fold.output.code[0].idx = 0: SRC_LVAL has 0 lanes", lambda f: push(f, "output", 0, capi.SRC_LVAL))
    bad("fold.output.code[0].kind = 6 is not a source kind", lambda f: push(f, "output", 0, capi.SRC_WEIGHT))
    bad("fold.output.code[0].idx = 3: SRC_ACC has 1 words", lambda f: push(f, "output", 0, capi.SRC_ACC, 3))
    bad("fold.output.n_insn = 65 exceeds 64", lambda f: setattr(f.output, "n_insn", 65))
    bad("fold.output.out_schema must have 1..8 lanes", lambda f: setattr(f.output.out_schema, "n_val_lanes", 0))

    def keyed(f):
        f.output.out_schema.n_key_lanes, f.output.out_schema.n_val_lanes = 1, 0
    bad("fold.output.out_schema has key lanes", keyed)
    bad("fold.output ends with stack depth 2, needs 3", lambda f: setattr(f.output.out_schema, "n_val_lanes", 2))
    bad("delta and in_trace differ in schema", in_tr=Spine(be, Schema("i", "ui")))
    bad("delta and out_trace differ in key lanes", out_tr=Spine(be, Schema("u", "u")))
    bad("out_trace must have fold.output's value lanes", out_tr=Spine(be, Schema("i", "uu")))
    bad("out_trace must have fold.output's value lanes", out_tr=Spine(be, Schema("i", "i")))
    # the other calls keep their texts: ACC and WEIGHT are outside the enum there
    from dbsp_b200._capi import CRowFn

    fn = CRowFn()
    fn.out_schema = Schema("i", "u").c()
    fn.n_insn = 3
    for i, k in enumerate((capi.SRC_KEY, capi.SRC_LVAL, capi.SRC_CONST)):
        fn.code[i].op, fn.code[i].kind = capi.FN_PUSH, k
    fn.code[2].cst = 1
    for kind in (capi.SRC_ACC, capi.SRC_WEIGHT):
        fn.code[1].kind = kind
        refused(be, "map_index_fn", be.ctx, d.h, ctypes.byref(fn), _ref(o),
                names=f"map_index_fn: fn.code[1].kind = {kind} is not a source kind", status=INVALID, outs=[o])
        refused(be, "map_index_fanout", be.ctx, d.h, ctypes.byref(fn), 2, _ref(o),
                names=f"map_index_fanout: fn.code[1].kind = {kind} is not a source kind", status=INVALID, outs=[o])


def run_python_refusals(be):
    """Fold and Stream.aggregate refuse what cannot run, before any step; what only the library checks raises
    DbspError at the step"""
    with pytest.raises(ValueError, match="init has 2 accumulator words and step gives 1"):
        Fold([0, 0], [acc(0)])
    with pytest.raises(ValueError, match="an accumulator has 1..15"):
        Fold([0] * 16, [acc(0)] * 16, output=Proj(Schema("", "u"), [acc(0)]))
    with pytest.raises(ValueError, match="an accumulator has 1..15"):
        Fold([], [])
    with pytest.raises(ValueError, match="instructions"):
        Fold([0], [sum((lval(0) for _ in range(40)), acc(0))])
    with pytest.raises(ValueError, match="needs an output of at most 8 lanes"):
        Fold([0] * 9, [acc(0)] * 9)
    with pytest.raises(ValueError, match="key lanes"):
        Fold([0], [acc(0)], output=Proj(Schema("u", "u"), [key(0), acc(0)]))
    with pytest.raises(ValueError, match="fan-out"):
        Fold([0], [acc(0)], output=Proj(Schema("", "u"), [acc(0)], fanout=2))
    c = RootCircuit(be)
    st = {}
    s = Schema("u", "u")
    src = c.add_source(lambda: st["d"], s)
    with pytest.raises(ValueError, match="not a semigroup"):
        src.aggregate(f_sum(), local=True)
    # the library's rules: a value lane the input lacks, in the step and in the output
    for fold in (Fold([0], [acc(0) + lval(3)]), Fold([0], [acc(0)], output=Proj(Schema("", "u"), [lval(0)])),
                 Fold([0], [acc(0)], output=Proj(Schema("", "u"), [acc(2)]))):
        c = RootCircuit(be)
        src = c.add_source(lambda: st["d"], s)
        src.aggregate(fold)
        st["d"] = be.batch_from_columns(s, [np.array([1], np.uint64), np.array([2], np.uint64)])
        with pytest.raises(DbspError, match="aggregate_fold failed: DBSP_ERR_INVALID"):
            c.step()


def run_plain_oracle_lacks(oracle):
    """the dbsp_proj oracle has no dbsp_aggregate_fold: aggregate(Fold) names the missing call"""
    assert not oracle.api.exports("aggregate_fold")
    c = RootCircuit(oracle)
    src = c.add_source(lambda: None, Schema("u", "u"))
    with pytest.raises(DbspError, match="orc_aggregate_fold: this library does not export it"):
        src.aggregate(f_sum())
    with pytest.raises(DbspError, match="orc_aggregate_fold: this library does not export it"):
        src.stream_aggregate(f_sum())


def run_profile_class(be):
    s = Schema("i", "uu")
    rng = np.random.default_rng(4)
    T = [rows_full(rng, s, 1000, 100)]
    fold = f_weight()
    tr, ot = Spine(be, s), Spine(be, out_schema_of(s, fold))
    tr.insert(upload(be, s, T[0]))
    d = upload(be, s, T[0])
    be.profile(True)
    be.aggregate_fold(d, tr, ot, fold)
    prof = be.profile_read()
    be.profile(False)
    n, keys = len(T[0][1]), len(np.unique(T[0][0][0]))
    assert prof["agg_fold"]["launches"] == 1, prof
    assert prof["agg_fold"]["alg_bytes"] == n * (s.nl + 1) * 8 + keys * 3 * 8, prof


# ---- Nexmark q18 and q6 ---------------------------------------------------------------------------------------------
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _set(handles, tables):
    for k in ("person", "auction", "bid"):
        rows = tables.get(k, [])
        handles[k].set([np.array(x, np.uint64) for x in zip(*rows)] if rows else [np.zeros(0, np.uint64)] * 5)


def run_golden(be, query):
    """the reference's q18.rs / q6.rs tests: every step's output equals the expected Z-set"""
    from dbsp_b200.nexmark import queries as nq

    for case in golden()[query]:
        c = RootCircuit(be)
        inp, handles = nq.add_nexmark_input(c)
        o = nq.QUERIES[query](inp).output()
        for t, step in enumerate(case["steps"]):
            _set(handles, {"bid": step["bids"], "auction": step.get("auctions", [])})
            c.step()
            assert o.value.rows() == sorted(tuple(r) for r in step["expect"]), (case["name"], t, o.value.rows())


def m_q18(bids):
    """GROUP BY (auction, bidder): the first bid in (price, date_time, extra) order among those with the latest
    date_time, or the zero bid when every date_time is 0 (Bid::default() is never replaced)"""
    best = {}
    for b, w in sorted(bids.items()):
        if w == 0:
            continue
        k = b[:2]
        cur = best.get(k, (0, 0, 0, 0, 0))
        if b[3] > cur[3]:
            best[k] = b
        else:
            best.setdefault(k, cur)
    return {v: 1 for v in best.values()}


def m_q6(auctions, bids):
    """per seller, the average of the winning prices (max bid in [date_time, expires]) of its last 10 auctions by id"""
    win = {}
    for a in auctions:
        for b in bids.get(a[0], ()):
            if a[3] <= b[3] <= a[4]:
                k = (a[0], a[1])
                win[k] = max(win.get(k, 0), b[2])
    by_seller = {}
    for (aid, seller), p in sorted(win.items()):
        by_seller.setdefault(seller, []).append((aid, p))
    return {(s, sum(p for _, p in sorted(v)[-10:]) // len(sorted(v)[-10:])): 1 for s, v in by_seller.items()}


def run_generated(be, query, n_events=40_000, steps=3):
    """q18 / q6 on generated events, the integral of the output against the GROUP BY model after every step"""
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.nexmark import queries as nq

    gen = NexmarkGenerator(0x7FC359184519C0AA, first_event_rate=50)
    c = RootCircuit(be)
    inp, handles = nq.add_nexmark_input(c)
    integral = nq.QUERIES[query](inp).integrate().output()
    bids, auctions, by_auction = {}, [], {}
    for s in range(steps):
        t = gen.tables(s * n_events, n_events)
        for k in ("person", "auction", "bid"):
            handles[k].set(t[k])
        c.step()
        for b in zip(*[x.tolist() for x in t["bid"]]):
            bids[b] = bids.get(b, 0) + 1
            by_auction.setdefault(b[0], []).append(b)
        auctions += list(zip(*[x.tolist() for x in t["auction"]]))
        want = m_q18(bids) if query == "q18" else m_q6(auctions, by_auction)
        got = {r[:-1]: r[-1] for r in integral.value.rows()}
        assert got == want, (query, s, len(got), len(want))
    assert len(want) > 10


def run_nexmark_pair(be, ref, query, n_events=5_000_000, steps=5):
    import parity_util

    total = parity_util.run_nexmark_pair(be, ref, query, n_events * steps, n_events)
    assert total > 0


ALL_CASES = {}
for _s in (Schema("i", "iu"), Schema("uu", "ui")):
    for _f in FOLDS:
        ALL_CASES[f"direct_{_s.key}_{_s.val}_{_f}"] = lambda be, ref=None, s=_s, f=_f: run_direct(be, ref, s, f)
ALL_CASES["cancel_across_batches"] = run_cancel_across_batches
ALL_CASES["many_batches"] = run_many_batches
ALL_CASES["keyless"] = run_keyless
ALL_CASES["hot_key"] = run_hot_key
ALL_CASES["stream_aggregate"] = run_stream_aggregate
ALL_CASES["builtin_equivalents"] = run_builtin_equivalents
for _seed in range(6):
    ALL_CASES[f"random_{_seed}"] = lambda be, ref=None, seed=_seed: run_circuit_random(
        be, ref, Schema("iu", "ui") if seed % 2 else Schema("u", "iuu"),
        random_fold(seed, Schema("iu", "ui") if seed % 2 else Schema("u", "iuu")), steps=4, seed=seed,
        what=f"random fold {seed}")
for _name in FOLDS:
    ALL_CASES[f"circuit_{_name}"] = lambda be, ref=None, name=_name: run_circuit_random(
        be, ref, Schema("i", "iu"), FOLDS[name](), what=f"circuit {name}")
for _p in hc.PAIRS:
    for _r in ("growth", "churn", "hot"):
        ALL_CASES[f"regime_{_r}_{_p}"] = lambda be, ref=None, r=_r, p=_p: run_regime(be, ref, r, p)
