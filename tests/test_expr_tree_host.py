"""The TREE form of the expression program (csrc/expr_tree.h) without a GPU: `flockgpu_selftest_eval_tree` compiles
expressions to the register program the kernels run and interprets it on the host with the kernels' own interpreter.

The judge is a row-at-a-time restatement of the semantics in this file (`ref_eval`: DataFusion 6 / arrow-rs rules --
wrapping integers, truncated division, one IEEE rounding per Float64 node, Kleene logic, SQL CASE and IN), itself checked
against Arrow compute on the shapes Arrow compute expresses."""
import math
import re

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
from flock_b200 import _ffi, col, lit, case
from test_tpch_host import LIKE_PATTERNS

I32, I64, U64, F64, TS, UTF8, BOOL = fb.INT32, fb.INT64, fb.UINT64, fb.FLOAT64, fb.TIMESTAMP, fb.UTF8, fb.BOOL
U32, D32 = fb.UINT32, fb.DATE32


# ---- the reference: a postfix stack machine over python values (value, is_null, divided_by_zero) ----------------------
class DivideByZero(Exception):
    pass


def _wrap(v, dt):
    if dt in (I32, D32):
        return ((int(v) + (1 << 31)) & 0xffffffff) - (1 << 31)
    if dt == fb.UINT32:
        return int(v) & 0xffffffff
    if dt == U64:
        return int(v) & ((1 << 64) - 1)
    return ((int(v) + (1 << 63)) & ((1 << 64) - 1)) - (1 << 63)


def _rank(dt):
    return {I32: 1, fb.UINT32: 2, I64: 3, TS: 3, U64: 4}[dt]


def _promote(a, b):
    if a == b:
        return a
    if F64 in (a, b):
        return F64
    return a if _rank(a) >= _rank(b) else b


_RANGE = {I32: (-(1 << 31), (1 << 31) - 1), U32: (0, (1 << 32) - 1), I64: (-(1 << 63), (1 << 63) - 1), TS: (-(1 << 63), (1 << 63) - 1),
          U64: (0, (1 << 64) - 1)}


def _convert(v, frm, to, cast=False):
    """frm -> to.  Implicit conversions (coercion to a common type) wrap; an explicit CAST (cast=True) gives None where
    `to` cannot hold the value, as arrow-rs's numeric cast (num::cast::cast) does: NaN, +-inf, a float out of range
    once truncated toward zero, an integer out of range."""
    if frm == to or v is None or BOOL in (frm, to):
        return v
    if to == F64:
        return float(v)
    if frm == F64:
        if not math.isfinite(v):
            return None if cast else 0
        v = math.trunc(v)
    if cast:
        lo, hi = _RANGE[to]
        return v if lo <= v <= hi else None
    return _wrap(v, to)


def _arith(op, a, b, dt):
    if dt == F64:
        with np.errstate(all="ignore"):
            x, y = np.float64(a), np.float64(b)
            r = {fb.OP_ADD: x + y, fb.OP_SUB: x - y, fb.OP_MUL: x * y, fb.OP_DIV: x / y}[op]
        return float(r), False
    if op in (fb.OP_DIV, fb.OP_MOD):
        if b == 0:
            return 0, True
        q = abs(a) // abs(b) * (1 if (a < 0) == (b < 0) else -1)
        return _wrap(q if op == fb.OP_DIV else a - q * b, dt), False
    return _wrap({fb.OP_ADD: a + b, fb.OP_SUB: a - b, fb.OP_MUL: a * b}[op], dt), False


def _compare(op, a, b, lt, rt):
    if lt == UTF8:
        a, b = a.encode(), b.encode()
    elif F64 in (lt, rt):
        a, b = float(a), float(b)
        if math.isnan(a) or math.isnan(b):
            return op == fb.OP_NE
    elif U64 in (lt, rt) or fb.UINT32 in (lt, rt):
        a, b = a & ((1 << 64) - 1), b & ((1 << 64) - 1)
    return {fb.OP_EQ: a == b, fb.OP_NE: a != b, fb.OP_LT: a < b, fb.OP_LE: a <= b, fb.OP_GT: a > b, fb.OP_GE: a >= b}[op]


def _kleene(op, a, b):
    (va, na, ea, _), (vb, nb, eb, _) = a, b
    dom = op == fb.OP_OR
    decided = (not na and bool(va) == dom) or (not nb and bool(vb) == dom)
    if decided:
        return (dom, False, ea or eb, BOOL)
    return (None, True, ea or eb, BOOL) if (na or nb) else (not dom, False, ea or eb, BOOL)


def _like(s, pattern):
    """SQL LIKE without an escape character: '%' any run of code points, '_' exactly one."""
    rx = "".join(".*" if ch == "%" else "." if ch == "_" else re.escape(ch) for ch in pattern)
    return re.fullmatch(rx, s, re.DOTALL) is not None


def ref_eval_row(tokens, row, dtypes):
    st = []
    for op, dt, c, i64, f64, s in tokens:
        if op == fb.OP_COLUMN:
            st.append((row[c], row[c] is None, False, dtypes[c]))
        elif op == fb.OP_LIT_I64:
            st.append((_wrap(i64, dt), False, False, dt))
        elif op == fb.OP_LIT_F64:
            st.append((f64, False, False, F64))
        elif op == fb.OP_LIT_UTF8:
            st.append((s.decode(), False, False, UTF8))
        elif op == fb.OP_LIT_NULL:
            st.append((None, True, False, dt))
        elif op == fb.OP_CAST:
            v, n, e, t = st.pop()
            v = _convert(v, t, dt, cast=True)
            st.append((v, v is None, e, dt))
        elif op in (fb.OP_LIKE, fb.OP_NOT_LIKE):
            (p, np_, ep, _), (v, n, e, t) = st.pop(), st.pop()
            st.append((None, True, e or ep, BOOL) if n or np_ else (_like(v, p) != (op == fb.OP_NOT_LIKE), False, e or ep, BOOL))
        elif op == fb.OP_NEG:
            v, n, e, t = st.pop()
            st.append((None if n else (-v if t == F64 else _wrap(-v, t)), n, e, t))
        elif op == fb.OP_NOT:
            v, n, e, t = st.pop()
            st.append((None if n else not v, n, e, BOOL))
        elif op in (fb.OP_IS_NULL, fb.OP_IS_NOT_NULL):
            v, n, e, t = st.pop()
            st.append((n == (op == fb.OP_IS_NULL), False, e, BOOL))
        elif op in (fb.OP_AND, fb.OP_OR):
            b = st.pop()
            a = st.pop()
            st.append(_kleene(op, a, b))
        elif fb.OP_ADD <= op <= fb.OP_MOD:
            (vb, nb, eb, tb), (va, na, ea, ta) = st.pop(), st.pop()
            T = _promote(ta, tb)
            if na or nb:
                st.append((None, True, ea or eb, T))
            else:
                v, e = _arith(op, _convert(va, ta, T), _convert(vb, tb, T), T)
                st.append((v, False, ea or eb or e, T))
        elif fb.OP_EQ <= op <= fb.OP_GE:
            (vb, nb, eb, tb), (va, na, ea, ta) = st.pop(), st.pop()
            st.append((None, True, ea or eb, BOOL) if na or nb else (_compare(op, va, vb, ta, tb), False, ea or eb, BOOL))
        elif op == fb.OP_CASE:
            has_base, has_else = c & 1, c & 2
            need = 2 * i64 + (1 if has_base else 0) + (1 if has_else else 0)
            kids = st[len(st) - need:]
            del st[len(st) - need:]
            base = kids.pop(0) if has_base else None
            branches = [kids[2 * k + 1] for k in range(i64)] + ([kids[-1]] if has_else else [])
            T = None
            for v, n, e, t in branches:
                T = t if T is None else (T if BOOL in (T, t) else _promote(T, t))
            result, err = (None, True, False, T), False
            for k in range(i64):
                w, th = kids[2 * k], kids[2 * k + 1]
                if has_base:
                    w = (None, True, base[2] or w[2], BOOL) if base[1] or w[1] else (_compare(fb.OP_EQ, base[0], w[0], base[3], w[3]), False, base[2] or w[2], BOOL)
                err = err or w[2]
                if not w[1] and w[0]:
                    result = th
                    break
            else:
                if has_else:
                    result = kids[-1]
            v, n, e, t = result
            st.append((_convert(v, t, T), n, err or e, T))
        elif op == fb.OP_IN_LIST:
            kids = st[len(st) - (i64 + 1):]
            del st[len(st) - (i64 + 1):]
            x = kids[0]
            acc = None
            for l in kids[1:]:
                eq = (None, True, x[2], BOOL) if x[1] or l[1] else (_compare(fb.OP_EQ, x[0], l[0], x[3], l[3]), False, x[2], BOOL)
                acc = eq if acc is None else _kleene(fb.OP_OR, acc, eq)
            if c:
                acc = (None if acc[1] else not acc[0], acc[1], acc[2], BOOL)
            st.append(acc)
        else:
            raise AssertionError(op)
    assert len(st) == 1
    return st[0]


def ref_eval(e, batch):
    dtypes = [{pa.int32(): I32, pa.int64(): I64, pa.uint64(): U64, pa.uint32(): U32, pa.float64(): F64, pa.string(): UTF8, pa.date32(): D32}.get(f.type, TS)
              for f in batch.schema]
    cols = [c.to_pylist() for c in [pc.cast(c, pa.int64()) if pa.types.is_timestamp(c.type) else pc.cast(c, pa.int32()) if c.type == pa.date32() else c
                                    for c in batch.columns]]
    out = []
    for r in range(batch.num_rows):
        v, n, err, t = ref_eval_row(fb.E.wrap(e).tokens, [c[r] for c in cols], dtypes)
        if err:
            raise DivideByZero()
        out.append(None if n else v)
    return out


def same(got, valid, want, dtype):
    assert len(want) == len(valid)
    for r, w in enumerate(want):
        assert bool(valid[r]) == (w is not None), (r, w, got[r], valid[r])
        if w is None:
            continue
        if dtype == F64:
            g = float(got[r])
            assert (math.isnan(g) and math.isnan(w)) or np.float64(g).view(np.int64) == np.float64(w).view(np.int64), (r, w, g)
        else:
            assert int(got[r]) == (w if dtype != U64 else w & ((1 << 64) - 1)), (r, w, got[r])


def batch(n=64, seed=0, nulls=True):
    rng = np.random.default_rng(seed)
    mask = lambda k: (rng.integers(0, k, n) == 0) if nulls else None
    return pa.RecordBatch.from_arrays([
        pa.array(rng.integers(-50, 50, n).astype(np.int32), mask=mask(5)),
        pa.array(rng.integers(-(1 << 40), 1 << 40, n)),
        pa.array(rng.integers(0, 1 << 63, n, dtype=np.uint64) * np.uint64(2) + np.uint64(1)),
        pa.array(np.round(rng.normal(0, 100, n), 2), mask=mask(7)),
        pa.array(rng.integers(1_436_918_400_000, 1_436_918_500_000, n), pa.timestamp("ms")),
        pa.array([None if nulls and k == 7 else ["MAIL", "SHIP", "AIR", "RAIL", "1-URGENT", "2-HIGH", "", "x"][k] for k in rng.integers(0, 8, n)], pa.string()),
        pa.array(rng.integers(-3, 4, n).astype(np.int32)),
        pa.array(rng.integers(0, 11, n) / 100.0),
    ], names=["a", "l", "u", "f", "t", "s", "z", "d"])


# ---- the edge relation: the columns of batch() (same indices) plus UInt32, Date32 and a row id --------------------------
I32_MIN, I32_MAX, I64_MIN, I64_MAX = -(1 << 31), (1 << 31) - 1, -(1 << 63), (1 << 63) - 1
NEG_NAN = float(np.uint64(0xfff8000000000000).view(np.float64))
EDGE_POOLS = [
    [I32_MIN, I32_MAX, -1, 0, 1, I32_MIN + 1],                                                        # a   Int32
    [I64_MIN, I64_MAX, -1, 0, (1 << 53) + 1, -(1 << 53) - 1, I64_MIN + 1],                            # l   Int64
    [1 << 63, (1 << 64) - 1, 0, 1, (1 << 63) + 1, (1 << 63) - 1],                                      # u   UInt64
    [0.0, -0.0, math.inf, -math.inf, math.nan, NEG_NAN, 5e-324, -5e-324, 1.5e-310, 1e308, -1e308, 0.1,
     2.0 ** 63, -2.0 ** 63, 2.0 ** 64, 2147483647.9, -2147483648.9, 4294967295.5, -0.5, 9.3e18],        # f   Float64
    [-1, -86_400_000 * 365 * 30 - 7, I64_MIN, I64_MAX, 0, -1_000_000_000_000_001],                    # t   Timestamp(ms), before 1970
    ["", "é", "日本語", "a" * 70, "a" * 71, "PROMO", "PROMO BRUSHED", "PROMO BRUSHED TIN", "%", "_", "aé", "abab"],  # s   Utf8
    [-1, 1, I32_MIN, -1, 1],                                                                          # z   Int32 divisor (no 0)
    [0.0, -0.0, 0.1, 1e308, -5e-324],                                                                 # d   Float64
    [1 << 31, (1 << 32) - 1, 0, (1 << 31) - 1, (1 << 31) + 1],                                        # w   UInt32
    [0, -1, I32_MIN, I32_MAX, -719_162, 2_932_896],                                                   # day Date32
]
EDGE_BLOCK = 24                                 # rows of the fixed edge block: at the start, in the middle and at the end
WORDS = ["MAIL", "SHIP", "AIR", "RAIL", "1-URGENT", "2-HIGH", "", "x", "PROMO PLATED", "STANDARD PROMO", "promo x", "éa", "a%b", "a_b",
         "xxabxxab", "日本語"]
NULLABLE = (0, 2, 3, 5, 8, 9)                   # a, u, f, s, w, day; the rest never hold NULLs


def edge_relation(n, seed, nulls=7):
    """`n` rows: ~30 % of each column from its edge pool, the rest ordinary; one fixed edge block at the start, in the
    middle and in the last rows.  nulls: 0 none, 7 one row in 7, -1 every row but one (in the nullable columns)."""
    rng = np.random.default_rng(seed)
    ordinary = [rng.integers(-1000, 1000, n), rng.integers(-(1 << 40), 1 << 40, n), rng.integers(0, 1 << 64, n, dtype=np.uint64),
                np.round(rng.normal(0, 100, n), 2), rng.integers(1_436_918_400_000, 1_436_918_500_000, n), None,
                rng.choice([2, 3, -7, 1000, -1, 1], n), rng.integers(0, 11, n) / 100.0, rng.integers(0, 1 << 32, n, dtype=np.uint64),
                rng.integers(8000, 11000, n)]
    types = [np.int32, np.int64, np.uint64, np.float64, np.int64, object, np.int32, np.float64, np.uint32, np.int32]
    arrow = [pa.int32(), pa.int64(), pa.uint64(), pa.float64(), pa.timestamp("ms"), pa.string(), pa.int32(), pa.float64(), pa.uint32(), pa.date32()]
    starts = sorted({0, (n // 2) & ~3, max(n - EDGE_BLOCK, 0)})
    arrays = []
    for c, pool in enumerate(EDGE_POOLS):
        pool = np.array(pool, dtype=object if types[c] in (object, np.uint64) else types[c])
        if c == 5:
            v = np.array(WORDS + EDGE_POOLS[5], dtype=object)[rng.integers(0, len(WORDS) + len(EDGE_POOLS[5]), n)]
        else:
            v = ordinary[c].astype(types[c])
        edge = rng.random(n) < 0.3
        v = v.astype(object) if types[c] is np.uint64 else v
        v[edge] = pool[rng.integers(0, len(pool), int(edge.sum()))]
        for s in starts:
            k = min(EDGE_BLOCK, n - s)
            v[s:s + k] = pool[(np.arange(k) + c) % len(pool)]
        mask = None
        if c in NULLABLE and nulls and n:
            mask = rng.integers(0, nulls, n) == 0 if nulls > 0 else np.arange(n) != int(rng.integers(0, n))
        arrays.append(pa.array(v if types[c] is not np.uint64 else v.tolist(), arrow[c], mask=mask))
    arrays.append(pa.array(np.arange(n, dtype=np.int64)))
    return pa.RecordBatch.from_arrays(arrays, names=["a", "l", "u", "f", "t", "s", "z", "d", "w", "day", "rid"])


# ---- random trees ------------------------------------------------------------------------------------------------------
INT_TYPES = ("int32", "uint32", "int64", "uint64")


def random_tree(rng, depth, kind, edges=False):
    """kind: 'int' | 'float' | 'bool'.  edges=False: the columns of batch() and mild literals.  edges=True (the edge
    relation): also UInt32 / Date32 columns, the edge literals, division by the divisor column, Int32 results that
    wrap, comparisons across Int64 / UInt64 / Float64, NaN operands, explicit casts that can give NULL, CASE with a base
    expression and LIKE."""
    pick = lambda *xs: xs[int(rng.integers(0, len(xs)))]
    sub = lambda k: random_tree(rng, depth - 1, k, edges)
    if edges and rng.random() < 0.3:
        if depth == 0 or rng.random() < 0.4:
            if kind == "int":
                return pick(col(8), col(2), lit(I32_MIN, "int32"), lit(I32_MAX, "int32"), lit(I64_MIN), lit(I64_MAX), lit((1 << 53) + 1),
                            lit((1 << 64) - 1, "uint64"), lit(1 << 31, "uint32"), lit(-1), col(3).cast(pick(*INT_TYPES)),
                            col(1).cast(pick("int32", "uint32", "uint64")), col(2).cast(pick("int64", "int32")), col(8).cast("int32"),
                            col(0).cast(pick("uint32", "uint64")))
            if kind == "float":
                return pick(col(3), lit(math.nan), lit(NEG_NAN), lit(math.inf), lit(-math.inf), lit(-0.0), lit(5e-324), lit(1e308), lit(-1e308),
                            lit(0.1), col(2).cast("float64"), col(1).cast("float64"), col(8).cast("float64"))
            return pick(col(3) == math.nan, col(3) < lit(NEG_NAN), col(3) != math.nan, col(5).like(pick(*LIKE_PATTERNS), rng.random() < 0.4),
                        col(9) < lit(int(rng.integers(-2, 11000)), "date32"), col(9).isin([lit(0, "date32"), lit(-1, "date32"), lit(I32_MIN, "date32")]),
                        col(1) < col(2), col(2) >= col(3), col(1) == col(3), col(8) > col(0), col(8) <= col(1))
        r = rng.random()
        if kind == "int":
            if r < 0.3:
                return pick(sub("int") / col(6), sub("int") % col(6), sub("int") / col(6).cast("int64"), sub("int") % col(6).cast("int64"))
            if r < 0.5:
                return pick(col(0) * col(0), col(0) + lit(I32_MAX, "int32"), -col(0), col(0) * col(6) - lit(I32_MIN, "int32"), col(8) * col(8))
            if r < 0.75:
                return pick(sub("float").cast(pick(*INT_TYPES)), sub("int").cast(pick("int32", "uint32", "uint64")))
            return case([(int(rng.integers(-2, 3)), sub("int")), (lit(1 << 31, "uint32"), sub("int"))], base=pick(col(8), col(0), sub("int")),
                        otherwise=sub("int") if rng.random() < 0.6 else None)
        if kind == "float":
            return pick(sub("float") / sub("float"), sub("float") * sub("int"), sub("int").cast("float64") - sub("float"))
        if r < 0.5:
            a, b = pick(sub("int"), sub("float"), col(2), col(8)), pick(sub("int"), sub("float"), col(2), col(1))
            return pick(a == b, a != b, a < b, a <= b, a > b, a >= b)
        if r < 0.7:
            return col(5).like(pick(*LIKE_PATTERNS), rng.random() < 0.4) | sub("bool")
        return pick(sub("int"), sub("float")).isin([I64_MIN, -1, None] if rng.random() < 0.5 else [0, 1 << 31], negated=rng.random() < 0.4)
    if depth == 0 or rng.random() < 0.15:
        if kind == "int":
            return pick(col(0), col(1), col(6), col(0).cast("int64"), lit(int(rng.integers(-9, 10))), col(4).cast("int64"))
        if kind == "float":
            return pick(col(3), col(7), lit(float(np.round(rng.normal(0, 5), 2))), col(0).cast("float64"))
        return pick(col(0) > int(rng.integers(-20, 20)), col(5) == pick("MAIL", "SHIP", ""), col(3).is_null(), col(7) <= 0.05, col(5) < "RAIL")
    r = rng.random()
    if kind in ("int", "float"):
        if r < 0.5:
            a, b = sub(kind), sub(kind)
            ops = [lambda: a + b, lambda: a - b, lambda: a * b, lambda: a / b] + ([lambda: a % b] if kind == "int" else [])
            return ops[int(rng.integers(0, len(ops)))]()
        if r < 0.6:
            return -(sub(kind).cast("int64") if edges and kind == "int" else sub(kind))   # unary minus takes no unsigned operand
        if r < 0.85:
            n = int(rng.integers(1, 3))
            return case([(sub("bool"), sub(kind)) for _ in range(n)], otherwise=sub(kind) if rng.random() < 0.7 else None)
        if r < 0.92 and kind == "int":
            return case([(int(rng.integers(-3, 4)), sub("int")), (col(0), sub("int"))], base=col(6), otherwise=sub("int"))
        return sub("int").cast("float64") if kind == "float" else sub(kind)
    if r < 0.35:
        k = pick("int", "float")
        a, b = sub(k), sub(k)
        return pick(a == b, a != b, a < b, a <= b, a > b, a >= b)
    if r < 0.6:
        return pick(sub("bool") & sub("bool"), sub("bool") | sub("bool"))
    if r < 0.7:
        return ~sub("bool")
    if r < 0.8:
        return pick(sub("int"), sub("float")).is_null() if rng.random() < 0.5 else pick(sub("int"), sub("float")).is_not_null()
    if r < 0.9:
        return col(5).isin(["MAIL", "SHIP", None] if rng.random() < 0.3 else ["MAIL", "1-URGENT", ""], negated=rng.random() < 0.4)
    return sub("int").isin([int(v) for v in rng.integers(-5, 6, 3)] + ([None] if rng.random() < 0.3 else []), negated=rng.random() < 0.4)


@pytest.mark.parametrize("seed", [42, 7, 1234])
def test_random_trees_match_the_reference(seed):
    rng = np.random.default_rng(seed)
    ran = refused = failed = 0
    for k in range(120):
        b = batch(48, seed=seed * 1000 + k, nulls=k % 3 != 0)
        kind = ["int", "float", "bool"][k % 3]
        e = random_tree(rng, int(rng.integers(2, 7)), kind)
        try:
            want = ref_eval(e, b)
        except DivideByZero:
            want = None
        try:
            if kind == "bool":
                got, _ = fb.selftest_eval_tree(b, e, predicate=True)
            else:
                (got, valid, dt), = fb.selftest_eval_tree(b, [e])[0]
        except fb.FlockGpuError as err:
            if err.code == _ffi.ERR_UNSUPPORTED and ("registers" in err.message or "instructions" in err.message):
                refused += 1
                continue
            assert err.code == _ffi.ERR_EXECUTION and want is None, (err, e.tokens)
            failed += 1
            continue
        assert want is not None, e.tokens
        if kind == "bool":
            assert list(got) == [w is True for w in want], e.tokens       # FilterExec keeps the rows whose predicate is TRUE
        elif got is not None:                                             # None: the tree is a plain column
            same(got, valid, want, dt)
        ran += 1
    assert ran >= 80 and refused <= 30, (ran, refused, failed)   # the deepest trees exceed the register budget: refused by name


# ---- the reference against Arrow compute -------------------------------------------------------------------------------
def test_reference_and_tree_agree_with_arrow_compute():
    b = batch(200, seed=5)
    A, L, F, S, D = b.column(0), b.column(1), b.column(3), b.column(5), b.column(7)
    A64 = pc.cast(A, pa.int64())
    cases = [
        (case([(col(0) > 3, col(1)), (col(3) < 0.0, col(1) * 2)], otherwise=lit(0)),
         pc.case_when(pc.make_struct(pc.greater(A, 3), pc.less(F, 0.0)), L, pc.multiply(L, 2), pa.scalar(0, pa.int64()))),
        (case([(col(0) > 3, col(3))]), pc.case_when(pc.make_struct(pc.greater(A, 3)), F)),                    # no ELSE: NULL
        (col(3) * (1.0 - col(7)) * (1.0 + col(7)), pc.multiply(pc.multiply(F, pc.subtract(1.0, D)), pc.add(1.0, D))),   # TPC-H q1
        (-col(3), pc.negate(F)),
        (-col(0), pc.negate(A)),
        (case([((col(5) == "1-URGENT") | (col(5) == "2-HIGH"), lit(1))], otherwise=lit(0)),                  # TPC-H q12
         pc.if_else(pc.fill_null(pc.or_kleene(pc.equal(S, "1-URGENT"), pc.equal(S, "2-HIGH")), False), 1, 0)),
    ]
    for e, arrow in cases:
        want = ref_eval(e, b)
        assert want == arrow.to_pylist(), e.tokens
        (got, valid, dt), = fb.selftest_eval_tree(b, [e])[0]
        same(got, valid, want, dt)
    preds = [
        (col(5).isin(["MAIL", "SHIP"]), pc.is_in(S, value_set=pa.array(["MAIL", "SHIP"]))),
        (col(5).isin(["MAIL", "SHIP"], negated=True), None),
        (col(0).cast("int64").isin([1, 2, 3]).is_null(), pc.is_null(pc.equal(A64, 1))),
        (col(3).is_null() | (col(0) > 0), pc.or_kleene(pc.is_null(F), pc.greater(A, 0))),
        ((col(7) >= lit(0.06) - 0.01) & (col(7) <= lit(0.06) + 0.01), pc.and_(pc.greater_equal(D, 0.06 - 0.01), pc.less_equal(D, 0.06 + 0.01))),  # q6 BETWEEN
    ]
    for e, arrow in preds:
        keep = [w is True for w in ref_eval(e, b)]
        got, _ = fb.selftest_eval_tree(b, e, predicate=True)
        assert list(got) == keep, e.tokens
        if arrow is not None:
            assert keep == [x is True for x in arrow.to_pylist()], e.tokens
    # NOT IN over a NULL value is NULL (the row is dropped), which pc.is_in (NULL -> false -> inverted true) does not say
    e = col(5).isin(["MAIL", "SHIP"], negated=True)
    keep, _ = fb.selftest_eval_tree(b, e, predicate=True)
    assert not any(k for k, s in zip(keep, S.to_pylist()) if s is None) and any(keep)


# ---- hand-written edges ------------------------------------------------------------------------------------------------
def test_null_tables_of_every_opcode():
    t = pa.array([True, True, True, False, False, False, None, None, None])
    u = pa.array([True, False, None] * 3)
    x = pa.array([1 if v else 0 if v is not None else None for v in t.to_pylist()], pa.int32())
    y = pa.array([1 if v else 0 if v is not None else None for v in u.to_pylist()], pa.int32())
    b = pa.RecordBatch.from_arrays([x, y], names=["x", "y"])
    P, Q = col(0) == 1, col(1) == 1
    as_value = lambda p: case([(p, lit(1)), (~p, lit(0))])                # TRUE -> 1, FALSE -> 0, NULL -> NULL
    for e, arrow in [(P & Q, pc.and_kleene(t, u)), (P | Q, pc.or_kleene(t, u)), (~P, pc.invert(t)), (P.is_null(), pc.is_null(t)),
                     (P.is_not_null(), pc.is_valid(t)), (~(P & ~Q) | P.is_null(), pc.or_kleene(pc.invert(pc.and_kleene(t, pc.invert(u))), pc.is_null(t)))]:
        (got, valid, dt), = fb.selftest_eval_tree(b, [as_value(e)])[0]
        want = [None if v is None else int(v) for v in arrow.to_pylist()]
        same(got, valid, want, dt)
    for e, want in [(col(0) + col(1), [2, 1, None, 1, 0, None, None, None, None]), (-col(0), [-1, -1, -1, 0, 0, 0, None, None, None]),
                    (col(0).isin([1, None]), None)]:
        if want is None:
            keep, _ = fb.selftest_eval_tree(b, e, predicate=True)
            assert list(keep) == [True] * 3 + [False] * 6                 # 0 IN (1, NULL) is NULL, not FALSE; both drop the row
            (got, valid, dt), = fb.selftest_eval_tree(b, [as_value(e)])[0]
            same(got, valid, [1, 1, 1, None, None, None, None, None, None], dt)
        else:
            (got, valid, dt), = fb.selftest_eval_tree(b, [e])[0]
            same(got, valid, want, dt)


def test_case_shapes_and_division_by_zero():
    b = batch(64, seed=9)
    z = b.column(6).to_pylist()
    l = b.column(1).to_pylist()
    # CASE with a base expression, no ELSE
    (got, valid, dt), = fb.selftest_eval_tree(b, [case([(0, lit(10)), (1, col(1))], base=col(6))])[0]
    same(got, valid, [10 if v == 0 else l[r] if v == 1 else None for r, v in enumerate(z)], dt)
    # 1 / 0 in a branch that is never taken gives a result ...
    guarded = case([(col(6) != 0, col(1) / col(6).cast("int64"))], otherwise=lit(-1))
    (got, valid, dt), = fb.selftest_eval_tree(b, [guarded])[0]
    same(got, valid, ref_eval(guarded, b), dt)
    assert 0 in z
    # ... and FLOCKGPU_ERR_EXECUTION in one that is
    with pytest.raises(fb.FlockGpuError, match="Divide by zero") as info:
        fb.selftest_eval_tree(b, [case([(col(6) >= 0, col(1) / col(6).cast("int64"))], otherwise=lit(-1))])
    assert info.value.code == _ffi.ERR_EXECUTION
    with pytest.raises(fb.FlockGpuError, match="Divide by zero"):
        fb.selftest_eval_tree(b, (col(1) + col(1)) % (col(6) - col(6)).cast("int64") == 0, predicate=True)
    # a NULL divisor raises nothing: the quotient is NULL
    null_divisor = (col(1) + 1) / case([(col(6) != 0, col(6).cast("int64"))])
    (got, valid, dt), = fb.selftest_eval_tree(b, [null_divisor])[0]
    want = ref_eval(null_divisor, b)
    assert None in want
    same(got, valid, want, dt)


def test_limits_are_refused_by_name():
    b = batch(8, seed=1)
    deep = col(1)
    for k in range(12):                                                      # a right-deep comb: every level holds a register
        deep = (col(1) + k) * (deep - (col(0).cast("int64") * k))
    wide = col(1) + 1
    for k in range(80):                                                      # 80 different products: few registers, many instructions
        wide = wide + (col(1) + k) * (col(1) - k)
    for e in (deep, wide):
        try:
            fb.selftest_eval_tree(b, [e])
        except fb.FlockGpuError as err:
            assert err.code == _ffi.ERR_UNSUPPORTED and ("registers" in err.message or "instructions" in err.message)
    with pytest.raises(fb.FlockGpuError, match="more than") as info:
        fb.selftest_eval_tree(b, [wide])
    assert info.value.code == _ffi.ERR_UNSUPPORTED
    with pytest.raises(fb.FlockGpuError, match="Utf8") as info:              # a CASE that returns strings
        fb.selftest_eval_tree(b, [case([(col(0) > 0, lit("a"))], otherwise=lit("b"))])
    assert info.value.code == _ffi.ERR_UNSUPPORTED
    with pytest.raises(fb.FlockGpuError, match="boolean") as info:           # tables have no Boolean type
        fb.selftest_eval_tree(b, [col(0) > 0])
    assert info.value.code == _ffi.ERR_UNSUPPORTED
    for bad in (fb.E(col(0).tokens + [(fb.OP_CASE, 0, fb.CASE_HAS_ELSE, 1, 0.0, None)]),            # CASE short of operands
                fb.E(col(0).tokens + lit(1).tokens + [(fb.OP_CASE, 0, 8, 1, 0.0, None)]),               # unknown flag bits
                fb.E(col(0).tokens + [(fb.OP_IN_LIST, 0, 0, 3, 0.0, None)]),                            # IN short of operands
                fb.E(col(0).tokens + col(1).tokens + [(fb.OP_IN_LIST, 0, 0, 1, 0.0, None)])):           # IN over a non-literal
        with pytest.raises(fb.FlockGpuError) as info:
            fb.selftest_eval_tree(b, [bad])
        assert info.value.code == _ffi.ERR_INVALID, bad.tokens


def test_common_subexpressions_are_computed_once():
    """TPC-H q1 sums l_extendedprice * (1 - l_discount) and that product times (1 + l_tax): one program, the shared product once."""
    b = batch(32, seed=2)
    disc_price = col(3) * (1.0 - col(7))
    _, alone = fb.selftest_eval_tree(b, [disc_price])
    out, both = fb.selftest_eval_tree(b, [disc_price, disc_price * (1.0 + col(7))])
    assert both == alone + 3                                                 # add, multiply, store: the literal 1.0 is shared too
    same(out[0][0], out[0][1], ref_eval(disc_price, b), F64)
    same(out[1][0], out[1][1], ref_eval(disc_price * (1.0 + col(7)), b), F64)
    out, _ = fb.selftest_eval_tree(b, [col(4), col(1) + 1])                  # plain columns stay plain columns
    assert out[0][0] is None and out[0][2] == TS and out[1][2] == I64


def test_old_forms_still_win():
    """Everything the chain / term forms evaluate exactly keeps them: same fast kinds, same pass-through answers as
    before.  What they cannot evaluate exactly, such as a lossy CAST, they refuse."""
    b = batch(64, seed=3, nulls=False)
    for e, fast in [(col(0).cast("int64") % 123 == 0, 1), (col(0).cast("int64") == 10, 2), (~(col(0).cast("int64") < 5), 2),
                    ((col(5) == "MAIL") | (col(5) == "SHIP"), 0), ((col(1) + 5) * 3 > col(0).cast("int64"), 0)]:
        got, kind = fb.selftest_eval_predicate(b, e)
        assert kind == fast
        tree, _ = fb.selftest_eval_tree(b, e, predicate=True)                 # and the tree form gives the same rows
        assert np.array_equal(got, tree)
    v, dt = fb.selftest_eval_value(b, col(4))
    assert v is None and dt == TS
    v, dt = fb.selftest_eval_value(b, 0.908 * col(0).cast("float64"))
    (tv, valid, tdt), = fb.selftest_eval_tree(b, [0.908 * col(0).cast("float64")])[0]
    assert dt == tdt == F64 and np.array_equal(v.view(np.int64), tv.view(np.int64))
    for e in (case([(col(0) > 0, lit(1))], otherwise=lit(0)), -col(1), col(1) * (col(1) + 1) * (col(1) - 1) * (col(0).cast("int64") + col(1))):
        with pytest.raises(fb.FlockGpuError) as info:                        # the chain form keeps refusing what it refused
            fb.selftest_eval_value(b, e)
        assert info.value.code == _ffi.ERR_UNSUPPORTED


# ---- the edge relation: the host interpreter against the reference, the reference against Arrow compute ----------------
def run_tree(b, e, kind):
    """The host build of the tree form: ('ok', mask | (values, valid, dtype)), ('refused', None) for a tree over the
    compiler's register / instruction budget, ('raised', None) for "Divide by zero"."""
    try:
        if kind == "bool":
            return "ok", fb.selftest_eval_tree(b, e, predicate=True)[0]
        return "ok", fb.selftest_eval_tree(b, [e])[0][0]
    except fb.FlockGpuError as err:
        if err.code == _ffi.ERR_UNSUPPORTED and ("registers" in err.message or "instructions" in err.message):
            return "refused", None
        assert err.code == _ffi.ERR_EXECUTION and "Divide by zero" in err.message, (err, e.tokens)
        return "raised", None


def check_against_reference(b, e, kind, got):
    """`got` (run_tree over `b`) against ref_eval over the same rows."""
    status, res = got
    try:
        want = ref_eval(e, b)
    except DivideByZero:
        assert status == "raised", e.tokens
        return
    assert status == "ok", (status, e.tokens)
    if kind == "bool":
        assert list(res) == [w is True for w in want], e.tokens
    elif res[0] is not None:
        same(res[0], res[1], want, res[2])


@pytest.mark.parametrize("seed", [42, 7, 1234])
def test_random_edge_trees_match_the_reference(seed):
    rng = np.random.default_rng(seed)
    counts = {"ok": 0, "refused": 0, "raised": 0}
    for k in range(90):
        b = edge_relation(300, seed=seed * 1000 + k, nulls=[0, 7, -1][k % 3])
        kind = ["int", "float", "bool"][k % 3]
        e = random_tree(rng, int(rng.integers(2, 6)), kind, edges=True)
        got = run_tree(b, e, kind)
        counts[got[0]] += 1
        if got[0] != "refused":
            check_against_reference(b, e, kind, got)
    assert counts["ok"] >= 55 and counts["refused"] <= 20, counts


def test_edge_reference_agrees_with_arrow_compute():
    b = edge_relation(400, seed=3)
    A, L, U, F, S, W = (b.column(i) for i in (0, 1, 2, 3, 5, 8))
    keep = lambda e: [w is True for w in ref_eval(e, b)]
    arrow = lambda x: [w is True for w in x.to_pylist()]
    for p in LIKE_PATTERNS:
        for negated in (False, True):
            want = pc.match_like(S, p)
            assert keep(col(5).like(p, negated)) == arrow(pc.invert(want) if negated else want), p
    P, Q = col(0) > 0, col(3) < 0.5
    AP, AQ = pc.greater(A, 0), pc.less(F, 0.5)
    for e, x in [(P & Q, pc.and_kleene(AP, AQ)), (P | Q, pc.or_kleene(AP, AQ)), (~(P & ~Q), pc.invert(pc.and_kleene(AP, pc.invert(AQ)))),
                 (col(1).isin([I64_MIN, -1, 0, (1 << 53) + 1]), pc.is_in(L, value_set=pa.array([I64_MIN, -1, 0, (1 << 53) + 1]))),
                 (col(8).isin([lit(1 << 31, "uint32"), lit(0, "uint32")]), pc.is_in(W, value_set=pa.array([1 << 31, 0], pa.uint32()))),
                 (col(2).isin([lit((1 << 64) - 1, "uint64")]), pc.is_in(U, value_set=pa.array([(1 << 64) - 1], pa.uint64()))),
                 (col(3) == math.nan, pc.equal(F, math.nan)), (col(3) >= 0.1, pc.greater_equal(F, 0.1))]:
        assert keep(e) == arrow(x), e.tokens
    # Int32 arithmetic wraps (arrow's unchecked kernels); the integer CASTs agree with Arrow's checked cast (Arrow's
    # Float64 -> integer cast cannot be the judge: it truncates only with its range check switched off)
    assert ref_eval(col(0) * col(0), b) == pc.multiply(A, A).to_pylist()
    for src, to, dt in [(1, "int32", pa.int32()), (2, "int64", pa.int64()), (8, "int32", pa.int32()), (0, "uint64", pa.uint64())]:
        got = ref_eval(col(src).cast(to), b)
        for r, v in enumerate(got):
            w = b.column(src).slice(r, 1)
            if v is not None:
                assert [v] == pc.cast(w, dt).to_pylist()
            elif w.null_count == 0:                                        # NULL only where Arrow's checked cast refuses the value
                with pytest.raises(pa.ArrowInvalid):
                    pc.cast(w, dt)


def test_lossy_cast_is_null_in_the_tree_form_and_refused_by_the_chain():
    """CAST(Float64 AS an integer type) and narrowing integer CASTs: NULL where the target cannot hold the value
    (arrow-rs's numeric cast), truncation toward zero otherwise.  The chain and term forms have no NULLs of their own:
    they refuse such a cast, and the operators evaluate it in the tree form."""
    f = [0.0, -0.0, math.inf, -math.inf, math.nan, NEG_NAN, 2.5, -2.5, 2147483647.9, 2147483648.0, -2147483648.9, -2147483649.0, -0.5, -1.0,
         4294967295.5, 4294967296.0, 2.0 ** 63, -2.0 ** 63, 9223372036854774784.0, 2.0 ** 64, 18446744073709549568.0, 1e308, 5e-324]
    i = [0, -1, I32_MIN, I32_MAX, I32_MAX + 1, I32_MIN - 1, (1 << 32) - 1, 1 << 32, I64_MIN, I64_MAX]
    u = [0, 1, I32_MAX, 1 << 31, (1 << 32) - 1, 1 << 32, I64_MAX, 1 << 63, (1 << 64) - 1, 5]
    b = pa.record_batch([pa.array(f), pa.array(i + [7] * (len(f) - len(i))), pa.array(u + [7] * (len(f) - len(u)), pa.uint64())], ["f", "i", "u"])
    fits = {"int32": lambda v: I32_MIN <= v <= I32_MAX, "uint32": lambda v: 0 <= v < 1 << 32, "int64": lambda v: I64_MIN <= v <= I64_MAX,
            "uint64": lambda v: 0 <= v < 1 << 64}
    for src in range(3):
        for to in INT_TYPES:
            e = col(src).cast(to)
            want = ref_eval(e, b)
            for v, w in zip(b.column(src).to_pylist(), want):
                t = math.trunc(v) if isinstance(v, float) and math.isfinite(v) else v
                assert w == (t if isinstance(t, int) and fits[to](t) else None), (src, to, v, w)
            if src == 1 and to == "int64" or src == 2 and to == "uint64":
                continue                                                   # no cast at all: a plain column
            (vals, valid, dt), = fb.selftest_eval_tree(b, [e])[0]
            same(vals, valid, want, dt)
            mask, _ = fb.selftest_eval_tree(b, e.is_null(), predicate=True)         # IS NULL sees the NULLs of the cast
            assert list(mask) == [w is None for w in want]
            for chain_form in (lambda: fb.selftest_eval_value(b, e), lambda: fb.selftest_eval_predicate(b, e > 0)):
                with pytest.raises(fb.FlockGpuError, match="a CAST that can give NULL") as info:
                    chain_form()
                assert info.value.code == _ffi.ERR_UNSUPPORTED
    # widening casts and implicit coercion keep wrapping, and keep the chain form
    v, dt = fb.selftest_eval_value(b, col(1).cast("float64") + col(2).cast("float64"))
    assert dt == F64
    v, dt = fb.selftest_eval_value(b, col(1) + col(2))                     # Int64 + UInt64: both as UInt64, wrapping
    assert dt == U64 and [int(x) for x in v] == [(x + y) & ((1 << 64) - 1) for x, y in zip(b.column(1).to_pylist(), b.column(2).to_pylist())]
