"""The inner hash join at the edges of its key types, against `ref_join`, a plain dict-of-rows reference.

Decided semantics (SURVEY.md Appendix C.8): two key tuples match when every component pair is non-NULL and equal;
Float64 components are equal when their bit patterns are and neither is NaN (NaN matches nothing, -0.0 does not meet
+0.0, +inf meets +inf); the key columns of the two sides must have one type, Timestamp unit and zone included, or the
join fails with FLOCKGPU_ERR_UNSUPPORTED before any fast path runs.

Which path of hash_join.cu each case reaches.  The launch profile names the kernels, not their KW instantiation, so
the rule that picks it is stated here: one key column of 4 bytes -> KW 4, of 8 bytes -> KW 8, two columns of 4 bytes
or anything else -> KW 0 (two 4-byte columns packed into one word, otherwise row keys); the side with fewer rows is
hashed, and a hashed side of ONE row with a 4- or 8-byte key, no validity on either key and no Float64 key runs
`join_one_kernel` instead of build / count / emit.
  * join_*_kernel<4> (16-byte slot table)      one Int32, UInt32 or Date32 key             test_single_key_edges
  * join_*_kernel<8> (representative-row table) one Int64, UInt64, Timestamp (s/ms/us/ns, with and without zone) or
                                                 Float64 key                               test_single_key_edges
  * join_*_kernel<0>, packed                    (Int32, Int32), (Int32, Date32), (UInt32, Int32)  test_multi_key_edges
  * join_*_kernel<0>, row keys                  (Int64, Int64), (Int64, Int32), Utf8, (Utf8, Int32), 3 and 8 keys
                                                 test_multi_key_edges; 9 keys refused in test_nine_keys_refused
  * join_one_kernel<4> / <8>                    test_one_build_row (and where it must not run: a NULL on the single
                                                 row, NULLs on the probe side, a Float64 key)
  * table capacity and probe-chain wrap-around  test_sizes, test_crafted_collisions_wrap_the_probe
  * count scan, both grid-prefix protocols      test_sizes (compact_mode 0 and 1)
  * the 2^32 - 2 pair limit                     test_pair_count_limit
  * DeferredAgg::select_equal                   test_select_equal_fast_path (dense_argmax_kernel / no join kernel)
  * DeferredGroups::select_group_match          test_select_group_match_fast_path (group_match_kernel)
  * the one-pass join count (dim_count_kernel)  test_join_count_plan_refuses_unlike_timestamp_units
  * hash_partition then join part by part       test_partitioned_join
The tests without the `gpu` mark check the reference itself against the oracle and Acero, and the crafted
collisions against sharding.fmix64."""
import collections

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import oracle
from flock_b200 import plans, sharding

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
ERR_UNSUPPORTED = -2
JOIN_KERNELS = ("join_one_kernel", "join_build_kernel", "join_count_scan_kernel", "join_emit_kernel")


def f64(bits: int) -> float:
    return float(np.array([bits], np.uint64).view(np.float64)[0])


FLOAT_EDGES = [0.0, -0.0, np.inf, -np.inf, f64(0x7FF8000000000000), f64(0xFFF8000000000000), f64(0x7FF0000000000001),
               f64(0xFFF4000000000123), 5e-324, -5e-324, 2.2250738585072009e-308, 1.5, -1.5, 2.0 ** 53]
UTF8_EDGES = ["", "a", "a\0", "\0", "abcdefg", "abcdefgh", "abcdefghi", "o" * 15, "o" * 16, "o" * 17, "o" * 16 + "p",
              "o" * 16 + "q", "é", "日本語", "\U0001F600x", "L" * 69 + "a", "L" * 69 + "b"]
TS_UNITS = [("s", None), ("ms", None), ("us", None), ("ns", None), ("s", "UTC"), ("ms", "UTC"), ("us", "Europe/Paris"), ("ns", "UTC")]
TS_EDGES = [I64_MIN, I64_MIN + 1, -86_400_000_123, -1, 0, 1, 86_400_000, I64_MAX]

# key kind -> (Arrow type, edge values, how to draw filler values)
KEY_KINDS = {
    "int32": (pa.int32(), [I32_MIN, -1, 0, I32_MAX, 7], lambda r, n: r.integers(I32_MIN, I32_MAX, n, dtype=np.int64)),
    "uint32": (pa.uint32(), [0, 1, 1 << 31, (1 << 32) - 1, (1 << 31) - 1], lambda r, n: r.integers(0, 1 << 32, n, dtype=np.int64)),
    "date32": (pa.date32(), [-719_162, -25_567, -1, 0, 1, 2_932_896], lambda r, n: r.integers(-800_000, 3_000_000, n)),
    "int64": (pa.int64(), [I64_MIN, I64_MAX, 5, (1 << 32) + 5, (3 << 32) + 5, -1, (1 << 32) - 1, (1 << 53) + 1, 1 << 53],
              lambda r, n: r.integers(I64_MIN, I64_MAX, n, dtype=np.int64)),
    "uint64": (pa.uint64(), [1 << 63, (1 << 64) - 1, (1 << 63) + 1, 0, 5, (1 << 32) + 5],
               lambda r, n: r.integers(0, 1 << 64, n, dtype=np.uint64)),
    "float64": (pa.float64(), FLOAT_EDGES, lambda r, n: r.standard_normal(n) * 1e6),
    "utf8": (pa.utf8(), UTF8_EDGES, lambda r, n: ["s%x" % v for v in r.integers(0, 1 << 40, n)]),
}
for _u, _tz in TS_UNITS:
    KEY_KINDS["ts_%s_%s" % (_u, _tz or "naive")] = (pa.timestamp(_u, _tz), TS_EDGES, lambda r, n: r.integers(-(1 << 50), 1 << 50, n))


def rb(**cols):
    return pa.RecordBatch.from_arrays(list(cols.values()), names=list(cols.keys()))


def make_array(typ: pa.DataType, values, null_mask=None) -> pa.Array:
    """An array of `typ` from Python / numpy values; NULL slots of a fixed-width array keep the value under them."""
    if pa.types.is_string(typ):
        return pa.array([None if null_mask is not None and null_mask[i] else v for i, v in enumerate(values)], pa.utf8())
    if pa.types.is_floating(typ):
        raw = pa.array(np.asarray(values, np.float64))
    elif pa.types.is_date32(typ):
        raw = pa.array(np.asarray(values, np.int64).astype(np.int32))
    elif pa.types.is_timestamp(typ):
        raw = pa.array(np.asarray(values, np.int64))
    else:
        raw = pa.array(np.asarray(values).astype(typ.to_pandas_dtype()))
    if null_mask is None or not np.any(null_mask):
        return raw.view(typ) if not raw.type.equals(typ) else raw
    bitmap = pa.array(~np.asarray(null_mask, bool)).buffers()[1]
    return pa.Array.from_buffers(typ, len(raw), [bitmap, raw.buffers()[1]])


def draw_keys(kind: str, n: int, rng, edge_share: float, filler=None):
    """n values of `kind`: edge values (each many times) mixed with filler values drawn at random."""
    typ, edges, draw = KEY_KINDS[kind]
    fill = draw(rng, n) if filler is None else filler
    pick = rng.integers(0, len(edges), n)
    use_edge = rng.random(n) < edge_share
    if pa.types.is_string(typ):
        return [edges[p] if e else f for p, e, f in zip(pick, use_edge, fill)]
    edge_arr = np.array(edges, dtype=np.float64 if pa.types.is_floating(typ) else (np.uint64 if typ == pa.uint64() else np.int64))
    fill = np.asarray(fill).astype(edge_arr.dtype)
    return np.where(use_edge, edge_arr[pick], fill)


def payload(n: int, rng, tag: int) -> dict:
    """Columns of every type, some nullable, and `id`: the row's position, unique on its side."""
    ids = np.arange(n, dtype=np.int64)
    null = ids % 7 == 3
    return {
        "id": pa.array(ids),
        "p_i32": make_array(pa.int32(), (ids * 2654435761) % (1 << 31) - (1 << 30)),
        "p_u32": make_array(pa.uint32(), (ids * 40503 + tag) % (1 << 32), null),
        "p_u64": make_array(pa.uint64(), (ids.astype(np.uint64) << np.uint64(40)) | np.uint64(tag)),
        "p_f64": make_array(pa.float64(), np.where(ids % 5 == 0, -0.0, ids * 0.25 - 7.0), ids % 11 == 1),
        "p_d32": make_array(pa.date32(), ids % 40_000 - 20_000, null),
        "p_ts": make_array(pa.timestamp("us"), ids * 1_000_003 - (1 << 40)),
        "p_s": make_array(pa.utf8(), ["v%d%s" % (i, "w" * int(i % 23)) for i in ids], ids % 9 == 2),
    }


def side(kinds, n, rng, prefix, null_every=None, filler=None, keys_first=True, with_payload=True, edge_share=0.1):
    """A relation with key columns of `kinds` (named <prefix>k<i>) and payload columns; `null_every[i]` puts a NULL in
    key i every that many rows (values under the NULLs are live keys)."""
    keys = {}
    for i, kind in enumerate(kinds):
        vals = draw_keys(kind, n, rng, edge_share, None if filler is None else filler[i])
        mask = None
        if null_every and null_every[i]:
            mask = (np.arange(n) % null_every[i]) == (i % null_every[i])
        keys["%sk%d" % (prefix, i)] = make_array(KEY_KINDS[kind][0], vals, mask)
    pay = {prefix + k: v for k, v in payload(n, rng, len(prefix)).items()} if with_payload else {prefix + "id": pa.array(np.arange(n, dtype=np.int64))}
    cols = {**keys, **pay} if keys_first else {**pay, **keys}
    b = rb(**cols)
    key_idx = [b.schema.names.index("%sk%d" % (prefix, i)) for i in range(len(kinds))]
    return b, key_idx


# ---- the reference ------------------------------------------------------------------------------------------------------
def key_components(arr) -> list:
    """One hashable per row, or None where the row can match nothing (NULL, or a NaN Float64)."""
    arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
    valid = np.asarray(arr.is_valid())
    t = arr.type
    if pa.types.is_floating(t):
        vals = arr.fill_null(0.0).to_numpy(zero_copy_only=False)
        bits = vals.view(np.uint64).tolist()
        nan = np.isnan(vals)
        return [b if v and not z else None for b, v, z in zip(bits, valid, nan)]
    if pa.types.is_string(t):
        return [None if s is None else s.encode() for s in arr.to_pylist()]
    if pa.types.is_date32(t):
        vals = arr.view(pa.int32()).fill_null(0).to_numpy(zero_copy_only=False).tolist()
    elif pa.types.is_timestamp(t):
        vals = arr.view(pa.int64()).fill_null(0).to_numpy(zero_copy_only=False).tolist()
    else:
        vals = arr.fill_null(0).to_numpy(zero_copy_only=False).tolist()
    return [x if v else None for x, v in zip(vals, valid)]


def key_tuples(batch, keys) -> list:
    comps = [key_components(batch.column(k)) for k in keys]
    return [None if any(c is None for c in t) else t for t in zip(*comps)]


def ref_pairs(left, right, lkeys, rkeys):
    build = collections.defaultdict(list)
    for i, k in enumerate(key_tuples(left, lkeys)):
        if k is not None:
            build[k].append(i)
    li, ri = [], []
    for j, k in enumerate(key_tuples(right, rkeys)):
        rows = build.get(k) if k is not None else None
        if rows:
            li.extend(rows)
            ri.extend([j] * len(rows))
    return np.array(li, np.int64), np.array(ri, np.int64)


def ref_join(left, right, lkeys, rkeys) -> pa.Table:
    """left JOIN right ON left.lkeys = right.rkeys (Inner): a dict from key tuple to build rows, materialised with take
    as left ++ right."""
    li, ri = ref_pairs(left, right, lkeys, rkeys)
    cols = [c.take(pa.array(li)) for c in left.columns] + [c.take(pa.array(ri)) for c in right.columns]
    return pa.Table.from_arrays(cols, schema=pa.schema(list(left.schema) + list(right.schema)))


def expected_pairs(left, right, lkeys, rkeys) -> int:
    """sum over keys of (build rows x probe rows), from np.unique over the key tuples."""
    def counts(batch, keys):
        tups = [repr(t) for t in key_tuples(batch, keys) if t is not None]
        if not tups:
            return {}
        u, c = np.unique(np.array(tups, dtype=object), return_counts=True)
        return dict(zip(u.tolist(), c.tolist()))
    lc, rc = counts(left, lkeys), counts(right, rkeys)
    return int(sum(c * rc.get(k, 0) for k, c in lc.items()))


def comparable(col) -> pa.Array:
    col = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    if pa.types.is_floating(col.type):
        return pa.Array.from_buffers(pa.uint64(), len(col), col.buffers(), offset=col.offset)   # bits, validity kept
    if pa.types.is_timestamp(col.type) or pa.types.is_date32(col.type):
        return col.view(pa.int64() if pa.types.is_timestamp(col.type) else pa.int32())
    return col


def canonical(t: pa.Table, ids=None) -> pa.Table:
    cols = [comparable(c) for c in t.columns]
    if t.num_rows == 0:
        return pa.Table.from_arrays(cols, names=t.schema.names)
    if ids is not None:     # (left id, right id) names one output row
        order = np.lexsort((t.column(ids[1]).to_numpy(), t.column(ids[0]).to_numpy()))
    else:
        tmp = pa.table({"c%d" % i: c for i, c in enumerate(cols)})
        order = pc.sort_indices(tmp, sort_keys=[("c%d" % i, "ascending") for i in range(len(cols))]).to_numpy()
    return pa.Table.from_arrays([c.take(pa.array(order)) for c in cols], names=t.schema.names)


def assert_same_rows(got: pa.Table, want: pa.Table, ids=None):
    """Equal as multisets of rows, Float64 compared by bits; same column names and types."""
    assert got.schema.names == want.schema.names
    assert [f.type for f in got.schema] == [f.type for f in want.schema], (got.schema, want.schema)
    assert got.num_rows == want.num_rows, (got.num_rows, want.num_rows)
    g, w = canonical(got, ids), canonical(want, ids)
    for name, a, b in zip(g.schema.names, g.columns, w.columns):
        assert a.equals(b), "column %s differs" % name


def id_cols(left, right):
    return [left.schema.names.index(next(n for n in left.schema.names if n.endswith("id"))),
            left.num_columns + right.schema.names.index(next(n for n in right.schema.names if n.endswith("id")))]


# ---- crafted collisions: keys that share home slot 1023 of a 1024-slot table ---------------------------------------------
def home(keys) -> np.ndarray:
    return sharding.fmix64(np.asarray(keys).astype(np.int64).view(np.uint64) if np.asarray(keys).dtype.kind == "i" else np.asarray(keys, np.uint64)) & np.uint64(1023)


def colliding_int32(count: int) -> np.ndarray:
    """Int32 keys (negative ones included) whose 4-byte key, zero-extended as the KW 4 table hashes it, homes in slot 1023."""
    cand = np.arange(-(1 << 21), 1 << 21, dtype=np.int64)
    u32 = cand.astype(np.int32).view(np.uint32).astype(np.uint64)
    hit = cand[(sharding.fmix64(u32) & np.uint64(1023)) == 1023]
    return np.concatenate([hit[hit < 0][: count // 2], hit[hit >= 0][: count - count // 2]]).astype(np.int32)


def colliding_int64(count: int) -> np.ndarray:
    """Int64 keys homing in slot 1023 that share their low 32 bits: k, k + j * 2^32, ... (and some negative)."""
    j = np.arange(-(1 << 19), 1 << 19, dtype=np.int64)
    cand = (j << 32) + 5
    hit = cand[(sharding.fmix64(cand.view(np.uint64)) & np.uint64(1023)) == 1023]
    return hit[:count]


def test_crafted_collisions_share_slot_1023():
    k32 = colliding_int32(24)
    assert len(k32) == 24 and (k32 < 0).any() and (k32 >= 0).any()
    assert np.all(sharding.fmix64(k32.view(np.uint32).astype(np.uint64)) & np.uint64(1023) == 1023)
    k64 = colliding_int64(24)
    assert len(k64) == 24 and np.all(k64 & 0xFFFFFFFF == 5) and len(np.unique(k64)) == 24
    assert np.all(sharding.fmix64(k64.view(np.uint64)) & np.uint64(1023) == 1023)


# ---- the CPU half: the reference against the oracle and Acero ---------------------------------------------------------
CPU_CASES = [["int32"], ["uint32"], ["int64"], ["uint64"], ["float64"], ["utf8"], ["ts_ms_naive"], ["ts_ns_UTC"],
             ["int32", "int32"], ["int64", "int32"], ["utf8", "int32"], ["int64", "utf8", "float64"]]


def cpu_pair(kinds, seed, nulls, with_payload=True):
    rng = np.random.default_rng(seed)
    ne = [5 + i for i in range(len(kinds))] if nulls else None
    l, lk = side(kinds, 3000, rng, "l_", null_every=ne, edge_share=0.5, with_payload=with_payload)
    r, rk = side(kinds, 2000, rng, "r_", null_every=None, keys_first=False, edge_share=0.5, with_payload=with_payload)
    return l, r, lk, rk


@pytest.mark.parametrize("kinds", CPU_CASES, ids=lambda k: "-".join(k))
def test_reference_matches_oracle(kinds):
    """The oracle refuses NULLs and Date32, so this runs the null-free relations; it pins the oracle's NaN rule."""
    l, r, lk, rk = cpu_pair(kinds, 3, nulls=False, with_payload=False)
    want = pa.Table.from_batches([oracle.hash_join(l, r, lk, rk)])
    got = ref_join(l, r, lk, rk)
    assert got.num_rows == expected_pairs(l, r, lk, rk) > 0
    assert_same_rows(got, want, id_cols(l, r))


@pytest.mark.parametrize("kinds", [k for k in CPU_CASES if "float64" not in k] + [["date32"], ["int32", "date32"]], ids=lambda k: "-".join(k))
@pytest.mark.parametrize("nulls", [False, True])
def test_reference_matches_acero(kinds, nulls):
    l, r, lk, rk = cpu_pair(kinds, 4, nulls)
    got = ref_join(l, r, lk, rk)
    want = pa.Table.from_batches([l]).join(pa.Table.from_batches([r]), [l.schema.names[k] for k in lk], [r.schema.names[k] for k in rk],
                                           join_type="inner", coalesce_keys=False)
    want = want.select(got.schema.names)
    assert got.num_rows == expected_pairs(l, r, lk, rk) > 0
    assert_same_rows(got, want, id_cols(l, r))


def test_reference_float_key_rules():
    """NaN meets nothing, -0.0 does not meet +0.0, +inf meets +inf, subnormals meet themselves."""
    nan2 = f64(0x7FF0000000000001)
    l = rb(a=pa.array([0.0, -0.0, np.inf, np.nan, nan2, 5e-324, -np.inf]), x=pa.array(np.arange(7)))
    r = rb(b=pa.array([-0.0, np.nan, nan2, np.inf, 5e-324, 0.0, 0.0]), y=pa.array(np.arange(7)))
    got = ref_join(l, r, [0], [0])
    assert sorted(zip(got["x"].to_pylist(), got["y"].to_pylist())) == [(0, 5), (0, 6), (1, 0), (2, 3), (5, 4)]
    assert oracle.hash_join(l, r, [0], [0]).num_rows == 5


# ======================================================================================================================
# the GPU half
# ======================================================================================================================
def gpu_join(ctx, left, right, lkeys, rkeys, left_t=None, right_t=None):
    """(result as Arrow, {kernel: launches} of the join)."""
    lt = left_t if left_t is not None else ctx.import_batches([left])
    rt = right_t if right_t is not None else ctx.import_batches([right])
    ctx.profile_begin()
    try:
        out = ctx.hash_join(lt, rt, lkeys, rkeys)
        got = out.to_arrow()
    finally:
        prof = ctx.profile_end()
    return got, {k: v["launches"] for k, v in prof.items()}


def check_join(ctx, left, right, lkeys, rkeys, path=None):
    """The GPU join equals ref_join as a multiset of rows and has Σ build x probe rows; `path` = the kernels that ran."""
    got, ran = gpu_join(ctx, left, right, lkeys, rkeys)
    n = expected_pairs(left, right, lkeys, rkeys)
    assert got.num_rows == n
    assert_same_rows(got, ref_join(left, right, lkeys, rkeys), id_cols(left, right))
    joined = [k for k in JOIN_KERNELS if ran.get(k)]
    if path == "table":
        assert joined == ["join_build_kernel", "join_count_scan_kernel"] + (["join_emit_kernel"] if n else []), ran
    elif path == "one":
        assert joined == ["join_one_kernel"], ran
    return got, ran


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KEY_KINDS))
def test_single_key_edges(gpu_ctx, kind):
    """One key column: KW 4 for Int32 / UInt32 / Date32, KW 8 for the 8-byte types, KW 0 (row keys) for Utf8.  NULLs on
    the left (over live key values), none on the right but a nullable-free side next to it; both orientations."""
    rng = np.random.default_rng(len(kind) * 7)
    l, lk = side([kind], 5000, rng, "l_", null_every=[4])
    r, rk = side([kind], 3000, rng, "r_", keys_first=False)
    got, _ = check_join(gpu_ctx, l, r, lk, rk, path="table")
    if kind == "float64":
        bits = comparable(got["l_k0"]).to_numpy(zero_copy_only=False)
        assert not np.isnan(got["l_k0"].to_numpy()).any()
        assert np.array_equal(bits, comparable(got["r_k0"]).to_numpy(zero_copy_only=False))       # -0.0 never met +0.0
        assert (bits == 0x8000000000000000).any() and (got["l_k0"].to_numpy() == np.inf).any()
    check_join(gpu_ctx, r, l, rk, lk, path="table")          # the other side hashed, output still left ++ right
    # equal sizes, and an all-NULL key column on one side
    r2, rk2 = side([kind], 5000, rng, "r_")
    check_join(gpu_ctx, l, r2, lk, rk2, path="table")
    l_null, _ = side([kind], 700, rng, "l_", null_every=[1])
    got, _ = check_join(gpu_ctx, l_null, r, lk, rk)
    assert got.num_rows == 0


MULTI_KINDS = [["int32", "int32"], ["int32", "date32"], ["uint32", "int32"],                      # packed
               ["int64", "int64"], ["int64", "int32"], ["utf8", "int32"], ["float64", "utf8"],     # row keys
               ["int32", "int64", "utf8"], ["int32", "uint32", "int64", "uint64", "date32", "ts_us_naive", "utf8", "float64"]]


def narrow(filler_n, rng, kinds):
    """Filler values from ranges small enough that keys of every width meet a few times without being edge values."""
    span = max(3, round(2000 ** (1 / len(kinds))))
    out = []
    for kind in kinds:
        v = rng.integers(0, span, filler_n)
        out.append(["s%d" % x for x in v] if kind == "utf8" else (v - span // 2) * 0.5 if kind == "float64" else v)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kinds", MULTI_KINDS, ids=lambda k: "-".join(k))
def test_multi_key_edges(gpu_ctx, kinds):
    """Two 4-byte keys pack into one word (hi:lo); everything else compares rows.  A NULL in either component of a key
    (over a value that would match) skips the row."""
    rng = np.random.default_rng(len(kinds))
    n_l, n_r = 4000, 6000
    share = 0.3 if len(kinds) <= 2 else 0.03
    l, lk = side(kinds, n_l, rng, "l_", null_every=[5 + 2 * i for i in range(len(kinds))], filler=narrow(n_l, rng, kinds), edge_share=share)
    r, rk = side(kinds, n_r, rng, "r_", keys_first=False, filler=narrow(n_r, rng, kinds), edge_share=share)
    got, _ = check_join(gpu_ctx, l, r, lk, rk, path="table")
    assert got.num_rows > 300
    check_join(gpu_ctx, r, l, rk, lk, path="table")


ONE_ROW_KINDS = ["int32", "uint32", "date32", "int64", "uint64", "ts_ns_UTC", "ts_s_naive"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ONE_ROW_KINDS + ["float64"])
def test_one_build_row(gpu_ctx, kind):
    """A hashed side of one row with a 4- or 8-byte key is an equality filter (join_one_kernel), on either side, for
    every edge value; a NULL on the single row or on the probe side, and a Float64 key, take the table instead."""
    rng = np.random.default_rng(99)
    big, bk = side([kind], 20_001, rng, "b_", edge_share=0.3)
    typ, edges, _ = KEY_KINDS[kind]
    for value in edges + [12345]:                      # 12345: absent
        one = rb(o_k0=make_array(typ, [value]), o_id=pa.array([0], pa.int64()), o_s=pa.array(["only"]))
        expect = "table" if kind == "float64" else "one"
        check_join(gpu_ctx, one, big, [0], bk, path=expect)
        check_join(gpu_ctx, big, one, bk, [0], path=expect)
    if kind == "float64":
        return
    value = edges[0]
    one_null = rb(o_k0=make_array(typ, [value], [True]), o_id=pa.array([0], pa.int64()))
    got, _ = check_join(gpu_ctx, one_null, big, [0], bk, path="table")
    assert got.num_rows == 0
    big_nulls, bk2 = side([kind], 20_001, rng, "b_", null_every=[3], edge_share=0.3)
    one = rb(o_k0=make_array(typ, [value]), o_id=pa.array([0], pa.int64()))
    got, _ = check_join(gpu_ctx, big_nulls, one, bk2, [0], path="table")
    assert got.num_rows > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["int32", "int64", "utf8"])
def test_sizes(gpu_ctx, kind):
    """Build sides of 1, 2, 511, 512, 513 rows (table capacity 1024 up to 512 rows, 2048 at 513) against probe sides
    of 0, 1, 1023, 1024, 1025 rows (JC_TILE = 1024), smaller side left, right and equal; then 100 K against 3 M rows
    under both grid-prefix protocols of the count scan."""
    rng = np.random.default_rng(8)
    kinds = [kind]
    for nb, npr in [(1, 1025), (2, 1024), (511, 1023), (512, 1025), (513, 1024), (2, 0), (1, 1), (1024, 1024), (513, 513)]:
        b, bk = side(kinds, nb, rng, "b_", filler=narrow(nb, rng, kinds), edge_share=0.2)
        p, pk = side(kinds, npr, rng, "p_", null_every=[6], filler=narrow(npr, rng, kinds), edge_share=0.2)
        path = None if npr == 0 else "table" if nb > 1 or kind == "utf8" else None
        check_join(gpu_ctx, b, p, bk, pk, path=path)
        check_join(gpu_ctx, p, b, pk, bk, path=path)
    if kind == "utf8":
        return
    nb, npr = 100_000, 3_000_000
    b, bk = side(kinds, nb, rng, "b_", null_every=[9], edge_share=0.0005)
    # the probe side draws from the build side's keys (NULLs included, as values), so most probe rows match
    p = rb(p_id=pa.array(np.arange(npr, dtype=np.int64)), p_k0=b.column(bk[0]).fill_null(0).take(pa.array(rng.integers(0, nb, npr))))
    want = ref_join(b, p, bk, [1])
    assert want.num_rows == expected_pairs(b, p, bk, [1]) > npr // 2
    for mode in (0, 1):
        gpu_ctx.set_option("compact_mode", mode)
        try:
            got, ran = gpu_join(gpu_ctx, b, p, bk, [1])
        finally:
            gpu_ctx.set_option("compact_mode", 0)
        assert [k for k in JOIN_KERNELS if ran.get(k)] == ["join_build_kernel", "join_count_scan_kernel", "join_emit_kernel"]
        assert_same_rows(got, want, id_cols(b, p))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["int32", "int64"])
def test_crafted_collisions_wrap_the_probe(gpu_ctx, kind):
    """A build side of <= 512 rows (capacity 1024) whose keys all home in slot 1023: the linear probe wraps to slot 0.
    Int64 keys of the cluster differ only in their high half; absent probe keys home into the same cluster."""
    keys = colliding_int32(40) if kind == "int32" else colliding_int64(40)
    present, absent = keys[:24], keys[24:]
    rng = np.random.default_rng(5)
    nb = 300
    bvals = np.concatenate([np.repeat(present, 3), rng.integers(0, 1 << 20, nb - 72)]).astype(keys.dtype)
    pvals = np.concatenate([np.repeat(present, 5), np.repeat(absent, 5), rng.integers(0, 1 << 20, 2000)]).astype(keys.dtype)
    rng.shuffle(bvals)
    rng.shuffle(pvals)
    typ = pa.int32() if kind == "int32" else pa.int64()
    b = rb(b_k=pa.array(bvals, typ), b_id=pa.array(np.arange(nb, dtype=np.int64)))
    p = rb(p_id=pa.array(np.arange(len(pvals), dtype=np.int64)), p_k=pa.array(pvals, typ))
    got, _ = check_join(gpu_ctx, b, p, [0], [1], path="table")
    assert got.num_rows >= 24 * 3 * 5
    check_join(gpu_ctx, p, b, [1], [0], path="table")


@pytest.mark.gpu
def test_duplicates_cross_product(gpu_ctx):
    """3000 x 3000 rows of one key next to many singleton keys: 9 M output rows."""
    rng = np.random.default_rng(12)
    n = 3000 + 50_000
    lk = np.concatenate([np.full(3000, -7, np.int64), np.arange(50_000, dtype=np.int64) * 3 + 1])
    rk = np.concatenate([np.full(3000, -7, np.int64), np.arange(50_000, dtype=np.int64) * 2 + 1])
    l, _ = side(["int64"], n, rng, "l_", filler=[lk], edge_share=0.0, with_payload=False)
    r, _ = side(["int64"], n, rng, "r_", filler=[rk], edge_share=0.0, keys_first=False, with_payload=False)
    got, _ = check_join(gpu_ctx, l, r, [0], [r.schema.names.index("r_k0")], path="table")
    assert got.num_rows == 3000 * 3000 + len(np.intersect1d(lk[3000:], rk[3000:]))


@pytest.mark.gpu
def test_pair_count_limit(gpu_ctx):
    """65 536 x 65 537 rows of one key is 2^32 + 65 536 pairs, more than 2^32 - 2: refused after the count scan, before
    any output is allocated.  The context then joins normally."""
    import flock_b200 as fb
    l = rb(k=pa.array(np.full(65_536, 3, np.int32)))
    r = rb(k=pa.array(np.full(65_537, 3, np.int32)))
    with pytest.raises(fb.FlockGpuError) as info:
        gpu_join(gpu_ctx, l, r, [0], [0])
    assert info.value.code == ERR_UNSUPPORTED and "2^32-2" in str(info.value)
    ll, rr = l.slice(0, 1000), r.slice(0, 999)
    check_join(gpu_ctx, rb(k=ll["k"], id=pa.array(np.arange(1000))), rb(k=rr["k"], id=pa.array(np.arange(999))), [0], [0], path="table")


REFUSED = [(pa.int32(), pa.uint32()), (pa.int32(), pa.date32()), (pa.int64(), pa.timestamp("ms")),
           (pa.timestamp("ms"), pa.timestamp("us")), (pa.timestamp("ns"), pa.timestamp("ns", "UTC")),
           (pa.timestamp("s", "UTC"), pa.timestamp("s", "Europe/Paris"))]


@pytest.mark.gpu
@pytest.mark.parametrize("types", REFUSED, ids=lambda t: "%s-%s" % t)
def test_refusals(gpu_ctx, types):
    """Key columns of unlike type, Timestamp unit or zone are refused, naming both formats, whichever side is larger."""
    import flock_b200 as fb
    lt, rt = types
    l = rb(a=make_array(lt, [1, 2, 3]), id=pa.array([1, 2, 3]))
    r = rb(b=make_array(rt, [1, 2, 3, 3]))
    for a, b in ((l, r), (r, l)):
        with pytest.raises(fb.FlockGpuError) as info:
            gpu_join(gpu_ctx, a, b, [0], [0])
        assert info.value.code == ERR_UNSUPPORTED and "key types differ" in str(info.value)
    # the same types join
    check_join(gpu_ctx, l, rb(b=make_array(lt, [1, 2, 3, 3]), id=pa.array([0, 1, 2, 3])), [0], [0])


@pytest.mark.gpu
def test_nine_keys_refused(gpu_ctx):
    import flock_b200 as fb
    b = rb(**{"c%d" % i: pa.array([1, 2], pa.int32()) for i in range(9)})
    with pytest.raises(fb.FlockGpuError) as info:
        gpu_join(gpu_ctx, b, b, list(range(9)), list(range(9)))
    assert info.value.code == ERR_UNSUPPORTED and "more than 8 key columns" in str(info.value)


# ---- the deferred fast paths ------------------------------------------------------------------------------------------
def dense_keys(n, rng, base):
    return (base + np.arange(n) // 5 + rng.integers(0, 30, n)).astype(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("base", [-150_000, I32_MAX - 200_000])
def test_select_equal_fast_path(gpu_ctx, base):
    """count = MAX(count) over a COUNT(*) by one Int32 key still in its direct-address table: fused (dense_argmax_kernel,
    no join kernel) and against a resolved one-row UInt64 relation, in both argument orders."""
    rng = np.random.default_rng(17)
    n = 700_000
    k = dense_keys(n, rng, base)
    t = gpu_ctx.import_batches([rb(k=pa.array(k), v=pa.array(np.arange(n, dtype=np.int64)))])
    agg = lambda: gpu_ctx.hash_aggregate(t, [0], [("count", -1, "n")], "single")
    whole = agg().to_arrow()
    top = int(whole["n"].to_numpy().max())
    one_max = rb(m=pa.array([top], pa.uint64()))
    whole_b = whole.combine_chunks().to_batches()[0]                 # (k, n), materialised from a second aggregate
    for swap in (False, True):
        d = agg()
        mx = gpu_ctx.hash_aggregate(d, [], [("max", 1, "m")], "single")
        if swap:
            got, ran = gpu_join(gpu_ctx, None, None, [0], [1], left_t=mx, right_t=d)
        else:
            got, ran = gpu_join(gpu_ctx, None, None, [1], [0], left_t=d, right_t=mx)
        assert ran.get("dense_argmax_kernel") == 1 and not any(ran.get(x) for x in JOIN_KERNELS), ran
        want = ref_join(one_max, whole_b, [0], [1]) if swap else ref_join(whole_b, one_max, [1], [0])
        assert got.num_rows > 0
        assert_same_rows(got.rename_columns(want.schema.names), want)
        # a resolved one-row UInt64 relation: a count present, one absent, and 1
        for value in (top, top + 1, 1):
            ob = rb(m=pa.array([value], pa.uint64()), tag=pa.array([-1], pa.int32()))
            d = agg()
            one = gpu_ctx.import_batches([ob])
            if swap:
                got, ran = gpu_join(gpu_ctx, None, None, [0], [1], left_t=one, right_t=d)
            else:
                got, ran = gpu_join(gpu_ctx, None, None, [1], [0], left_t=d, right_t=one)
            assert not any(ran.get(x) for x in JOIN_KERNELS), ran
            want = ref_join(ob, whole_b, [0], [1]) if swap else ref_join(whole_b, ob, [1], [0])
            assert_same_rows(got, want)


def group_inputs(rng, n, val_type, null_vals):
    k = dense_keys(n, rng, 40_000)      # the direct-address table spans the keys' unsigned range: no negative keys
    if val_type == pa.int32():
        v = rng.integers(-5, 5, n).astype(np.int64)
        v[::97] = I32_MIN
        v[::101] = I32_MAX
    else:
        v = rng.integers(-5, 5, n).astype(np.int64)
        v[::97] = I64_MIN
        v[::101] = I64_MAX
    mask = (np.arange(n) % 13 == 0) if null_vals else None
    return rb(k=pa.array(k), v=make_array(val_type, v, mask))


@pytest.mark.gpu
@pytest.mark.parametrize("func", ["max", "min"])
@pytest.mark.parametrize("val_type", [pa.int32(), pa.int64()], ids=str)
def test_select_group_match_fast_path(gpu_ctx, func, val_type):
    """NEXMark q9's shape: other JOIN (key, MAX(v)) ON (key, v) as one selection (group_match_kernel) over the other
    side.  The other side holds NULL keys, NULL values, keys outside the table, values of the other extreme."""
    rng = np.random.default_rng(23)
    n = 400_000
    src = group_inputs(rng, n, val_type, null_vals=True)
    t = gpu_ctx.import_batches([src])
    groups = gpu_ctx.hash_aggregate(t, [0], [(func, 1, "m")], "single").to_arrow().combine_chunks().to_batches()[0]
    m = 300_000
    gk = groups["k"].to_numpy()
    gv = groups["m"].to_numpy(zero_copy_only=False) if groups["m"].null_count == 0 else groups["m"].fill_null(0).to_numpy()
    pick = rng.integers(0, len(gk), m)
    ok = gk[pick].astype(np.int64)
    ov = np.where(rng.random(m) < 0.5, gv[pick], rng.integers(-5, 5, m)).astype(np.int64)
    ok[::41] = gk.max() + 1 + np.arange(len(ok[::41])) % 7          # outside the table
    ok[::43] = I32_MIN
    ov[::47] = I64_MIN if val_type == pa.int64() else I32_MIN
    ov[::53] = I64_MAX if val_type == pa.int64() else I32_MAX
    other = rb(o_id=pa.array(np.arange(m, dtype=np.int64)), o_k=make_array(pa.int32(), ok, np.arange(m) % 17 == 0),
               o_v=make_array(val_type, ov, np.arange(m) % 19 == 0))
    want = ref_join(other, groups, [1, 2], [0, 1])
    for swap in (False, True):
        d = gpu_ctx.hash_aggregate(t, [0], [(func, 1, "m")], "single")
        ot = gpu_ctx.import_batches([other])
        got, ran = gpu_join(gpu_ctx, None, None, [0, 1], [1, 2], left_t=d, right_t=ot) if swap else \
            gpu_join(gpu_ctx, None, None, [1, 2], [0, 1], left_t=ot, right_t=d)
        assert ran.get("group_match_kernel") == 1 and not any(ran.get(x) for x in JOIN_KERNELS), ran
        w = ref_join(groups, other, [0, 1], [1, 2]) if swap else want
        assert got.num_rows == w.num_rows > 1000
        assert_same_rows(got.rename_columns(w.schema.names), w)


@pytest.mark.gpu
def test_deferred_fast_paths_refuse_unlike_timestamps(gpu_ctx):
    """(key, MAX(ts[ms])) against (key, ts[us]) would take select_group_match by dtype alone: it is refused before any
    fast path.  Matching units take the fast path."""
    import flock_b200 as fb
    rng = np.random.default_rng(31)
    n = 400_000
    k = dense_keys(n, rng, 1000)
    v = rng.integers(-(1 << 40), 1 << 40, n)
    t = gpu_ctx.import_batches([rb(k=pa.array(k), v=make_array(pa.timestamp("ms"), v))])
    for unit, tz in (("us", None), ("ms", "UTC")):
        other = gpu_ctx.import_batches([rb(o_k=pa.array(k[:1000]), o_v=make_array(pa.timestamp(unit, tz), v[:1000]))])
        for swap in (False, True):
            d = gpu_ctx.hash_aggregate(t, [0], [("max", 1, "m")], "single")
            with pytest.raises(fb.FlockGpuError) as info:
                if swap:
                    gpu_ctx.hash_join(d, other, [0, 1], [0, 1])
                else:
                    gpu_ctx.hash_join(other, d, [0, 1], [0, 1])
            assert info.value.code == ERR_UNSUPPORTED and "tsm:" in str(info.value)
    other = rb(o_k=pa.array(k[:1000]), o_v=make_array(pa.timestamp("ms"), v[:1000]))
    d = gpu_ctx.hash_aggregate(t, [0], [("max", 1, "m")], "single")
    got, ran = gpu_join(gpu_ctx, other, None, [0, 1], [0, 1], right_t=d)
    assert ran.get("group_match_kernel") == 1
    groups = gpu_ctx.hash_aggregate(t, [0], [("max", 1, "m")], "single").to_arrow().combine_chunks().to_batches()[0]
    want = ref_join(other, groups, [0, 1], [0, 1])
    assert_same_rows(got.rename_columns(want.schema.names), want)


# ---- the one-pass join count of a YSB-shaped plan -----------------------------------------------------------------------
def ts_count_plan(fact_type, dim_type):
    """SELECT g, COUNT(*) FROM fact JOIN dim ON fact.t = dim.t GROUP BY g, g a column of the dimension."""
    fact = pa.schema([pa.field("t", fact_type, False), pa.field("x", pa.int64(), False)])
    dim = pa.schema([pa.field("dt", dim_type, False), pa.field("g", pa.utf8(), False)])
    f = plans.coalesce_batches_exec(plans.repartition_hash(plans.repartition_rr(plans.memory_exec(fact, None), 4), [plans.column("t", 0)], 4))
    d = plans.coalesce_batches_exec(plans.repartition_hash(plans.repartition_rr(plans.memory_exec(dim, None), 4), [plans.column("dt", 0)], 4))
    join = plans.hash_join_exec(f, d, [(plans.column("t", 0), plans.column("dt", 0))])   # t 0, x 1, dt 2, g 3
    return plans.two_phase_aggregate([("g", 3)], [plans._ysb_count()], plans.coalesce_batches_exec(join), 4), fact, dim


@pytest.mark.gpu
@pytest.mark.parametrize("dim_unit", [("ms", None), ("us", None), ("ms", "UTC")], ids=str)
def test_join_count_plan_refuses_unlike_timestamp_units(gpu_ctx, dim_unit):
    """A fact key of Timestamp(ms) against a dimension key of another unit or zone is refused, not counted by
    dim_count_kernel; the same unit is counted in one pass and equals the reference."""
    import flock_b200 as fb
    rng = np.random.default_rng(3)
    plan, fs, ds = ts_count_plan(pa.timestamp("ms"), pa.timestamp(*dim_unit))
    dv = np.arange(-50, 50, dtype=np.int64) * 1000
    fv = rng.choice(dv, 20_000)
    fact = pa.RecordBatch.from_arrays([make_array(pa.timestamp("ms"), fv), pa.array(np.arange(20_000, dtype=np.int64))], schema=fs)
    dim = pa.RecordBatch.from_arrays([make_array(pa.timestamp(*dim_unit), dv), pa.array(["g%d" % (i % 7) for i in range(100)])], schema=ds)
    ec = fb.ExecutionContext(gpu_ctx, plan)
    try:
        ec.feed_data_sources([[[fact]], [[dim]]])
        gpu_ctx.profile_begin()
        try:
            if dim_unit == ("ms", None):
                got = pa.Table.from_batches(ec.execute()[0])
            else:
                with pytest.raises(fb.FlockGpuError) as info:
                    ec.execute()
                assert info.value.code == ERR_UNSUPPORTED and "key types differ" in str(info.value)
        finally:
            prof = gpu_ctx.profile_end()
        ec.clean_data_sources()
    finally:
        ec.close()
    if dim_unit != ("ms", None):
        assert prof.get("dim_count_kernel", {}).get("launches", 0) == 0, sorted(prof)
        return
    assert prof.get("dim_count_kernel", {}).get("launches", 0) == 1, sorted(prof)
    joined = ref_join(fact, dim, [0], [0])
    want = collections.Counter(joined["g"].to_pylist())
    assert dict(zip(got["g"].to_pylist(), got[got.schema.names[-1]].to_pylist())) == dict(want)


# ---- Flock's Partitioned mode: hash_partition both sides, join part i with part i -------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kinds", [["int32"], ["int64"], ["float64"], ["utf8"], ["int32", "utf8"]], ids=lambda k: "-".join(k))
@pytest.mark.parametrize("n_parts", [1, 3, 8])
def test_partitioned_join(gpu_ctx, kinds, n_parts):
    """Keys at different column positions on the two sides, NULLs on one side only: equal keys must be routed to the
    same part whatever their position and validity, so the union of the part joins is the whole join."""
    rng = np.random.default_rng(n_parts)
    l, lk = side(kinds, 20_000, rng, "l_", null_every=[5 + i for i in range(len(kinds))], filler=narrow(20_000, rng, kinds) if len(kinds) > 1 else None, edge_share=0.05)
    r, rk = side(kinds, 30_000, rng, "r_", keys_first=False, filler=narrow(30_000, rng, kinds) if len(kinds) > 1 else None, edge_share=0.05)
    lp = gpu_ctx.hash_partition(gpu_ctx.import_batches([l]), lk, n_parts)
    rp = gpu_ctx.hash_partition(gpu_ctx.import_batches([r]), rk, n_parts)
    parts = [gpu_ctx.hash_join(a, b, lk, rk).to_arrow() for a, b in zip(lp, rp)]
    got = pa.concat_tables(parts)
    want = ref_join(l, r, lk, rk)
    assert got.num_rows == expected_pairs(l, r, lk, rk) > 0
    assert_same_rows(got, want, id_cols(l, r))
