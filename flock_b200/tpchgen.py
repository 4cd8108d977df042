"""TPC-H tables in Flock's schemas (flock/src/datasource/tpch/mod.rs), generated from a seed with vectorised numpy.

The value rules are those of the TPC-H specification, section 4.2.3, wherever the predicates of q1, q3, q5 to q10,
q12 and q14 can see them: cardinalities per scale factor, sparse order keys (the first 8 of every 32), customer keys
never divisible by 3, the date ranges (STARTDATE 1992-01-01, CURRENTDATE 1995-06-17, ENDDATE 1998-12-31) with the
ship, commit and receipt offsets, return flag and line status against CURRENTDATE, the quantity, discount and tax
ranges, P_RETAILPRICE's formula, L_EXTENDEDPRICE = L_QUANTITY * P_RETAILPRICE, L_SUPPKEY from the part's four
partsupp suppliers, the segment, priority, ship mode, ship instruction, P_TYPE syllable, container and brand lists, the
fixed 25 nations and 5 regions, P_NAME's five distinct colour words, and O_TOTALPRICE / O_ORDERSTATUS derived from the
order's lines.  Money is integer cents divided by 100.  Comments, addresses and phone digits come from a small
vocabulary instead of the specification's text grammar (no query here reads them except as opaque group keys).  Dates
are Date32: days since 1970-01-01.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa

STARTDATE, CURRENTDATE, ENDDATE = (int(np.datetime64(d, "D").astype(np.int64)) for d in ("1992-01-01", "1995-06-17", "1998-12-31"))

REGIONS = ["AFRICA", "AMERICA", "ASIA", "EUROPE", "MIDDLE EAST"]
NATIONS = [("ALGERIA", 0), ("ARGENTINA", 1), ("BRAZIL", 1), ("CANADA", 1), ("EGYPT", 4), ("ETHIOPIA", 0), ("FRANCE", 3), ("GERMANY", 3),
           ("INDIA", 2), ("INDONESIA", 2), ("IRAN", 4), ("IRAQ", 4), ("JAPAN", 2), ("JORDAN", 4), ("KENYA", 0), ("MOROCCO", 0),
           ("MOZAMBIQUE", 0), ("PERU", 1), ("CHINA", 2), ("ROMANIA", 3), ("SAUDI ARABIA", 4), ("VIETNAM", 2), ("RUSSIA", 3),
           ("UNITED KINGDOM", 3), ("UNITED STATES", 1)]
SEGMENTS = ["AUTOMOBILE", "BUILDING", "FURNITURE", "MACHINERY", "HOUSEHOLD"]
PRIORITIES = ["1-URGENT", "2-HIGH", "3-MEDIUM", "4-NOT SPECIFIED", "5-LOW"]
SHIPMODES = ["REG AIR", "AIR", "RAIL", "SHIP", "TRUCK", "MAIL", "FOB"]
INSTRUCTIONS = ["DELIVER IN PERSON", "COLLECT COD", "NONE", "TAKE BACK RETURN"]
TYPE_S1 = ["STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO"]
TYPE_S2 = ["ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED"]
TYPE_S3 = ["TIN", "NICKEL", "BRASS", "STEEL", "COPPER"]
CONTAINER_S1 = ["SM", "LG", "MED", "JUMBO", "WRAP"]
CONTAINER_S2 = ["CASE", "BOX", "BAG", "JAR", "PKG", "PACK", "CAN", "DRUM"]
# P_NAME's words (the specification's 4.2.3 colour list)
COLORS = ("almond antique aquamarine azure beige bisque black blanched blue blush brown burlywood burnished chartreuse chiffon "
          "chocolate coral cornflower cornsilk cream cyan dark deep dim dodger drab firebrick floral forest frosted gainsboro ghost "
          "goldenrod green grey honeydew hot indian ivory khaki lace lavender lawn lemon light lime linen magenta maroon medium "
          "metallic midnight mint misty moccasin navajo navy olive orange orchid pale papaya peach peru pink plum powder puff purple "
          "red rose rosy royal saddle salmon sandy seashell sienna sky slate smoke snow spring steel tan thistle tomato turquoise "
          "violet wheat white yellow").split()
WORDS = ["furiously", "carefully", "quickly", "slyly", "blithely", "final", "regular", "special", "pending", "express", "ironic",
         "bold", "even", "silent", "unusual", "deposits", "requests", "accounts", "packages", "theodolites", "instructions", "foxes"]

_I32, _F64, _S, _D = pa.int32(), pa.float64(), pa.utf8(), pa.date32()
SCHEMAS = {
    "part": pa.schema([("p_partkey", _I32), ("p_name", _S), ("p_mfgr", _S), ("p_brand", _S), ("p_type", _S), ("p_size", _I32),
                       ("p_container", _S), ("p_retailprice", _F64), ("p_comment", _S)]),
    "supplier": pa.schema([("s_suppkey", _I32), ("s_name", _S), ("s_address", _S), ("s_nationkey", _I32), ("s_phone", _S),
                           ("s_acctbal", _F64), ("s_comment", _S)]),
    "partsupp": pa.schema([("ps_partkey", _I32), ("ps_suppkey", _I32), ("ps_availqty", _I32), ("ps_supplycost", _F64), ("ps_comment", _S)]),
    "customer": pa.schema([("c_custkey", _I32), ("c_name", _S), ("c_address", _S), ("c_nationkey", _I32), ("c_phone", _S),
                           ("c_acctbal", _F64), ("c_mktsegment", _S), ("c_comment", _S)]),
    "orders": pa.schema([("o_orderkey", _I32), ("o_custkey", _I32), ("o_orderstatus", _S), ("o_totalprice", _F64), ("o_orderdate", _D),
                         ("o_orderpriority", _S), ("o_clerk", _S), ("o_shippriority", _I32), ("o_comment", _S)]),
    "lineitem": pa.schema([("l_orderkey", _I32), ("l_partkey", _I32), ("l_suppkey", _I32), ("l_linenumber", _I32), ("l_quantity", _F64),
                           ("l_extendedprice", _F64), ("l_discount", _F64), ("l_tax", _F64), ("l_returnflag", _S), ("l_linestatus", _S),
                           ("l_shipdate", _D), ("l_commitdate", _D), ("l_receiptdate", _D), ("l_shipinstruct", _S), ("l_shipmode", _S),
                           ("l_comment", _S)]),
    "nation": pa.schema([("n_nationkey", _I32), ("n_name", _S), ("n_regionkey", _I32), ("n_comment", _S)]),
    "region": pa.schema([("r_regionkey", _I32), ("r_name", _S), ("r_comment", _S)]),
}
TABLES = list(SCHEMAS)


def schema(table: str) -> pa.Schema:
    return SCHEMAS[table]


def cardinalities(scale: float) -> dict[str, int]:
    """Rows per table at a scale factor (lineitem varies: 1 to 7 lines per order)."""
    return {"part": int(200_000 * scale), "supplier": max(int(10_000 * scale), 4), "customer": int(150_000 * scale),
            "orders": int(1_500_000 * scale), "nation": 25, "region": 5}


def _pick(rng, words: list[str], n: int) -> pa.Array:
    return pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(words), n).astype(np.int32)), pa.array(words)).dictionary_decode()


def _fmt(prefix: str, keys: np.ndarray) -> pa.Array:
    return pa.array(np.char.add(prefix, np.char.zfill(keys.astype(str), 9)).astype(object), _S)


def _phones(rng, nationkeys: np.ndarray) -> pa.Array:
    n = len(nationkeys)
    parts = [(nationkeys + 10).astype(str), rng.integers(100, 1000, n).astype(str), rng.integers(100, 1000, n).astype(str),
             rng.integers(1000, 10000, n).astype(str)]
    out = parts[0]
    for p in parts[1:]:
        out = np.char.add(np.char.add(out, "-"), p)
    return pa.array(out.astype(object), _S)


def _money(cents: np.ndarray) -> np.ndarray:
    return cents.astype(np.float64) / 100.0


def retailprice_cents(partkey: np.ndarray) -> np.ndarray:
    partkey = partkey.astype(np.int64)
    return 90000 + (partkey // 10) % 20001 + 100 * (partkey % 1000)


def order_keys(n: int) -> np.ndarray:
    """Sparse keys: of every 32 consecutive keys only the first 8 are used."""
    i = np.arange(n, dtype=np.int64)
    return (i // 8) * 32 + (i % 8) + 1


def part_names(seed: int, n: int) -> np.ndarray:
    """P_NAME: five distinct words of COLORS, drawn from a generator derived from `seed`."""
    rng = np.random.default_rng([seed, 1])
    words = rng.integers(0, len(COLORS), (n, 5))
    while True:
        s = np.sort(words, axis=1)
        dup = np.any(s[:, 1:] == s[:, :-1], axis=1)
        if not dup.any():
            break
        words[dup] = rng.integers(0, len(COLORS), (int(dup.sum()), 5))
    w = np.array(COLORS)[words]
    out = w[:, 0]
    for k in range(1, 5):
        out = np.char.add(np.char.add(out, " "), w[:, k])
    return out


def generate(scale: float = 0.01, seed: int = 42, columns: dict[str, list[str]] | None = None) -> dict[str, pa.Table]:
    """All eight tables (or, with `columns`, only the listed tables and columns) at scale factor `scale`."""
    rng = np.random.default_rng(seed)
    card = cardinalities(scale)
    P, S, C, O = card["part"], card["supplier"], card["customer"], card["orders"]
    out: dict[str, dict[str, pa.Array]] = {}

    out["region"] = {"r_regionkey": pa.array(np.arange(5, dtype=np.int32)), "r_name": pa.array(REGIONS, _S), "r_comment": _pick(rng, WORDS, 5)}
    out["nation"] = {"n_nationkey": pa.array(np.arange(25, dtype=np.int32)), "n_name": pa.array([n for n, _ in NATIONS], _S),
                     "n_regionkey": pa.array(np.array([r for _, r in NATIONS], np.int32)), "n_comment": _pick(rng, WORDS, 25)}

    pk = np.arange(1, P + 1, dtype=np.int32)
    t1, t2, t3 = rng.integers(0, 6, P), rng.integers(0, 5, P), rng.integers(0, 5, P)
    types = np.char.add(np.char.add(np.char.add(np.char.add(np.array(TYPE_S1)[t1], " "), np.array(TYPE_S2)[t2]), " "), np.array(TYPE_S3)[t3])
    m, b = rng.integers(1, 6, P), rng.integers(1, 6, P)
    containers = np.char.add(np.char.add(np.array(CONTAINER_S1)[rng.integers(0, 5, P)], " "), np.array(CONTAINER_S2)[rng.integers(0, 8, P)])
    # Names once took two words of 24 from this stream.  Those draws stay, unused, so that every other column keeps its
    # values for a seed; the names come from a generator of their own.
    rng.integers(0, 24, P)
    rng.integers(0, 24, P)
    names = part_names(seed, P)
    p_price_cents = retailprice_cents(pk)
    out["part"] = {"p_partkey": pa.array(pk), "p_name": pa.array(names.astype(object), _S),
                   "p_mfgr": pa.array(np.char.add("Manufacturer#", m.astype(str)).astype(object), _S),
                   "p_brand": pa.array(np.char.add(np.char.add("Brand#", m.astype(str)), b.astype(str)).astype(object), _S),
                   "p_type": pa.array(types.astype(object), _S), "p_size": pa.array(rng.integers(1, 51, P).astype(np.int32)),
                   "p_container": pa.array(containers.astype(object), _S), "p_retailprice": pa.array(_money(p_price_cents)),
                   "p_comment": _pick(rng, WORDS, P)}

    sk = np.arange(1, S + 1, dtype=np.int32)
    s_nat = rng.integers(0, 25, S).astype(np.int32)
    out["supplier"] = {"s_suppkey": pa.array(sk), "s_name": _fmt("Supplier#", sk), "s_address": _pick(rng, WORDS, S),
                       "s_nationkey": pa.array(s_nat), "s_phone": _phones(rng, s_nat),
                       "s_acctbal": pa.array(_money(rng.integers(-99999, 1000000, S))), "s_comment": _pick(rng, WORDS, S)}

    # partsupp: supplier i (0..3) of part p is (p + i * (S/4 + (p-1)/S)) % S + 1
    ps_part = np.repeat(pk.astype(np.int64), 4)
    ps_i = np.tile(np.arange(4, dtype=np.int64), P)
    ps_supp = (ps_part + ps_i * (S // 4 + (ps_part - 1) // S)) % S + 1
    out["partsupp"] = {"ps_partkey": pa.array(ps_part.astype(np.int32)), "ps_suppkey": pa.array(ps_supp.astype(np.int32)),
                       "ps_availqty": pa.array(rng.integers(1, 10000, 4 * P).astype(np.int32)),
                       "ps_supplycost": pa.array(_money(rng.integers(100, 100001, 4 * P))), "ps_comment": _pick(rng, WORDS, 4 * P)}

    ck = np.arange(1, C + 1, dtype=np.int32)
    c_nat = rng.integers(0, 25, C).astype(np.int32)
    out["customer"] = {"c_custkey": pa.array(ck), "c_name": _fmt("Customer#", ck), "c_address": _pick(rng, WORDS, C),
                       "c_nationkey": pa.array(c_nat), "c_phone": _phones(rng, c_nat),
                       "c_acctbal": pa.array(_money(rng.integers(-99999, 1000000, C))), "c_mktsegment": _pick(rng, SEGMENTS, C),
                       "c_comment": _pick(rng, WORDS, C)}

    # orders: a customer key drawn uniformly from those not divisible by 3
    ok = order_keys(O)
    non3 = ck[ck % 3 != 0]
    o_cust = non3[rng.integers(0, len(non3), O)]
    o_date = rng.integers(STARTDATE, ENDDATE - 151 + 1, O).astype(np.int32)
    n_lines = rng.integers(1, 8, O)
    L = int(n_lines.sum())
    order_of = np.repeat(np.arange(O), n_lines)
    starts = np.cumsum(n_lines) - n_lines
    linenumber = (np.arange(L) - starts[order_of] + 1).astype(np.int32)
    l_part = rng.integers(1, P + 1, L).astype(np.int64)
    l_supp = (l_part + rng.integers(0, 4, L) * (S // 4 + (l_part - 1) // S)) % S + 1
    qty = rng.integers(1, 51, L)
    ext_cents = qty * retailprice_cents(l_part)
    disc = rng.integers(0, 11, L)          # hundredths
    tax = rng.integers(0, 9, L)
    ship = o_date[order_of] + rng.integers(1, 122, L)
    commit = o_date[order_of] + rng.integers(30, 91, L)
    receipt = ship + rng.integers(1, 31, L)
    status_o = ship > CURRENTDATE
    rflag = np.where(receipt <= CURRENTDATE, np.where(rng.integers(0, 2, L) == 0, "R", "A"), "N")
    out["lineitem"] = {"l_orderkey": pa.array(ok[order_of].astype(np.int32)), "l_partkey": pa.array(l_part.astype(np.int32)),
                       "l_suppkey": pa.array(l_supp.astype(np.int32)), "l_linenumber": pa.array(linenumber),
                       "l_quantity": pa.array(qty.astype(np.float64)), "l_extendedprice": pa.array(_money(ext_cents)),
                       "l_discount": pa.array(disc / 100.0), "l_tax": pa.array(tax / 100.0),
                       "l_returnflag": pa.array(rflag.astype(object), _S), "l_linestatus": pa.array(np.where(status_o, "O", "F").astype(object), _S),
                       "l_shipdate": pa.array(ship.astype(np.int32), _D), "l_commitdate": pa.array(commit.astype(np.int32), _D),
                       "l_receiptdate": pa.array(receipt.astype(np.int32), _D), "l_shipinstruct": _pick(rng, INSTRUCTIONS, L),
                       "l_shipmode": _pick(rng, SHIPMODES, L), "l_comment": _pick(rng, WORDS, L)}

    # O_TOTALPRICE = sum(L_EXTENDEDPRICE * (1 + L_TAX) * (1 - L_DISCOUNT)) in cents; O_ORDERSTATUS F / O / P
    line_total = ext_cents * (100 + tax) * (100 - disc) / 10000.0
    total_cents = np.round(np.bincount(order_of, weights=line_total, minlength=O))
    n_open = np.bincount(order_of, weights=status_o, minlength=O)
    ostatus = np.where(n_open == 0, "F", np.where(n_open == n_lines, "O", "P"))
    out["orders"] = {"o_orderkey": pa.array(ok.astype(np.int32)), "o_custkey": pa.array(o_cust.astype(np.int32)),
                     "o_orderstatus": pa.array(ostatus.astype(object), _S), "o_totalprice": pa.array(_money(total_cents)),
                     "o_orderdate": pa.array(o_date, _D), "o_orderpriority": _pick(rng, PRIORITIES, O),
                     "o_clerk": _fmt("Clerk#", rng.integers(1, max(int(1000 * scale), 1) + 1, O)),
                     "o_shippriority": pa.array(np.zeros(O, np.int32)), "o_comment": _pick(rng, WORDS, O)}

    tables = {}
    for name, cols in out.items():
        if columns is not None and name not in columns:
            continue
        sch = SCHEMAS[name]
        keep = columns[name] if columns is not None else sch.names
        tables[name] = pa.table([cols[c] for c in keep], schema=pa.schema([sch.field(c) for c in keep]))
    return tables
