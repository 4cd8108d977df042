"""Synthetic NEXMark record batches with the reference's schemas and value distributions.

This is the *input generator* for tests and bench.py.  It reproduces the distributions of the
reference generator (flock/src/datasource/nexmark/event.rs:83-97, :152-207, :247-311, :354-371 and
config.rs:121-252) with numpy's PCG64 -- it is distribution-faithful, not bit-faithful to Rust's
``SmallRng`` stream (the generators are out of scope, SURVEY.md section 8d).  All columns are
non-null, exactly like the reference schemas (event.rs:130-149, :220-245, :336-352).

Event ``n`` (single generator, first_event_id = 0) is a person when ``n % 50 == 0``, an auction when
``n % 50 in 1..3`` and a bid otherwise (config.rs:135-138, event.rs:84-96).
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa

BATCH_ROWS = 65536                      # 64 Ki-row batches (BASELINE.json metric)
BASE_TIME = 1_436_918_400_000           # config.rs: base_time
PROPORTION_DENOMINATOR = 50
PERSON_PROPORTION, AUCTION_PROPORTION, BID_PROPORTION = 1, 3, 46
FIRST_PERSON_ID = FIRST_AUCTION_ID = 1000
FIRST_CATEGORY_ID, NUM_CATEGORIES = 10, 5
ACTIVE_PEOPLE, IN_FLIGHT_AUCTIONS = 1000, 100
PERSON_ID_LEAD = AUCTION_ID_LEAD = 10
HOT_SELLER_RATIO, HOT_AUCTION_RATIO, HOT_BIDDER_RATIO = 4, 2, 4
HOT_RATIO_2 = 100
EVENTS_PER_SECOND = 10_000

US_STATES = "az,ca,id,or,wa,wy".split(",")
US_CITIES = "phoenix,los angeles,san francisco,boise,portland,bend,redmond,seattle,kent,cheyenne".split(",")
FIRST_NAMES = "peter,paul,luke,john,saul,vicky,kate,julie,sarah,deiter,walter".split(",")
LAST_NAMES = "shultz,abrams,spencer,white,bartels,walton,smith,jones,noris".split(",")

TS = pa.timestamp("ms")


def bid_schema() -> pa.Schema:
    """event.rs:336-352"""
    return pa.schema(
        [pa.field("auction", pa.int32(), False), pa.field("bidder", pa.int32(), False),
         pa.field("price", pa.int32(), False), pa.field("b_date_time", TS, False)],
        metadata={"name": "bid"})


def auction_schema() -> pa.Schema:
    """event.rs:220-245"""
    return pa.schema(
        [pa.field("a_id", pa.int32(), False), pa.field("item_name", pa.utf8(), False),
         pa.field("description", pa.utf8(), False), pa.field("initial_bid", pa.int32(), False),
         pa.field("reserve", pa.int32(), False), pa.field("a_date_time", TS, False),
         pa.field("expires", TS, False), pa.field("seller", pa.int32(), False),
         pa.field("category", pa.int32(), False)],
        metadata={"name": "auction"})


def person_schema() -> pa.Schema:
    """event.rs:130-149"""
    return pa.schema(
        [pa.field("p_id", pa.int32(), False), pa.field("name", pa.utf8(), False),
         pa.field("email_address", pa.utf8(), False), pa.field("credit_card", pa.utf8(), False),
         pa.field("city", pa.utf8(), False), pa.field("state", pa.utf8(), False),
         pa.field("p_date_time", TS, False)],
        metadata={"name": "person"})


# ------------------------------------------------------------------------------------------------
# id arithmetic (event.rs:171-186 Person::{next_id,last_id}; :283-306 Auction::{next_id,last_id})
# ------------------------------------------------------------------------------------------------
def _event_timestamp(n: np.ndarray) -> np.ndarray:
    # config.rs:248-252 with a constant rate: delay = 1e6 / eps microseconds per event.  (The reference
    # rounds in f32; f64 is used here so that timestamps stay monotone beyond 2^24 events.)
    delay_us = 1_000_000.0 / EVENTS_PER_SECOND
    return BASE_TIME + np.round(n.astype(np.float64) * delay_us / 1000.0).astype(np.int64)


def _last_person_id(ev: np.ndarray) -> np.ndarray:
    return ev // PROPORTION_DENOMINATOR          # offset clamps to 0 for every non-person event


def _last_auction_id(ev: np.ndarray) -> np.ndarray:
    epoch = ev // PROPORTION_DENOMINATOR
    off = ev % PROPORTION_DENOMINATOR
    is_person = off < PERSON_PROPORTION
    epoch = np.where(is_person, epoch - 1, epoch)
    off = np.where(is_person | (off >= PERSON_PROPORTION + AUCTION_PROPORTION),
                   AUCTION_PROPORTION - 1, off - PERSON_PROPORTION)
    return epoch * AUCTION_PROPORTION + off


def _next_person_id(ev: np.ndarray, rng: np.random.Generator) -> np.ndarray:
    people = _last_person_id(ev) + 1
    active = np.minimum(people, ACTIVE_PEOPLE)
    return people - active + (rng.random(ev.size) * (active + PERSON_ID_LEAD)).astype(np.int64)


def _next_auction_id(ev: np.ndarray, rng: np.random.Generator) -> np.ndarray:
    mx = _last_auction_id(ev)
    mn = np.maximum(mx - IN_FLIGHT_AUCTIONS, 0)
    return mn + (rng.random(ev.size) * (mx - mn + 1 + AUCTION_ID_LEAD)).astype(np.int64)


def _price(n: int, rng: np.random.Generator) -> np.ndarray:
    u = rng.random(n, dtype=np.float32)
    return np.round(np.power(np.float32(10.0), u * np.float32(6.0)) * np.float32(100.0)).astype(np.int64)


def _choice_strings(words: list[str], n: int, rng: np.random.Generator) -> pa.Array:
    idx = rng.integers(0, len(words), n).astype(np.int32)
    return pa.DictionaryArray.from_arrays(pa.array(idx), pa.array(words)).dictionary_decode()


def _gen_strings(n: int, max_len: int, rng: np.random.Generator) -> pa.Array:
    """event.rs:34-51: len ~ U[3,max), chars a-z with 1/13 spaces, then trimmed."""
    if n == 0:
        return pa.array([], pa.utf8())
    lens = rng.integers(3, max_len, n)
    width = int(max_len)
    chars = rng.integers(0, 26, (n, width)).astype(np.uint8) + ord("a")
    chars[rng.integers(0, 13, (n, width)) == 0] = ord(" ")
    col = np.arange(width)[None, :]
    inside = col < lens[:, None]
    nonsp = inside & (chars != ord(" "))
    any_ns = nonsp.any(axis=1)
    first = np.where(any_ns, nonsp.argmax(axis=1), 0)
    last = np.where(any_ns, width - 1 - nonsp[:, ::-1].argmax(axis=1), -1)
    keep = (col >= first[:, None]) & (col <= last[:, None])
    out_len = np.where(any_ns, last - first + 1, 0)
    offsets = np.zeros(n + 1, np.int32)
    np.cumsum(out_len, out=offsets[1:])
    data = chars[keep]
    return pa.Array.from_buffers(pa.utf8(), n, [None, pa.py_buffer(offsets), pa.py_buffer(data)])


# ------------------------------------------------------------------------------------------------
# relations
# ------------------------------------------------------------------------------------------------
def _bid_event_numbers(first: int, n: int) -> np.ndarray:
    k = np.arange(first, first + n, dtype=np.int64)
    return (k // BID_PROPORTION) * PROPORTION_DENOMINATOR + PERSON_PROPORTION + AUCTION_PROPORTION + k % BID_PROPORTION


def _auction_event_numbers(first: int, n: int) -> np.ndarray:
    k = np.arange(first, first + n, dtype=np.int64)
    return (k // AUCTION_PROPORTION) * PROPORTION_DENOMINATOR + PERSON_PROPORTION + k % AUCTION_PROPORTION


def _person_event_numbers(first: int, n: int) -> np.ndarray:
    return np.arange(first, first + n, dtype=np.int64) * PROPORTION_DENOMINATOR


def bids(n_bids: int, seed: int = 42, first_bid: int = 0, columns: list[str] | None = None) -> pa.RecordBatch:
    """``n_bids`` consecutive bid events (event.rs:354-371) as one RecordBatch.  ``columns`` restricts the schema (the
    100 M-bid configuration scans `auction` only); the random draws happen in schema order, so a restricted batch
    carries exactly the values the full batch would."""
    rng = np.random.default_rng([seed, 3, first_bid])
    ev = _bid_event_numbers(first_bid, n_bids)
    full = bid_schema()
    want = [f.name for f in full] if columns is None else list(columns)
    last = max(full.get_field_index(c) for c in want)
    arrays = {}
    hot_a = rng.integers(0, HOT_AUCTION_RATIO, n_bids) > 0
    auction = np.where(hot_a, (_last_auction_id(ev) // HOT_RATIO_2) * HOT_RATIO_2, _next_auction_id(ev, rng))
    arrays["auction"] = pa.array((auction + FIRST_AUCTION_ID).astype(np.int32))
    del hot_a, auction
    if last >= 1:
        hot_b = rng.integers(0, HOT_BIDDER_RATIO, n_bids) > 0
        bidder = np.where(hot_b, (_last_person_id(ev) // HOT_RATIO_2) * HOT_RATIO_2 + 1, _next_person_id(ev, rng))
        arrays["bidder"] = pa.array((bidder + FIRST_PERSON_ID).astype(np.int32))
    if last >= 2:
        arrays["price"] = pa.array(_price(n_bids, rng).astype(np.int32))
    if last >= 3:
        arrays["b_date_time"] = pa.array(_event_timestamp(ev), TS)
    fields = [full.field(c) for c in want]
    return pa.RecordBatch.from_arrays([arrays[c] for c in want], schema=pa.schema(fields, metadata=full.metadata))


def auctions(n_auctions: int, seed: int = 42, first_auction: int = 0, columns: list[str] | None = None) -> pa.RecordBatch:
    """``n_auctions`` consecutive auction events (event.rs:247-311).  ``columns`` restricts the schema
    (feed_data_sources matches leaves by field-name subset, context.rs:402-416), which keeps the
    1 B-event configuration from materialising 6 GB of item descriptions nobody scans."""
    rng = np.random.default_rng([seed, 2, first_auction])
    ev = _auction_event_numbers(first_auction, n_auctions)
    want = set(columns) if columns is not None else None
    time = _event_timestamp(ev)
    initial = _price(n_auctions, rng)
    hot = rng.integers(0, HOT_SELLER_RATIO, n_auctions) > 0
    seller = np.where(hot, (_last_person_id(ev) // HOT_RATIO_2) * HOT_RATIO_2, _next_person_id(ev, rng))
    reserve = initial + _price(n_auctions, rng)
    events_for_auctions = (IN_FLIGHT_AUCTIONS * PROPORTION_DENOMINATOR) // AUCTION_PROPORTION
    horizon = _event_timestamp(ev + events_for_auctions) - time
    expires = time + 1 + (rng.random(n_auctions) * np.maximum(horizon * 2, 1)).astype(np.int64)
    category = FIRST_CATEGORY_ID + rng.integers(0, NUM_CATEGORIES, n_auctions)
    full = auction_schema()
    arrays, fields = [], []
    for f in full:
        if want is not None and f.name not in want:
            continue
        if f.name == "a_id":
            a = pa.array((_last_auction_id(ev) + FIRST_AUCTION_ID).astype(np.int32))
        elif f.name == "item_name":
            a = _gen_strings(n_auctions, 20, rng)
        elif f.name == "description":
            a = _gen_strings(n_auctions, 100, rng)
        elif f.name == "initial_bid":
            a = pa.array(initial.astype(np.int32))
        elif f.name == "reserve":
            a = pa.array(reserve.astype(np.int32))
        elif f.name == "a_date_time":
            a = pa.array(time, TS)
        elif f.name == "expires":
            a = pa.array(expires, TS)
        elif f.name == "seller":
            a = pa.array((seller + FIRST_PERSON_ID).astype(np.int32))
        else:
            a = pa.array(category.astype(np.int32))
        arrays.append(a)
        fields.append(f)
    return pa.RecordBatch.from_arrays(arrays, schema=pa.schema(fields, metadata=full.metadata))


def persons(n_persons: int, seed: int = 42, first_person: int = 0, columns: list[str] | None = None) -> pa.RecordBatch:
    """``n_persons`` consecutive person events (event.rs:152-169)."""
    rng = np.random.default_rng([seed, 1, first_person])
    ev = _person_event_numbers(first_person, n_persons)
    want = set(columns) if columns is not None else None
    full = person_schema()
    arrays, fields = [], []
    for f in full:
        if want is not None and f.name not in want:
            continue
        if f.name == "p_id":
            a = pa.array((_last_person_id(ev) + FIRST_PERSON_ID).astype(np.int32))
        elif f.name == "name":
            combos = [f"{a} {b}" for a in FIRST_NAMES for b in LAST_NAMES]
            a = _choice_strings(combos, n_persons, rng)
        elif f.name == "email_address":
            u, d = _gen_strings(n_persons, 7, rng), _gen_strings(n_persons, 5, rng)
            a = pa.compute.binary_join_element_wise(u, d, pa.scalar("@"))
            a = pa.compute.binary_join_element_wise(a, pa.scalar("com"), pa.scalar("."))
        elif f.name == "credit_card":
            digits = rng.integers(0, 10, (n_persons, 19)).astype(np.uint8) + ord("0")
            digits[:, [4, 9, 14]] = ord(" ")
            a = pa.Array.from_buffers(pa.utf8(), n_persons, [
                None, pa.py_buffer(np.arange(0, 19 * (n_persons + 1), 19, dtype=np.int32)),
                pa.py_buffer(np.ascontiguousarray(digits).reshape(-1))])
        elif f.name == "city":
            a = _choice_strings(US_CITIES, n_persons, rng)
        elif f.name == "state":
            a = _choice_strings(US_STATES, n_persons, rng)
        else:
            a = pa.array(_event_timestamp(ev), TS)
        arrays.append(a)
        fields.append(f)
    return pa.RecordBatch.from_arrays(arrays, schema=pa.schema(fields, metadata=full.metadata))


TS_NS_UTC = pa.timestamp("ns", tz="UTC")


def bid_ptime_schema() -> pa.Schema:
    """The bid columns plus the processing time q12 groups by: ``SELECT *, now() AS p_time FROM bid``."""
    return pa.schema(list(bid_schema()) + [pa.field("p_time", TS_NS_UTC, False)], metadata={"name": "bid"})


def bids_ptime(n_bids: int, seed: int = 42, first_bid: int = 0) -> pa.RecordBatch:
    """``bids(n_bids, seed, first_bid)`` with a ``p_time`` column.  The reference stamps every bid with ``now()`` as its
    source function reads it; here the stamp is deterministic: it advances by 1 us every 4 bids (monotone in the bid's
    position, 4 bids per stamp), so each bidder's MIN and MAX are stamps of different bids."""
    b = bids(n_bids, seed, first_bid)
    k = np.arange(first_bid, first_bid + n_bids, dtype=np.int64)
    p_time = pa.array(BASE_TIME * 1_000_000 + (k // 4) * 1_000, TS_NS_UTC)
    return pa.RecordBatch.from_arrays(list(b.columns) + [p_time], schema=bid_ptime_schema())


def side_input_schema() -> pa.Schema:
    """event.rs:375-385"""
    return pa.schema([pa.field("key", pa.int32(), False), pa.field("value", pa.int32(), False)], metadata={"name": "side_input"})


def side_input(n_auctions: int, seed: int = 42) -> pa.RecordBatch:
    """q13's side input, SYNTHETIC: the reference downloads a CSV of (key, value) pairs; this table is generated from
    ``seed`` instead.  Keys are the auction ids a window of ``n_auctions`` auctions produces, ascending, with about one
    in eight left out so that some bids find no match; values are uniform in [0, 2^20)."""
    rng = np.random.default_rng([seed, 4])
    ids = np.arange(FIRST_AUCTION_ID, FIRST_AUCTION_ID + n_auctions, dtype=np.int32)
    keys = ids[rng.random(ids.size) >= 0.125]
    values = rng.integers(0, 1 << 20, keys.size).astype(np.int32)
    return pa.RecordBatch.from_arrays([pa.array(keys), pa.array(values)], schema=side_input_schema())


def bids_chunked(n_bids: int, seed: int = 42, columns: list[str] | None = None, first_bid: int = 0, chunk: int = 4_000_000,
                 threads: int = 16, batch_rows: int = BATCH_ROWS) -> list[pa.RecordBatch]:
    """``n_bids`` consecutive bids generated ``chunk`` at a time on a thread pool (numpy releases the interpreter lock
    in its array kernels) and cut into ``batch_rows``-row batches.  Chunk c is seeded by its first bid number, so the
    stream does not depend on the thread count.  100 M `auction` values take seconds instead of a minute."""
    from concurrent.futures import ThreadPoolExecutor
    starts = list(range(0, max(n_bids, 1), chunk))
    def one(o):
        return bids(min(chunk, n_bids - o), seed, first_bid + o, columns)
    if len(starts) == 1:
        parts = [one(0)]
    else:
        with ThreadPoolExecutor(max_workers=min(threads, len(starts))) as ex:
            parts = list(ex.map(one, starts))
    out: list[pa.RecordBatch] = []
    for part in parts:          # chunk is a multiple of batch_rows only by luck: re-cut over the concatenation
        out.append(part)
    tbl = pa.Table.from_batches(out).combine_chunks()
    return split_batches(tbl.to_batches()[0] if tbl.num_rows else parts[0], batch_rows)


def split_batches(batch: pa.RecordBatch, rows: int = BATCH_ROWS) -> list[pa.RecordBatch]:
    """Cut a relation into ``rows``-row record batches (last one short), SURVEY.md section 8d."""
    if batch.num_rows == 0:
        return [batch]
    return [batch.slice(o, min(rows, batch.num_rows - o)) for o in range(0, batch.num_rows, rows)]


def relation_counts(n_events: int) -> tuple[int, int, int]:
    """(persons, auctions, bids) among the first ``n_events`` events."""
    full, rem = divmod(n_events, PROPORTION_DENOMINATOR)
    p = full * PERSON_PROPORTION + min(rem, PERSON_PROPORTION)
    a = full * AUCTION_PROPORTION + min(max(rem - PERSON_PROPORTION, 0), AUCTION_PROPORTION)
    return p, a, n_events - p - a


def generate(n_events: int, seed: int = 42, batch_rows: int = BATCH_ROWS,
             relations: tuple[str, ...] = ("person", "auction", "bid"),
             columns: dict[str, list[str]] | None = None, chunk: int = 4_000_000) -> dict[str, list[pa.RecordBatch]]:
    """First ``n_events`` NEXMark events as lists of ``batch_rows``-row batches per relation."""
    n_p, n_a, n_b = relation_counts(n_events)
    columns = columns or {}
    out: dict[str, list[pa.RecordBatch]] = {}

    def chunks(total, fn, cols=None):
        parts = []
        for first in range(0, max(total, 1), chunk):
            n = min(chunk, total - first)
            parts.append(fn(n, seed, first, cols) if cols is not None or fn is not bids else fn(n, seed, first))
        tbl = pa.Table.from_batches(parts).combine_chunks()
        return split_batches(tbl.to_batches()[0] if tbl.num_rows else parts[0], batch_rows)

    if "person" in relations:
        out["person"] = chunks(n_p, persons, columns.get("person", None) or [f.name for f in person_schema()])
    if "auction" in relations:
        out["auction"] = chunks(n_a, auctions, columns.get("auction", None) or [f.name for f in auction_schema()])
    if "bid" in relations:
        out["bid"] = chunks(n_b, bids)
    return out
