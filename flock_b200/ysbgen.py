"""Yahoo Streaming Benchmark inputs, vectorised with numpy.

Follows the distributions of the reference generator (flock/src/datasource/ysb/{event.rs,generator.rs}), not its RNG
bits: `campaigns` campaigns of `ads` ads each, every id a random (version 4) UUID string; every event picks its ad
uniformly, its ad type uniformly from five and its event type uniformly from three; `ip_address` is "0.0.0.0" and
`event_time` (milliseconds) advances by 1000 / events_per_second from 1.  Every column is Utf8 but the time.
"""
from __future__ import annotations

import json

import numpy as np
import pyarrow as pa

AD_TYPES = ["banner", "modal", "sponsored-search", "mail", "mobile"]
EVENT_TYPES = ["view", "click", "purchase"]
EVENTS_PER_SECOND = 1000          # generator.rs: config "events-per-second"
TS = pa.timestamp("ms")
UUID_LEN = 36


def ad_event_schema() -> pa.Schema:
    """event.rs: AdEvent::schema()."""
    return pa.schema([pa.field("user_id", pa.utf8(), False), pa.field("page_id", pa.utf8(), False),
                      pa.field("ad_id", pa.utf8(), False), pa.field("ad_type", pa.utf8(), False),
                      pa.field("event_type", pa.utf8(), False), pa.field("event_time", TS, False),
                      pa.field("ip_address", pa.utf8(), False)], metadata={"name": "ysb_ad_events"})


def campaign_schema() -> pa.Schema:
    """event.rs: Campaign::schema()."""
    return pa.schema([pa.field("c_ad_id", pa.utf8(), False), pa.field("campaign_id", pa.utf8(), False)],
                     metadata={"name": "ysb_campaigns"})


_HEX = np.frombuffer(b"0123456789abcdef", np.uint8)
_DASHES = (8, 13, 18, 23)
_DIGIT_POS = np.array([i for i in range(UUID_LEN) if i not in _DASHES])


def uuid_bytes(n: int, rng: np.random.Generator) -> np.ndarray:
    """`n` random UUIDs (Uuid::new_v4) as an (n, 36) array of their lowercase 8-4-4-4-12 hex text."""
    raw = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    raw[:, 6] = (raw[:, 6] & 0x0F) | 0x40      # version 4
    raw[:, 8] = (raw[:, 8] & 0x3F) | 0x80      # variant 10xx (RFC 4122)
    nibbles = np.empty((n, 32), np.uint8)
    nibbles[:, 0::2] = raw >> 4
    nibbles[:, 1::2] = raw & 0x0F
    out = np.full((n, UUID_LEN), ord("-"), np.uint8)
    out[:, _DIGIT_POS] = _HEX[nibbles]
    return out


def _fixed_strings(chars: np.ndarray) -> pa.Array:
    """(n, w) bytes -> a Utf8 array of n strings of w bytes each."""
    n, w = chars.shape
    offsets = (np.arange(n + 1, dtype=np.int64) * w).astype(np.int32)
    return pa.Array.from_buffers(pa.utf8(), n, [None, pa.py_buffer(offsets), pa.py_buffer(np.ascontiguousarray(chars))])


def _choice(words: list[str], idx: np.ndarray) -> pa.Array:
    return pa.DictionaryArray.from_arrays(pa.array(idx.astype(np.int32)), pa.array(words)).dictionary_decode()


def campaigns(n_campaigns: int = 100, ads: int = 10, seed: int = 42) -> pa.RecordBatch:
    """generator.rs:43-55: `ads` ad ids per campaign id, one row (c_ad_id, campaign_id) per ad, grouped by campaign."""
    rng = np.random.default_rng([seed, 11])
    camp = uuid_bytes(n_campaigns, rng)
    ad = uuid_bytes(n_campaigns * ads, rng)
    return pa.RecordBatch.from_arrays([_fixed_strings(ad), _fixed_strings(np.repeat(camp, ads, axis=0))], schema=campaign_schema())


def ad_events(n_events: int, campaigns: pa.RecordBatch, seed: int = 42, columns: list[str] | None = None,
              events_per_second: int = EVENTS_PER_SECOND) -> pa.RecordBatch:
    """`n_events` ad events over the ads of `campaigns`.  Each column has its own random stream, so a batch restricted by
    `columns` (the benchmark scans ad_id and event_type only) carries exactly the values the full batch would."""
    full = ad_event_schema()
    want = [f.name for f in full] if columns is None else list(columns)
    ad_ids = campaigns.column(campaigns.schema.get_field_index("c_ad_id")).to_pylist()
    ad_chars = np.frombuffer("".join(ad_ids).encode(), np.uint8).reshape(len(ad_ids), UUID_LEN)

    def rng(i):
        return np.random.default_rng([seed, 13, i])
    arrays = {}
    for c in want:
        i = full.get_field_index(c)
        if c in ("user_id", "page_id"):
            arrays[c] = _fixed_strings(uuid_bytes(n_events, rng(i)))
        elif c == "ad_id":
            arrays[c] = _fixed_strings(ad_chars[rng(i).integers(0, len(ad_ids), n_events)])
        elif c == "ad_type":
            arrays[c] = _choice(AD_TYPES, rng(i).integers(0, len(AD_TYPES), n_events))
        elif c == "event_type":
            arrays[c] = _choice(EVENT_TYPES, rng(i).integers(0, len(EVENT_TYPES), n_events))
        elif c == "event_time":
            step = 1000.0 / events_per_second
            arrays[c] = pa.array(np.floor(1.0 + np.arange(n_events) * step).astype(np.int64), TS)
        elif c == "ip_address":
            arrays[c] = _choice(["0.0.0.0"], np.zeros(n_events, np.int32))
        else:
            raise KeyError(c)
    return pa.RecordBatch.from_arrays([arrays[c] for c in want], schema=pa.schema([full.field(c) for c in want], metadata=full.metadata))


def to_ndjson(batch: pa.RecordBatch) -> bytes:
    """The events as the source function sends them (generator.rs: next_epoch): serde_json of each AdEvent, fields in
    declaration order, the time as an integer, one event per line."""
    names = [f.name for f in ad_event_schema()]
    cols = {n: (batch.column(batch.schema.get_field_index(n)).cast(pa.int64()) if n == "event_time" else batch.column(batch.schema.get_field_index(n))).to_pylist()
            for n in names}
    lines = []
    for i in range(batch.num_rows):
        lines.append(json.dumps({n: cols[n][i] for n in names}, separators=(",", ":")))
    return ("\n".join(lines) + "\n").encode() if lines else b""
