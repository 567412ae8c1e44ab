"""The fast-field value images of sort columns (fast_value_to_u64 / u64_to_fast_value against common/src/lib.rs's i64_to_u64 and
f64_to_u64, restated here bit by bit), and the sort entry points of the C ABI: exported by the library and mirrored by _abi.py,
tq_stats' new fields appended at its end."""
import ctypes as C
import os
import re
import struct
import subprocess

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import _abi
from tantivy_b200.lib import LIB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = 1 << 63


def i64_to_u64(v):  # (val as u64) ^ HIGHEST_BIT
    return (v & (2**64 - 1)) ^ H


def f64_to_u64(v):  # bits ^ HIGHEST_BIT when the sign is positive, else !bits
    bits = struct.unpack("<Q", struct.pack("<d", v))[0]
    return bits ^ H if not bits >> 63 else bits ^ (2**64 - 1)


F64 = [-np.inf, -1e308, -2.5, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0, 2.5, 1e308, np.inf]
I64 = [-2**63, -2**63 + 1, -5, -1, 0, 1, 7, 2**63 - 2, 2**63 - 1]


def test_f64_images():
    got = T.fast_value_to_u64(np.array(F64), "f64")
    assert [int(x) for x in got] == [f64_to_u64(v) for v in F64]
    assert all(int(a) < int(b) for a, b in zip(got[:-1], got[1:]))  # monotonic, -0.0 below +0.0
    back = T.u64_to_fast_value(got, "f64")
    assert [struct.pack("<d", x) for x in back] == [struct.pack("<d", x) for x in F64]  # (the sign of zero survives)


def test_f64_nan():
    for bits in (0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001):
        v = np.array([bits], np.uint64).view(np.float64)
        img = T.fast_value_to_u64(v, "f64")
        assert int(img[0]) == (bits ^ H if not bits >> 63 else bits ^ (2**64 - 1))
        assert int(T.u64_to_fast_value(img, "f64").view(np.uint64)[0]) == bits
    pos_nan = int(T.fast_value_to_u64(np.array([0x7FF8000000000000], np.uint64).view(np.float64), "f64")[0])
    assert pos_nan > int(T.fast_value_to_u64(np.array([np.inf]), "f64")[0])  # a positive NaN sorts above +inf


def test_i64_and_date_images():
    got = T.fast_value_to_u64(np.array(I64, np.int64), "i64")
    assert [int(x) for x in got] == [i64_to_u64(v) for v in I64]
    assert got[0] == 0 and got[-1] == 2**64 - 1 and got[4] == H
    assert all(int(a) < int(b) for a, b in zip(got[:-1], got[1:]))
    assert list(T.u64_to_fast_value(got, "i64")) == I64
    dates = np.array(["1960-03-01T00:00:00", "1970-01-01", "2024-05-06T07:08:09.123456789"], dtype="datetime64[ns]")
    img = T.fast_value_to_u64(dates, "date")
    assert [int(x) for x in img] == [i64_to_u64(int(d)) for d in dates.view(np.int64)]
    assert np.array_equal(T.fast_value_to_u64(dates[:2].astype("datetime64[s]"), "date"), img[:2])  # any unit: nanoseconds
    assert np.array_equal(T.u64_to_fast_value(img, "date"), dates)


def test_u64_and_bool_images():
    u = np.array([0, 1, 2**63, 2**64 - 1], np.uint64)
    assert np.array_equal(T.fast_value_to_u64(u, "u64"), u)
    assert np.array_equal(T.u64_to_fast_value(u, "u64"), u)
    assert list(T.fast_value_to_u64(np.array([False, True]), "bool")) == [0, 1]
    assert list(T.u64_to_fast_value(np.array([0, 1], np.uint64), "bool")) == [False, True]
    with pytest.raises(ValueError):
        T.fast_value_to_u64(u, "i32")


def test_random_round_trip_and_order():
    rng = np.random.default_rng(3)
    f = np.concatenate([rng.normal(0, 1e3, 2000), rng.normal(0, 1e-300, 100), [0.0, -0.0]])
    img = T.fast_value_to_u64(f, "f64")
    assert np.array_equal(T.u64_to_fast_value(img, "f64").view(np.uint64), f.view(np.uint64))
    o = np.argsort(img, kind="stable")
    assert np.all(np.diff(f[o]) >= 0)
    i = rng.integers(-2**63, 2**63 - 1, 2000, dtype=np.int64, endpoint=True)
    img = T.fast_value_to_u64(i, "i64")
    assert np.array_equal(T.u64_to_fast_value(img, "i64"), i)
    assert np.array_equal(np.argsort(img, kind="stable"), np.argsort(i, kind="stable"))


def test_abi_symbols_and_specs():
    for name in ("tq_sort_column_register", "tq_sort_column_unregister", "tq_sort_batch"):
        assert hasattr(LIB, name)
    hdr = open(os.path.join(ROOT, "include", "tantivy_b200.h")).read()
    assert re.search(r"#define TQ_ORDER_DESC 0u", hdr) and re.search(r"#define TQ_ORDER_ASC 1u", hdr)
    assert (_abi.TQ_ORDER_DESC, _abi.TQ_ORDER_ASC) == (0, 1)
    assert C.sizeof(_abi.SortSpec) == 8


def _header_stats_fields():
    hdr = open(os.path.join(ROOT, "include", "tantivy_b200.h")).read()
    body = hdr[hdr.index("typedef struct {\n  uint64_t lists_cached;"):hdr.index("} tq_stats;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.replace("typedef struct {", "").strip()
        if not decl:
            continue
        for part in decl.split(" ", 1)[1].split(","):
            names.append(re.sub(r"\[\d+\]", "", part).strip())
    return names


def test_stats_layout_mirrored():
    names = _header_stats_fields()
    assert names == [n for n, _ in _abi.Stats._fields_]
    assert names[-4:] == ["sort_ms", "units_sort", "sort_tiles_seen", "sort_tiles_skipped"]


def test_stats_offsets_match_the_compiler(tmp_path):
    """offsetof / sizeof of tq_stats as a C compiler lays it out equal the ctypes mirror's."""
    src = tmp_path / "off.c"
    fields = [n for n, _ in _abi.Stats._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tantivy_b200.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(tq_stats, {n}));\n' for n in fields)
                   + '  printf("%zu\\n", sizeof(tq_stats));\n  return 0;\n}\n')
    exe = tmp_path / "off"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [getattr(_abi.Stats, n).offset for n in fields] + [C.sizeof(_abi.Stats)]
