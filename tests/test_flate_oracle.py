"""The inflate oracle (oracle/orc_flate.c) against Python's zlib on a seeded pool, on hand-written invalid streams, and on
every truncation of a few streams."""
import random
import zlib

import pytest

import flate_util as F


def test_pool_equals_zlib():
    for fmt, s, data, multi in F.pool():
        r, out = F.orc_decode(fmt, s, len(data) + 16, multi)
        assert r == len(data) and out == data, (fmt, len(data), r)


def test_dst_one_byte_short():
    for fmt, s, data, multi in F.pool(n=40):
        if data:
            assert F.orc_decode(fmt, s, len(data) - 1, multi)[0] == -4


@pytest.mark.parametrize("case", F.invalid_streams(), ids=lambda c: "%d-%s" % (c[0], c[1][:6].hex()))
def test_invalid_streams(case):
    fmt, s, want = case[:3]
    multi = case[3] if len(case) > 3 else True
    assert F.orc_decode(fmt, s, 1 << 16, multi)[0] == want


@pytest.mark.parametrize("case", F.stale_streams(), ids=lambda c: "%d-%d" % (c[0], len(c[1])))
def test_stale_tables(case):
    # an empty code keeps the table of its slot; the fixed code has a slot of its own
    fmt, s, want = case
    r = F.orc_decode(fmt, s, 1 << 16)[0]
    assert r == want if want is not None else r < 0


def test_reference_fixtures():
    n = 0
    for name, fmt, s, want in F.fixture_streams():
        r, out = F.orc_decode(fmt, s, 1 << 20)
        if want is None:
            assert r < 0, name
        elif isinstance(want, int):
            assert r == want, (name, r)
        else:
            assert r == len(want) and out == want, (name, r)
        n += 1
    assert n > 120


def test_truncations():
    rng = random.Random(3)
    data = F.text(rng, 3000)
    for fmt in (F.RAW, F.ZLIB, F.GZIP):
        for level in (0, 1, 9):
            s = F.deflate(data, fmt, level)
            for i in range(len(s)):
                r = F.orc_decode(fmt, s[:i], 4000)[0]
                if fmt == F.RAW:
                    # a raw stream cut inside the extra bits of a length or distance ends there without error
                    assert r == -12 or (r >= 0 and data.startswith(F.orc_decode(fmt, s[:i], 4000)[1])), (fmt, level, i, r)
                else:
                    assert r == -12, (fmt, level, i, r)


def test_mutations_agree_with_zlib_on_success():
    # every mutated zlib stream that zlib decodes, the oracle decodes to the same bytes (zlib's error messages do not map
    # onto the reference's classes, so failures are compared between the oracle and the device instead)
    rng = random.Random(11)
    base = [F.deflate(F.text(rng, n), F.ZLIB, lv) for n, lv in ((2000, 1), (5000, 6), (800, 9), (3000, 0))]
    for _ in range(600):
        s = F.mutate(rng, rng.choice(base))
        try:
            want = zlib.decompress(s)
        except zlib.error:
            want = None
        r, out = F.orc_decode(F.ZLIB, s, 1 << 16)
        if want is not None:
            assert r == len(want) and out == want
