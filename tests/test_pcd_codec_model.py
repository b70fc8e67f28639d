"""CPU: the ASCII PCD codec's per-token arithmetic (erasor_b200/csrc/pcd_codec.h, compiled for the host into
liberasor_b200_hostcheck.so) against numpy and Python.

- Parse: every token gives np.float32(float(tok)) bit for bit -- the correctly rounded double, then float, which is what
  read_pcd_ascii (np.loadtxt + astype) and the C++ load_pcd (istream >> double + (float)) compute -- and rejects exactly what
  np.loadtxt rejects.  Tokens the fast path cannot decide take the exact big-integer path, and some must.
- Format: every float gives Python's "%.8g" % float(f) (glibc printf's "%.8g"), NaN spelled "nan" whatever its sign.
The token and value sets are shared with tests/test_gpu_pcd_codec.py, which holds the kernels to the same references.
"""
import ctypes
import io
import os
import random
import warnings
from decimal import Decimal, getcontext
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTCHECK = os.path.join(ROOT, "erasor_b200", "_lib", "liberasor_b200_hostcheck.so")

KIND_FAST, KIND_SLOW, KIND_INVALID = 0, 1, 2

# numpy's loadtxt rejects each of these (as a whole token)
INVALID_TOKENS = ["0x10", "1_0", "1d5", "--1", "1e", ".", "e5", "+", "-", "1e+", "1e-", "1.2.3", "infinit", "infx", "nan(1)", "1e5.5",
                  "+-1", "1..", "..1", "in", "na", "nanx", "0b1", "1f", "1,5", "1e5e5", "+.", "-.e1", "1_000.5", "inf1", "e", "E3",
                  "1.5x", "x1", "１"]
SPECIAL_TOKENS = ["nan", "NaN", "NAN", "-nan", "+nan", "+NaN", "inf", "-inf", "+inf", "Inf", "-iNf", "infinity", "-Infinity",
                  "+INFINITY", "iNfInItY"]
PLAIN_TOKENS = ["0", "-0", "+0", "0.0", "-0.0", "-0e5", "0e-999", "-0.000e+400", "1.", ".5", "+.5e-3", "-.5E+3", "00012", "0001.2500",
                "1e99999999999999999999", "-1e99999999999999999999", "1e-99999999999", "1E5", "1e+05", "1e-05", "123456789",
                "3.4028235e38", "3.4028236e38", "3.40282357e38", "3.4028235677973366e38", "3.402823567797337e38", "-3.4028237e38",
                "1.17549435e-38", "1.1754942e-38", "1.4e-45", "1.401298464324817e-45", "7e-46", "7.006492321624085e-46",
                "7.0064923216240861e-46", "7.00649232162408e-46", "1e-46", "0.1", "0.2", "0.3", "1e23", "8.98846567431158e307",
                "9007199254740993", "9007199254740992", "9007199254740994", "9007199254740995", "18014398509481987",
                "2.2250738585072011e-308", "2.2250738585072012e-308", "2.2250738585072014e-308", "2.225073858507201e-308",
                "4.9406564584124654e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "3e-324", "5e-324", "1e-324",
                "1e-310", "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "1.797693134862315807e308",
                "1e308", "-1e308", "1e309", "1e-308", "1e-323", "1e342", "1e-342", "1e400", "-1e-400", "1e-400", "1e324", "-1e-324",
                "123.456e-7", "0.000000000000000000000000000000000000000000001401298464324817", "100000000000000000000000",
                "1" + "0" * 30 + "e-30", "0." + "0" * 40 + "1e40"]

# read_pcd_ascii parses with np.loadtxt and converts with astype(float32)
def np_reference(tokens):
    """float32 bit patterns np.loadtxt + astype give for valid tokens (one token per line)"""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a = np.loadtxt(io.StringIO("\n".join(tokens) + "\n"), dtype=np.float64, ndmin=1)
    with np.errstate(over="ignore"):
        return a.astype(np.float32).view(np.uint32)


def loadtxt_rejects(tok: str) -> bool:
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            np.loadtxt(io.StringIO(tok + "\n"), dtype=np.float64)
        return False
    except ValueError:
        return True


def midpoint_tokens(n, seed):
    """Decimals within 1e-30 (relative) of the midpoint between two neighbouring floats: a direct decimal -> float rounding and
    the decimal -> double -> float rounding disagree on the ones above a midpoint whose lower float is even, and both sides of
    the midpoint are taken.  Also the exact midpoints, and midpoints of subnormal floats."""
    getcontext().prec = 80
    rng = np.random.default_rng(seed)
    bits = rng.integers(1, 0x7F7FFFFF, n, dtype=np.uint32)
    bits[: n // 8] = rng.integers(1, 0x007FFFFF, n // 8, dtype=np.uint32)          # subnormals
    out = []
    for b in bits:
        f = np.uint32(b).view(np.float32)
        g = np.nextafter(f, np.float32(np.inf))
        mid = (Fraction(float(f)) + Fraction(float(g))) / 2
        d = Decimal(mid.numerator) / Decimal(mid.denominator)
        eps = d * Decimal("1e-30")
        for v in (d, d + eps, d - eps):
            out.append(f"{v:.45e}")
    return out


def long_mantissa_tokens(seed):
    rng = random.Random(seed)
    out = []
    for nd in (17, 19, 20, 25, 800):
        for _ in range(12):
            digits = str(rng.randint(1, 9)) + "".join(rng.choice("0123456789") for _ in range(nd - 1))
            e = rng.randint(-60, 40)
            pos = rng.randint(1, nd)
            out.append(f"{digits[:pos]}.{digits[pos:]}e{e - pos}")
            out.append(f"-{digits}e{rng.randint(-nd - 40, 30)}")
    # double halfway cases written with many digits: 2^53 + 1 and friends, and a 800-digit token on a double midpoint
    out += ["9007199254740993" + "0" * 20, "9007199254740993." + "0" * 780 + "1", "9007199254740993." + "0" * 790,
            "9007199254740992." + "9" * 800, "2.2250738585072011" + "0" * 784 + "1e-308"]
    return out


def exponent_tokens(seed):
    rng = random.Random(seed)
    out = []
    for e in (308, -308, 324, -324, 342, -342, 400, -400, 309, -323, -325, 38, -38, -45, -46):
        for _ in range(6):
            m = rng.choice(["1", "9.999999", "4.94065645841246544", "2.47032822920623272", "1.7976931348623157",
                            str(rng.randint(1, 10 ** 18))])
            out.append(f"{m}e{e}")
            out.append(f"-{m}e{e - len(m)}")
    return out


def random_tokens(n, seed):
    """what writers produce: %.8g, %.9g and repr of random floats of every binade, and random doubles"""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 0x7F800000, n, dtype=np.uint32).view(np.float32)
    d = rng.standard_normal(n) * np.exp(rng.uniform(-40, 40, n))
    out = [("%.8g" % float(v)) for v in f[: n // 3]] + [("%.9g" % float(v)) for v in f[n // 3:]] + [repr(float(v)) for v in d]
    return out


def adversarial_tokens():
    """every valid token kind the codec must get right (shared with the GPU test's adversarial file)"""
    return SPECIAL_TOKENS + PLAIN_TOKENS + midpoint_tokens(400, 7) + long_mantissa_tokens(8) + exponent_tokens(9)


def format_values(seed=3, per_binade=64):
    """float32 values for the formatter: a random sample of every binade (both signs), the %f / %e switch at 1e-4 / 1e-5 and
    1e7 / 1e8 and at every power of ten, every float whose eight-digit rounding carries into the next power of ten (with
    neighbours), and the special values."""
    rng = np.random.default_rng(seed)
    vals = []
    for be in range(256 - 1):
        m = rng.integers(0, 1 << 23, per_binade, dtype=np.uint32)
        b = (np.uint32(be) << np.uint32(23)) | m
        b[: per_binade // 2] |= np.uint32(0x80000000)
        vals.append(b.view(np.float32))
    around = []
    for x in range(-45, 39):
        for p in (10.0 ** x, 9.99999995 * 10.0 ** x, 9.9999999 * 10.0 ** x, 9.99999999 * 10.0 ** x):
            with np.errstate(over="ignore"):
                c = np.float32(p)
            if not np.isfinite(c) or c == 0:
                continue
            lo = hi = c
            for _ in range(40):
                lo = np.nextafter(lo, np.float32(0))
                hi = np.nextafter(hi, np.float32(np.inf))
            v = lo
            while v <= hi and np.isfinite(v):
                around.append(v)
                v = np.nextafter(v, np.float32(np.inf))
    vals.append(np.array(around, dtype=np.float32))
    vals.append(np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1e-4, 1e-5, 1e7, 1e8, 9.9999999747e-07, 999999995904.0,
                          1234567.25, 1234567.75, 0.5, 1.5, 2.5], dtype=np.float32))
    vals.append(np.array([1, 0x80000001, 0x7F7FFFFF, 0xFF7FFFFF, 0x00800000, 0x007FFFFF, 0x7FC00000, 0xFFC00000, 0x7F800001],
                         dtype=np.uint32).view(np.float32))
    return np.concatenate(vals)


def tie_values():
    """every float of a few binades whose exact value lies halfway between two eight-digit decimals (printf rounds it to even)"""
    out = []
    for e in (-5, 0, 3, 6, 10, 13):
        lo_b, hi_b = 2.0 ** e, 2.0 ** (e + 1)
        for X in range(int(np.floor(np.log10(lo_b))), int(np.floor(np.log10(hi_b))) + 1):
            t = 7 - X
            sh = 22 - e - t
            if sh < 0:
                continue
            step = 1 << sh
            k = np.arange(step, 1 << 24, 2 * step, dtype=np.int64)
            k = k[k >= (1 << 23)]
            v = (k.astype(np.float64) * 2.0 ** (e - 23))
            v = v[(v >= 10.0 ** X) & (v < 10.0 ** (X + 1))]
            out.append(v.astype(np.float32))
    return np.concatenate(out)


def py_format(v: np.ndarray):
    return ["nan" if np.isnan(x) else "%.8g" % float(x) for x in v]


# ---- the host build of pcd_codec.h ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    if not os.path.exists(HOSTCHECK):
        pytest.skip("build first: erasor_b200/csrc/build.sh")
    return ctypes.CDLL(HOSTCHECK)


def host_parse(L, tokens, want_value=True):
    raw = [t.encode() for t in tokens]
    offs = np.zeros(len(raw) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(r) for r in raw])
    text = np.frombuffer(b"".join(raw) + b"\0", dtype=np.uint8)
    bits = np.zeros(len(raw), dtype=np.uint32)
    kind = np.zeros(len(raw), dtype=np.int32)
    assert L.erasor_hostcheck_pcd_parse(text.ctypes.data_as(ctypes.c_void_p), offs.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(raw)),
                                        ctypes.c_int(1 if want_value else 0), bits.ctypes.data_as(ctypes.c_void_p),
                                        kind.ctypes.data_as(ctypes.c_void_p)) == 0
    return bits, kind


def host_format(L, vals):
    v = np.ascontiguousarray(vals, dtype=np.float32)
    buf = ctypes.create_string_buffer(16 * len(v) + 1)
    lens = np.zeros(len(v), dtype=np.int32)
    assert L.erasor_hostcheck_pcd_format(v.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(v)), buf, lens.ctypes.data_as(ctypes.c_void_p)) == 0
    raw = buf.raw
    return [raw[16 * i: 16 * i + lens[i]].decode() for i in range(len(v))]


def check_parse(L, tokens):
    bits, kind = host_parse(L, tokens)
    assert (kind != KIND_INVALID).all(), [t for t, k in zip(tokens, kind) if k == KIND_INVALID][:5]
    ref = np_reference(tokens)
    bad = np.nonzero(bits != ref)[0]
    assert len(bad) == 0, [(tokens[i][:60], hex(bits[i]), hex(ref[i])) for i in bad[:5]]
    # the Python reference of the other reader (float() then float32) agrees too: one rounding to double, then one to float
    with np.errstate(over="ignore"):
        for t, b in zip(tokens[:200], bits[:200]):
            assert np.float32(float(t)).view(np.uint32) == b, t
    return kind


def test_invalid_tokens_are_rejected_like_loadtxt(L):
    for t in INVALID_TOKENS:
        assert loadtxt_rejects(t), t
    _, kind = host_parse(L, INVALID_TOKENS)
    assert (kind == KIND_INVALID).all(), [t for t, k in zip(INVALID_TOKENS, kind) if k != KIND_INVALID]


def test_unkept_columns_are_checked_alone(L):
    """a column that is not kept only goes through the grammar check (want_value = false): it rejects the same tokens and accepts
    every valid one, without the slow path"""
    _, kind = host_parse(L, INVALID_TOKENS, want_value=False)
    assert (kind == KIND_INVALID).all(), [t for t, k in zip(INVALID_TOKENS, kind) if k != KIND_INVALID]
    valid = adversarial_tokens()
    bits, kind = host_parse(L, valid, want_value=False)
    assert (kind == KIND_FAST).all(), [t[:40] for t, k in zip(valid, kind) if k != KIND_FAST][:5]
    assert not bits.any()


def test_special_and_plain_tokens(L):
    for t in SPECIAL_TOKENS + PLAIN_TOKENS:
        assert not loadtxt_rejects(t), t
    kind = check_parse(L, SPECIAL_TOKENS + PLAIN_TOKENS)
    slow = {t for t, k in zip(SPECIAL_TOKENS + PLAIN_TOKENS, kind) if k == KIND_SLOW}
    # these cannot be decided by Clinger's fast path and must have gone through the big-integer comparison
    for t in ("9007199254740993", "2.2250738585072011e-308", "2.4703282292062327e-324", "1.7976931348623159e308", "1e-400", "1e342"):
        assert t in slow, t
    assert "0.1" not in slow and "123.456e-7" not in slow and "1e23" not in slow


def test_tokens_near_float_midpoints(L):
    toks = midpoint_tokens(400, 7)
    kind = check_parse(L, toks)
    assert (kind == KIND_SLOW).sum() > len(toks) // 2


def test_double_rounding_differs_from_direct_rounding(L):
    """the tokens just above an exact midpoint between two floats, with the lower float even: decimal -> double lands exactly on the
    midpoint and the float rounding goes to even (down), where a direct decimal -> float rounding goes up"""
    getcontext().prec = 80
    f = np.float32(1.0)
    g = np.nextafter(f, np.float32(2))
    mid = (Decimal(float(f)) + Decimal(float(g))) / 2
    tok = f"{mid + mid * Decimal('1e-30'):.40e}"
    bits, kind = host_parse(L, [tok])
    assert bits[0] == np.float32(1.0).view(np.uint32)      # double rounding: to the even float below
    assert kind[0] == KIND_SLOW


def test_long_mantissas_and_extreme_exponents(L):
    toks = long_mantissa_tokens(8) + exponent_tokens(9)
    kind = check_parse(L, toks)
    n800 = [k for t, k in zip(toks, kind) if len(t) > 700]
    assert n800 and all(k == KIND_SLOW for k in n800)


def test_random_writer_tokens(L):
    toks = random_tokens(30000, 11)
    kind = check_parse(L, toks)
    assert (kind == KIND_FAST).mean() > 0.4


def test_format_every_binade_and_boundaries(L):
    v = format_values()
    got, ref = host_format(L, v), py_format(v)
    bad = [(float(x), g, r) for x, g, r in zip(v, got, ref) if g != r]
    assert not bad, bad[:10]


def test_format_carries_into_power_of_ten(L):
    v = np.array([9.9999999747e-07, 999999995904.0], dtype=np.float32)
    assert host_format(L, v) == ["1e-06", "1e+12"]
    # every float whose eight-digit rounding reaches the next power of ten, at every decade
    carries = []
    for x in range(-46, 39):
        lo, hi = Fraction(999999995, 100000000) * Fraction(10) ** x, Fraction(10) ** (x + 1)
        with np.errstate(over="ignore"):
            c = np.float32(float(lo))
        if not np.isfinite(c):
            continue
        while Fraction(float(c)) >= lo:
            c = np.nextafter(c, np.float32(0))
        c = np.nextafter(c, np.float32(np.inf))
        while np.isfinite(c) and Fraction(float(c)) < hi:
            carries.append(c)
            c = np.nextafter(c, np.float32(np.inf))
    carries = np.array(carries, dtype=np.float32)
    assert len(carries) >= 5 and np.float32(9.9999999747e-07) in carries and np.float32(999999995904.0) in carries
    got = host_format(L, carries)
    assert got == py_format(carries)
    assert all(g.startswith("1e") or g.rstrip("0").rstrip(".") in ("1", "10", "100", "1000", "10000", "100000", "1000000", "10000000")
               or g.startswith("0.") for g in got)


def test_format_ties_round_to_even(L):
    v = tie_values()
    assert len(v) > 10000
    assert host_format(L, np.array([1234567.25], dtype=np.float32)) == ["1234567.2"]
    got, ref = host_format(L, v), py_format(v)
    bad = [(float(x), g, r) for x, g, r in zip(v, got, ref) if g != r]
    assert not bad, bad[:10]


def test_format_special_values(L):
    v = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan], dtype=np.float32)
    v = np.concatenate([v, np.array([1, 0x80000001, 0x7F7FFFFF], dtype=np.uint32).view(np.float32)])
    assert host_format(L, v) == ["0", "-0", "inf", "-inf", "nan", "nan", "1.4012985e-45", "-1.4012985e-45", "3.4028235e+38"]


def test_format_then_parse_round_trips_the_writers_text(L):
    """parse(format(x)) equals what read_pcd_ascii makes of write_pcd_ascii's text for the same floats"""
    v = format_values(per_binade=16)
    text = host_format(L, v)
    assert text == py_format(v)
    bits, kind = host_parse(L, text)
    assert (kind != KIND_INVALID).all()
    ref = np_reference(text)
    assert np.array_equal(bits, ref)
