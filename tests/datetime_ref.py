"""Python restatement of the date-time and bitmap transforms of app/vmselect/promql/transform.go, the reference of vmb_transform's
ids 64..74 (csrc/go_conv.cuh).

Date-time (newTransformFuncDateTime :333): a NaN stays; else s = int64(v) and the field of time.Unix(s, 0).UTC().
Bitmap (newTransformBitmap :2724): NaN if v or w is NaN, else float64(op(uint64(v), uint64(w))).

Go's float -> integer conversions are those of amd64: int64(v) is CVTTSD2SQ (trunc(v) in [-2^63, 2^63), else -2^63, +-Inf
included), uint64(v) the ssagen float64ToUint64 lowering on top of it.  Go's time fields are restated from Go 1.26's time.go:
abs = uint64(s + unixToAbsolute) seconds since March 1 of year -absoluteYears, then days.split, ayday.split and friends, in
wrapping uint64 arithmetic (Python integers reduced mod 2^64 where Go's would wrap).  The scalar form works in Python integers;
the numpy form does the same in uint64 arrays, whose arithmetic wraps like Go's."""
import math

import numpy as np

NAN = float("nan")
GO_NAN = np.frombuffer(np.uint64(0x7FF8000000000001).tobytes(), dtype=np.float64)[0]  # math.NaN(): the result of a NaN bitmap
M64 = (1 << 64) - 1
I64_MIN = -(1 << 63)

ABSOLUTE_YEARS = 292277022400  # time.go absoluteYears (a multiple of 400): the absolute zero instant is March 1 of -absoluteYears
UNIX_TO_INTERNAL = (1969 * 365 + 1969 // 4 - 1969 // 100 + 1969 // 400) * 86400
INTERNAL_TO_ABSOLUTE = (ABSOLUTE_YEARS // 400 * 146097 + 306) * 86400  # absoluteYears*365.2425 + marchThruDecember days
UNIX_TO_ABSOLUTE = UNIX_TO_INTERNAL + INTERNAL_TO_ABSOLUTE           # 9223372028741760000

DATETIME_FUNCS = ["hour", "minute", "day_of_month", "day_of_week", "day_of_year", "days_in_month", "month", "year"]
BITMAP_FUNCS = ["bitmap_and", "bitmap_or", "bitmap_xor"]
DAYS_IN_MONTH = [0, 31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]  # transform.go:2884

# app/vmselect/promql/exec_test.go, as written there: time() at 1000 ... 2000 s, step 200 s
T = np.arange(1000, 2001, 200, dtype=np.float64)
EXEC_TEST_DATETIME = [
    ("minute", T, [16, 20, 23, 26, 30, 33]),                                           # exec_test.go:825 minute()
    ("day_of_month", T * 1e4, [26, 19, 12, 5, 28, 20]),                                # :836
    ("day_of_week", T * 1e4, [0, 2, 5, 0, 2, 4]),                                      # :847
    ("day_of_year", T * 1e4, [116, 139, 163, 186, 209, 232]),                          # :858
    ("days_in_month", T * 2e4, [31, 31, 30, 31, 28, 30]),                              # :869
    ("hour", T * 1e4, [17, 21, 0, 4, 8, 11]),                                          # :880
    ("month", T * 1e4, [4, 5, 6, 7, 7, 8]),                                            # :891
    ("year", T * 1e5, [1973, 1973, 1974, 1975, 1975, 1976]),                          # :902
    ("minute", 30 * 60 + T, [46, 50, 53, 56, 0, 3]),                                   # :913
    ("minute", np.where((T <= 1200) | (T > 1600), T, NAN), [16, 20, NAN, NAN, 30, 33]),  # :924
]
EXEC_TEST_BITMAP = [
    ("bitmap_and", 0xB3, 0x11, [17] * 6),                       # exec_test.go:229
    ("bitmap_and", T, 0x11, [0, 16, 16, 0, 0, 16]),             # :240
    ("bitmap_and", NAN, 1, [NAN] * 6),                          # :251 (every point NaN: no series)
    ("bitmap_and", 1, NAN, [NAN] * 6),                          # :256
    ("bitmap_or", 0xA2, 0x11, [179] * 6),                       # :272
    ("bitmap_or", T, 0x11, [1017, 1201, 1401, 1617, 1817, 2001]),  # :283
    ("bitmap_or", NAN, 1, [NAN] * 6),                           # :294
    ("bitmap_xor", 0xB3, 0x11, [162] * 6),                      # :310
    ("bitmap_xor", T, 0x11, [1017, 1185, 1385, 1617, 1817, 1985]),  # :321
    ("bitmap_xor", NAN, 1, [NAN] * 6),                          # :332
]


def go_int64(v):
    """int64(v) on amd64 (CVTTSD2SQ); v not NaN"""
    if -2.0 ** 63 <= v < 2.0 ** 63:
        return int(v)
    return I64_MIN


def go_uint64(v):
    """uint64(v) on amd64 (float64ToUint64): exact on [0, 2^64) after truncation; else through int64's indefinite value"""
    if v < 2.0 ** 63:
        return go_int64(v) & M64
    return (go_int64(v - 2.0 ** 63) & M64) | (1 << 63)


def is_leap_u32(y):
    """isLeapYear(uint32(y)) transform.go:2874, y a Go int"""
    y &= 0xFFFFFFFF
    if y % 4 != 0:
        return False
    if y % 100 != 0:
        return True
    return y % 400 == 0


def go_time_fields(s):
    """the fields of time.Unix(s, 0).UTC() for an int64 s, in Go 1.26's arithmetic"""
    abs_ = (s + UNIX_TO_ABSOLUTE) & M64                      # absSeconds(sec + unixToAbsolute): wraps below -unixToAbsolute
    days = abs_ // 86400
    sod = abs_ % 86400
    d = 4 * days + 3                                          # days.split
    century = d // 146097
    cday = (d % 146097) // 4
    cd = 4 * cday + 3
    cyear, ayday = cd // 1461, cd % 1461 // 4
    janfeb = 1 if ayday >= 306 else 0                         # marchThruDecember
    md = 2141 * ayday + 197913                                # ayday.split
    month = (md >> 16) - 12 * janfeb
    mday = 1 + (md & 0xFFFF) // 2141
    year = (((century * 100 - ABSOLUTE_YEARS) & M64) ^ (1 << 63)) - (1 << 63) + cyear + janfeb  # int(uint64(century)*100-absoluteYears)
    leap = 1 if cyear % 4 == 0 and (cyear != 0 or century % 4 == 0) else 0
    yday = ayday + 60 + (leap & (1 - janfeb)) - 365 * janfeb
    dim = 29 if month == 2 and is_leap_u32(year) else DAYS_IN_MONTH[month]
    return {"hour": sod // 3600, "minute": sod % 3600 // 60, "day_of_month": mday, "day_of_week": (days + 3) % 7,
            "day_of_year": yday, "days_in_month": dim, "month": month, "year": year}


def time_field(name, v):
    """one value of hour(q) ... year(q)"""
    if math.isnan(v):
        return v
    return float(go_time_fields(go_int64(v))[name])


def bitmap(name, v, w):
    """one value of bitmap_and / or / xor(q, w); float(int) rounds half to even like Go's float64(uint64)"""
    if math.isnan(v) or math.isnan(w):
        return GO_NAN
    a, b = go_uint64(v), go_uint64(w)
    return float({"bitmap_and": a & b, "bitmap_or": a | b, "bitmap_xor": a ^ b}[name])


# ---- numpy forms, for matrices
def np_int64(v):
    v = np.asarray(v, dtype=np.float64)
    ok = (v >= -2.0 ** 63) & (v < 2.0 ** 63)
    s = np.where(ok, v, 0.0).astype(np.int64)
    s[~ok] = I64_MIN
    return s


def np_uint64(v):
    v = np.asarray(v, dtype=np.float64)
    lo = v < 2.0 ** 63
    a = np_int64(np.where(lo, v, 0.0)).view(np.uint64)
    with np.errstate(invalid="ignore"):
        b = np_int64(np.where(lo, 0.0, v - 2.0 ** 63)).view(np.uint64) | np.uint64(1 << 63)
    return np.where(lo, a, b)


def np_time_field(name, m):
    """time_field over an array (NaNs kept as they are)"""
    m = np.asarray(m, dtype=np.float64)
    nan = np.isnan(m)
    s = np_int64(np.where(nan, 0.0, m))
    u = np.uint64
    abs_ = s.view(u) + u(UNIX_TO_ABSOLUTE)
    days = abs_ // u(86400)
    sod = abs_ - days * u(86400)
    if name == "hour":
        out = sod // u(3600)
    elif name == "minute":
        out = sod % u(3600) // u(60)
    elif name == "day_of_week":
        out = (days + u(3)) % u(7)
    else:
        d = u(4) * days + u(3)
        century = d // u(146097)
        cday = d % u(146097) // u(4)
        cd = u(4) * cday + u(3)
        cyear, ayday = cd // u(1461), cd % u(1461) // u(4)
        janfeb = (ayday >= u(306)).astype(np.uint64)
        md = u(2141) * ayday + u(197913)
        month = (md >> u(16)) - u(12) * janfeb
        if name == "day_of_month":
            out = u(1) + (md & u(0xFFFF)) // u(2141)
        elif name == "month":
            out = month
        else:
            year = (century * u(100) - u(ABSOLUTE_YEARS)).view(np.int64) + cyear.astype(np.int64) + janfeb.astype(np.int64)
            if name == "year":
                out = year
            elif name == "day_of_year":
                leap = ((cyear % u(4) == 0) & ((cyear != 0) | (century % u(4) == 0))).astype(np.uint64)
                out = ayday + u(60) + (leap & (u(1) - janfeb)) - u(365) * janfeb
            else:
                y = year.view(np.uint64) & u(0xFFFFFFFF)
                leap = (y % u(4) == 0) & ((y % u(100) != 0) | (y % u(400) == 0))
                out = np.asarray(DAYS_IN_MONTH, dtype=np.uint64)[month.astype(np.int64)]
                out = np.where((month == 2) & leap, u(29), out)
    out = out.astype(np.int64).astype(np.float64)
    return np.where(nan, m, out)


def np_bitmap(name, m, w):
    """bitmap over a matrix [rows x points] with w a number or a per-point array"""
    m = np.asarray(m, dtype=np.float64)
    w = np.broadcast_to(np.asarray(w, dtype=np.float64), m.shape)
    a, b = np_uint64(m), np_uint64(w)
    r = {"bitmap_and": a & b, "bitmap_or": a | b, "bitmap_xor": a ^ b}[name]
    return np.where(np.isnan(m) | np.isnan(w), GO_NAN, r.astype(np.float64))


def np_ref(name, m, w=None):
    return np_bitmap(name, m, w) if name in BITMAP_FUNCS else np_time_field(name, m)
