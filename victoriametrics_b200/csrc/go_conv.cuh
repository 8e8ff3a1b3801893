// Go's float64 -> integer conversions and Go's UTC calendar, restated for the date-time and bitmap transforms of transform.inc
// (newTransformFuncDateTime transform.go:333, newTransformBitmap :2724).
//
// Conversions: the Go spec leaves out-of-range float -> integer conversions to the implementation.  These follow amd64 at the
// default GOAMD64 level: int64(v) is CVTTSD2SQ, which truncates and gives 0x8000000000000000 for every value outside
// [-2^63, 2^63), +-Inf and NaN included (CUDA's cvt.rzi.s64.f64 saturates instead, so the range is tested here); uint64(v) is the
// ssagen float64ToUint64 lowering: v < 2^63 ? uint64(int64(v)) : uint64(int64(v - 2^63)) | 2^63.
//
// Calendar: time.Unix(s, 0).UTC() keeps s, and every field reads abs = uint64(s + unixToAbsolute), seconds since the "absolute
// zero instant", March 1 of year -absoluteYears (time.go of Go 1.26: absoluteYears = 292277022400, a multiple of 400, and
// unixToAbsolute = (absoluteYears * 365.2425 + 306 + 719162) * 86400 = 9223372028741760000).  The constant and the split
// below (days.split, ayday.split, century.year, century.leap, weekday) restate Go 1.26's time.go without a Go toolchain or Go's
// sources to check them against: UNVERIFIED.  They only matter below s = -unixToAbsolute (the bottom
// 8.1e9 s of int64, -2^63 included), where s + unixToAbsolute wraps and the fields are those of a day near year 2.9e11; at and
// above it every formula is the proleptic Gregorian calendar, which tests/test_datetime_ref.py checks against Python's datetime.
#pragma once
#include <stdint.h>

#define GO_ABS_YEARS 292277022400ll
#define GO_UNIX_TO_ABS 9223372028741760000ull

__device__ __forceinline__ int64_t go_f64_to_i64(double v) {
    return v >= -9223372036854775808.0 && v < 9223372036854775808.0 ? __double2ll_rz(v) : (int64_t)0x8000000000000000ull;
}

__device__ __forceinline__ uint64_t go_f64_to_u64(double v) {
    if (v < 9223372036854775808.0) return (uint64_t)go_f64_to_i64(v);
    return (uint64_t)go_f64_to_i64(__dsub_rn(v, 9223372036854775808.0)) | 0x8000000000000000ull;  // exact below 2^64
}

__device__ __forceinline__ bool go_leap_u32(uint32_t y) { return y % 4 == 0 && (y % 100 != 0 || y % 400 == 0); }  // transform.go:2874

// The fields of time.Unix(s, 0).UTC() that go_time_field reads.  sod: second of the day; wday: Weekday (Sunday 0); Go's absolute
// date split (days.split): century = (4 * days + 3) / 146097, cday the day in it, c400: the century is a multiple of 4,
// cent_year: int(uint64(century)*100 - absoluteYears), the year that starts the century.
struct GoCal {
    uint32_t sod, wday, cday;
    bool c400;
    int64_t cent_year;
};

__device__ __forceinline__ GoCal go_cal_split(int64_t s) {
    GoCal g;
    const uint64_t abs = (uint64_t)s + GO_UNIX_TO_ABS, days = abs / 86400;  // wraps below -unixToAbsolute, as Go's does
    g.sod = (uint32_t)(abs - days * 86400);
    g.wday = (uint32_t)((days + 3) % 7);  // March 1 of the absolute zero year, a multiple of 400, is a Wednesday
    const uint64_t d = 4 * days + 3, century = d / 146097;
    g.cday = (uint32_t)(d % 146097) / 4;
    g.c400 = century % 4 == 0;
    g.cent_year = (int64_t)(century * 100 - (uint64_t)GO_ABS_YEARS);
    return g;
}

// ops: 0 hour, 1 minute, 2 day_of_month, 3 day_of_week, 4 day_of_year, 5 days_in_month, 6 month, 7 year
__device__ __forceinline__ double go_time_field(int op, int64_t s) {
    const GoCal g = go_cal_split(s);
    if (op == 0) return (double)(g.sod / 3600);
    if (op == 1) return (double)(g.sod / 60 % 60);
    if (op == 3) return (double)g.wday;
    const uint32_t cd = 4 * g.cday + 3, cyear = cd / 1461, ayday = cd % 1461 / 4;  // ayday: days since March 1
    const uint32_t janfeb = ayday >= 306;
    const uint32_t md = 2141 * ayday + 197913, month = (md >> 16) - 12 * janfeb;
    const int64_t year = g.cent_year + cyear + janfeb;
    switch (op) {
        case 2: return (double)(1 + (md & 0xffff) / 2141);
        case 4:  // ayday.yday: + leap &^ janFeb; a March-based year is a leap year when the calendar year it starts is
            return (double)(ayday + 60 + (!janfeb && cyear % 4 == 0 && (cyear != 0 || g.c400)) - 365 * janfeb);
        case 5:  // daysInMonth[m] (transform.go:2884) is 30 + ((m + m / 8) & 1) outside February
            return month == 2 ? (go_leap_u32((uint32_t)year) ? 29.0 : 28.0) : (double)(30 + ((month + (month >> 3)) & 1));
        case 6: return (double)month;
    }
    return (double)year;
}
