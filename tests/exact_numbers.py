"""IEEE-754 bit patterns computed exactly, with Python integers and fractions only: the reference the schema resolution
tests hold the promotions and the numeric default constants to.

Nothing here goes through a Python float or a hardware conversion (numpy's casts use the same x86 instructions as the
host code under test, and CPython's struct quiets signalling NaNs), so it is independent of what it checks.
  int_to_f32_bits / int_to_f64_bits   an int64 rounded to nearest even (int / long -> float / double)
  widen_f32_bits                      float -> double, exact; a NaN keeps its payload and gets the quiet bit
  decimal_text_to_f64_bits / _f32_    a JSON number's text as a double, and as that double rounded to float
  int32_of_varint                     the `as i32` of a zigzag varint's value taken mod 2^64 (an int's decode)"""
from fractions import Fraction

M64 = (1 << 64) - 1

# (precision in bits incl. the implicit one, exponent bias, exponent field width)
F32 = (24, 127, 8)
F64 = (53, 1023, 11)


def _pack(fmt, sign: int, q: int, e: int) -> int:
    """Bits of (-1)^sign * q * 2^e, where q < 2^p is already rounded and e >= the subnormal exponent; infinity when the
    value is beyond the finite range."""
    p, bias, ew = fmt
    mant_bits, top = p - 1, (1 << ew) - 1
    if q >= 1 << p:   # (only 2^p itself, after a round-up)
        q, e = q >> 1, e + 1
    if q == 0:
        return sign << (ew + mant_bits)
    if q < 1 << mant_bits:   # subnormal: the exponent is the smallest one
        biased = 0
    else:
        biased = e + mant_bits + bias
        if biased >= top:
            return (sign << (ew + mant_bits)) | (top << mant_bits)
        q -= 1 << mant_bits
    return (sign << (ew + mant_bits)) | (biased << mant_bits) | q


def _round_fraction(fmt, x: Fraction, sign: int) -> int:
    """x >= 0 to nearest, ties to even."""
    p, bias, _ = fmt
    if x == 0:
        return _pack(fmt, sign, 0, 0)
    e = x.numerator.bit_length() - x.denominator.bit_length()   # 2^e <= x < 2^(e+1) after the adjustment
    if Fraction(2) ** e > x:
        e -= 1
    e = max(e, 1 - bias)                                        # below the normal range: the subnormal spacing
    ulp_e = e - (p - 1)
    scaled = x / Fraction(2) ** ulp_e
    q = scaled.numerator // scaled.denominator
    rem = scaled - q
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and q & 1):
        q += 1
    return _pack(fmt, sign, q, ulp_e)


def _int_bits(fmt, v: int) -> int:
    assert -(1 << 63) <= v < (1 << 63)
    return _round_fraction(fmt, Fraction(abs(v)), 1 if v < 0 else 0)


def int_to_f32_bits(v: int) -> int:
    return _int_bits(F32, v)


def int_to_f64_bits(v: int) -> int:
    return _int_bits(F64, v)


def widen_f32_bits(u: int) -> int:
    s, e, m = u >> 31, (u >> 23) & 0xFF, u & 0x7FFFFF
    sign = s << 63
    if e == 0xFF:
        return sign | (0x7FF << 52) | (((1 << 51) | (m << 29)) if m else 0)
    if e == 0:
        if m == 0:
            return sign
        n = m.bit_length()                       # value m * 2^-149, leading bit at 2^(n - 150)
        return sign | ((n - 150 + 1023) << 52) | ((m - (1 << (n - 1))) << (53 - n))
    return sign | ((e - 127 + 1023) << 52) | (m << 29)


def bits_value(fmt, b: int) -> Fraction:
    """The exact value of finite bits `b`."""
    p, bias, ew = fmt
    mb = p - 1
    s, e, m = b >> (ew + mb), (b >> mb) & ((1 << ew) - 1), b & ((1 << mb) - 1)
    assert e != (1 << ew) - 1
    v = Fraction(m, 1 << mb) * Fraction(2) ** (1 - bias) if e == 0 else Fraction((1 << mb) | m, 1 << mb) * Fraction(2) ** (e - bias)
    return -v if s else v


def decimal_text_to_f64_bits(text: str) -> int:
    t = text.strip()
    sign = 1 if t.startswith("-") else 0
    return _round_fraction(F64, Fraction(t.lstrip("+-")), sign)


def decimal_text_to_f32_bits(text: str) -> int:
    """Two roundings: the text to the nearest double, then that double to the nearest float."""
    d = decimal_text_to_f64_bits(text)
    sign = d >> 63
    if (d >> 52) & 0x7FF == 0x7FF:
        return (sign << 31) | 0x7F800000
    return _round_fraction(F32, abs(bits_value(F64, d)), sign)


def int32_of_varint(z: int) -> int:
    z &= M64
    v = (z >> 1) ^ -(z & 1)
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)
