"""TEST INFRASTRUCTURE (oracle): Jubjub point decoding restated with Python integers, independent of the device code.

  curve        -x^2 + y^2 = 1 + d x^2 y^2 over Fr            core/jubjub/src/curve/mod.rs:198-210
  Point::read  y = low 255 bits (< r or NotInField), x^2 = (y^2 - 1) / (d y^2 + 1), square root (none: NotOnCurve),
               x negated when its parity differs from bit 255      core/jubjub/src/curve/edwards.rs:92-164
  as_prime_order  [r_J] P == O                                   edwards.rs:319-325
  into_xy      affine (x, y)                                     edwards.rs:341-352

Affine twisted-Edwards addition (with its two field divisions) and a plain double-and-add; the square root is
Tonelli-Shanks with Euler's criterion deciding which elements have none.  Status codes are those of zk_jubjub_into_xy."""
from __future__ import annotations

R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001          # Fr modulus (the Jubjub base field)
D = 19257038036680949359750312669786877991949435402254120286184196891950884077233    # mod.rs:204, d = -(10240/10241)
R_J = 0x0e7db4ea6533afa906673b0101343b00a6682093ccc81082d0970e5ed6f72cb7        # fs.rs:14, the prime subgroup order
COFACTOR = 8
OK, NOT_IN_FIELD, NOT_ON_CURVE, NOT_PRIME_ORDER = 0, 1, 2, 3
IDENTITY = (0, 1)

assert D == (-10240 * pow(10241, -1, R)) % R


def is_square(a: int) -> bool:
    a %= R
    return a == 0 or pow(a, (R - 1) // 2, R) == 1


def sqrt(a: int):
    """A square root of a in Fr, or None.  Tonelli-Shanks with r - 1 = 2^32 t."""
    a %= R
    if a == 0:
        return 0
    if not is_square(a):
        return None
    s, t = 0, R - 1
    while t % 2 == 0:
        s, t = s + 1, t // 2
    z = 2
    while is_square(z):
        z += 1
    m, c, x, b = s, pow(z, t, R), pow(a, (t + 1) // 2, R), pow(a, t, R)
    while b != 1:
        i, b2 = 0, b
        while b2 != 1:
            b2, i = b2 * b2 % R, i + 1
        e = pow(c, 1 << (m - i - 1), R)
        m, c, x, b = i, e * e % R, x * e % R, b * e * e % R
    assert x * x % R == a
    return x


def on_curve(p) -> bool:
    x, y = p
    return (-x * x + y * y - 1 - D * x * x % R * y * y) % R == 0


def add(p, q):
    """Affine twisted-Edwards addition with a = -1 (complete: the denominators never vanish on the curve)."""
    (x1, y1), (x2, y2) = p, q
    k = D * x1 * x2 % R * y1 * y2 % R
    x3 = (x1 * y2 + y1 * x2) * pow((1 + k) % R, -1, R) % R
    y3 = (y1 * y2 + x1 * x2) * pow((1 - k) % R, -1, R) % R
    return x3, y3


def neg(p):
    return (-p[0]) % R, p[1]


def mul(p, k: int):
    acc = IDENTITY
    for bit in bin(k)[2:] if k else "":
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, p)
    return acc


def read(enc: bytes):
    """Point::read: (status, point or None)."""
    assert len(enc) == 32
    v = int.from_bytes(enc, "little")
    sign, y = v >> 255, v & ((1 << 255) - 1)
    if y >= R:
        return NOT_IN_FIELD, None
    u = (y * y - 1) * pow((D * y * y + 1) % R, -1, R) % R
    x = sqrt(u)
    if x is None:
        return NOT_ON_CURVE, None
    if (x & 1) != sign:
        x = (-x) % R
    return OK, (x, y)


def into_xy(enc: bytes):
    """read + as_prime_order + into_xy: (status, x, y); x = y = 0 when rejected."""
    st, p = read(enc)
    if st != OK:
        return st, 0, 0
    if mul(p, R_J) != IDENTITY:
        return NOT_PRIME_ORDER, 0, 0
    return OK, p[0], p[1]


def encode(p) -> bytes:
    """The write side (edwards.rs:190-206): y little-endian with the parity of x in bit 255."""
    x, y = p
    return (y | ((x & 1) << 255)).to_bytes(32, "little")


def point_for_y(y: int, sign: int = 0):
    """The curve point with this y and x parity, or None."""
    x = sqrt((y * y - 1) * pow((D * y * y + 1) % R, -1, R))
    if x is None:
        return None
    return ((-x) % R if (x & 1) != sign else x), y


def torsion_point(order: int):
    """A point of exact order 2, 4 or 8 (the cofactor part of the group)."""
    if order == 2:
        return 0, R - 1
    y = 2
    while True:
        p = point_for_y(y)
        if p is not None:
            t = mul(p, R_J)                       # kills the prime part: t has order dividing 8
            o = next(k for k in (1, 2, 4, 8) if mul(t, k) == IDENTITY)
            if o >= order:
                return mul(t, o // order)
        y += 1


def prime_order_point(seed: int):
    """[8] P for the first curve point P with y >= seed: a point of the prime-order subgroup (or the identity)."""
    y = seed % R
    while True:
        p = point_for_y(y, seed & 1)
        if p is not None:
            q = mul(p, COFACTOR)
            if q != IDENTITY:
                return q
        y = (y + 1) % R
