#!/usr/bin/env python3
"""Generates constants.cuh: field / curve constants as 32-bit limb tables.

Every constant is derived here from its mathematical definition (moduli are the published
curve parameters; Montgomery constants and ristretto square roots are computed). The values the
reference hard-codes (sxt/field25/base/constants.h:37-56, sxt/fieldgk/base/constants.h:16-35,
sxt/field12/base/constants.h:33-69, sxt/field51/constant/{d,sqrtm1,invsqrtamd}.h) are the same
numbers in 64-bit / radix-2^51 limbs; tests/test_constants.py checks the ones that have a sign
choice against RFC 9496's decimal values.

Limb tables are emitted as `switch` functions so that, after loop unrolling, every use folds to an
immediate operand (no constant-bank or register traffic).
"""
import math
import os

P25519 = 2**255 - 19
BN254_Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
BN254_R = 21888242871839275222246405745257275088548364400416034343698204186575808495617
BLS_Q = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab


def limbs(v, n):
    return [(v >> (32 * i)) & 0xFFFFFFFF for i in range(n)]


def table(name, v, n):
    ls = limbs(v, n)
    out = [f"__host__ __device__ __forceinline__ constexpr u32 {name}(int i) {{", "  switch (i) {"]
    for i, l in enumerate(ls):
        out.append(f"  case {i}: return 0x{l:08x}u;")
    out += ["  default: return 0u;", "  }", "}"]
    return "\n".join(out)


def sqrt25519(x):
    p = P25519
    sqrtm1 = pow(2, (p - 1) // 4, p)
    r = pow(x, (p + 3) // 8, p)
    if (r * r - x) % p:
        r = r * sqrtm1 % p
    assert (r * r - x) % p == 0
    return r


def sqrt_mod(n, p):
    """Tonelli-Shanks; returns the smaller of the two roots."""
    assert pow(n, (p - 1) // 2, p) == 1
    q, s = p - 1, 0
    while q % 2 == 0:
        q //= 2
        s += 1
    z = 2
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    m, c, t, r = s, pow(z, q, p), pow(n, q, p), pow(n, (q + 1) // 2, p)
    while t != 1:
        i, t2 = 0, t
        while t2 != 1:
            t2 = t2 * t2 % p
            i += 1
        b = pow(c, 1 << (m - i - 1), p)
        m, c = i, b * b % p
        t, r = t * c % p, r * b % p
    return min(r, p - r)


# subgroup generators the reference multiplies its benchmark / test points from
# (sxt/curve_g1/constant/generator.h:34-66, curve_bng1/constant/generator.h:34-60,
#  curve_gk/constant/generator.h:34-60): bls12-381 the standard G1 generator, bn254 (1, 2),
# grumpkin (1, sqrt(-16)) with the smaller root
BLS_GX = 3685416753713387016781088315183077757961620795782546409894578378688607592378376318836054947676345821548104185464507
BLS_GY = 1339506544944476473020471379941921221584933875938349620426543736416511423956333506472724655353366534992391756441569
# the G2 generator of bls12-381 (IETF BLS signatures / zcash), coordinates c0 + c1 u in Fp2 = Fp[u]/(u^2 + 1)
BLS2_GX = (0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
           0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e)
BLS2_GY = (0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
           0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be)
# the G2 generator of bn254 (EIP-197, which lists the u coefficient first), as c0 + c1 u; its twist is
# y^2 = x^3 + 3 / (9 + u)
BN2_GX = (10857046999023057135944570762232829481370756359578518086990519993285655852781,
          11559732032986387107991004021392285783925812861821192530917403151452391805634)
BN2_GY = (8495653923123431417604973247489272438418190587263600148770280649306958101930,
          4082367875863433681332203403145435568316851327593401208105741076214120093531)
BN2_B = (27 * pow(82, -1, BN254_Q) % BN254_Q, -3 * pow(82, -1, BN254_Q) % BN254_Q)  # 3 (9 - u) / 82


def mont_block(prefix, p, n, b, gx, gy):
    R = 1 << (32 * n)
    assert (gy * gy - gx ** 3 - b) % p == 0
    out = [f"// ---- {prefix}: p = 0x{p:x}, R = 2^{32 * n}, curve y^2 = x^3 + ({b})"]
    out.append(table(f"{prefix}_P", p, n))
    out.append(table(f"{prefix}_ONE", R % p, n))          # 1 in Montgomery form
    out.append(table(f"{prefix}_R2", R * R % p, n))        # to-Montgomery multiplier
    out.append(table(f"{prefix}_B3", (3 * b % p) * R % p, n))  # 3b in Montgomery form
    out.append(table(f"{prefix}_B", (b % p) * R % p, n))
    inv = (-pow(p, -1, 1 << 32)) % (1 << 32)
    out.append(f"constexpr u32 {prefix}_INV = 0x{inv:08x}u;  // -p^-1 mod 2^32")
    out.append(table(f"{prefix}_PM2", p - 2, n))           # inversion exponent
    out.append(table(f"{prefix}_HALF", (p - 1) // 2, n))   # lexicographic-largest threshold
    out.append(table(f"{prefix}_GX", gx * R % p, n))        # subgroup generator, Montgomery form
    out.append(table(f"{prefix}_GY", gy * R % p, n))
    return "\n".join(out)


def fp2_block(prefix, p, n, b, gx, gy, b3=False):
    """The generator of a curve y^2 = x^3 + b over Fp2 = Fp[u]/(u^2 + 1), b and the coordinates as
    (c0, c1): 2n limbs per coordinate, the Montgomery c0 (R = 2^(32 n)) then c1; with b3, also 3b
    (for twists where multiplying by 3b takes an Fp2 product rather than additions)."""
    def mul(x, y):
        return ((x[0] * y[0] - x[1] * y[1]) % p, (x[0] * y[1] + x[1] * y[0]) % p)
    x3 = mul(mul(gx, gx), gx)
    assert mul(gy, gy) == ((x3[0] + b[0]) % p, (x3[1] + b[1]) % p)
    R = 1 << (32 * n)

    def mont(v):
        return v[0] * R % p + (v[1] * R % p << (32 * n))
    out = [f"// ---- {prefix}: generator of y^2 = x^3 + ({b[0]} + {b[1]} u) over Fp2, p = 0x{p:x}",
           table(f"{prefix}_GX", mont(gx), 2 * n), table(f"{prefix}_GY", mont(gy), 2 * n)]
    if b3:
        out.append(table(f"{prefix}_B3", mont((3 * b[0] % p, 3 * b[1] % p)), 2 * n))
    return "\n".join(out)


BLS_R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
# the curve parameters x of the two pairing-friendly families (bls12-381: x < 0; bn254: x > 0)
BLS_X = -0xd201000000010000
BN_X = 0x44e992b44a6909f1


def tower_block(prefix, p, r, n, xi0, x):
    """Constants of the pairing tower Fp6 = Fp2[v] / (v^3 - xi), Fp12 = Fp6[w] / (w^2 - v) over
    Fp2 = Fp[u] / (u^2 + 1), xi = xi0 + u (pairing.cuh): the Frobenius coefficients
    gamma_{k,i} = xi^(i (p^k - 1) / 6) of w^i (k = 1..3, i = 1..5, flattened as ((k-1) 5 + i-1) 2n
    limbs, Montgomery c0 then c1), 1/2, the Miller loop count, |x|, the hard part of the final
    exponentiation and, for bn254, the twist Frobenius constants of pi(Q)."""
    def mul(a, b):
        return ((a[0] * b[0] - a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)

    def pw(a, e):
        acc = (1, 0)
        for bit in bin(e)[2:]:
            acc = mul(acc, acc)
            if bit == "1":
                acc = mul(acc, a)
        return acc
    R = 1 << (32 * n)

    def mont(v):
        return v[0] * R % p + (v[1] * R % p << (32 * n))
    xi = (xi0, 1)
    assert p % 4 == 3 and (p - 1) % 6 == 0
    # the tower is a field: xi is neither a square nor a cube in Fp2
    assert pw(xi, (p * p - 1) // 2) != (1, 0) and pw(xi, (p * p - 1) // 3) != (1, 0)
    flat = 0
    for k in (1, 2, 3):
        for i in range(1, 6):
            g = pw(xi, i * (p ** k - 1) // 6)
            if k == 2:  # the p^2 coefficients lie in Fp and are sixth roots of unity
                assert g[1] == 0 and pw(g, 6) == (1, 0)
            flat |= mont(g) << (64 * n * ((k - 1) * 5 + i - 1))
    loop = abs(x) if x < 0 else 6 * x + 2  # bls12-381: the ate loop |x|; bn254: the optimal ate 6x + 2
    hard = (p ** 4 - p ** 2 + 1) // r
    assert (p ** 4 - p ** 2 + 1) % r == 0
    if x < 0:  # bls12-381: lambda_3 = (x - 1)^2 / 3, lambda_2 = lambda_3 x, lambda_1 = lambda_2 x - lambda_3,
        assert (x - 1) ** 2 % 3 == 0  # lambda_0 = lambda_1 x + 1
        l3 = (x - 1) ** 2 // 3
        l2 = l3 * x
        l1 = l2 * x - l3
        l0 = l1 * x + 1
    else:  # bn254 (Devegili-Scott-Dahab)
        l3, l2 = 1, 6 * x * x + 1
        l1 = -36 * x ** 3 - 18 * x ** 2 - 12 * x + 1
        l0 = -36 * x ** 3 - 30 * x ** 2 - 18 * x - 2
    assert l0 + l1 * p + l2 * p ** 2 + l3 * p ** 3 == hard
    out = [f"// ---- {prefix}: pairing tower over Fp2 of p = 0x{p:x}, xi = {xi0} + u, x = {x}",
           f"constexpr u32 {prefix}_XI0 = {xi0}u;  // xi = {xi0} + u",
           table(f"{prefix}_FROB", flat, 30 * n),
           table(f"{prefix}_TWO_INV", (p + 1) // 2 * R % p, n),
           f"constexpr u64 {prefix}_LOOP_LO = 0x{loop & (2**64 - 1):016x}ull;  // Miller loop count",
           f"constexpr u64 {prefix}_LOOP_HI = 0x{loop >> 64:x}ull;",
           f"constexpr int {prefix}_LOOP_BITS = {loop.bit_length()};",
           f"constexpr u64 {prefix}_X_ABS = 0x{abs(x):016x}ull;",
           f"constexpr bool {prefix}_X_NEG = {'true' if x < 0 else 'false'};",
           f"constexpr u64 {prefix}_LAMBDA3_LO = 0x{l3 & (2**64 - 1):016x}ull;  // hard part, lambda_3",
           f"constexpr u64 {prefix}_LAMBDA3_HI = 0x{l3 >> 64:016x}ull;"]
    if x > 0:  # pi(x', y') = (conj(x') xi^((p-1)/3), conj(y') xi^((p-1)/2)) on the D-type twist
        out.append(table(f"{prefix}_TWIST_FROB_X", mont(pw(xi, (p - 1) // 3)), 2 * n))
        out.append(table(f"{prefix}_TWIST_FROB_Y", mont(pw(xi, (p - 1) // 2)), 2 * n))
    return "\n".join(out)


def fp2_ops(p):
    """(mul, inv, pow) of Fp2 = Fp[u] / (u^2 + 1) on pairs (c0, c1); an Fp element is (c, 0)."""
    def mul(a, b):
        return ((a[0] * b[0] - a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)

    def inv(a):
        n = pow((a[0] * a[0] + a[1] * a[1]) % p, p - 2, p)
        return (a[0] * n % p, -a[1] * n % p)

    def pw(a, e):
        acc = (1, 0)
        for bit in bin(e)[2:]:
            acc = mul(acc, acc)
            if bit == "1":
                acc = mul(acc, a)
        return acc
    return mul, inv, pw


def ec_mul(p, k, pt):
    """[k] pt on y^2 = x^3 + b over Fp2 (affine, None = identity, k of either sign)."""
    mul, inv, _ = fp2_ops(p)

    def sub(a, b):
        return ((a[0] - b[0]) % p, (a[1] - b[1]) % p)

    def add(a, b):
        if a is None or b is None:
            return b if a is None else a
        if a[0] == b[0]:
            if sub((0, 0), a[1]) == b[1]:
                return None
            x2 = mul(a[0], a[0])
            lam = mul((3 * x2[0] % p, 3 * x2[1] % p), inv((2 * a[1][0] % p, 2 * a[1][1] % p)))
        else:
            lam = mul(sub(b[1], a[1]), inv(sub(b[0], a[0])))
        x3 = sub(sub(mul(lam, lam), a[0]), b[0])
        return (x3, sub(mul(lam, sub(a[0], x3)), a[1]))
    acc = None
    for bit in bin(abs(k))[2:]:
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, pt)
    return acc if k >= 0 or acc is None else (acc[0], sub((0, 0), acc[1]))


def sextic_twist_order(p, t, r):
    """#E'(Fp2) of the sextic twist whose order r divides, for a curve over Fp of trace t."""
    t2 = t * t - 2 * p  # the trace over Fp2
    f2 = (4 * p * p - t2 * t2) // 3
    f = math.isqrt(f2)
    assert f * f == f2
    orders = [p * p + 1 - s for s in ((t2 + 3 * f) // 2, (t2 - 3 * f) // 2, (-t2 + 3 * f) // 2,
                                      (-t2 - 3 * f) // 2)]
    hits = [n for n in orders if n % r == 0]
    assert len(hits) == 1
    return hits[0]


def points_block():
    """Constants of the point checks and decoding (points.cuh): the square-root exponents of the
    bls12-381 Fp ((p + 1) / 4) and Fp2 ((p - 3) / 4), b' = 4 (1 + u) of its G2 for decompression, and
    the endomorphisms of the subgroup checks. Each eigenvalue relation is asserted on the generator,
    and every group order h r is asserted odd: the complete RCB16 formulas the checks multiply with
    then never meet a point of order 2."""
    p, r, x = BLS_Q, BLS_R, BLS_X
    mul, inv, pw = fp2_ops(p)
    assert p % 4 == 3
    g1 = ((BLS_GX, 0), (BLS_GY, 0))
    # bls12-381 G1 (Scott 2021): phi(x, y) = (beta x, y) = [-x^2] P on the order-r subgroup
    beta = pow(2, (p - 1) // 3, p)
    assert beta != 1 and pow(beta, 3, p) == 1
    minus_x2 = ec_mul(p, -x * x, g1)
    assert (mul((beta, 0), g1[0]), g1[1]) == minus_x2
    assert (mul((beta * beta % p, 0), g1[0]), g1[1]) != minus_x2
    n1 = p + 1 - (x + 1)
    assert n1 % r == 0 and n1 % 2 == 1
    # bls12-381 G2 (M-type twist): psi(x, y) = (conj(x) cx, conj(y) cy) = [x] Q
    cx = inv(pw((1, 1), (p - 1) // 3))
    cy = inv(pw((1, 1), (p - 1) // 2))
    g2 = (BLS2_GX, BLS2_GY)

    def psi(pt, gx, gy):
        return (mul((pt[0][0], -pt[0][1] % p), gx), mul((pt[1][0], -pt[1][1] % p), gy))
    assert psi(g2, cx, cy) == ec_mul(p, x, g2)
    n2 = sextic_twist_order(p, x + 1, r)
    assert n2 % 2 == 1
    # bn254 G2 (D-type twist): psi = pi of the Miller loop, xi^((p-1)/3), xi^((p-1)/2), = [6 x^2] Q
    q = BN254_Q
    bmul, _, bpw = fp2_ops(q)
    bx, by = bpw((9, 1), (q - 1) // 3), bpw((9, 1), (q - 1) // 2)
    bg2 = (BN2_GX, BN2_GY)
    assert (bmul((bg2[0][0], -bg2[0][1] % q), bx), bmul((bg2[1][0], -bg2[1][1] % q), by)) == \
        ec_mul(q, 6 * BN_X * BN_X, bg2)
    n5 = sextic_twist_order(q, 6 * BN_X * BN_X + 1, BN254_R)
    assert n5 % 2 == 1 and n5 == (2 * q - BN254_R) * BN254_R
    R = 1 << 384

    def mont2(v):
        return v[0] * R % p + (v[1] * R % p << 384)
    return "\n".join([
        "// ---- point checks and decoding (points.cuh)",
        table("BLS_SQRT_EXP", (p + 1) // 4, 12),   # Fp square root candidate a^((p+1)/4)
        table("BLS2_SQRT_EXP", (p - 3) // 4, 12),  # Fp2 square root (Adj-Rodriguez-Henriquez alg. 9)
        table("BLS_BETA", beta * R % p, 12),        # cube root of unity of phi on G1, Montgomery
        table("BLS2_B", mont2((4, 4)), 24),         # b' = 4 (1 + u)
        table("BLS2_PSI_X", mont2(cx), 24),         # (1 + u)^(-(p-1)/3)
        table("BLS2_PSI_Y", mont2(cy), 24)])        # (1 + u)^(-(p-1)/2)


L25519 = 2**252 + 27742317777372353535851937790883648493  # order of the ristretto255 group


def scalar_block(prefix, p, n):
    """Montgomery constants of a scalar field (no curve attached)."""
    R = 1 << (32 * n)
    out = [f"// ---- {prefix}: scalar field, p = 0x{p:x}, R = 2^{32 * n}"]
    out.append(table(f"{prefix}_P", p, n))
    out.append(table(f"{prefix}_ONE", R % p, n))
    out.append(table(f"{prefix}_R2", R * R % p, n))
    inv = (-pow(p, -1, 1 << 32)) % (1 << 32)
    out.append(f"constexpr u32 {prefix}_INV = 0x{inv:08x}u;  // -p^-1 mod 2^32")
    out.append(table(f"{prefix}_PM2", p - 2, n))
    out.append(table(f"{prefix}_HALF", (p - 1) // 2, n))
    return "\n".join(out)


def main():
    p = P25519
    d = (-121665 * pow(121666, -1, p)) % p
    sqrtm1 = pow(2, (p - 1) // 4, p)
    a = p - 1
    sqrtadm1 = sqrt25519((a * d - 1) % p)
    if sqrtadm1 % 2 == 0:  # RFC 9496 SQRT_AD_MINUS_ONE is the odd root
        sqrtadm1 = p - sqrtadm1
    invsqrtamd = pow(sqrt25519((a - d) % p), -1, p)
    if invsqrtamd % 2 == 1:  # RFC 9496 INVSQRT_A_MINUS_D is the even root
        invsqrtamd = p - invsqrtamd
    parts = ["// GENERATED by gen_constants.py — do not edit.", "#pragma once", "#include <cstdint>",
             "namespace b200 {", "typedef uint32_t u32;", "typedef uint64_t u64;",
             "// ---- curve25519 base field, p = 2^255 - 19 (plain residues, 8 x 32-bit limbs)"]
    for name, v in [("F25_P", p), ("F25_D", d), ("F25_D2", 2 * d % p), ("F25_INVD", pow(d, -1, p)),
                    ("F25_SQRTM1", sqrtm1),
                    ("F25_ONEMSQD", (1 - d * d) % p), ("F25_SQDMONE", (d - 1) ** 2 % p),
                    ("F25_SQRTADM1", sqrtadm1), ("F25_INVSQRTAMD", invsqrtamd)]:
        parts.append(table(name, v, 8))
    parts.append(mont_block("BN", BN254_Q, 8, 3, 1, 2))
    parts.append(mont_block("GK", BN254_R, 8, -17, 1, sqrt_mod(-16 % BN254_R, BN254_R)))
    parts.append(mont_block("BLS", BLS_Q, 12, 4, BLS_GX, BLS_GY))
    parts.append(fp2_block("BLS2", BLS_Q, 12, (4, 4), BLS2_GX, BLS2_GY))
    parts.append(fp2_block("BN2", BN254_Q, 8, BN2_B, BN2_GX, BN2_GY, b3=True))
    parts.append(scalar_block("SC25", L25519, 8))
    parts.append(tower_block("BLS12", BLS_Q, BLS_R, 12, 1, BLS_X))
    parts.append(tower_block("BN12", BN254_Q, BN254_R, 8, 9, BN_X))
    parts.append(points_block())
    parts.append("}  // namespace b200")
    here = os.path.dirname(os.path.abspath(__file__))
    path, text = os.path.join(here, "constants.cuh"), "\n".join(parts) + "\n"
    if not os.path.exists(path) or open(path).read() != text:  # keep the mtime: incremental builds
        with open(path, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
