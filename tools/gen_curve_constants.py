#!/usr/bin/env python3
"""Generates libecc_b200/csrc/curve_constants.inc — per-curve device constants as 32-bit little-endian words.

The inputs are the published domain parameters (p, a, b, q, Gx, Gy) of the three curves BASELINE.json names;
everything else (Montgomery constants for p and for q) is derived here with Python integers, independently of the
oracle's C derivation.  tests/test_constants.py cross-checks the generated values against the reference
(oracle/_ref: ref_curve_info, which reads the reference's src/curves/known/ec_params_*.h) and against the oracle.

Reference counterparts: fp_ctx {p, mpinv, r, r_square} (src/fp/fp.h:31-57); ec_shortw_crv {a, b, order}
(src/curves/ec_shortw.h:25-36); ec_params.ec_gen / ec_gen_order (src/curves/ec_params.h:51-87).
"""
import os

CURVES = {
    # name: (libecc ec_curve_type id (src/lib_ecc_types.h:147-), p, a, b, q, gx, gy)
    "SECP256R1": (4,
        0xffffffff00000001000000000000000000000000ffffffffffffffffffffffff,
        0xffffffff00000001000000000000000000000000fffffffffffffffffffffffc,
        0x5ac635d8aa3a93e7b3ebbd55769886bc651d06b0cc53b0f63bce3c3e27d2604b,
        0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551,
        0x6b17d1f2e12c4247f8bce6e563a440f277037d812deb33a0f4a13945d898c296,
        0x4fe342e2fe1a7f9b8ee7eb4a7c0f9e162bce33576b315ececbb6406837bf51f5),
    "FRP256V1": (1,
        0xf1fd178c0b3ad58f10126de8ce42435b3961adbcabc8ca6de8fcf353d86e9c03,
        0xf1fd178c0b3ad58f10126de8ce42435b3961adbcabc8ca6de8fcf353d86e9c00,
        0xee353fca5428a9300d4aba754a44c00fdfec0c9ae4b1a1803075ed967b7bb73f,
        0xf1fd178c0b3ad58f10126de8ce42435b53dc67e140d2bf941ffdd459c6d655e1,
        0xb6b3d4c356c139eb31183d4749d423958c27d2dcaf98b70164c97a2dd98f5cff,
        0x6142e0f7c8b204911f9271f0f3ecef8c2701c307e8e4c9e183115a1554062cfb),
    "SECP384R1": (5,
        0xfffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffeffffffff0000000000000000ffffffff,
        0xfffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffeffffffff0000000000000000fffffffc,
        0xb3312fa7e23ee7e4988e056be3f82d19181d9c6efe8141120314088f5013875ac656398d8a2ed19d2a85c8edd3ec2aef,
        0xffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973,
        0xaa87ca22be8b05378eb1c71ef320ad746e1d3b628ba79b9859f741e082542a385502f25dbf55296c3a545e3872760ab7,
        0x3617de4a96262c6f5d9e98bf9292dc29f8f41dbd289a147ce9da3113b5f0b8c00a60b1ce1d7e819d7a431d7c90ea0e5f),
    # generic-a (Brainpool) and a = 0 (secp256k1) curves: the "other short-Weierstrass curves" row (SURVEY.md §8f.4)
    "BRAINPOOLP256R1": (8,
        0xa9fb57dba1eea9bc3e660a909d838d726e3bf623d52620282013481d1f6e5377,
        0x7d5a0975fc2c3057eef67530417affe7fb8055c126dc5c6ce94a4b44f330b5d9,
        0x26dc5c6ce94a4b44f330b5d9bbd77cbf958416295cf7e1ce6bccdc18ff8c07b6,
        0xa9fb57dba1eea9bc3e660a909d838d718c397aa3b561a6f7901e0e82974856a7,
        0x8bd2aeb9cb7e57cb2c4b482ffc81b7afb9de27e1e3bd23c23a4453bd9ace3262,
        0x547ef835c3dac4fd97f8461a14611dc9c27745132ded8e545c1d54c72f046997),
    "BRAINPOOLP384R1": (12,
        0x8cb91e82a3386d280f5d6f7e50e641df152f7109ed5456b412b1da197fb71123acd3a729901d1a71874700133107ec53,
        0x7bc382c63d8c150c3c72080ace05afa0c2bea28e4fb22787139165efba91f90f8aa5814a503ad4eb04a8c7dd22ce2826,
        0x04a8c7dd22ce28268b39b55416f0447c2fb77de107dcd2a62e880ea53eeb62d57cb4390295dbc9943ab78696fa504c11,
        0x8cb91e82a3386d280f5d6f7e50e641df152f7109ed5456b31f166e6cac0425a7cf3ab6af6b7fc3103b883202e9046565,
        0x1d1c64f068cf45ffa2a63a81b7c13f6b8847a3e77ef14fe3db7fcafe0cbd10e8e826e03436d646aaef87b2e247d4af1e,
        0x8abe1d7520f9c2a45cb1eb8e95cfd55262b70b29feec5864e19c054ff99129280e4646217791811142820341263c5315),
    "SECP256K1": (19,
        0xfffffffffffffffffffffffffffffffffffffffffffffffffffffffefffffc2f,
        0x0,
        0x7,
        0xfffffffffffffffffffffffffffffffebaaedce6af48a03bbfd25e8cd0364141,
        0x79be667ef9dcbbac55a06295ce870b07029bfcdb2dce28d959f2815b16f81798,
        0x483ada7726a3c4655da4fbfc0e1108a8fd17b448a68554199c47d08ffb10d4b8),
    # 521-bit instantiation (SURVEY.md §8f.4): 9 reference limbs = 18 device words, byte lengths (66) not a multiple of 4
    "SECP521R1": (6,
        (1 << 521) - 1,
        (1 << 521) - 4,
        0x0051953eb9618e1c9a1f929a21a0b68540eea2da725b99b315f3b8b489918ef109e156193951ec7e937b1652c0bd3bb1bf073573df883d2c34f1ef451fd46b503f00,
        0x01fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffa51868783bf2f966b7fcc0148f709a5d03bb5c9b8899c47aebb6fb71e91386409,
        0x00c6858e06b70404e9cd9e3ecb662395b4429c648139053fb521f828af606b4d3dbaa14b5e77efe75928fe1dc127a2ffa8de3348b3c1856a429bf97e7e31c2e5bd66,
        0x011839296a789a3bc0045c8a5fb42c7d1bd998f54449579b446817afbd17273e662c97ee72995ef42640c550b9013fad0761353c7086a272c24088be94769fd16650),
    # more of the reference's short-Weierstrass parameter sets (src/curves/known/): SM2, the largest Brainpool prime
    # (16 words), and the two small NIST primes (224 bits: 28-byte fields in 8 words; 192 bits: 6 words)
    "SM2P256V1": (17,
        0xfffffffeffffffffffffffffffffffffffffffff00000000ffffffffffffffff,
        0xfffffffeffffffffffffffffffffffffffffffff00000000fffffffffffffffc,
        0x28e9fa9e9d9f5e344d5a9e4bcf6509a7f39789f515ab8f92ddbcbd414d940e93,
        0xfffffffeffffffffffffffffffffffff7203df6b21c6052b53bbf40939d54123,
        0x32c4ae2c1f1981195f9904466a39c9948fe30bbff2660be1715a4589334c74c7,
        0xbc3736a2f4f6779c59bdcee36b692153d0a9877cc62a474002df32e52139f0a0),
    "BRAINPOOLP512R1": (9,
        0xaadd9db8dbe9c48b3fd4e6ae33c9fc07cb308db3b3c9d20ed6639cca703308717d4d9b009bc66842aecda12ae6a380e62881ff2f2d82c68528aa6056583a48f3,
        0x7830a3318b603b89e2327145ac234cc594cbdd8d3df91610a83441caea9863bc2ded5d5aa8253aa10a2ef1c98b9ac8b57f1117a72bf2c7b9e7c1ac4d77fc94ca,
        0x3df91610a83441caea9863bc2ded5d5aa8253aa10a2ef1c98b9ac8b57f1117a72bf2c7b9e7c1ac4d77fc94cadc083e67984050b75ebae5dd2809bd638016f723,
        0xaadd9db8dbe9c48b3fd4e6ae33c9fc07cb308db3b3c9d20ed6639cca70330870553e5c414ca92619418661197fac10471db1d381085ddaddb58796829ca90069,
        0x81aee4bdd82ed9645a21322e9c4c6a9385ed9f70b5d916c1b43b62eef4d0098eff3b1f78e2d0d48d50d1687b93b97d5f7c6d5047406a5e688b352209bcb9f822,
        0x7dde385d566332ecc0eabfa9cf7822fdf209f70024a57b1aa000c55b881f8111b2dcde494a5f485e5bca4bd88a2763aed1ca2b2fa8f0540678cd1e0f3ad80892),
    "SECP224R1": (3,
        0xffffffffffffffffffffffffffffffff000000000000000000000001,
        0xfffffffffffffffffffffffffffffffefffffffffffffffffffffffe,
        0xb4050a850c04b3abf54132565044b0b7d7bfd8ba270b39432355ffb4,
        0xffffffffffffffffffffffffffff16a2e0b8f03e13dd29455c5c2a3d,
        0xb70e0cbd6bb4bf7f321390b94a03c1d356c21122343280d6115c1d21,
        0xbd376388b5f723fb4c22dfe6cd4375a05a07476444d5819985007e34),
    "SECP192R1": (2,
        0xfffffffffffffffffffffffffffffffeffffffffffffffff,
        0xfffffffffffffffffffffffffffffffefffffffffffffffc,
        0x64210519e59c80e70fa7e9ab72243049feb8deecc146b9b1,
        0xffffffffffffffffffffffff99def836146bc9b1b4d22831,
        0x188da80eb03090f67cbf20eb43a18800f4ff0afd82ff1012,
        0x07192b95ffc8da78631011ed6b24cdd573f977a11e794811),
}


def nwords(p):
    """Device words per element: two per 64-bit limb of the reference (nn wlen), so that R = 2^(32N) is the reference's."""
    return 2 * ((p.bit_length() + 63) // 64)


def words(x, n):
    return ", ".join("0x%08xu" % ((x >> (32 * i)) & 0xffffffff) for i in range(n))


def tonelli_shanks_params(p):
    """(s, Q, z) with p - 1 = Q * 2^s, Q odd, and z the smallest non-residue counting up from 0: the choices of the
    reference's fp_sqrt (src/fp/fp_sqrt.c:167-199)."""
    s, Q = 0, p - 1
    while Q % 2 == 0:
        s, Q = s + 1, Q // 2
    z = 0
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    return s, Q, z


def field_block(tag, mod, n, sqrt=False):
    R = 1 << (32 * n)
    m0 = (-pow(mod, -1, 1 << 32)) % (1 << 32)
    out = []
    out.append("struct %s {" % tag)
    out.append("    static constexpr int N = %d;" % n)
    out.append("    static constexpr int BITS = %d;" % mod.bit_length())
    out.append("    static constexpr int BYTES = %d;  /* wire length (big-endian) */" % ((mod.bit_length() + 7) // 8))
    out.append("    static constexpr uint32_t M0 = 0x%08xu;  /* -mod^-1 mod 2^32 */" % m0)
    out.append("    ECC_CONST_ARRAY(P, %d, %s);      /* modulus */" % (n, words(mod, n)))
    out.append("    ECC_CONST_ARRAY(ONE, %d, %s);    /* R mod m */" % (n, words(R % mod, n)))
    out.append("    ECC_CONST_ARRAY(RR, %d, %s);     /* R^2 mod m */" % (n, words(R * R % mod, n)))
    out.append("    ECC_CONST_ARRAY(PM2, %d, %s);    /* m - 2 (Fermat exponent) */" % (n, words(mod - 2, n)))
    if sqrt:
        # Tonelli-Shanks (Field::sqrt, fp.cuh): m - 1 = Q * 2^SQRT_S; used only where SQRT_S > 1
        s, Q, z = tonelli_shanks_params(mod)
        out.append("    static constexpr int SQRT_S = %d;  /* 2-adicity of m - 1 */" % s)
        out.append("    ECC_CONST_ARRAY(SQRT_QH, %d, %s);  /* (Q - 1) / 2, Q the odd part of m - 1 */"
                   % (n, words((Q - 1) // 2, n)))
        out.append("    ECC_CONST_ARRAY(SQRT_C, %d, %s);   /* z^Q * R mod m, z = %d the smallest non-residue */"
                   % (n, words(pow(z, Q, mod) * R % mod, n), z))
    out.append("};")
    return out


def main():
    lines = ["/* GENERATED by tools/gen_curve_constants.py — do not edit. 32-bit little-endian words. */", ""]
    for name, (cid, p, a, b, q, gx, gy) in CURVES.items():
        n = nwords(p)
        assert nwords(q) == n
        a_kind = 0 if a == p - 3 else (1 if a == 0 else 2)   # selects the doubling formula in ec.cuh
        assert (gy * gy - (gx ** 3 + a * gx + b)) % p == 0
        R = 1 << (32 * n)
        lines += field_block("Fp_%s" % name, p, n, sqrt=True)
        lines += field_block("Fq_%s" % name, q, n)
        lines.append("struct Curve_%s {" % name)
        lines.append("    typedef Fp_%s Fp;" % name)
        lines.append("    typedef Fq_%s Fq;" % name)
        lines.append("    static constexpr int ID = %d;  /* libecc ec_curve_type */" % cid)
        lines.append("    static constexpr int N = %d;" % n)
        lines.append("    static constexpr int PLEN = %d;  /* bytes of p */" % ((p.bit_length() + 7) // 8))
        lines.append("    static constexpr int QLEN = %d;  /* bytes of q */" % ((q.bit_length() + 7) // 8))
        lines.append("    static constexpr int QBITS = %d;" % q.bit_length())
        lines.append("    static constexpr int A_KIND = %d;  /* 0: a = -3, 1: a = 0, 2: generic a */" % a_kind)
        lines.append("    ECC_CONST_ARRAY(A_MONT, %d, %s);   /* a*R mod p */" % (n, words(a * R % p, n)))
        lines.append("    static const char *name() { return \"%s\"; }" % name)
        lines.append("    ECC_CONST_ARRAY(B_MONT, %d, %s);   /* b*R mod p */" % (n, words(b * R % p, n)))
        lines.append("    ECC_CONST_ARRAY(GX_MONT, %d, %s);  /* Gx*R mod p */" % (n, words(gx * R % p, n)))
        lines.append("    ECC_CONST_ARRAY(GY_MONT, %d, %s);  /* Gy*R mod p */" % (n, words(gy * R % p, n)))
        lines.append("    ECC_CONST_ARRAY(GX, %d, %s);" % (n, words(gx, n)))
        lines.append("    ECC_CONST_ARRAY(GY, %d, %s);" % (n, words(gy, n)))
        lines.append("};")
        lines.append("")
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "libecc_b200", "csrc",
                        "curve_constants.inc")
    with open(path, "w") as f:
        f.write("\n".join(lines))
    print("wrote", os.path.normpath(path))


if __name__ == "__main__":
    main()
