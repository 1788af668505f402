"""BIGN and DBIGN without a GPU: the host build of the device code (tests/hostsim/bign.cpp: belt.cuh, bash.cuh and the
BIGN cores of ec.cuh) against the standard's test vectors, the reference's belt_encrypt / BELT-HASH / BASH, its BIGN and
DBIGN signer and its ec_verify (oracle/_ref/libecc_ref_bign.so, built by oracle/ref_bign.mk)."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, ROOT, golden, random_scalars, rng, _buf

from libecc_b200 import bign_adata

HASH_IDS = {"SHA224": 1, "SHA256": 2, "SHA384": 3, "SHA512": 4, "SHA3_224": 5, "SHA3_256": 6, "SHA3_384": 7,
            "SHA3_512": 8, "SM3": 11, "BELT_HASH": 16, "BASH224": 17, "BASH256": 18, "BASH384": 19, "BASH512": 20}
DIGEST = {"SHA224": 28, "SHA256": 32, "SHA384": 48, "SHA512": 64, "SHA3_224": 28, "SHA3_256": 32, "SHA3_384": 48,
          "SHA3_512": 64, "SM3": 32, "BELT_HASH": 32, "BASH224": 28, "BASH256": 32, "BASH384": 48, "BASH512": 64}
RATE = {"BELT_HASH": 32, "BASH224": 136, "BASH256": 128, "BASH384": 96, "BASH512": 64}
COMB_W = 6  # comb window of the host build (small: the table is built on the CPU)
OID_SHA256 = bytes.fromhex("608648016503040201")  # DER content of 2.16.840.1.101.3.4.2.1

HOSTSIM_SRC = os.path.join(ROOT, "tests", "hostsim", "bign.cpp")
HOSTSIM_SO = os.path.join(ROOT, "tests", "hostsim", "_build", "libecc_hostsim_bign.so")
REF_BIGN_SO = os.path.join(ROOT, "oracle", "_ref", "libecc_ref_bign.so")
_libs = {}


def hostsim_lib() -> ctypes.CDLL:
    """the host build of the BIGN code, built on demand like test_decdsa_host.hostsim_lib"""
    if "hostsim" not in _libs:
        deps = [HOSTSIM_SRC, os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")] + [
            os.path.join(ROOT, "libecc_b200", "csrc", f) for f in
            ("fp.cuh", "ec.cuh", "msm_core.cuh", "curve_constants.inc", "sha2.cuh", "sha2_constants.inc", "sha3.cuh",
             "sha3_constants.inc", "sm3.cuh", "hmac.cuh", "belt.cuh", "bash.cuh", "bash_constants.inc")]
        if not os.path.exists(HOSTSIM_SO) or os.path.getmtime(HOSTSIM_SO) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(HOSTSIM_SO), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", HOSTSIM_SRC, "-o", HOSTSIM_SO],
                           check=True, capture_output=True)
        lib = ctypes.CDLL(HOSTSIM_SO)
        vp, u32, u64, ci = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int
        lib.hostsim_belt_encrypt.argtypes = [u32, vp, vp, vp]
        lib.hostsim_bign_hash.argtypes = [ci, vp, u64, vp]
        lib.hostsim_belt_sbox.argtypes = [vp]
        lib.hostsim_bign_det_nonce.argtypes = [vp, ci, vp, vp, ci, vp]
        lib.hostsim_bign_theta.argtypes = [vp, u32, vp, u32, vp, u32, vp]
        lib.hostsim_bign_sign.argtypes = [ci, ci, ci, ci, u32, vp, vp, vp, vp, vp, vp, vp, vp]
        lib.hostsim_bign_verify.argtypes = [ci, ci, ci, u32, vp, vp, vp, vp, vp, vp, vp]
        _libs["hostsim"] = lib
    return _libs["hostsim"]


def ref_bign():
    """oracle/_ref/libecc_ref_bign.so (the reference's BIGN code), or None where it was not built"""
    if "ref" not in _libs:
        lib = None
        if os.path.exists(REF_BIGN_SO):
            lib = ctypes.CDLL(REF_BIGN_SO)
            vp, u32, ci, cp = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_char_p
            lib.ref_bign_sign.argtypes = [cp, ci, cp, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, ci]
            lib.ref_bign_verify.argtypes = [cp, cp, u32, vp, vp, vp, vp, vp, vp, vp, ci]
            lib.ref_belt_encrypt.argtypes = [u32, vp, vp, vp]
            lib.ref_bign_hash.argtypes = [cp, vp, u32, vp]
        _libs["ref"] = lib
    return _libs["ref"]


def need_ref():
    lib = ref_bign()
    if lib is None:
        pytest.skip("the reference's BIGN wrapper (oracle/_ref/libecc_ref_bign.so) is not built here")
    return lib


def pack(items):
    blob = np.frombuffer(b"".join(items) + b"\0", dtype=np.uint8).copy()
    off = np.zeros(len(items) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in items])
    return blob, off


def host_hash(name, msg):
    out = np.zeros(64, np.uint8)
    m = np.frombuffer(msg + b"\0", np.uint8)
    assert hostsim_lib().hostsim_bign_hash(HASH_IDS[name], _buf(m), len(msg), _buf(out)) == DIGEST[name]
    return out[:DIGEST[name]].tobytes()


def ref_hash(name, msg):
    out = np.zeros(64, np.uint8)
    m = np.frombuffer(msg + b"\0", np.uint8)
    assert need_ref().ref_bign_hash(name.encode(), _buf(m), len(msg), _buf(out)) == DIGEST[name]
    return out[:DIGEST[name]].tobytes()


def host_sign(curve, alg, hash_name, priv, msgs, adata, nonces=None):
    cid, _, qlen = ALL_CURVES[curve]
    n = len(msgs)
    blob, off = pack(msgs)
    ab, aoff = pack(adata)
    sigs = np.zeros((n, qlen // 2 + qlen), np.uint8)
    st = np.zeros(n, np.int8)
    k = np.ascontiguousarray(nonces) if nonces is not None else None
    assert hostsim_lib().hostsim_bign_sign(cid, COMB_W, 18 if alg == "BIGN" else 19, HASH_IDS[hash_name], n,
                                           _buf(priv), _buf(k) if k is not None else None, _buf(blob), _buf(off),
                                           _buf(ab), _buf(aoff), _buf(sigs), _buf(st)) == 0
    return sigs, st


def ref_sign(curve, alg, hash_name, priv, msgs, adata, nonces=None):
    _, plen, qlen = ALL_CURVES[curve]
    n = len(msgs)
    blob, off = pack(msgs)
    ab, aoff = pack(adata)
    sigs = np.zeros((n, qlen // 2 + qlen), np.uint8)
    pubs = np.zeros((n, 2 * plen), np.uint8)
    st = np.zeros(n, np.int8)
    k = np.ascontiguousarray(nonces) if nonces is not None else None
    assert need_ref().ref_bign_sign(curve.encode(), 1 if alg == "DBIGN" else 0, hash_name.encode(), n,
                                    _buf(np.ascontiguousarray(priv)), _buf(k) if k is not None else None, _buf(blob),
                                    _buf(off), _buf(ab), _buf(aoff), _buf(sigs), _buf(pubs), _buf(st), 8) == 0
    return sigs, pubs, st


def host_verify(curve, hash_name, sigs, pubs, msgs, adata):
    cid = ALL_CURVES[curve][0]
    n = len(msgs)
    blob, off = pack(msgs)
    ab, aoff = pack(adata)
    v = np.zeros(n, np.int8)
    assert hostsim_lib().hostsim_bign_verify(cid, COMB_W, HASH_IDS[hash_name], n, _buf(np.ascontiguousarray(sigs)),
                                             _buf(np.ascontiguousarray(pubs)), _buf(blob), _buf(off), _buf(ab),
                                             _buf(aoff), _buf(v)) == 0
    return v


def ref_verify(curve, hash_name, sigs, pubs, msgs, adata):
    n = len(msgs)
    blob, off = pack(msgs)
    ab, aoff = pack(adata)
    v = np.zeros(n, np.int8)
    assert need_ref().ref_bign_verify(curve.encode(), hash_name.encode(), n, _buf(np.ascontiguousarray(sigs)),
                                      _buf(np.ascontiguousarray(pubs)), _buf(blob), _buf(off), _buf(ab), _buf(aoff),
                                      _buf(v), 8) == 0
    return v


def be(v, nbytes):
    return np.frombuffer(int(v).to_bytes(nbytes, "big"), np.uint8)


# ------------------------------------------------------------------------------ BELT, BELT-HASH and BASH


def test_standard_vectors():
    key = bytes.fromhex("E9DEE72C8F0C0FA62DDB49F46F73964706075316ED247A3739CBA38303A98BF6")
    blk = bytes.fromhex("B194BAC80A08F53B366D008E584A5DE4")
    out = np.zeros(16, np.uint8)
    hostsim_lib().hostsim_belt_encrypt(1, _buf(np.frombuffer(key, np.uint8)), _buf(np.frombuffer(blk, np.uint8)),
                                       _buf(out))
    assert out.tobytes().hex().upper() == "69CCA1C93557C9E3D66BC3E0FA88FA6E"
    assert host_hash("BELT_HASH", bytes.fromhex("B194BAC80A08F53B366D008E58")).hex().upper() == \
        "ABEF9725D4C5A83597A367D14494CC2542F20F659DDFECC961A3EC550CBA8C75"
    assert host_hash("BASH256", b"").hex().upper() == \
        "114C3DFAE373D9BCBC3602D6386F2D6A2059BA1BF9048DBAA5146A6CB775709D"


def test_sbox_matches_reference():
    """every entry of H: belt-block with a key of zeros reads the table through G only, so compare it cipher-wide on
    blocks that walk every byte value through every G input position, and the table bytes as BELT-HASH's IV"""
    ref = need_ref()
    sbox = np.zeros(256, np.uint8)
    hostsim_lib().hostsim_belt_sbox(_buf(sbox))
    n = 256
    keys = np.zeros((n, 32), np.uint8)
    blocks = np.repeat(np.arange(256, dtype=np.uint8)[:, None], 16, axis=1)
    for kk in (keys, rng(70).integers(0, 256, size=(n, 32), dtype=np.uint8)):
        got, want = np.zeros((n, 16), np.uint8), np.zeros((n, 16), np.uint8)
        hostsim_lib().hostsim_belt_encrypt(n, _buf(kk), _buf(blocks), _buf(got))
        ref.ref_belt_encrypt(n, _buf(kk), _buf(blocks), _buf(want))
        assert (got == want).all()
    # the first 32 entries are BELT-HASH's initial value; the hash of the empty message depends on them only
    assert host_hash("BELT_HASH", b"") == ref_hash("BELT_HASH", b"")


def test_belt_encrypt_random_vs_reference():
    ref = need_ref()
    n = 4096
    g = rng(71)
    keys = g.integers(0, 256, size=(n, 32), dtype=np.uint8)
    blocks = g.integers(0, 256, size=(n, 16), dtype=np.uint8)
    got, want = np.zeros((n, 16), np.uint8), np.zeros((n, 16), np.uint8)
    hostsim_lib().hostsim_belt_encrypt(n, _buf(keys), _buf(blocks), _buf(got))
    ref.ref_belt_encrypt(n, _buf(keys), _buf(blocks), _buf(want))
    assert (got == want).all()


@pytest.mark.parametrize("name", sorted(RATE))
def test_belt_bash_vs_reference_at_block_edges(name):
    r = RATE[name]
    g = rng(72)
    lengths = sorted({0, 1} | {b * r + d for b in range(4) for d in (-1, 0, 1) if b * r + d >= 0} | {3 * r + 1})
    for ln in lengths:
        msg = g.integers(0, 256, size=ln, dtype=np.uint8).tobytes()
        assert host_hash(name, msg) == ref_hash(name, msg), (name, ln)


@pytest.mark.parametrize("name", ["SHA224", "SHA256", "SHA3_224", "SHA3_512"])
def test_other_hashes_through_bign_front_end(name):
    msg = b"bign front end"
    assert host_hash(name, msg) == hashlib.new(name.lower().replace("_", "-").replace("sha3-", "sha3_"),
                                               msg).digest()


def test_bash_constants_generated():
    """bash_constants.inc is what tools/gen_bash_constants.py writes, and the LFSR gives the table the reference uses
    (its first and last constants)"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen_bash", os.path.join(ROOT, "tools", "gen_bash_constants.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rc = mod.round_constants()
    assert rc[0] == 0x3BF5080AC8BA94B1 and rc[1] == 0xC1D1659C1BBD92F6 and rc[23] == 0xDE8082CD72DEBC78
    with open(os.path.join(ROOT, "libecc_b200", "csrc", "bash_constants.inc")) as f:
        text = f.read()
    for v in rc:
        assert "0x%016xull" % v in text
    assert "{ 8, 53, 14, 1 }" in text and "{ 56, 35, 2, 55 }" in text


# ------------------------------------------------------------------------------ adata and the DBIGN nonce


def test_bign_adata_layout():
    assert bign_adata(b"\x06\x01", b"xyz") == b"\x00\x02\x00\x03\x06\x01xyz"
    assert bign_adata(b"") == b"\x00\x00\x00\x00"
    with pytest.raises(ValueError):
        bign_adata(b"a" * 65532)


def py_det_nonce(q, theta, h):
    """the DBIGN nonce in Python, on host_belt for the block cipher: (k, rounds)"""
    qbits = q.bit_length()
    qlen = (qbits + 7) // 8
    n = max(2, len(h) // 16)
    r = bytearray(h) + bytes(16 * n - len(h))
    blocks = [bytes(r[16 * j:16 * j + 16]) for j in range(n)]
    i = 1
    while True:
        s = bytes(16)
        for j in range(n - 1):
            s = bytes(a ^ b for a, b in zip(s, blocks[j]))
        e = host_belt(theta, s)
        e = bytes(a ^ b for a, b in zip(e, blocks[n - 1]))
        e = bytes(a ^ b for a, b in zip(e, i.to_bytes(16, "little")))
        blocks = blocks[1:n - 1] + [e, s]
        rb = b"".join(blocks)
        if qlen < 16 * n:
            k = int.from_bytes(rb[:qlen], "little") & ((1 << qbits) - 1)
        else:
            k = int.from_bytes(rb, "little")
        if i >= 2 * n and 0 < k < q:
            return k, i
        i += 1


def host_belt(key, blk):
    out = np.zeros(16, np.uint8)
    hostsim_lib().hostsim_belt_encrypt(1, _buf(np.frombuffer(key, np.uint8)), _buf(np.frombuffer(blk, np.uint8)),
                                       _buf(out))
    return out.tobytes()


@pytest.mark.parametrize("curve", ["SECP256R1", "BRAINPOOLP256R1", "SECP521R1", "SECP224R1"])
@pytest.mark.parametrize("hlen", [28, 32, 48, 64])
def test_det_nonce_vs_python(curve, hlen):
    q = ORDER[curve]
    qlen = (q.bit_length() + 7) // 8
    g = rng(73)
    for _ in range(8):
        theta = g.integers(0, 256, size=32, dtype=np.uint8).tobytes()
        h = g.integers(0, 256, size=hlen, dtype=np.uint8).tobytes()
        k = np.zeros(qlen, np.uint8)
        rounds = hostsim_lib().hostsim_bign_det_nonce(_buf(be(q, qlen)), q.bit_length(), _buf(np.frombuffer(theta, np.uint8)),
                                                      _buf(np.frombuffer(h, np.uint8)), hlen, _buf(k))
        want, want_rounds = py_det_nonce(q, theta, h)
        assert int.from_bytes(k.tobytes(), "big") == want and rounds == want_rounds


# ------------------------------------------------------------------------------ signatures and verdicts


CURVE_HASHES = [(c, h) for c in ALL_CURVES for h in ("BELT_HASH", "SHA256", "BASH384")] + \
    [("SECP521R1", h) for h in ("SHA224", "SHA3_224", "SHA512", "BASH512", "SM3", "SHA384")] + \
    [("SECP256R1", h) for h in ("SHA224", "SHA384", "SHA512", "SHA3_224", "SHA3_256", "SHA3_384", "SHA3_512", "SM3",
                                "BASH224", "BASH256", "BASH512")]


def sign_inputs(curve, n, tag):
    q = ORDER[curve]
    qlen = ALL_CURVES[curve][2]
    g = rng(tag)
    priv = random_scalars(curve, n, tag=tag)
    for i, v in enumerate([1, 2, q - 1]):
        priv[i] = be(v, qlen)
    nonces = random_scalars(curve, n, tag=tag + 1)
    msgs = [g.integers(0, 256, size=int(g.integers(0, 300)), dtype=np.uint8).tobytes() for _ in range(n)]
    msgs[0] = b""
    oids = [b"", OID_SHA256, bytes(range(11))]
    adata = [bign_adata(oids[i % 3], g.integers(0, 256, size=int(g.integers(0, 400)), dtype=np.uint8).tobytes())
             for i in range(n)]
    adata[4] = adata[4] + b"trailing"
    return priv, nonces, msgs, adata


@pytest.mark.parametrize("curve,hash_name", CURVE_HASHES)
@pytest.mark.parametrize("alg", ["BIGN", "DBIGN"])
def test_sign_vs_reference(curve, hash_name, alg):
    need_ref()
    q = ORDER[curve]
    qlen = ALL_CURVES[curve][2]
    n = 24
    priv, nonces, msgs, adata = sign_inputs(curve, n, 80)
    # ERR items: keys 0 and q, nonces 0 and q (BIGN), malformed adata records
    priv[5] = be(0, qlen)
    priv[6] = be(q, qlen)
    nonces[7] = be(0, qlen)
    nonces[8] = be(q, qlen)
    adata[9] = b""
    adata[10] = b"\x00\x01\x00"
    adata[11] = b"\x00\x05\x00\x05abcdefghi"  # oid_len + t_len = 10 > 9
    adata[12] = bign_adata(b"\x01", b"") + b"\x00" * (0x10000 - 5)  # 65536 bytes: longer than a u16 can say
    got, gst = host_sign(curve, alg, hash_name, priv, msgs, adata, nonces if alg == "BIGN" else None)
    want, pubs, wst = ref_sign(curve, alg, hash_name, priv, msgs, adata, nonces)
    assert (gst == wst).all(), (gst, wst)
    assert (got == want).all()
    bad = [5, 6, 9, 10, 11, 12] + ([7, 8] if alg == "BIGN" else [])
    assert (gst[bad] == -1).all() and (np.delete(gst, bad) == 0).all()
    # the signatures verify, on the host build and in the reference
    ok = np.delete(np.arange(n), bad)
    sel = lambda a: [a[i] for i in ok]
    assert (host_verify(curve, hash_name, got[ok], pubs[ok], sel(msgs), sel(adata)) == 0).all()
    assert (ref_verify(curve, hash_name, got[ok], pubs[ok], sel(msgs), sel(adata)) == 0).all()


def corrupted_set(curve, hash_name, tag):
    """signed items and one-bit / range / format corruptions of them: (sigs, pubs, msgs, adata)"""
    q = ORDER[curve]
    _, plen, qlen = ALL_CURVES[curve]
    l = qlen // 2
    priv, nonces, msgs, adata = sign_inputs(curve, 16, tag)
    sigs, pubs, st = ref_sign(curve, "BIGN", hash_name, priv, msgs, adata, nonces)
    assert (st == 0).all()
    S, P, M, A = [], [], [], []

    def add(s, p, m, a):
        S.append(np.frombuffer(bytes(s), np.uint8))
        P.append(np.frombuffer(bytes(p), np.uint8))
        M.append(bytes(m))
        A.append(bytes(a))

    g = rng(tag + 5)
    for i in range(16):
        s, p, m, a = bytearray(sigs[i].tobytes()), bytearray(pubs[i].tobytes()), msgs[i], adata[i]
        add(s, p, m, a)                                                        # valid
        s0 = bytearray(s); s0[int(g.integers(0, l))] ^= 1 << int(g.integers(0, 8)); add(s0, p, m, a)
        s1 = bytearray(s); s1[l + int(g.integers(0, qlen))] ^= 1 << int(g.integers(0, 8)); add(s1, p, m, a)
        add(s, p, m + b"\x01", a)                                              # message
        pk = bytearray(p); pk[int(g.integers(0, 2 * plen))] ^= 1; add(s, pk, m, a)   # key (off the curve)
        oid_len = int.from_bytes(a[:2], "big")
        if oid_len:
            aa = bytearray(a); aa[4] ^= 0x80; add(s, p, m, aa)                 # OID
        sq = bytearray(s); sq[l:] = q.to_bytes(qlen, "little"); add(sq, p, m, a)   # s1 = q
        add(s, p, m, a[:3])                                                    # malformed adata
    if qlen == 66:                                                             # s0[32] != 0 on SECP521R1
        s = bytearray(sigs[0].tobytes()); s[32] = 1; add(s, pubs[0].tobytes(), msgs[0], adata[0])
    return np.stack(S), np.stack(P), M, A


@pytest.mark.parametrize("curve,hash_name", [("SECP256R1", "BELT_HASH"), ("SECP521R1", "SHA256"),
                                             ("BRAINPOOLP384R1", "BASH384"), ("SECP192R1", "SHA3_224")])
def test_verify_vs_reference(curve, hash_name):
    need_ref()
    sigs, pubs, msgs, adata = corrupted_set(curve, hash_name, 90)
    got = host_verify(curve, hash_name, sigs, pubs, msgs, adata)
    want = ref_verify(curve, hash_name, sigs, pubs, msgs, adata)
    assert (got == want).all()
    assert (got == 0).sum() >= 16 and (got == -1).sum() > 16


# ------------------------------------------------------------------------------ the reference's 15 known answers


def _ec_mul(k, P, a, p):
    """k*P on y^2 = x^3 + a*x + b over F_p, affine, None for infinity (plain Python: test reference only)"""
    def add(P1, P2):
        if P1 is None:
            return P2
        if P2 is None:
            return P1
        (x1, y1), (x2, y2) = P1, P2
        if x1 == x2 and (y1 + y2) % p == 0:
            return None
        lam = ((3 * x1 * x1 + a) * pow(2 * y1, -1, p) if P1 == P2 else (y2 - y1) * pow(x2 - x1, -1, p)) % p
        x3 = (lam * lam - x1 - x2) % p
        return x3, (lam * (x1 - x3) - y1) % p
    R = None
    for bit in bin(k)[2:]:
        R = add(R, R)
        if bit == "1":
            R = add(R, P)
    return R


def host_belt_hash3(a, b, c):
    """BELT-HASH(a || b || c) through the host build's three-segment source"""
    out = np.zeros(32, np.uint8)
    bufs = [np.frombuffer(x + b"\0", np.uint8) for x in (a, b, c)]
    hostsim_lib().hostsim_bign_theta(_buf(bufs[0]), len(a), _buf(bufs[1]), len(b), _buf(bufs[2]), len(c), _buf(out))
    return out.tobytes()


@pytest.mark.parametrize("kat", golden("bign_kat.json"), ids=lambda k: k["name"])
def test_known_answers(kat):
    """every BIGN / DBIGN vector of the reference (STB curves) through the host build's hashes: s0 recomputed from
    W = k*G evaluated here; s1 from k; for DBIGN, k recovered from the signature equals the host build's nonce
    derivation run with that curve's q"""
    p, a, q = (int(kat[f], 16) for f in ("p", "a", "q"))
    plen, qlen = len(kat["p"]) // 2, len(kat["q"]) // 2
    l = qlen // 2
    g = bytes.fromhex(kat["g"])
    G = (int.from_bytes(g[:plen], "big"), int.from_bytes(g[plen:], "big"))
    x = int(kat["priv"], 16)
    msg, ad, sig = (bytes.fromhex(kat[f]) for f in ("msg", "adata", "sig"))
    oid_len, t_len = int.from_bytes(ad[:2], "big"), int.from_bytes(ad[2:4], "big")
    oid, t = ad[4:4 + oid_len], ad[4 + oid_len:4 + oid_len + t_len]
    h = host_hash(kat["hash"], msg)
    hbar = int.from_bytes(h, "little") % q
    s0, s1 = sig[:l], int.from_bytes(sig[l:], "little")
    b = int.from_bytes(s0, "little") + (1 << (8 * l))
    k_sig = (s1 + hbar + b * x) % q
    if kat["alg"] == "BIGN":
        assert int(kat["nonce"], 16) == k_sig
    else:
        theta = host_belt_hash3(oid, x.to_bytes(qlen, "little")[:2 * l], t)
        k = np.zeros(qlen, np.uint8)
        assert hostsim_lib().hostsim_bign_det_nonce(_buf(be(q, qlen)), q.bit_length(),
                                                    _buf(np.frombuffer(theta, np.uint8)),
                                                    _buf(np.frombuffer(h, np.uint8)), len(h), _buf(k)) > 0
        assert int.from_bytes(k.tobytes(), "big") == k_sig
    W = _ec_mul(k_sig, G, a, p)
    assert host_belt_hash3(oid, W[0].to_bytes(plen, "little")[:2 * l], h)[:l] == s0
