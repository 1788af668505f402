"""Deterministic ECDSA (RFC 6979) and ECDSA of raw messages without a GPU: the host build of the device algorithm
(tests/hostsim/decdsa.cpp: SHA-224, HMAC, the nonce derivation and the whole signer) against hashlib / Python's hmac,
the reference's hmac, an independent RFC 6979 written here, the reference's DECDSA signer (ref_sig_sign_batch with
ec_sign and rand == NULL), its 32 known answers (tests/golden/ecdsa_kat.json) and the oracle's ECDSA digest signer."""
import ctypes
import hashlib
import hmac
import os
import subprocess

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, ROOT, golden, oracle_sign, random_scalars, ref_lib, rng, _buf

HASH_IDS = {"SHA224": 1, "SHA256": 2, "SHA384": 3, "SHA512": 4, "SHA3_224": 5, "SHA3_256": 6, "SHA3_384": 7,
            "SHA3_512": 8, "SM3": 11}


def _sm3(*a):
    return hashlib.new("sm3", *a)


HASHLIB = {"SHA224": hashlib.sha224, "SHA256": hashlib.sha256, "SHA384": hashlib.sha384, "SHA512": hashlib.sha512,
           "SHA3_224": hashlib.sha3_224, "SHA3_256": hashlib.sha3_256, "SHA3_384": hashlib.sha3_384,
           "SHA3_512": hashlib.sha3_512, "SM3": _sm3}
DIGEST = {h: f().digest_size for h, f in HASHLIB.items()}
BLOCK = {"SHA224": 64, "SHA256": 64, "SHA384": 128, "SHA512": 128, "SHA3_224": 144, "SHA3_256": 136,
         "SHA3_384": 104, "SHA3_512": 72, "SM3": 64}
COMB_W = 6  # comb window of the host build (small: the table is built on the CPU)

HOSTSIM_SRC = os.path.join(ROOT, "tests", "hostsim", "decdsa.cpp")
HOSTSIM_SO = os.path.join(ROOT, "tests", "hostsim", "_build", "libecc_hostsim_decdsa.so")
_libs = {}


def hostsim_lib() -> ctypes.CDLL:
    """the host build of the signer, built on demand like test_sign_msgs_host.hostsim_lib"""
    if "hostsim" not in _libs:
        deps = [HOSTSIM_SRC, os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")] + [
            os.path.join(ROOT, "libecc_b200", "csrc", f) for f in
            ("fp.cuh", "ec.cuh", "msm_core.cuh", "curve_constants.inc", "sha2.cuh", "sha2_constants.inc", "sha3.cuh",
             "sha3_constants.inc", "sm3.cuh", "hmac.cuh")]
        if not os.path.exists(HOSTSIM_SO) or os.path.getmtime(HOSTSIM_SO) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(HOSTSIM_SO), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", HOSTSIM_SRC, "-o", HOSTSIM_SO],
                           check=True, capture_output=True)
        lib = ctypes.CDLL(HOSTSIM_SO)
        vp, u32, u64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64
        lib.hostsim_decdsa_hash.argtypes = [ctypes.c_int, vp, u64, vp]
        lib.hostsim_hmac.argtypes = [ctypes.c_int, vp, u32, vp, u64, vp]
        lib.hostsim_rfc6979_nonce.argtypes = [ctypes.c_int, ctypes.c_int, u32, vp, vp, vp, vp]
        lib.hostsim_ecdsa_det_sign.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, u32, vp, vp, vp,
                                               vp, vp, vp, vp]
        _libs["hostsim"] = lib
    return _libs["hostsim"]


def pack(msgs):
    blob = np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8).copy()
    off = np.zeros(len(msgs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    return blob, off


def be(v, nbytes):
    return np.frombuffer(int(v).to_bytes(nbytes, "big"), np.uint8)


# ------------------------------------------------------------------------------------------ RFC 6979 in Python


def py_rfc6979(curve, hash_name, x, h):
    """(k, retries): RFC 6979 §3.2 on Python's hmac, with the reference's acceptance of k (k < q only)"""
    q = ORDER[curve]
    qbits = q.bit_length()
    qlen = (qbits + 7) // 8
    hf = HASHLIB[hash_name]
    hs = hf().digest_size
    mac = lambda key, m: hmac.new(key, m, hf).digest()

    def bits2int(b):
        v = int.from_bytes(b, "big")
        return v >> (8 * len(b) - qbits) if 8 * len(b) > qbits else v

    xo = x.to_bytes(qlen, "big")
    ho = (bits2int(h) % q).to_bytes(qlen, "big")
    V, K = b"\x01" * hs, b"\x00" * hs
    K = mac(K, V + b"\x00" + xo + ho)
    V = mac(K, V)
    K = mac(K, V + b"\x01" + xo + ho)
    V = mac(K, V)
    retries = 0
    while True:
        T = b""
        while len(T) < qlen:
            V = mac(K, V)
            T += V
        k = bits2int(T[:qlen])
        if k < q:
            return k, retries
        K = mac(K, V + b"\x00")
        V = mac(K, V)
        retries += 1


def have_sm3():
    try:
        hashlib.new("sm3")
        return True
    except ValueError:
        return False


PY_HASHES = [h for h in HASH_IDS if h != "SM3" or have_sm3()]


# ------------------------------------------------------------------------------------------ SHA-224 and HMAC


def test_sha224_block_edges():
    lib = hostsim_lib()
    data = rng(700).bytes(300)
    out = ctypes.create_string_buffer(64)
    for n in list(range(0, 130)) + [183, 184, 191, 192, 193, 255, 256, 299]:
        assert lib.hostsim_decdsa_hash(1, data[:n], n, out) == 28
        assert out.raw[:28] == hashlib.sha224(data[:n]).digest(), n


def test_unsupported_hash_is_refused():
    out = ctypes.create_string_buffer(64)
    for ht in (0, 9, 10, 12, -1):
        assert hostsim_lib().hostsim_decdsa_hash(ht, b"", 0, out) == -1
        assert hostsim_lib().hostsim_hmac(ht, b"k", 1, b"", 0, out) == -1


def hmac_lengths(hash_name):
    bs, ds = BLOCK[hash_name], DIGEST[hash_name]
    keys = sorted({0, 1, ds - 1, ds, ds + 1, bs - 1, bs, bs + 1, 2 * bs + 3})
    msgs = sorted({0, 1, 55, 56, 63, 64, 65, max(0, bs - ds - 9), bs - 1, bs, bs + 1, 2 * bs - 1, 200})
    return keys, msgs


@pytest.mark.parametrize("hash_name", PY_HASHES)
def test_hmac_against_python(hash_name):
    lib = hostsim_lib()
    g = rng(701)
    key, data = g.bytes(400), g.bytes(400)
    out = ctypes.create_string_buffer(64)
    keys, msgs = hmac_lengths(hash_name)
    for kl in keys:
        for ml in msgs:
            ds = lib.hostsim_hmac(HASH_IDS[hash_name], key[:kl], kl, data[:ml], ml, out)
            assert ds == DIGEST[hash_name]
            assert out.raw[:ds] == hmac.new(key[:kl], data[:ml], HASHLIB[hash_name]).digest(), (kl, ml)


@pytest.mark.parametrize("hash_name", list(HASH_IDS))
def test_hmac_against_reference(hash_name):
    """the reference's hmac (hash/hmac.c) for all nine hashes, SM3 included"""
    ref = ref_lib()
    if ref is None:
        pytest.skip("the compiled reference (oracle/_ref/libecc_ref.so) is not available")
    lib = hostsim_lib()
    g = rng(702)
    key, data = g.bytes(400), g.bytes(400)
    out = ctypes.create_string_buffer(64)
    ref_out = ctypes.create_string_buffer(64)
    keys, msgs = hmac_lengths(hash_name)
    for kl in keys:
        for ml in msgs:
            ds = lib.hostsim_hmac(HASH_IDS[hash_name], key[:kl], kl, data[:ml], ml, out)
            olen = ctypes.c_uint8(64)
            assert ref.hmac(key[:kl], ctypes.c_uint32(kl), ctypes.c_int(HASH_IDS[hash_name]), data[:ml],
                            ctypes.c_uint32(ml), ref_out, ctypes.byref(olen)) == 0
            assert olen.value == ds and out.raw[:ds] == ref_out.raw[:ds], (kl, ml)


# ------------------------------------------------------------------------------------------ the nonce


def hostsim_nonce(curve, hash_name, privs, digests):
    _, _, qlen = ALL_CURVES[curve]
    n = len(privs)
    k = np.zeros((n, qlen), np.uint8)
    retries = np.zeros(n, np.int32)
    assert hostsim_lib().hostsim_rfc6979_nonce(ALL_CURVES[curve][0], HASH_IDS[hash_name], n, _buf(privs),
                                               _buf(np.ascontiguousarray(digests)), _buf(k), _buf(retries)) == 0
    return k, retries


def nonce_workload(curve, hash_name, n, tag):
    _, _, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    ds = DIGEST[hash_name]
    privs = random_scalars(curve, n, tag=tag)
    digests = rng(tag + 1).integers(0, 256, size=(n, ds), dtype=np.uint8)
    digests[0] = 0xFF      # h >= q before the reduction of bits2octets
    digests[1] = 0x00
    privs[2] = be(1, qlen)
    privs[3] = be(q - 1, qlen)
    return privs, digests


NONCE_CASES = [(c, h) for c in ALL_CURVES for h in PY_HASHES]


@pytest.mark.parametrize("curve,hash_name", NONCE_CASES)
def test_nonce_against_python(curve, hash_name):
    n = 12
    q = ORDER[curve]
    privs, digests = nonce_workload(curve, hash_name, n, 7100 + NONCE_CASES.index((curve, hash_name)))
    k, retries = hostsim_nonce(curve, hash_name, privs, digests)
    for i in range(n):
        want, wr = py_rfc6979(curve, hash_name, int.from_bytes(privs[i].tobytes(), "big"), digests[i].tobytes())
        assert int.from_bytes(k[i].tobytes(), "big") == want and retries[i] == wr, i
        assert want < q


@pytest.mark.parametrize("curve,hash_name", [("BRAINPOOLP256R1", "SHA256"), ("BRAINPOOLP384R1", "SHA384"),
                                             ("BRAINPOOLP512R1", "SHA3_256"), ("FRP256V1", "SHA256")])
def test_retry_loop_is_exercised(curve, hash_name):
    """P(k >= q) per attempt: 0.34 / 0.45 / 0.33 on the brainpool curves, 0.055 on FRP256V1; the retry counts the
    Python side observes are the host build's, and on the brainpool curves many items retry, some three times"""
    n = 300
    privs, digests = nonce_workload(curve, hash_name, n, 7300)
    k, retries = hostsim_nonce(curve, hash_name, privs, digests)
    want = [py_rfc6979(curve, hash_name, int.from_bytes(privs[i].tobytes(), "big"), digests[i].tobytes())
            for i in range(n)]
    assert [int.from_bytes(k[i].tobytes(), "big") for i in range(n)] == [w[0] for w in want]
    assert list(retries) == [w[1] for w in want]
    if curve.startswith("BRAINPOOL"):
        assert (retries >= 1).sum() >= n // 5 and (retries >= 3).sum() >= 3, np.bincount(retries)
    else:
        assert (retries >= 1).sum() >= 3, np.bincount(retries)


@pytest.mark.parametrize("curve,hash_name,blocks", [("SECP521R1", "SHA224", 3), ("SECP521R1", "SHA256", 3),
                                                    ("SECP521R1", "SHA3_224", 3), ("SECP384R1", "SHA256", 2),
                                                    ("BRAINPOOLP512R1", "SHA3_256", 2), ("SECP192R1", "SHA512", 1)])
def test_multi_block_t_and_shifted_h1(curve, hash_name, blocks):
    """T takes `blocks` V blocks; SECP192R1 with SHA-512 shifts h right by 320 bits before the reduction"""
    _, _, qlen = ALL_CURVES[curve]
    assert -(-qlen // DIGEST[hash_name]) == blocks
    n = 40
    privs, digests = nonce_workload(curve, hash_name, n, 7400 + blocks)
    k, retries = hostsim_nonce(curve, hash_name, privs, digests)
    for i in range(n):
        want, wr = py_rfc6979(curve, hash_name, int.from_bytes(privs[i].tobytes(), "big"), digests[i].tobytes())
        assert int.from_bytes(k[i].tobytes(), "big") == want and retries[i] == wr, i


def test_key_out_of_range_gives_no_nonce():
    curve = "SECP256R1"
    q = ORDER[curve]
    privs, digests = nonce_workload(curve, "SHA256", 4, 7500)
    privs[0] = be(0, 32)
    privs[1] = be(q, 32)
    k, retries = hostsim_nonce(curve, "SHA256", privs, digests)
    assert not k[:2].any() and list(retries[:2]) == [-1, -1] and k[2:].any(axis=1).all()


# ------------------------------------------------------------------------------------------ signatures


def hostsim_sign(curve, sig_type, hash_name, privs, nonces=None, digests=None, msgs=None):
    _, _, qlen = ALL_CURVES[curve]
    n = len(privs)
    sigs = np.full((n, 2 * qlen), 0xAA, np.uint8)
    st = np.full(n, 7, np.int8)
    blob, off = pack(msgs) if msgs is not None else (None, None)
    rc = hostsim_lib().hostsim_ecdsa_det_sign(
        ALL_CURVES[curve][0], COMB_W, sig_type, HASH_IDS[hash_name], n, _buf(privs),
        _buf(nonces) if nonces is not None else None, _buf(np.ascontiguousarray(digests)) if digests is not None else None,
        _buf(blob) if blob is not None else None, _buf(off) if off is not None else None, _buf(sigs), _buf(st))
    assert rc == 0
    return sigs, st


def ref_decdsa(curve, hash_name, privs, msgs, nthreads=8):
    """(sigs, pubs, status) of the reference's ec_sign(…, DECDSA, hash, NULL, 0): RFC 6979 nonces"""
    ref = ref_lib()
    if ref is None:
        pytest.skip("the compiled reference (oracle/_ref/libecc_ref.so) is not available")
    _, plen, qlen = ALL_CURVES[curve]
    n = len(msgs)
    blob, off = pack(msgs)
    sigs = np.zeros((n, 2 * qlen), np.uint8)
    pubs = np.zeros((n, 2 * plen), np.uint8)
    st = np.zeros(n, np.int8)
    assert ref.ref_sig_sign_batch(curve.encode(), b"DECDSA", hash_name.encode(), n, _buf(privs), _buf(blob), _buf(off),
                                  _buf(sigs), _buf(pubs), _buf(st), nthreads) == 0
    return sigs, pubs, st


def sign_workload(curve, n, tag):
    """random keys and messages of 0 to 300 bytes; then keys 1, 2, q - 1 and the invalid 0 and q"""
    _, _, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    g = rng(tag)
    privs = random_scalars(curve, n, tag=tag + 1)
    msgs = [g.bytes(int(g.integers(0, 301))) for _ in range(n)]
    msgs[5] = b""
    for j, v in enumerate((1, 2, q - 1, 0, q)):
        privs[j] = be(v, qlen)
    return privs, msgs


SIGN_CASES = [(c, h) for c in ALL_CURVES for h in HASH_IDS]


@pytest.mark.parametrize("curve,hash_name", SIGN_CASES)
def test_decdsa_against_reference(curve, hash_name):
    """both forms of the host build against the reference's DECDSA signer; keys 0 and q are ECCB200_ERR"""
    n = 10
    privs, msgs = sign_workload(curve, n, 7600 + SIGN_CASES.index((curve, hash_name)))
    want, _, wst = ref_decdsa(curve, hash_name, privs, msgs)
    got, st = hostsim_sign(curve, 14, hash_name, privs, msgs=msgs)
    assert list(st) == [0, 0, 0, -1, -1] + [0] * (n - 5)
    assert (st == wst).all() and (got == want).all()
    digests = np.stack([np.frombuffer(HASHLIB[hash_name](m).digest(), np.uint8) for m in msgs]) \
        if hash_name in PY_HASHES else None
    if digests is not None:
        got2, st2 = hostsim_sign(curve, 14, hash_name, privs, digests=digests)
        assert (st2 == st).all() and (got2 == got).all()


def test_kat_fixture_contents():
    kats = [k for k in golden("ecdsa_kat.json") if k["alg"] == "DECDSA"]
    assert len(kats) == 32
    assert {k["hash"] for k in kats} == {"SHA224", "SHA256", "SHA384", "SHA512"}
    assert {k["curve"] for k in kats} == {"SECP192R1", "SECP256R1", "SECP384R1", "SECP521R1"}


@pytest.mark.parametrize("kat", [k for k in golden("ecdsa_kat.json") if k["alg"] == "DECDSA"], ids=lambda k: k["name"])
def test_kat(kat):
    curve, hash_name = kat["curve"], kat["hash"]
    _, _, qlen = ALL_CURVES[curve]
    priv = be(int(kat["priv"], 16), qlen).copy().reshape(1, qlen)
    msg = bytes.fromhex(kat["msg"])
    assert HASHLIB[hash_name](msg).hexdigest() == kat["digest"]
    for kw in ({"msgs": [msg]}, {"digests": np.frombuffer(bytes.fromhex(kat["digest"]), np.uint8).reshape(1, -1)}):
        sigs, st = hostsim_sign(curve, 14, hash_name, priv, **kw)
        assert st[0] == 0 and sigs[0].tobytes().hex() == kat["sig"]


@pytest.mark.parametrize("curve,hash_name", [("SECP256R1", "SHA256"), ("SECP521R1", "SHA3_512"),
                                             ("BRAINPOOLP384R1", "SHA224"), ("SECP192R1", "SHA512"),
                                             ("SM2P256V1", "SM3")])
def test_ecdsa_message_form_equals_digest_signer(curve, hash_name):
    """ECDSA of raw messages with the caller's nonces equals the oracle's ECDSA digest signer on hashlib digests"""
    if hash_name not in PY_HASHES:
        pytest.skip("hashlib has no SM3 here")
    n = 24
    privs, msgs = sign_workload(curve, n, 7700)
    privs = privs[5:]
    msgs = msgs[5:]
    nonces = random_scalars(curve, len(msgs), tag=7701)
    digests = np.stack([np.frombuffer(HASHLIB[hash_name](m).digest(), np.uint8) for m in msgs])
    want, wst = oracle_sign(curve, privs, nonces, digests, DIGEST[hash_name])
    got, st = hostsim_sign(curve, 1, hash_name, privs, nonces=nonces, msgs=msgs)
    assert (st == 0).all() and (wst == 0).all() and (got == want).all()


def test_ecdsa_kat_with_nonces():
    """the reference's ECDSA known answers (caller's nonce) through the message form"""
    ran = 0
    for kat in golden("ecdsa_kat.json"):
        if kat["alg"] != "ECDSA":
            continue
        curve, hash_name = kat["curve"], kat["hash"]
        if curve not in ALL_CURVES:
            continue
        _, _, qlen = ALL_CURVES[curve]
        priv = be(int(kat["priv"], 16) % (1 << (8 * qlen)), qlen).copy().reshape(1, qlen)
        nonce = be(int(kat["nonce"], 16), qlen).copy().reshape(1, qlen)
        sigs, st = hostsim_sign(curve, 1, hash_name, priv, nonces=nonce, msgs=[bytes.fromhex(kat["msg"])])
        assert st[0] == 0 and sigs[0].tobytes().hex() == kat["sig"], kat["name"]
        ran += 1
    assert ran >= 10
