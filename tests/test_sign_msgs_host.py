"""ECKCDSA / ECGDSA / ECRDSA / SM2 signing of raw messages without a GPU: the host build of the device algorithm
(tests/hostsim/sign.cpp: SM3, the three-segment hash, SM2's Z, comb, scheme core) against hashlib and the reference's
hash, against the reference's signer with injected nonces (oracle/ref_sign_adata.c:
ref_sig_sign_with_randomness_adata), against the reference's own known-answer vectors (tests/golden/sign_kat.json),
and on crafted vectors that reach the restart and key-range branches."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, ROOT, golden, hx, random_scalars, ref_lib, rng, _buf

ALGS = {"ECKCDSA": 2, "ECGDSA": 6, "ECRDSA": 7, "SM2": 8}
HASH_IDS = {"SHA256": 2, "SHA384": 3, "SHA512": 4, "SHA3_224": 5, "SHA3_256": 6, "SHA3_384": 7, "SHA3_512": 8,
            "SM3": 11}
HASHLIB = {"SHA224": hashlib.sha224, "SHA256": hashlib.sha256, "SHA384": hashlib.sha384, "SHA512": hashlib.sha512,
           "SHA3_224": hashlib.sha3_224, "SHA3_256": hashlib.sha3_256, "SHA3_384": hashlib.sha3_384,
           "SHA3_512": hashlib.sha3_512, "SM3": lambda *a: hashlib.new("sm3", *a)}
COMB_W = 6  # comb window of the host build (small: the table is built on the CPU)
ID_LENS = (0, 1, 18, 200, 8191)

HOSTSIM_SRC = os.path.join(ROOT, "tests", "hostsim", "sign.cpp")
HOSTSIM_SO = os.path.join(ROOT, "tests", "hostsim", "_build", "libecc_hostsim_sign.so")
REF_SIGN_SO = os.path.join(ROOT, "oracle", "_ref", "libecc_ref_sign_adata.so")
_libs = {}


def hostsim_lib() -> ctypes.CDLL:
    """the host build of the signer (the rest of the host build, tests/hostsim/hostsim.cpp, comes with it), built on
    demand like test_schnorr_sign_host.hostsim_lib"""
    if "hostsim" not in _libs:
        deps = [HOSTSIM_SRC, os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")] + [
            os.path.join(ROOT, "libecc_b200", "csrc", f) for f in
            ("fp.cuh", "ec.cuh", "msm_core.cuh", "curve_constants.inc", "sha2.cuh", "sha2_constants.inc", "sha3.cuh",
             "sha3_constants.inc", "sm3.cuh")]
        if not os.path.exists(HOSTSIM_SO) or os.path.getmtime(HOSTSIM_SO) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(HOSTSIM_SO), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", HOSTSIM_SRC, "-o", HOSTSIM_SO],
                           check=True, capture_output=True)
        lib = ctypes.CDLL(HOSTSIM_SO)
        vp, u32, u64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64
        lib.hostsim_msg_hash_seg3.argtypes = [ctypes.c_int, vp, u32, vp, u64, vp, u64, vp]
        lib.hostsim_sm3.argtypes = [vp, u64, vp]
        _libs["hostsim"] = lib
    return _libs["hostsim"]


def ref_sign_lib():
    """oracle/_ref/libecc_ref_sign_adata.so (oracle/ref_sign_adata.mk, built by build() where the reference's sources
    lie and travelling prebuilt elsewhere), or None when it is not available"""
    if "ref" not in _libs:
        if not os.path.exists(REF_SIGN_SO) and os.path.exists("/root/reference/src/libsig.h"):
            oracle = os.path.join(ROOT, "oracle")
            subprocess.run(["make", "-C", oracle, "-j8", "ref"], check=True, capture_output=True)
            subprocess.run(["make", "-C", oracle, "-f", "ref_sign_adata.mk", "all"], check=True, capture_output=True)
        _libs["ref"] = ctypes.CDLL(REF_SIGN_SO) if os.path.exists(REF_SIGN_SO) else None
    return _libs["ref"]


def siglen(curve, alg, hash_name):
    _, plen, qlen = ALL_CURVES[curve]
    ds = HASHLIB[hash_name]().digest_size
    return min(ds, qlen) + qlen if alg == "ECKCDSA" else 2 * qlen


def pack(msgs):
    blob = np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8).copy()
    off = np.zeros(len(msgs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    return blob, off


def be(v, nbytes):
    return np.frombuffer(int(v).to_bytes(nbytes, "big"), np.uint8)


def hostsim_sign(curve, alg, hash_name, privs, nonces, msgs, pubs=None, ids=None):
    lib = hostsim_lib()
    n = len(msgs)
    blob, off = pack(msgs)
    iblob, ioff = pack(ids if ids is not None else [b""] * n)
    sigs = np.full((n, siglen(curve, alg, hash_name)), 0xAA, np.uint8)
    st = np.full(n, 7, np.int8)
    rc = lib.hostsim_sign_msgs(ALGS[alg], HASH_IDS[hash_name], ALL_CURVES[curve][0], COMB_W, n, _buf(privs),
                               _buf(pubs) if pubs is not None else None, _buf(nonces), _buf(blob), _buf(off),
                               _buf(iblob), _buf(ioff), _buf(sigs), _buf(st))
    assert rc == 0
    return sigs, st


def ref_sign(curve, alg, hash_name, privs, nonces, msgs, ids=None, nthreads=8):
    """(sigs, pubs, status) from the reference's _ec_sign with rand returning nonces[i] and item i's ID as adata; pubs
    is the scheme's public key (x^-1*G for ECKCDSA and ECGDSA)"""
    ref = ref_sign_lib()
    if ref is None:
        pytest.skip("the reference's signer (oracle/_ref/libecc_ref_sign_adata.so) is not available")
    _, plen, _ = ALL_CURVES[curve]
    n = len(msgs)
    blob, off = pack(msgs)
    iblob, ioff = pack(ids if ids is not None else [b""] * n)
    sigs = np.zeros((n, siglen(curve, alg, hash_name)), np.uint8)
    pubs = np.zeros((n, 2 * plen), np.uint8)
    st = np.zeros(n, np.int8)
    assert ref.ref_sig_sign_with_randomness_adata(
        curve.encode(), alg.encode(), hash_name.encode(), n, _buf(privs), _buf(nonces), _buf(blob), _buf(off),
        _buf(iblob), _buf(ioff), _buf(sigs), _buf(pubs), _buf(st), nthreads) == 0
    return sigs, pubs, st


def ref_verify(curve, alg, hash_name, sigs, pubs, msgs, ids=None, nthreads=8):
    ref = ref_sign_lib()
    if ref is None:
        pytest.skip("the reference's verifier (oracle/_ref/libecc_ref_sign_adata.so) is not available")
    n = len(msgs)
    blob, off = pack(msgs)
    iblob, ioff = pack(ids if ids is not None else [b""] * n)
    v = np.zeros(n, np.int8)
    assert ref.ref_sig_verify_adata_batch(curve.encode(), alg.encode(), hash_name.encode(), n, _buf(sigs), _buf(pubs),
                                          _buf(blob), _buf(off), _buf(iblob), _buf(ioff), _buf(v), nthreads) == 0
    return v


# ------------------------------------------------------------------------------------------ SM3 and the byte source


def test_sm3_against_hashlib_and_reference():
    lib = hostsim_lib()
    data = rng(300).bytes(300)
    out = ctypes.create_string_buffer(64)
    ref_out = ctypes.create_string_buffer(64)
    ref_len = ctypes.c_uint32(0)
    ref = ref_lib()
    for n in range(301):
        assert lib.hostsim_sm3(data[:n], n, out) == 32
        assert out.raw[:32] == hashlib.new("sm3", data[:n]).digest(), n
        if ref is not None:
            assert ref.ref_hash(b"SM3", data[:n], n, ref_out, ctypes.byref(ref_len)) == 0
            assert ref_len.value == 32 and ref_out.raw[:32] == out.raw[:32], n


@pytest.mark.parametrize("hash_name", list(HASH_IDS))
def test_seg3_block_edges(hash_name):
    lib = hostsim_lib()
    h = HASHLIB[hash_name]
    data = rng(301).bytes(400)
    out = ctypes.create_string_buffer(64)
    for n in (0, 1, 55, 56, 63, 64, 65, 119, 120, 127, 128, 135, 136, 143, 144, 200, 399):
        for cut in (0, 2, n // 2, n):
            if cut > n:
                continue
            a, b = data[:min(cut, 2)], data[min(cut, 2):cut]
            ds = lib.hostsim_msg_hash_seg3(HASH_IDS[hash_name], a, len(a), b, len(b), data[cut:n], n - cut, out)
            assert ds == h().digest_size
            assert out.raw[:ds] == h(data[:n]).digest(), (n, cut)


@pytest.mark.parametrize("hash_name", list(HASH_IDS))
def test_seg3_every_split(hash_name):
    """a short input split into pre || mid || post at every pair of positions"""
    lib = hostsim_lib()
    h = HASHLIB[hash_name]
    data = rng(302).bytes(21)
    want = h(data).digest()
    out = ctypes.create_string_buffer(64)
    for i in range(len(data) + 1):
        for j in range(i, len(data) + 1):
            ds = lib.hostsim_msg_hash_seg3(HASH_IDS[hash_name], data[:i], i, data[i:j], j - i, data[j:], len(data) - j,
                                           out)
            assert out.raw[:ds] == want, (i, j)


def test_unsupported_hash_is_refused():
    out = ctypes.create_string_buffer(64)
    for ht in (0, 1, 9, 10, 12):
        assert hostsim_lib().hostsim_msg_hash_seg3(ht, b"", 0, b"", 0, b"", 0, out) == -1


# ------------------------------------------------------------------------------------------ against the reference


def workload(curve, alg, n, tag):
    """random keys, nonces, messages of 0 to 300 bytes (one empty, one of several blocks) and SM2 IDs of 0, 1, 18,
    200 and 8191 bytes; then the edge inputs: x = 0, q - 1, q and k = 0, q"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    g = rng(tag)
    privs = random_scalars(curve, n, tag=tag + 1)
    nonces = random_scalars(curve, n, tag=tag + 2)
    msgs = [g.bytes(int(g.integers(0, 301))) for _ in range(n)]
    msgs[5] = b""
    msgs[6] = g.bytes(333)
    ids = [g.bytes(ID_LENS[i % len(ID_LENS)]) for i in range(n)]
    for j, v in enumerate((0, q - 1, q)):
        privs[j] = be(v, qlen)
    for j, v in enumerate((0, q)):
        nonces[3 + j] = be(v, qlen)
    return privs, nonces, msgs, ids


HASHES = ("SHA256", "SHA384", "SHA512", "SHA3_256", "SHA3_512", "SM3")
CASES = [(c, a, h) for c in ALL_CURVES for a in ALGS for h in HASHES]


@pytest.mark.parametrize("curve,alg,hash_name", CASES)
def test_hostsim_against_reference(curve, alg, hash_name):
    n = 16
    tag = 6000 + 10 * list(ALL_CURVES).index(curve) + list(ALGS).index(alg)
    privs, nonces, msgs, ids = workload(curve, alg, n, tag)
    want, pubs, wst = ref_sign(curve, alg, hash_name, privs, nonces, msgs, ids)
    got, st = hostsim_sign(curve, alg, hash_name, privs, nonces, msgs, pubs, ids)
    assert (st == wst).all(), (st, wst)
    assert (got == want).all()
    assert st[0] == -1 and st[2] == -1 and st[3] == -1 and st[4] == -1
    assert st[1] == (-1 if alg == "SM2" else 0)  # x = q - 1: outside SM2's [1, q-2]
    assert (st[5:] == 0).all()


@pytest.mark.parametrize("alg", ["ECKCDSA", "SM2"])
@pytest.mark.parametrize("curve", ["SECP256R1", "SECP521R1"])
def test_key_off_curve_is_an_error(curve, alg):
    _, plen, _ = ALL_CURVES[curve]
    privs, nonces, msgs, ids = workload(curve, alg, 10, 77)
    want, pubs, wst = ref_sign(curve, alg, "SHA256", privs, nonces, msgs, ids)
    pubs[7, plen - 1] ^= 1
    sigs, st = hostsim_sign(curve, alg, "SHA256", privs, nonces, msgs, pubs, ids)
    assert st[7] == -1 and not sigs[7].any()
    keep = np.arange(10) != 7
    assert (st[keep] == wst[keep]).all() and (sigs[keep] == want[keep]).all()


def test_eckcdsa_z_cut_to_block_size():
    """SECP521R1 with SHA-512: 2*plen = 132 > 128, so z is Y cut to the block size; with SHA3-512 (72) as well"""
    curve = "SECP521R1"
    for hash_name in ("SHA512", "SHA3_512", "SHA256"):
        privs, nonces, msgs, ids = workload(curve, "ECKCDSA", 12, 88)
        want, pubs, wst = ref_sign(curve, "ECKCDSA", hash_name, privs, nonces, msgs)
        got, st = hostsim_sign(curve, "ECKCDSA", hash_name, privs, nonces, msgs, pubs)
        assert (st == wst).all() and (got == want).all() and (st[5:] == 0).all()


def test_sm2_long_id_is_an_error():
    curve = "SM2P256V1"
    privs, nonces, msgs, ids = workload(curve, "SM2", 8, 99)
    want, pubs, wst = ref_sign(curve, "SM2", "SM3", privs, nonces, msgs, ids)
    ids[6] = bytes(8192)
    sigs, st = hostsim_sign(curve, "SM2", "SM3", privs, nonces, msgs, pubs, ids)
    assert st[6] == -1 and not sigs[6].any() and st[7] == wst[7] == 0


# ------------------------------------------------------------------------------------------ known answers


def kat_vectors():
    return golden("sign_kat.json")


def test_kat_fixture_contents():
    kats = kat_vectors()
    assert len(kats) == 13
    count = {a: sum(1 for k in kats if k["alg"] == a) for a in ALGS}
    assert count == {"ECKCDSA": 10, "ECGDSA": 2, "ECRDSA": 0, "SM2": 1}
    assert sum(1 for k in kats if k["hash"] == "SHA224") == 1
    assert any(k["alg"] == "SM2" and k["hash"] == "SM3" and k["curve"] == "SM2P256V1" for k in kats)


def py_eckcdsa_from_W(curve, hash_name, x, k, W, Y, msg):
    """ECKCDSA restated over hashlib (SHA-224, which the device does not compute), W = k*G given"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    h = HASHLIB[hash_name]
    bs = h().block_size
    ds = h().digest_size
    rlen = min(ds, qlen)
    z = (Y + bytes(bs))[:bs]
    hz = h(z + msg).digest()[ds - rlen:]
    r = h(W[:plen]).digest()[ds - rlen:]
    e = int.from_bytes(bytes(a ^ b for a, b in zip(r, hz)), "big") % q
    return r + (x * (k - e) % q).to_bytes(qlen, "big")


@pytest.mark.parametrize("kat", kat_vectors(), ids=lambda k: k["name"])
def test_kat(kat):
    curve, alg, hash_name = kat["curve"], kat["alg"], kat["hash"]
    _, plen, qlen = ALL_CURVES[curve]
    x = int(kat["priv"], 16)
    priv = be(x, qlen).copy().reshape(1, qlen)
    nonce = hx(kat["nonce"]).copy().reshape(1, qlen)
    msg = bytes.fromhex(kat["msg"])
    pub = hx(kat["pub"]).copy().reshape(1, 2 * plen)
    if hash_name in HASH_IDS:
        sigs, st = hostsim_sign(curve, alg, hash_name, priv, nonce, [msg], pub, [bytes.fromhex(kat["adata"])])
        assert st[0] == 0 and sigs[0].tobytes().hex() == kat["sig"]
        return
    assert alg == "ECKCDSA"
    W = np.zeros((1, 2 * plen), np.uint8)
    wst = np.zeros(1, np.int8)
    assert hostsim_lib().hostsim_prj_pt_mul_batch(ALL_CURVES[curve][0], COMB_W, 1, _buf(nonce), None, _buf(W),
                                                  _buf(wst)) == 0
    assert wst[0] == 0
    k = int(kat["nonce"], 16)
    assert py_eckcdsa_from_W(curve, hash_name, x, k, W[0].tobytes(), pub[0].tobytes(), msg).hex() == kat["sig"]


# ------------------------------------------------------------------------------------------ crafted vectors


def kG_x(curve, k):
    _, plen, qlen = ALL_CURVES[curve]
    W = np.zeros((1, 2 * plen), np.uint8)
    st = np.zeros(1, np.int8)
    assert hostsim_lib().hostsim_prj_pt_mul_batch(ALL_CURVES[curve][0], COMB_W, 1, _buf(be(k, qlen).copy()), None,
                                                  _buf(W), _buf(st)) == 0
    assert st[0] == 0
    return int.from_bytes(W[0, :plen].tobytes(), "big")


def ecrdsa_s_zero_vector(curve, hash_name, tag):
    """(x, k, msg) with s = r*x + k*e == 0 mod q: x = -k*e*r^-1 after r and e are known"""
    q = ORDER[curve]
    g = rng(tag)
    k = int.from_bytes(g.bytes(80), "big") % (q - 1) + 1
    msg = g.bytes(40)
    r = kG_x(curve, k) % q
    e = int.from_bytes(HASHLIB[hash_name](msg).digest()[::-1], "big") % q or 1
    x = (-k * e * pow(r, -1, q)) % q
    assert r != 0 and 0 < x < q and (r * x + k * e) % q == 0
    return x, k, msg


@pytest.mark.parametrize("hash_name", ["SHA256", "SHA3_512", "SM3"])
@pytest.mark.parametrize("curve", ["SECP256R1", "BRAINPOOLP384R1", "SECP521R1", "SECP192R1"])
def test_ecrdsa_s_zero_retries(curve, hash_name):
    _, plen, qlen = ALL_CURVES[curve]
    x, k, msg = ecrdsa_s_zero_vector(curve, hash_name, 31)
    privs = np.stack([be(x, qlen), be(x + 1, qlen)])
    nonces = np.stack([be(k, qlen), be(k, qlen)])
    msgs = [msg, msg]
    want, pubs, wst = ref_sign(curve, "ECRDSA", hash_name, privs, nonces, msgs)
    got, st = hostsim_sign(curve, "ECRDSA", hash_name, privs, nonces, msgs, pubs)
    assert list(wst) == [2, 0] and list(st) == [2, 0]
    assert (got == want).all() and not got[0].any()


@pytest.mark.parametrize("curve", ["SM2P256V1", "SECP256K1", "SECP521R1"])
def test_sm2_key_range(curve):
    """x = q - 1 is refused (sig/sm2.c:72-75), x = q - 2 signs; checked in Python integers: r and s satisfy the
    scheme's equations with e = H(Z || m)"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    g = rng(55)
    nonces = random_scalars(curve, 2, tag=56)
    privs = np.stack([be(q - 1, qlen), be(q - 2, qlen)])
    msgs = [b"message digest", g.bytes(100)]
    ids = [b"1234567812345678", b"ALICE123@YAHOO.COM"]
    want, pubs, wst = ref_sign(curve, "SM2", "SM3", privs, nonces, msgs, ids)
    got, st = hostsim_sign(curve, "SM2", "SM3", privs, nonces, msgs, pubs, ids)
    assert list(wst) == [-1, 0] and list(st) == [-1, 0]
    assert (got == want).all() and not got[0].any()
    r = int.from_bytes(got[1, :qlen].tobytes(), "big")
    s = int.from_bytes(got[1, qlen:].tobytes(), "big")
    k = int.from_bytes(nonces[1].tobytes(), "big")
    x = q - 2
    assert (s * (1 + x) - (k - r * x)) % q == 0
    assert (ref_verify(curve, "SM2", "SM3", got[1:], pubs[1:], msgs[1:], ids[1:]) == 0).all()
