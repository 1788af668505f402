"""Schnorr-family signing (ECSDSA, ECOSDSA, ECFSDSA, BIP0340) without a GPU: the host build of the device algorithm
(tests/hostsim/schnorr_sign.cpp: segmented hash, BIP0340 nonce, comb, scheme core) against hashlib, against the
reference's signer with injected randomness (oracle/ref_sign_rand.c: ref_sig_sign_with_randomness) and against the
reference's own known-answer vectors (tests/golden/schnorr_sign_kat.json)."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, ROOT, golden, hx, random_scalars, rng, _buf

ALGS = {"ECSDSA": 3, "ECOSDSA": 4, "ECFSDSA": 5, "BIP0340": 20}
HASH_IDS = {"SHA256": 2, "SHA384": 3, "SHA512": 4, "SHA3_224": 5, "SHA3_256": 6, "SHA3_384": 7, "SHA3_512": 8}
HASHLIB = {"SHA224": hashlib.sha224, "SHA256": hashlib.sha256, "SHA384": hashlib.sha384, "SHA512": hashlib.sha512,
           "SHA3_224": hashlib.sha3_224, "SHA3_256": hashlib.sha3_256, "SHA3_384": hashlib.sha3_384,
           "SHA3_512": hashlib.sha3_512}
TAGS = (b"BIP0340/aux", b"BIP0340/nonce", b"BIP0340/challenge")
COMB_W = 6  # comb window of the host build (small: the table is built on the CPU)

HOSTSIM_SRC = os.path.join(ROOT, "tests", "hostsim", "schnorr_sign.cpp")
HOSTSIM_SO = os.path.join(ROOT, "tests", "hostsim", "_build", "libecc_hostsim_schnorr.so")
REF_SIGN_SO = os.path.join(ROOT, "oracle", "_ref", "libecc_ref_sign.so")
_libs = {}


def hostsim_lib() -> ctypes.CDLL:
    """the host build of the signer (the rest of the host build, tests/hostsim/hostsim.cpp, comes with it), built on
    demand like common.hostsim_lib"""
    if "hostsim" not in _libs:
        deps = [HOSTSIM_SRC, os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")] + [
            os.path.join(ROOT, "libecc_b200", "csrc", f) for f in
            ("fp.cuh", "ec.cuh", "msm_core.cuh", "curve_constants.inc", "sha2.cuh", "sha2_constants.inc", "sha3.cuh",
             "sha3_constants.inc")]
        if not os.path.exists(HOSTSIM_SO) or os.path.getmtime(HOSTSIM_SO) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(HOSTSIM_SO), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", HOSTSIM_SRC, "-o", HOSTSIM_SO],
                           check=True, capture_output=True)
        _libs["hostsim"] = ctypes.CDLL(HOSTSIM_SO)
    return _libs["hostsim"]


def ref_sign_lib():
    """oracle/_ref/libecc_ref_sign.so (oracle/ref_sign_rand.mk, built by build() where the reference's sources lie and
    travelling prebuilt elsewhere), or None when it is not available"""
    if "ref" not in _libs:
        if not os.path.exists(REF_SIGN_SO) and os.path.exists("/root/reference/src/libsig.h"):
            oracle = os.path.join(ROOT, "oracle")
            subprocess.run(["make", "-C", oracle, "-j8", "ref"], check=True, capture_output=True)
            subprocess.run(["make", "-C", oracle, "-f", "ref_sign_rand.mk", "all"], check=True, capture_output=True)
        _libs["ref"] = ctypes.CDLL(REF_SIGN_SO) if os.path.exists(REF_SIGN_SO) else None
    return _libs["ref"]


def siglen(curve, alg, hash_name):
    _, plen, qlen = ALL_CURVES[curve]
    ds = HASHLIB[hash_name]().digest_size
    return {"ECFSDSA": 2 * plen + qlen, "BIP0340": plen + qlen}.get(alg, ds + qlen)


def pack(msgs):
    blob = np.frombuffer(b"".join(msgs) + b"\0", dtype=np.uint8).copy()
    off = np.zeros(len(msgs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    return blob, off


def hostsim_sign(curve, alg, hash_name, privs, rand, msgs, pubs=None):
    lib = hostsim_lib()
    n = len(msgs)
    blob, off = pack(msgs)
    sigs = np.full((n, siglen(curve, alg, hash_name)), 0xAA, np.uint8)
    st = np.full(n, 7, np.int8)
    rc = lib.hostsim_schnorr_sign(ALGS[alg], HASH_IDS[hash_name], ALL_CURVES[curve][0], COMB_W, n, _buf(privs),
                                  _buf(pubs) if pubs is not None else None, _buf(rand), _buf(blob), _buf(off),
                                  _buf(sigs), _buf(st))
    assert rc == 0
    return sigs, st


def ref_sign(curve, alg, hash_name, privs, rand, msgs):
    """(sigs, pubs = x*G, status) from the reference's _ec_sign with rand returning randomness[i]"""
    ref = ref_sign_lib()
    if ref is None:
        pytest.skip("the reference's signer (oracle/_ref/libecc_ref_sign.so) is not available")
    _, plen, _ = ALL_CURVES[curve]
    n = len(msgs)
    blob, off = pack(msgs)
    sigs = np.zeros((n, siglen(curve, alg, hash_name)), np.uint8)
    pubs = np.zeros((n, 2 * plen), np.uint8)
    st = np.zeros(n, np.int8)
    assert ref.ref_sig_sign_with_randomness(curve.encode(), alg.encode(), hash_name.encode(), n, _buf(privs), _buf(rand),
                                            _buf(blob), _buf(off), _buf(sigs), _buf(pubs), _buf(st), 8) == 0
    return sigs, pubs, st


def be(v, nbytes):
    return np.frombuffer(int(v).to_bytes(nbytes, "big"), np.uint8)


# ------------------------------------------------------------------------------------------ hashing


@pytest.mark.parametrize("hash_name", list(HASH_IDS))
def test_segmented_hash_against_hashlib(hash_name):
    lib = hostsim_lib()
    h = HASHLIB[hash_name]
    block = h().block_size
    g = rng(900)
    data = g.bytes(2 * block + 300 + 260)
    mlens = sorted({0, 1} | {max(0, k * block + d) for k in (1, 2) for d in (-9, -8, -1, 0, 1, 8)})
    out = ctypes.create_string_buffer(64)
    for npre in list(range(0, 201, 7)) + [55, 56, 63, 64, 111, 112, 127, 128, 135, 136, 143, 144, 200]:
        pre = data[:npre]
        for mlen in mlens:
            msg = data[260:260 + mlen]
            ds = lib.hostsim_hash_segments(HASH_IDS[hash_name], pre, npre, msg, mlen, out)
            assert ds == h().digest_size
            assert out.raw[:ds] == h(pre + msg).digest(), (npre, mlen)


@pytest.mark.parametrize("hash_name", list(HASH_IDS))
def test_tagged_hash_against_hashlib(hash_name):
    """BIP0340's H_tag(z) = H(H(tag) || H(tag) || z) (sig/bip0340.c:45-69) from the host build's tag digest and the
    segmented hash"""
    lib = hostsim_lib()
    h = HASHLIB[hash_name]
    tag_d = ctypes.create_string_buffer(64)
    out = ctypes.create_string_buffer(64)
    z = rng(901).bytes(300)
    for t, tag in enumerate(TAGS):
        ds = lib.hostsim_bip0340_tag_hash(HASH_IDS[hash_name], t, tag_d)
        assert tag_d.raw[:ds] == h(tag).digest()
        ht = tag_d.raw[:ds]
        for npre, mlen in ((2 * ds, 0), (2 * ds + 32, 0), (2 * ds + 66, 150), (2 * ds + 132, 300)):
            pre = (ht + ht + z)[:npre]
            assert lib.hostsim_hash_segments(HASH_IDS[hash_name], pre, npre, z, mlen, out) == ds
            assert out.raw[:ds] == h(ht + ht + z[:npre - 2 * ds] + z[:mlen]).digest()


def test_unsupported_hash_is_refused():
    out = ctypes.create_string_buffer(64)
    assert hostsim_lib().hostsim_hash_segments(1, b"", 0, b"", 0, out) == -1  # SHA224 is not computed on the device
    assert hostsim_lib().hostsim_hash_segments(9, b"", 0, b"", 0, out) == -1


# ------------------------------------------------------------------------------------------ against the reference


def workload(curve, alg, n, tag):
    """random keys (with both parities of y(P) among them), randomness and messages of 0 to 300 bytes, then the invalid
    inputs: x and k (the nonce; BIP0340: x only, its randomness is an auxiliary value) equal to 0, q and 2^(8 qlen) - 1"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    g = rng(tag)
    privs = random_scalars(curve, n, tag=tag + 1)
    if alg == "BIP0340":
        rand = g.integers(0, 256, size=(n, qlen), dtype=np.uint8)
    else:
        rand = random_scalars(curve, n, tag=tag + 2)
    msgs = [g.bytes(int(g.integers(0, 301))) for _ in range(n)]
    bad = [0, q, (1 << (8 * qlen)) - 1]
    for j, v in enumerate(bad):
        privs[j] = be(v, qlen)
        if alg != "BIP0340":
            rand[len(bad) + j] = be(v, qlen)
    return privs, rand, msgs


CASES = [(c, a, h) for c in ALL_CURVES for a in ALGS for h in ("SHA256", "SHA384", "SHA512", "SHA3_224", "SHA3_512")]


@pytest.mark.parametrize("curve,alg,hash_name", CASES)
def test_hostsim_against_reference(curve, alg, hash_name):
    n = 24
    tag = 5000 + 10 * list(ALL_CURVES).index(curve) + list(ALGS).index(alg)
    privs, rand, msgs = workload(curve, alg, n, tag)
    want, pubs, wst = ref_sign(curve, alg, hash_name, privs, rand, msgs)
    got, st = hostsim_sign(curve, alg, hash_name, privs, rand, msgs, pubs)
    assert (st == wst).all(), (st, wst)
    assert (got == want).all()
    assert (st[:3] == -1).all() and (st[3:] != 7).all()
    if alg != "BIP0340":
        assert (st[3:6] == -1).all()
    assert (st[6:] == 0).all()
    if alg == "BIP0340":  # keys of both parities took part
        assert len({int(p[-1]) & 1 for p, s in zip(pubs, st) if s == 0}) == 2


@pytest.mark.parametrize("curve", ["SECP256K1", "SECP521R1"])
def test_bip0340_key_off_curve_is_an_error(curve):
    _, plen, qlen = ALL_CURVES[curve]
    privs, rand, msgs = workload(curve, "BIP0340", 8, 77)
    _, pubs, wst = ref_sign(curve, "BIP0340", "SHA256", privs, rand, msgs)
    assert (wst[3:] == 0).all()
    pubs[4, plen - 1] ^= 1
    sigs, st = hostsim_sign(curve, "BIP0340", "SHA256", privs, rand, msgs, pubs)
    assert st[4] == -1 and not sigs[4].any()
    assert (st[5:] == 0).all()


# ------------------------------------------------------------------------------------------ known answers


def kat_vectors():
    return golden("schnorr_sign_kat.json")


def test_kat_fixture_contents():
    kats = kat_vectors()
    assert len(kats) == 28
    count = {a: sum(1 for k in kats if k["alg"] == a) for a in ALGS}
    assert count == {"ECSDSA": 8, "ECOSDSA": 8, "ECFSDSA": 8, "BIP0340": 4}
    assert sum(1 for k in kats if k["hash"] == "SHA224") == 3


def py_sign_from_W(curve, alg, hash_name, x, k, W, msg):
    """the scheme core restated over hashlib (the hashes the device does not compute, SHA-224), W = k*G given"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    h = HASHLIB[hash_name]
    wx, wy = W[:plen], W[plen:]
    if alg == "ECFSDSA":
        e = int.from_bytes(h(wx + wy + msg).digest(), "big") % q
        return wx + wy + ((k + e * x) % q).to_bytes(qlen, "big")
    r = h(wx + (wy if alg == "ECSDSA" else b"") + msg).digest()
    e = int.from_bytes(r, "big") % q
    return r + ((k + e * x) % q).to_bytes(qlen, "big")


@pytest.mark.parametrize("kat", kat_vectors(), ids=lambda k: k["name"])
def test_kat(kat):
    curve, alg, hash_name = kat["curve"], kat["alg"], kat["hash"]
    if curve not in ALL_CURVES:
        pytest.skip("curve outside the engine")
    _, plen, qlen = ALL_CURVES[curve]
    x = int(kat["priv"], 16)
    priv = be(x, qlen).copy().reshape(1, qlen)
    rand = hx(kat["randomness"]).copy().reshape(1, qlen)
    msg = bytes.fromhex(kat["msg"])
    pub = hx(kat["pub"]).copy().reshape(1, 2 * plen)
    if hash_name in HASH_IDS:
        sigs, st = hostsim_sign(curve, alg, hash_name, priv, rand, [msg], pub)
        assert st[0] == 0 and sigs[0].tobytes().hex() == kat["sig"]
        return
    assert alg != "BIP0340"
    W = np.zeros((1, 2 * plen), np.uint8)
    wst = np.zeros(1, np.int8)
    assert hostsim_lib().hostsim_prj_pt_mul_batch(ALL_CURVES[curve][0], COMB_W, 1, _buf(rand), None, _buf(W), _buf(wst)) == 0
    assert wst[0] == 0
    k = int(kat["randomness"], 16)
    assert py_sign_from_W(curve, alg, hash_name, x, k, W[0].tobytes(), msg).hex() == kat["sig"]
