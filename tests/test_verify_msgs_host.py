"""ECKCDSA / ECSDSA / ECOSDSA / ECGDSA / ECRDSA / SM2 verification of raw messages without a GPU: the host build of the
device algorithm (tests/hostsim/verify_msgs.cpp: prep core, one inversion per item, comb + signed window, acceptance
test) against the reference's ec_verify (ref_sig_verify_batch, and ref_sig_verify_adata_batch for SM2's IDs) on valid
and corrupted signatures made by the reference's signers, on the reference's known answers, and on crafted vectors
that reach the e = 0, r + s = q and W' = infinity branches."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, ROOT, golden, hx, random_scalars, ref_lib, rng, _buf
from test_sign_msgs_host import HASHLIB, HASH_IDS, be, pack
from test_sign_msgs_host import ref_sign as ref_sign_adata
from test_sign_msgs_host import ref_verify as ref_verify_adata
from test_schnorr_sign_host import ref_sign_lib as ref_sign_schnorr_lib

ALGS = {"ECKCDSA": 2, "ECSDSA": 3, "ECOSDSA": 4, "ECGDSA": 6, "ECRDSA": 7, "SM2": 8}
HASHES = ("SHA256", "SHA384", "SHA512", "SHA3_256", "SHA3_512", "SM3")
COMB_W = 6  # comb window of the host build (small: the table is built on the CPU)
SM2_ID_LENS = (0, 1, 200, 8191)

HOSTSIM_SRC = os.path.join(ROOT, "tests", "hostsim", "verify_msgs.cpp")
HOSTSIM_SO = os.path.join(ROOT, "tests", "hostsim", "_build", "libecc_hostsim_verify_msgs.so")
_libs = {}


def hostsim_lib() -> ctypes.CDLL:
    """the host build of the verifier (with the signer's and the rest of the host build), built on demand"""
    if "hostsim" not in _libs:
        deps = [HOSTSIM_SRC] + [os.path.join(ROOT, "tests", "hostsim", f) for f in ("hostsim.cpp", "sign.cpp")] + [
            os.path.join(ROOT, "libecc_b200", "csrc", f) for f in
            ("fp.cuh", "ec.cuh", "msm_core.cuh", "curve_constants.inc", "sha2.cuh", "sha2_constants.inc", "sha3.cuh",
             "sha3_constants.inc", "sm3.cuh")]
        if not os.path.exists(HOSTSIM_SO) or os.path.getmtime(HOSTSIM_SO) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(HOSTSIM_SO), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", HOSTSIM_SRC, "-o", HOSTSIM_SO],
                           check=True, capture_output=True)
        _libs["hostsim"] = ctypes.CDLL(HOSTSIM_SO)
    return _libs["hostsim"]


def digest_size(hash_name):
    return HASHLIB[hash_name]().digest_size


def vsiglen(curve, alg, hash_name):
    qlen = ALL_CURVES[curve][2]
    ds = digest_size(hash_name)
    return {"ECSDSA": ds, "ECOSDSA": ds, "ECKCDSA": min(ds, qlen)}.get(alg, qlen) + qlen


def rlen(curve, alg, hash_name):
    return vsiglen(curve, alg, hash_name) - ALL_CURVES[curve][2]


def hostsim_verify(curve, alg, hash_name, sigs, pubs, msgs, ids=None):
    n = len(msgs)
    blob, off = pack(msgs)
    iblob, ioff = pack(ids if ids is not None else [b""] * n)
    v = np.full(n, 7, np.int8)
    rc = hostsim_lib().hostsim_verify_msgs(ALGS[alg], HASH_IDS[hash_name], ALL_CURVES[curve][0], COMB_W, n,
                                           _buf(sigs), _buf(pubs), _buf(blob), _buf(off), _buf(iblob), _buf(ioff),
                                           _buf(v))
    assert rc == 0
    return v


def ref_verify(curve, alg, hash_name, sigs, pubs, msgs, ids=None):
    """verdicts of the reference's ec_verify (with item i's ID as ancillary data for SM2)"""
    if alg == "SM2":
        return ref_verify_adata(curve, alg, hash_name, sigs, pubs, msgs, ids)
    ref = ref_lib()
    if ref is None:
        pytest.skip("the reference (oracle/_ref/libecc_ref.so) is not available")
    blob, off = pack(msgs)
    v = np.full(len(msgs), 7, np.int8)
    assert ref.ref_sig_verify_batch(curve.encode(), alg.encode(), hash_name.encode(), len(msgs),
                                    _buf(np.ascontiguousarray(sigs)), _buf(np.ascontiguousarray(pubs)), _buf(blob),
                                    _buf(off), _buf(v), 8) == 0
    return v


def ref_sign(curve, alg, hash_name, privs, nonces, msgs, ids=None):
    """(sigs, pubs, status) from the reference's signer with injected nonces"""
    if alg not in ("ECSDSA", "ECOSDSA"):
        return ref_sign_adata(curve, alg, hash_name, privs, nonces, msgs, ids)
    ref = ref_sign_schnorr_lib()
    if ref is None:
        pytest.skip("the reference's signer (oracle/_ref/libecc_ref_sign.so) is not available")
    n = len(msgs)
    blob, off = pack(msgs)
    sigs = np.zeros((n, vsiglen(curve, alg, hash_name)), np.uint8)
    pubs = np.zeros((n, 2 * ALL_CURVES[curve][1]), np.uint8)
    st = np.zeros(n, np.int8)
    assert ref.ref_sig_sign_with_randomness(curve.encode(), alg.encode(), hash_name.encode(), n, _buf(privs),
                                            _buf(nonces), _buf(blob), _buf(off), _buf(sigs), _buf(pubs), _buf(st),
                                            8) == 0
    return sigs, pubs, st


def valid_batch(curve, alg, hash_name, n, tag):
    """n valid signatures from the reference: random keys and nonces, messages of 0 to 300 bytes (item 1 empty, item 2
    of several blocks), SM2 IDs of 0, 1, 200 and 8191 bytes"""
    g = rng(tag)
    privs = random_scalars(curve, n, tag=tag + 1)
    nonces = random_scalars(curve, n, tag=tag + 2)
    msgs = [g.bytes(int(g.integers(0, 301))) for _ in range(n)]
    msgs[1] = b""
    msgs[2] = g.bytes(333)
    ids = [g.bytes(SM2_ID_LENS[i % len(SM2_ID_LENS)]) for i in range(n)] if alg == "SM2" else None
    sigs, pubs, st = ref_sign(curve, alg, hash_name, privs, nonces, msgs, ids)
    assert (st == 0).all(), st
    return sigs, pubs, msgs, ids


def corrupt(curve, alg, hash_name, sigs, pubs, msgs, ids, tag):
    """items 3.. of a valid batch made invalid, one way each; returns the indices that must be rejected"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    g = rng(tag)
    rl = rlen(curve, alg, hash_name)
    bit = lambda nbytes: (int(g.integers(0, nbytes)), 1 << int(g.integers(0, 8)))
    j, m = bit(rl)
    sigs[3, j] ^= m                                   # one bit of r
    j, m = bit(qlen)
    sigs[4, rl + j] ^= m                              # one bit of s
    mb = bytearray(msgs[5] or b"\0")
    j, m = bit(len(mb))
    mb[j] ^= m
    msgs[5] = bytes(mb)                               # one bit of the message
    j, m = bit(2 * plen)
    pubs[6, j] ^= m                                   # one bit of the key
    sigs[7, rl:] = be(0, qlen)                        # s = 0
    sigs[8, rl:] = be(q, qlen)                        # s = q
    pubs[9, 2 * plen - 1] ^= 1                        # key off the curve
    bad = [3, 4, 5, 6, 7, 8, 9]
    if rl == qlen and alg not in ("ECKCDSA",):
        sigs[10, :rl] = be(0, qlen)                   # r = 0
        sigs[11, :rl] = be(q, qlen)                   # r = q
        bad += [10, 11]
    if alg == "SM2":
        ids[12] = ids[12] + b"!"                      # a changed ID
        ids[13] = bytes(8192)                         # longer than SM2_MAX_ID_LEN
        bad += [12, 13]
    return bad


CASES = [(c, a, h) for c in ALL_CURVES for a in ALGS for h in HASHES]


@pytest.mark.parametrize("curve,alg,hash_name", CASES)
def test_hostsim_against_reference(curve, alg, hash_name):
    n = 18
    tag = 10000 + 1000 * list(ALL_CURVES).index(curve) + 100 * list(ALGS).index(alg) + 10 * HASHES.index(hash_name)
    sigs, pubs, msgs, ids = valid_batch(curve, alg, hash_name, n, tag)
    bad = corrupt(curve, alg, hash_name, sigs, pubs, msgs, ids, tag + 5)
    want = ref_verify(curve, alg, hash_name, sigs, pubs, msgs, ids)
    got = hostsim_verify(curve, alg, hash_name, sigs, pubs, msgs, ids)
    assert (got == want).all(), (got, want)
    expect = np.zeros(n, np.int8)
    expect[bad] = -1
    assert (want == expect).all(), (want, bad)


@pytest.mark.parametrize("curve,hash_name", [("SECP521R1", "SHA512"), ("SECP384R1", "SHA3_512")])
def test_eckcdsa_z_cut_to_block_size(curve, hash_name):
    """2*plen > block size: z is the key cut to the block size; a key differing only past the cut then verifies too"""
    _, plen, _ = ALL_CURVES[curve]
    bs = HASHLIB[hash_name]().block_size
    assert 2 * plen > bs
    sigs, pubs, msgs, ids = valid_batch(curve, "ECKCDSA", hash_name, 6, 88)
    assert (hostsim_verify(curve, "ECKCDSA", hash_name, sigs, pubs, msgs) == 0).all()
    assert (ref_verify(curve, "ECKCDSA", hash_name, sigs, pubs, msgs) == 0).all()


def test_unsupported_sig_type_or_hash_is_refused():
    lib = hostsim_lib()
    z = np.zeros(4096, np.uint8)
    off = np.zeros(2, np.uint64)
    v = np.full(1, 5, np.int8)
    for st in (1, 5, 14, 20):
        assert lib.hostsim_verify_msgs(st, 2, 4, COMB_W, 1, _buf(z), _buf(z), _buf(z), _buf(off), _buf(z), _buf(off),
                                       _buf(v)) == -1
    for ht in (0, 1, 9, 10, 12):
        assert lib.hostsim_verify_msgs(3, ht, 4, COMB_W, 1, _buf(z), _buf(z), _buf(z), _buf(off), _buf(z), _buf(off),
                                       _buf(v)) == -1
    assert v[0] == 5


# ------------------------------------------------------------------------------------------ known answers


def kat_vectors():
    """the reference's self-test vectors of the six schemes: (curve, alg, hash, sig, pub, msg, id)"""
    out = [(k["curve"], k["alg"], k["hash"], k["sig"], k["pub"], k["msg"], k["adata"]) for k in golden("sign_kat.json")]
    out += [(k["curve"], k["alg"], k["hash"], k["sig"], k["pub"], k["msg"], "")
            for k in golden("schnorr_sign_kat.json") if k["alg"] in ("ECSDSA", "ECOSDSA")]
    return out


def test_kat_fixture_contents():
    kats = kat_vectors()
    assert len(kats) == 13 + 16
    assert sum(1 for k in kats if k[2] in HASH_IDS) == 12 + 14


@pytest.mark.parametrize("kat", kat_vectors(), ids=lambda k: f"{k[1]}-{k[0]}-{k[2]}")
def test_kat(kat):
    curve, alg, hash_name, sig, pub, msg, adata = kat
    sig, pub, msg, ids = hx(sig), hx(pub), bytes.fromhex(msg), [bytes.fromhex(adata)]
    sigs = np.stack([sig, sig.copy(), sig.copy()])
    pubs = np.stack([pub, pub, pub])
    sigs[1, -1] ^= 1                                  # s
    msgs = [msg, msg, msg + b"\0"]
    want = ref_verify(curve, alg, hash_name, sigs, pubs, msgs, ids * 3 if alg == "SM2" else None)
    assert list(want) == [0, -1, -1]
    if hash_name in HASH_IDS:
        got = hostsim_verify(curve, alg, hash_name, sigs, pubs, msgs, ids * 3 if alg == "SM2" else None)
        assert list(got) == [0, -1, -1]


# ------------------------------------------------------------------------------------------ crafted vectors


def kG(curve, k):
    """affine wire bytes of k*G (host build)"""
    _, plen, qlen = ALL_CURVES[curve]
    W = np.zeros((1, 2 * plen), np.uint8)
    st = np.zeros(1, np.int8)
    assert hostsim_lib().hostsim_prj_pt_mul_batch(ALL_CURVES[curve][0], COMB_W, 1, _buf(be(k, qlen).copy()), None,
                                                  _buf(W), _buf(st)) == 0
    assert st[0] == 0
    return W[0]


def ecgdsa_e(curve, hash_name, msg):
    q = ORDER[curve]
    h = HASHLIB[hash_name](msg).digest()
    shift = max(0, 8 * len(h) - q.bit_length())
    return (int.from_bytes(h, "big") >> shift) % q


def ecrdsa_h(curve, hash_name, msg):
    return int.from_bytes(HASHLIB[hash_name](msg).digest()[::-1], "big") % ORDER[curve] or 1


def crafted(curve, alg, hash_name, kind, tag):
    """(sig, pub, msg, id) of a crafted vector the reference must reject:
    kind "e0"   ECSDSA / ECOSDSA with r = 0 mod q (e = 0);
    kind "rs_q" SM2 with r + s = q;
    kind "inf"  W' = a*G + b*Y at infinity: the private key y is chosen after a and b are known, a + b*y = 0 mod q"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    g = rng(tag)
    rnd = lambda: int.from_bytes(g.bytes(qlen + 8), "big") % (q - 1) + 1
    msg = g.bytes(int(g.integers(0, 80)))
    ident = g.bytes(16) if alg == "SM2" else b""
    rl = rlen(curve, alg, hash_name)
    s = rnd()
    if kind == "e0":
        r = 0 if (tag & 1) or q >= 1 << (8 * rl) else q
        return be(r, rl).tobytes() + be(s, qlen).tobytes(), kG(curve, rnd()), msg, ident
    if kind == "rs_q":
        r = rnd()
        s = q - r
        return be(r, qlen).tobytes() + be(s, qlen).tobytes(), kG(curve, rnd()), msg, ident
    assert kind == "inf"
    if alg in ("ECSDSA", "ECOSDSA"):
        rb = g.bytes(rl)
        r = int.from_bytes(rb, "big") % q
        a, b = s, -r % q                              # W' = sG + eY, e = -(r mod q)
        sig = rb + be(s, qlen).tobytes()
    else:
        r = rnd()
        sig = be(r, qlen).tobytes() + be(s, qlen).tobytes()
        if alg == "ECGDSA":
            ri = pow(r, -1, q)
            a, b = ri * ecgdsa_e(curve, hash_name, msg) % q, ri * s % q
        elif alg == "ECRDSA":
            hi = pow(ecrdsa_h(curve, hash_name, msg), -1, q)
            a, b = hi * s % q, -hi * r % q
        else:
            a, b = s, (r + s) % q                     # SM2
    assert a and b
    y = -a * pow(b, -1, q) % q
    assert (a + b * y) % q == 0
    return sig, kG(curve, y), msg, ident


CRAFTED = ([(a, "e0") for a in ("ECSDSA", "ECOSDSA")] + [("SM2", "rs_q")] +
           [(a, "inf") for a in ("ECSDSA", "ECOSDSA", "ECGDSA", "ECRDSA", "SM2")])


def crafted_batch(curve, alg, hash_name, kind, count, tag):
    vs = [crafted(curve, alg, hash_name, kind, tag + i) for i in range(count)]
    sigs = np.stack([np.frombuffer(v[0], np.uint8) for v in vs])
    pubs = np.stack([v[1] for v in vs])
    return sigs, pubs, [v[2] for v in vs], [v[3] for v in vs] if alg == "SM2" else None


@pytest.mark.parametrize("hash_name", ["SHA256", "SHA3_512", "SM3"])
@pytest.mark.parametrize("alg,kind", CRAFTED)
@pytest.mark.parametrize("curve", ["SECP256R1", "FRP256V1", "SECP521R1", "SECP224R1", "SM2P256V1"])
def test_crafted_vectors_are_rejected(curve, alg, kind, hash_name):
    sigs, pubs, msgs, ids = crafted_batch(curve, alg, hash_name, kind, 4, 900 + CRAFTED.index((alg, kind)))
    assert (ref_verify(curve, alg, hash_name, sigs, pubs, msgs, ids) == -1).all()
    assert (hostsim_verify(curve, alg, hash_name, sigs, pubs, msgs, ids) == -1).all()
