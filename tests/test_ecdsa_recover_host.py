"""ECDSA public-key recovery without a GPU: the host build of the device algorithm (tests/hostsim/ecdsa_recover.cpp:
range checks, the reference's square root, u and v, comb + signed window, the two final additions) against the
reference's own __ecdsa_public_key_from_sig and aff_pt_y_from_x (oracle/_ref/libecc_ref_recover.so).

Covered: the square roots on all eleven curves (thousands of x, and on SECP224R1 enough of them that Tonelli-Shanks
takes many different paths); recovery parity for hlen of 20 to 64 bytes with valid signatures, r and s at the edges of
their range, r in [p, q) on FRP256V1, an r that is no x coordinate, the reference's restart quirk (r = x(P) - q is never
recovered from x = r + q), an all-zero digest, and crafted signatures whose keys are the point at infinity or come out
of the doubling branch of the final addition; the reference's ECDSA / DECDSA known answers; and that every finite key
verifies its signature."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, PRIME, ROOT, golden, oracle_sign, oracle_smul, oracle_verify, random_scalars, \
    rng, _buf
from test_rare_branches import CURVE_AB, b2i, be, digest_of_e, dsmul, ecdsa_e, neg, point_with_x, smul, sqrt_mod, \
    unwire, wire

HOST_W = 6  # comb window of the host build (small: the table is built on the CPU)
HLENS = (20, 28, 32, 48, 64)
Q_BELOW_P = [c for c in ALL_CURVES if ORDER[c] < PRIME[c]]

HOSTSIM_SRC = os.path.join(ROOT, "tests", "hostsim", "ecdsa_recover.cpp")
HOSTSIM_SO = os.path.join(ROOT, "tests", "hostsim", "_build", "libecc_hostsim_recover.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libecc_ref_recover.so")
_libs = {}


def hostsim_lib() -> ctypes.CDLL:
    """the host build of the recovery (on top of the rest of the host build), built on demand"""
    if "hostsim" not in _libs:
        deps = [HOSTSIM_SRC, os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")] + [
            os.path.join(ROOT, "libecc_b200", "csrc", f) for f in
            ("fp.cuh", "ec.cuh", "msm_core.cuh", "curve_constants.inc", "sha2.cuh", "sha2_constants.inc", "sha3.cuh",
             "sha3_constants.inc", "sm3.cuh")]
        if not os.path.exists(HOSTSIM_SO) or os.path.getmtime(HOSTSIM_SO) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(HOSTSIM_SO), exist_ok=True)
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", HOSTSIM_SRC, "-o", HOSTSIM_SO],
                           check=True, capture_output=True)
        _libs["hostsim"] = ctypes.CDLL(HOSTSIM_SO)
    return _libs["hostsim"]


def ref_recover_lib():
    """the reference's recovery wrapper, or None where it has not been built (oracle/ref_recover.mk)"""
    if "ref" not in _libs:
        if not os.path.exists(REF_SO) and os.path.exists("/root/reference/src/libsig.h"):
            subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "ref_recover.mk", "all"], check=True,
                           capture_output=True)
        _libs["ref"] = ctypes.CDLL(REF_SO) if os.path.exists(REF_SO) else None
    return _libs["ref"]


def need_ref():
    lib = ref_recover_lib()
    if lib is None:
        pytest.skip("the reference's recovery (oracle/_ref/libecc_ref_recover.so) is not available")
    return lib


def ref_recover(curve, sigs, digests, hlen):
    """(keys [n][2][2*plen], status [n][2]) from the reference's __ecdsa_public_key_from_sig"""
    plen = ALL_CURVES[curve][1]
    sigs, digests = np.ascontiguousarray(sigs, np.uint8), np.ascontiguousarray(digests, np.uint8)
    n = sigs.shape[0]
    keys = np.full((n, 2, 2 * plen), 0xAA, np.uint8)
    st = np.full((n, 2), 7, np.int8)
    assert need_ref().ref_ecdsa_recover_batch(curve.encode(), n, _buf(sigs), _buf(digests), hlen, _buf(keys),
                                              _buf(st)) == 0
    return keys, st


def host_recover(curve, sigs, digests, hlen):
    plen = ALL_CURVES[curve][1]
    sigs, digests = np.ascontiguousarray(sigs, np.uint8), np.ascontiguousarray(digests, np.uint8)
    n = sigs.shape[0]
    keys = np.full((n, 2, 2 * plen), 0xAA, np.uint8)
    st = np.full((n, 2), 7, np.int8)
    assert hostsim_lib().hostsim_ecdsa_recover(ALL_CURVES[curve][0], HOST_W, n, _buf(sigs), _buf(digests), hlen,
                                               _buf(keys), _buf(st)) == 0
    return keys, st


def sig_rows(curve, rs):
    qlen = ALL_CURVES[curve][2]
    return np.stack([np.concatenate([be(r, qlen), be(s, qlen)]) for r, s in rs])


# ------------------------------------------------------------------------------------------ square roots


def host_y_from_x(curve, xs):
    plen = ALL_CURVES[curve][1]
    n = xs.shape[0]
    y1, y2 = np.zeros((n, plen), np.uint8), np.zeros((n, plen), np.uint8)
    ok, loops = np.zeros(n, np.int8), np.zeros(n, np.int32)
    assert hostsim_lib().hostsim_y_from_x(ALL_CURVES[curve][0], n, _buf(xs), _buf(y1), _buf(y2), _buf(ok),
                                          _buf(loops)) == 0
    return y1, y2, ok, loops


def ref_y_from_x(curve, xs):
    plen = ALL_CURVES[curve][1]
    n = xs.shape[0]
    y1, y2, ok = np.zeros((n, plen), np.uint8), np.zeros((n, plen), np.uint8), np.zeros(n, np.int8)
    assert need_ref().ref_y_from_x(curve.encode(), n, _buf(xs), _buf(y1), _buf(y2), _buf(ok)) == 0
    return y1, y2, ok


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_square_roots_match_the_reference(curve):
    p, plen = PRIME[curve], ALL_CURVES[curve][1]
    count = 20000 if curve == "SECP224R1" else 2000
    g = rng(7100 + ALL_CURVES[curve][0])
    vals = [0, 1, p - 1] + [b2i(g.bytes(plen + 8)) % p for _ in range(count)]
    xs = np.stack([be(v, plen) for v in vals])
    h1, h2, hok, loops = host_y_from_x(curve, xs)
    r1, r2, rok = ref_y_from_x(curve, xs)
    assert (hok == rok).all()
    assert (h1 == r1).all() and (h2 == r2).all()
    a, b = CURVE_AB[curve]
    for v, y, ok in zip(vals[:200], h1[:200], hok[:200]):  # and the plain restatement in Python integers
        want = sqrt_mod(v ** 3 + a * v + b, p)
        assert (ok == 0) == (want is not None) and (want is None or b2i(y) == want)
    assert 0.4 < (hok == 0).mean() < 0.6
    if curve == "SECP224R1":
        reached = sorted(set(int(x) for x in loops[hok == 0]))
        print(f"SECP224R1 Tonelli-Shanks: {len(reached)} distinct loop counts, {reached[0]} to {reached[-1]}")
        assert len(reached) >= 20 and reached[-1] - reached[0] >= 25, reached
    else:
        assert (loops == 0).all()


# ------------------------------------------------------------------------------------------ recovery parity


def valid_items(curve, n, hlen, tag):
    """n signatures of the oracle's signer on random hlen-byte digests: (sigs, digests, pubs)"""
    d = random_scalars(curve, n, tag=tag)
    k = random_scalars(curve, n, tag=tag + 1)
    dg = rng(tag + 2).integers(0, 256, size=(n, hlen), dtype=np.uint8)
    pubs, st = oracle_smul(curve, d)
    assert (st == 0).all()
    sigs, st = oracle_sign(curve, d, k, dg, hlen)
    assert (st == 0).all()
    return sigs, dg, pubs


def edge_rows(curve, good):
    """r or s at 0, 1, q - 1 and q next to a valid partner, and (1, 1), (q-1, q-1)"""
    q = ORDER[curve]
    r0, s0 = good
    rows = [(v, s0) for v in (0, 1, q - 1, q)] + [(r0, v) for v in (0, 1, q - 1, q)] + [(1, 1), (q - 1, q - 1)]
    return rows


def not_an_x(curve, g, count):
    """r in [1, q-1] for which r^3 + ar + b is not a square"""
    p, q = PRIME[curve], ORDER[curve]
    a, b = CURVE_AB[curve]
    out = []
    while len(out) < count:
        r = 1 + b2i(g.bytes(80)) % (q - 1)
        if r < p and sqrt_mod(r ** 3 + a * r + b, p) is None:
            out.append(r)
    return out


def restart_quirk_rows(curve, g, count):
    """r = x(P) - q for curve points P with x(P) in [q, p): the signature of a nonce point with x >= q"""
    q, p = ORDER[curve], PRIME[curve]
    return [point_with_x(curve, q, p, g)[0] - q for _ in range(count)]


def parity_batch(curve, hlen, tag):
    q, qlen = ORDER[curve], ALL_CURVES[curve][2]
    g = rng(tag + 9)
    sigs, dg, _ = valid_items(curve, 8, hlen, tag)
    good = (b2i(sigs[0, :qlen]), b2i(sigs[0, qlen:]))
    rs = [(b2i(s[:qlen]), b2i(s[qlen:])) for s in sigs] + edge_rows(curve, good)
    rs += [(r, good[1]) for r in not_an_x(curve, g, 3)]
    if curve in Q_BELOW_P:
        rs += [(r, good[1]) for r in restart_quirk_rows(curve, g, 4)]
    else:  # FRP256V1: r in [p, q)
        p = PRIME[curve]
        rs += [(r, good[1]) for r in (p, p + 1, q - 1, p + b2i(g.bytes(40)) % (q - p))]
    digests = [dg[i % len(dg)] for i in range(len(rs))]
    rs.append(good)
    digests.append(np.zeros(hlen, np.uint8))  # all-zero digest: u = 0
    return sig_rows(curve, rs), np.stack(digests)


@pytest.mark.parametrize("hlen", HLENS)
@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_recovery_matches_the_reference(curve, hlen):
    sigs, dg = parity_batch(curve, hlen, 7300 + 10 * ALL_CURVES[curve][0] + HLENS.index(hlen))
    want_k, want_s = ref_recover(curve, sigs, dg, hlen)
    got_k, got_s = host_recover(curve, sigs, dg, hlen)
    assert (got_s == want_s).all(), (got_s, want_s)
    assert (got_k == want_k).all()
    assert (want_s[:8] == 0).all()            # the valid signatures
    assert (want_s[[8, 11, 12, 15]] == -1).all()  # r or s equal to 0 or q
    assert (want_s[18:21] == -1).all()        # no point with x = r
    assert (want_s[-1] == 0).all()            # u = 0: Y1 = v*R1, Y2 = -Y1
    assert (want_k[-1, 0, :ALL_CURVES[curve][1]] == want_k[-1, 1, :ALL_CURVES[curve][1]]).all()
    if curve not in Q_BELOW_P:
        assert (want_s[21:25] == -1).all()    # r >= p on FRP256V1


@pytest.mark.parametrize("curve", Q_BELOW_P)
def test_restart_quirk_never_uses_r_plus_q(curve):
    """a nonce point with x >= q: recovery works from x = r (or fails), never from x = r + q the signer used"""
    q, qlen, plen = ORDER[curve], ALL_CURVES[curve][2], ALL_CURVES[curve][1]
    g = rng(7500 + ALL_CURVES[curve][0])
    rows, digests, true_keys = [], [], []
    for _ in range(6):
        x, y = point_with_x(curve, q, PRIME[curve], g)
        r, s, e = x - q, 1 + b2i(g.bytes(80)) % (q - 1), b2i(g.bytes(80)) % q
        ri = pow(r, -1, q)
        (Y,), st = dsmul(curve, [-e * ri], [s * ri], [(x, y)])  # the key x = r + q would give
        rows.append((r, s))
        digests.append(digest_of_e(curve, e))
        true_keys.append((Y, st[0]))
    sigs, dg = sig_rows(curve, rows), np.stack(digests)
    want_k, want_s = ref_recover(curve, sigs, dg, qlen)
    got_k, got_s = host_recover(curve, sigs, dg, qlen)
    assert (got_s == want_s).all() and (got_k == want_k).all()
    for i, (Y, st) in enumerate(true_keys):
        assert st == 0
        for k in range(2):
            assert want_s[i, k] != 0 or unwire(curve, want_k[i, k]) not in (Y, neg(curve, Y))


def crafted_rows(curve, tag, count):
    """(sigs, digests, expect): r = x(kG), e = +-k*s, so one key is the point at infinity and the other 2*u*G comes out
    of the doubling branch of the final addition; both signs, so each key takes each role"""
    q, qlen = ORDER[curve], ALL_CURVES[curve][2]
    g = rng(tag)
    rows, digests, expect = [], [], []
    while len(rows) < count:
        k, s = 1 + b2i(g.bytes(80)) % (q - 1), 1 + b2i(g.bytes(80)) % (q - 1)
        (R,) = smul(curve, [k])
        if R[0] >= q:
            continue
        r = R[0]
        for sign in (1, -1):
            e = sign * k * s % q
            u = -e * pow(r, -1, q) % q
            rows.append((r, s))
            digests.append(digest_of_e(curve, e))
            expect.append(smul(curve, [2 * u])[0])
    return sig_rows(curve, rows), np.stack(digests), expect


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_crafted_infinity_and_doubling(curve):
    qlen = ALL_CURVES[curve][2]
    sigs, dg, expect = crafted_rows(curve, 7700 + ALL_CURVES[curve][0], 4)
    want_k, want_s = ref_recover(curve, sigs, dg, qlen)
    got_k, got_s = host_recover(curve, sigs, dg, qlen)
    assert (got_s == want_s).all() and (got_k == want_k).all()
    for i, Y in enumerate(expect):
        assert sorted(want_s[i].tolist()) == [0, 1]
        fin = int(np.argmin(want_s[i]))
        assert unwire(curve, want_k[i, fin]) == Y and not want_k[i, 1 - fin].any()
    assert {int(np.argmax(s)) for s in want_s} == {0, 1}  # Y1 = infinity and Y2 = infinity both occur


# ------------------------------------------------------------------------------------------ known answers, integers


def kat_vectors():
    return [v for v in golden("ecdsa_kat.json") if v["alg"] in ("ECDSA", "DECDSA")]


def test_kat_fixture_contents():
    assert len(kat_vectors()) == 47


@pytest.mark.parametrize("kat", kat_vectors(), ids=lambda v: v["name"])
def test_kat_recovers_the_signer(kat):
    curve = kat["curve"]
    plen = ALL_CURVES[curve][1]
    sig = np.frombuffer(bytes.fromhex(kat["sig"]), np.uint8)[None]
    dg = np.frombuffer(bytes.fromhex(kat["digest"]), np.uint8)[None]
    pub = bytes.fromhex(kat["pub"])
    half = len(pub) // 2
    pub = be(b2i(pub[:half]), plen).tobytes() + be(b2i(pub[half:]), plen).tobytes()
    want_k, want_s = ref_recover(curve, sig, dg, dg.shape[1])
    got_k, got_s = host_recover(curve, sig, dg, dg.shape[1])
    assert (got_s == want_s).all() and (got_k == want_k).all()
    assert (want_s == 0).all()
    assert pub in (want_k[0, 0].tobytes(), want_k[0, 1].tobytes())


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_every_finite_key_verifies(curve):
    """the integer property: both recovered keys of a valid signature verify it (the oracle's ECDSA verify)"""
    hlen = 32
    sigs, dg, pubs = valid_items(curve, 24, hlen, 7900 + ALL_CURVES[curve][0])
    keys, st = host_recover(curve, sigs, dg, hlen)
    assert (st == 0).all()
    for k in range(2):
        assert (oracle_verify(curve, sigs, keys[:, k], dg, hlen) == 0).all()
    assert all(pubs[i].tobytes() in (keys[i, 0].tobytes(), keys[i, 1].tobytes()) for i in range(len(pubs)))


def test_bad_digest_length_is_refused():
    z = np.zeros(4096, np.uint8)
    st = np.full(2, 5, np.int8)
    for hlen in (0, 129):
        assert hostsim_lib().hostsim_ecdsa_recover(4, HOST_W, 1, _buf(z), _buf(z), hlen, _buf(z), _buf(st)) == -1
    assert (st == 5).all()
