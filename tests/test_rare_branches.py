"""The rare branches of the per-item signers and verifiers, driven through the production entry points with crafted
inputs that an attacker or an unlucky signer could send:

  - the final addition of the double-scalar core (window_mul adds a*G last) in its doubling branch (aG == bY) and at
    infinity (aG == -bY): ECDSA, ECFSDSA, ECSDSA / ECOSDSA through the generic double-scalar launch, BIP0340;
  - ECDSA's x(W') >= q candidate and, on FRP256V1 (q > p), an r in [p, q), which must not be reduced mod p;
  - ECDSA with u = e/s = 0 (the digest is 0 or q);
  - BIP0340's odd y(W') with x(W') == r;
  - the signers' restarts: ECDSA on e == r*d and s == 0, ECSDSA / ECOSDSA / ECFSDSA on s == 0 (status 2, no signature).

No vector needs a discrete logarithm: the test picks the private key, the public key or the nonce after the hash is
known.  CPU: every vector has the property it claims (Python integers and the oracle's scalar multiplications), the
reference (or, for the digest-only kinds, the oracle) gives the intended verdict or status, and the host build of the
kernel algorithms agrees.  GPU (`-m gpu`): each kind at lanes 0, 1, 63, 64 and 127 of a CTA of valid items, as one
whole CTA, and as the last item of batches of 3*128 - 1 and 3*128 + 1 items; the neighbours' results must not move
(the kernels share inversions across the 128 threads of a CTA, the host build does not)."""
import ctypes
import functools
import hashlib
import importlib.util
import os

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, PRIME, ROOT, hostsim_lib, make_signatures, oracle_sign, oracle_smul, \
    oracle_verify, ref_lib, rng, _buf
from test_bip0340 import challenge, oracle_bip_verify
from test_schnorr import ecsdsa_verify, oracle_double_smul, ref_verify
from test_schnorr_sign_host import HASHLIB, hostsim_sign, ref_sign, ref_sign_lib

_spec = importlib.util.spec_from_file_location("gen_curve_constants",
                                               os.path.join(ROOT, "tools", "gen_curve_constants.py"))
_gcc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_gcc)
CURVE_AB = {c: (v[2], v[3]) for c, v in _gcc.CURVES.items()}  # (id, p, a, b, q, gx, gy)

M = 4             # distinct vectors of each kind per curve
NFILL = 48        # distinct valid items per family and curve (cycled to fill the batches)
LANES = (0, 1, 63, 64, 127)
HOST_W = 6        # comb window of the host build
HNAME = {c: "SHA256" if ALL_CURVES[c][2] <= 32 else ("SHA384" if ALL_CURVES[c][2] <= 48 else "SHA512")
         for c in ALL_CURVES}


# ------------------------------------------------------------------------------------------ integers and points


def be(v, n):
    return np.frombuffer(int(v).to_bytes(n, "big"), np.uint8)


def b2i(b):
    return int.from_bytes(bytes(b), "big")


def inv(a, q):
    return pow(a, -1, q)


def sqrt_mod(v, p):
    """a square root of v mod p, or None; Tonelli-Shanks where p = 1 mod 4 (SECP224R1)"""
    v %= p
    if v == 0:
        return 0
    if pow(v, (p - 1) // 2, p) != 1:
        return None
    if p % 4 == 3:
        return pow(v, (p + 1) // 4, p)
    q, s = p - 1, 0
    while q % 2 == 0:
        q, s = q // 2, s + 1
    z = 2
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    m, c, t, r = s, pow(z, q, p), pow(v, q, p), pow(v, (q + 1) // 2, p)
    while t != 1:
        i, t2 = 0, t
        while t2 != 1:
            t2, i = t2 * t2 % p, i + 1
        b = pow(c, 1 << (m - i - 1), p)
        m, c, t, r = i, b * b % p, t * b * b % p, r * b % p
    return r


def point_with_x(curve, lo, hi, g):
    """a curve point (x, y) with x drawn uniformly from [lo, hi)"""
    p = PRIME[curve]
    a, b = CURVE_AB[curve]
    while True:
        x = lo + b2i(g.bytes(80)) % (hi - lo)
        y = sqrt_mod(x ** 3 + a * x + b, p)
        if y is not None:
            return x, (y if g.integers(0, 2) else (p - y) % p)


def wire(curve, pts):
    plen = ALL_CURVES[curve][1]
    return np.stack([np.concatenate([be(x, plen), be(y, plen)]) for x, y in pts])


def unwire(curve, row):
    plen = ALL_CURVES[curve][1]
    return b2i(row[:plen]), b2i(row[plen:])


def smul(curve, ks, pts=None):
    """affine k*G (or k*P) through the oracle; every result finite"""
    qlen = ALL_CURVES[curve][2]
    out, st = oracle_smul(curve, np.stack([be(k % ORDER[curve], qlen) for k in ks]),
                          wire(curve, pts) if pts is not None else None)
    assert (st == 0).all()
    return [unwire(curve, o) for o in out]


def dsmul(curve, a, b, pts):
    """(a*G + b*P, status) through the oracle: status 0 finite, 1 infinity"""
    qlen = ALL_CURVES[curve][2]
    ab = np.stack([np.concatenate([be(x % ORDER[curve], qlen), be(y % ORDER[curve], qlen)]) for x, y in zip(a, b)])
    out, st = oracle_double_smul(curve, ab, wire(curve, pts))
    return [unwire(curve, o) for o in out], st


def neg(curve, P):
    return P[0], (PRIME[curve] - P[1]) % PRIME[curve]


def lift_even(curve, d, P):
    """BIP0340's key d' with an even y(d'G), and d'G"""
    return (d, P) if P[1] % 2 == 0 else (ORDER[curve] - d, neg(curve, P))


def ecdsa_e(curve, digest):
    """the leftmost bitlen(q) bits of the digest, mod q (__ecdsa_verify_finalize)"""
    q, qlen = ORDER[curve], ALL_CURVES[curve][2]
    take = min(len(digest), qlen)
    return (b2i(digest[:take]) >> max(0, 8 * take - q.bit_length())) % q


def digest_of_e(curve, e):
    """qlen digest bytes whose ECDSA scalar is e (shifted left by 7 bits on SECP521R1)"""
    q, qlen = ORDER[curve], ALL_CURVES[curve][2]
    return be(e << (8 * qlen - q.bit_length()), qlen)


class Draw:
    def __init__(self, curve, tag):
        self.q = ORDER[curve]
        self.g = rng(tag)

    def scalar(self):
        return 1 + b2i(self.g.bytes(80)) % (self.q - 1)

    def msg(self):
        return self.g.bytes(int(self.g.integers(0, 90)))


def objs(xs):
    xs = list(xs)
    a = np.empty(len(xs), object)
    a[:] = xs
    return a


def cat(a, b):
    return {k: np.concatenate([a[k], b[k]]) for k in a}


def take(cols, idx):
    return {k: v[idx] for k, v in cols.items()}


def layouts(m, f):
    """Index vectors into concat(special[m], valid[f]): the special items at LANES of the first CTA, a whole CTA of them,
    valid items after that and a special item last, in batches of 3*128 - 1 and 3*128 + 1 items."""
    out = []
    for n in (3 * 128 - 1, 3 * 128 + 1):
        idx = m + np.arange(n) % f
        idx[list(LANES)] = np.arange(len(LANES)) % m
        idx[128:256] = np.arange(128) % m
        idx[-1] = (n + 1) % m
        out.append(idx)
    return out


def batches(fam, kind):
    """(columns, expected) of every batch that places `kind` among the family's valid items"""
    sel = np.flatnonzero(fam["items"]["kind"] == kind)
    pool = cat(take(fam["items"], sel), fam["valid"])
    for idx in layouts(len(sel), len(fam["valid"]["kind"])):
        yield take(pool, idx)


def need_reference():
    if ref_lib() is None or ref_sign_lib() is None:
        pytest.skip("compiled reference not available")


# ------------------------------------------------------------------------------------------ ECDSA verification


@functools.lru_cache(None)
def ecdsa_family(curve):
    """Vectors that verify from a real message (hash HNAME[curve]).  Per item: sig, pub, msg, dg, want (the
    reference's verdict), kind, intended verdict, and (u, v, W') for the property checks."""
    cid, plen, qlen = ALL_CURVES[curve]
    p, q = PRIME[curve], ORDER[curve]
    H = HASHLIB[HNAME[curve]]
    dr = Draw(curve, 61000 + cid)
    rows = []  # kind, intended, r, s, d or Y, msg, W'
    for kind, sign in (("double", 1), ("infinity", -1)):
        for _ in range(M):
            m, s = dr.msg(), dr.scalar()
            e = ecdsa_e(curve, H(m).digest())
            u = e * inv(s, q) % q
            W = smul(curve, [2 * u])[0]
            r = W[0] % q
            rows.append((kind, 0 if sign > 0 else -1, r, s, sign * e * inv(r, q) % q, m, W))
    if q < p:
        specs = [("x_above_q", 0, q + 1, p, q)]                   # r = x - q
    else:
        specs = [("r_above_p", -1, 1, q - p, -p), ("r_above_p_twin", 0, 1, q - p, 0)]  # r = x + p, and r = x
    for kind, want, lo, hi, shift in specs:
        for _ in range(M):
            W = point_with_x(curve, lo, hi, dr.g)
            r, s, m = W[0] - shift, dr.scalar(), dr.msg()
            e = ecdsa_e(curve, H(m).digest())
            u, v = e * inv(s, q) % q, r * inv(s, q) % q
            Y = dsmul(curve, [-u * inv(v, q)], [inv(v, q)], [W])[0][0]  # Y = W'/v - (u/v) G
            rows.append((kind, want, r, s, Y, m, W))
    # the key d as a scalar or Y as a point
    ds = [x[4] for x in rows if isinstance(x[4], int)]
    dpts = iter(smul(curve, ds))
    pubs = [x[4] if isinstance(x[4], tuple) else next(dpts) for x in rows]
    msgs = [x[5] for x in rows]
    sigs = np.stack([np.concatenate([be(x[2], qlen), be(x[3], qlen)]) for x in rows])
    dg = np.stack([np.frombuffer(H(m).digest(), np.uint8) for m in msgs])
    items = {"sig": sigs, "pub": wire(curve, pubs), "msg": objs(msgs), "dg": dg,
             "kind": objs(x[0] for x in rows), "intended": np.array([x[1] for x in rows], np.int8)}
    items["want"] = ref_verify_ecdsa(curve, items)
    aux = []
    for x, Y in zip(rows, pubs):
        e = ecdsa_e(curve, H(x[5]).digest())
        w = inv(x[3], q)
        aux.append((e * w % q, x[2] * w % q, Y, x[6]))
    # valid items: the oracle's signer on the digests of random messages
    vm = [dr.msg() for _ in range(NFILL)]
    vd = [dr.scalar() for _ in range(NFILL)]
    vdg = np.stack([np.frombuffer(H(m).digest(), np.uint8) for m in vm])
    vs, st = oracle_sign(curve, np.stack([be(d, qlen) for d in vd]),
                         np.stack([be(dr.scalar(), qlen) for _ in range(NFILL)]), vdg, vdg.shape[1])
    assert (st == 0).all()
    valid = {"sig": vs, "pub": wire(curve, smul(curve, vd)), "msg": objs(vm), "dg": vdg,
             "kind": objs(["valid"] * NFILL), "intended": np.zeros(NFILL, np.int8)}
    valid["want"] = ref_verify_ecdsa(curve, valid)
    return {"items": items, "valid": valid, "aux": aux, "hlen": dg.shape[1]}


def ref_verify_ecdsa(curve, cols):
    msgs = list(cols["msg"])
    blob = np.frombuffer(b"".join(msgs) or b"\0", np.uint8).copy()
    off = np.zeros(len(msgs) + 1, np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    v = np.zeros(len(msgs), np.int8)
    assert ref_lib().ref_ecdsa_verify_batch(curve.encode(), HNAME[curve].encode(), len(msgs), _buf(cols["sig"]),
                                            _buf(cols["pub"]), _buf(blob), _buf(off), _buf(v), 8) == 0
    return v


@functools.lru_cache(None)
def ecdsa_u0_family(curve):
    """u = e/s = 0: the digest (qlen bytes) is 0 or q; W' = vY with r = x(W') mod q.  Judged by the oracle."""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    dr = Draw(curve, 62000 + cid)
    ks = [dr.scalar() for _ in range(M)]
    Ws = smul(curve, ks)
    rows = []
    for j, (k, W) in enumerate(zip(ks, Ws)):
        r, s = W[0] % q, dr.scalar()
        v = r * inv(s, q) % q
        rows.append((r, s, k * inv(v, q) % q, np.zeros(qlen, np.uint8) if j % 2 == 0 else digest_of_e(curve, q), W))
    pubs = smul(curve, [x[2] for x in rows])
    items = {"sig": np.stack([np.concatenate([be(x[0], qlen), be(x[1], qlen)]) for x in rows]),
             "pub": wire(curve, pubs), "dg": np.stack([x[3] for x in rows]), "kind": objs(["u_zero"] * M),
             "intended": np.zeros(M, np.int8)}
    items["want"] = oracle_verify(curve, items["sig"], items["pub"], items["dg"], qlen)
    aux = [(0, x[0] * inv(x[1], q) % q, Y, x[4]) for x, Y in zip(rows, pubs)]
    vs, vp, vdg, vwant = make_signatures(curve, NFILL, tag=62100 + cid, hlen=qlen)
    valid = {"sig": vs, "pub": vp, "dg": vdg, "kind": objs(["valid"] * NFILL), "intended": np.zeros(NFILL, np.int8),
             "want": vwant}
    return {"items": items, "valid": valid, "aux": aux, "hlen": qlen}


def check_ecdsa_claims(curve, fam):
    """the property each vector is built for, in integers and through the oracle's scalar multiplications"""
    p, q = PRIME[curve], ORDER[curve]
    kinds, sigs = fam["items"]["kind"], fam["items"]["sig"]
    qlen = ALL_CURVES[curve][2]
    aux = fam["aux"]
    uG = smul(curve, [a[0] if a[0] else 1 for a in aux])
    vY = smul(curve, [a[1] for a in aux], [a[2] for a in aux])
    W, st = dsmul(curve, [a[0] for a in aux], [a[1] for a in aux], [a[2] for a in aux])
    for i, kind in enumerate(kinds):
        r, s = b2i(sigs[i, :qlen]), b2i(sigs[i, qlen:])
        assert 0 < r < q and 0 < s < q
        Wp = aux[i][3]
        if kind == "double":
            assert uG[i] == vY[i] and st[i] == 0 and W[i] == Wp and Wp[0] % q == r
        elif kind == "infinity":
            assert uG[i] == neg(curve, vY[i]) and st[i] == 1
        elif kind == "x_above_q":
            assert st[i] == 0 and W[i] == Wp and q <= Wp[0] < p and r == Wp[0] - q
        elif kind == "r_above_p":
            assert st[i] == 0 and W[i] == Wp and p <= r < q and Wp[0] == r - p and Wp[0] % q != r
        elif kind == "r_above_p_twin":
            assert st[i] == 0 and W[i] == Wp and Wp[0] == r < q - p
        elif kind == "u_zero":
            assert aux[i][0] == 0 and ecdsa_e(curve, bytes(fam["items"]["dg"][i])) == 0
            assert st[i] == 0 and vY[i] == W[i] == Wp and Wp[0] % q == r
        else:
            raise AssertionError(kind)


def ecdsa_kind_names(curve):
    return list(dict.fromkeys(ecdsa_family(curve)["items"]["kind"]))


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_ecdsa_verify_vectors(curve):
    need_reference()
    for fam in (ecdsa_family(curve), ecdsa_u0_family(curve)):
        check_ecdsa_claims(curve, fam)
        for part in ("items", "valid"):
            cols = fam[part]
            assert (cols["want"] == cols["intended"]).all(), (part, cols["kind"][cols["want"] != cols["intended"]])
            assert (oracle_verify(curve, cols["sig"], cols["pub"], cols["dg"], fam["hlen"]) == cols["want"]).all()
            got = np.full(len(cols["want"]), 7, np.int8)
            assert hostsim_lib().hostsim_ecdsa_verify_batch(ALL_CURVES[curve][0], HOST_W, len(got), _buf(cols["sig"]),
                                                            _buf(cols["pub"]), _buf(cols["dg"]), fam["hlen"],
                                                            _buf(got)) == 0
            assert (got == cols["want"]).all()
    kinds = set(ecdsa_family(curve)["items"]["kind"])
    assert kinds == ({"double", "infinity", "x_above_q"} if ORDER[curve] < PRIME[curve] else
                     {"double", "infinity", "r_above_p", "r_above_p_twin"})


def test_frp256v1_is_the_only_curve_with_q_above_p():
    assert [c for c in ALL_CURVES if ORDER[c] > PRIME[c]] == ["FRP256V1"]


# ------------------------------------------------------------------------------------------ Schnorr-type verification


def pack_sigs(rows):
    return np.stack([np.concatenate(r) for r in rows])


@functools.lru_cache(None)
def ecfsdsa_family(curve):
    """ECFSDSA (hash HNAME[curve]): the doubling branch (d = -k/(2h), signed by the reference with nonce k) and
    W' = infinity (s = h*d forged on a reference signature).  dg = H(R || m), the device's input."""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    hname = HNAME[curve]
    H = HASHLIB[hname]
    dr = Draw(curve, 63000 + cid)
    ks = [dr.scalar() for _ in range(M)]
    Rs = smul(curve, ks)
    msgs = [dr.msg() for _ in range(2 * M)]
    hs = [b2i(H(bytes(wire(curve, [R])[0]) + m).digest()) % q for R, m in zip(Rs, msgs)]
    dbl_d = [-k * inv(2 * h, q) % q for k, h in zip(ks, hs)]
    inf_d = [dr.scalar() for _ in range(M)]
    privs = np.stack([be(d, qlen) for d in dbl_d + inf_d])
    rand = np.stack([be(k, qlen) for k in ks] + [be(dr.scalar(), qlen) for _ in range(M)])
    sigs, pubs, st = ref_sign(curve, "ECFSDSA", hname, privs, rand, msgs)
    assert (st == 0).all()
    for i in range(M, 2 * M):                                  # s = h*d: W' = hd G - hd G
        h = b2i(H(bytes(sigs[i, :2 * plen]) + msgs[i]).digest()) % q
        sigs[i, 2 * plen:] = be(h * inf_d[i - M] % q, qlen)
    items = {"sig": sigs, "pub": pubs, "msg": objs(msgs), "kind": objs(["double"] * M + ["infinity"] * M),
             "intended": np.array([0] * M + [-1] * M, np.int8)}
    vm = [dr.msg() for _ in range(NFILL)]
    vs, vp, st = ref_sign(curve, "ECFSDSA", hname, np.stack([be(dr.scalar(), qlen) for _ in range(NFILL)]),
                          np.stack([be(dr.scalar(), qlen) for _ in range(NFILL)]), vm)
    assert (st == 0).all()
    valid = {"sig": vs, "pub": vp, "msg": objs(vm), "kind": objs(["valid"] * NFILL),
             "intended": np.zeros(NFILL, np.int8)}
    for cols in (items, valid):
        cols["dg"] = np.stack([np.frombuffer(H(bytes(s[:2 * plen]) + m).digest(), np.uint8)
                               for s, m in zip(cols["sig"], cols["msg"])])
        cols["want"] = ref_verify(curve, "ECFSDSA", hname, cols["sig"], cols["pub"], list(cols["msg"]))
    return {"items": items, "valid": valid, "hlen": H().digest_size, "hash": hname}


@functools.lru_cache(None)
def bip0340_family(curve):
    """BIP0340 (SHA-256): W' = infinity (s = e*d' forged) and an odd y(W') with x(W') = r (s = k + e*d' for a k with
    y(kG) odd, not negated).  dg = the tagged challenge hash, the device's input."""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    dr = Draw(curve, 64000 + cid)
    ds = [dr.scalar() for _ in range(2 * M)]
    Ps = smul(curve, ds)
    ks = []
    while len(ks) < 2 * M:                                      # nonces with y(kG) odd (the W' = inf rows use its x)
        k = dr.scalar()
        if smul(curve, [k])[0][1] % 2:
            ks.append(k)
    Rs = smul(curve, ks)
    rows, msgs = [], []
    for j, (d, P, k, R) in enumerate(zip(ds, Ps, ks, Rs)):
        m = dr.msg()
        dl, _ = lift_even(curve, d, P)
        e = b2i(challenge("SHA256", be(R[0], plen), be(P[0], plen), m)) % q
        s = e * dl % q if j < M else (k + e * dl) % q
        rows.append((be(R[0], plen), be(s, qlen)))
        msgs.append(m)
    items = {"sig": pack_sigs(rows), "pub": wire(curve, Ps), "msg": objs(msgs),
             "kind": objs(["infinity"] * M + ["odd_y"] * M), "intended": np.full(2 * M, -1, np.int8)}
    from test_bip0340 import ref_sign as ref_bip_sign
    vm = [dr.msg() for _ in range(NFILL)]
    vs, vp = ref_bip_sign(curve, "SHA256", np.stack([be(dr.scalar(), qlen) for _ in range(NFILL)]), vm)
    valid = {"sig": vs, "pub": vp, "msg": objs(vm), "kind": objs(["valid"] * NFILL),
             "intended": np.zeros(NFILL, np.int8)}
    for cols in (items, valid):
        cols["dg"] = np.stack([challenge("SHA256", s[:plen], pk[:plen], m)
                               for s, pk, m in zip(cols["sig"], cols["pub"], cols["msg"])])
        cols["want"] = ref_verify(curve, "BIP0340", "SHA256", cols["sig"], cols["pub"], list(cols["msg"]))
    return {"items": items, "valid": valid, "hlen": 32, "hash": "SHA256", "ks": ks}


@functools.lru_cache(None)
def ecsdsa_family(curve):
    """ECSDSA and ECOSDSA (hash HNAME[curve]) in their doubling branch, d = -k/(2e) signed by the reference with
    nonce k, verified through the generic double-scalar multiplication; kind names carry the scheme."""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    hname = HNAME[curve]
    H = HASHLIB[hname]
    dr = Draw(curve, 65000 + cid)
    fam = {}
    for alg in ("ECSDSA", "ECOSDSA"):
        ks = [dr.scalar() for _ in range(M)]
        Ws = wire(curve, smul(curve, ks))
        msgs = [dr.msg() for _ in range(M)]
        pre = (lambda w: bytes(w)) if alg == "ECSDSA" else (lambda w: bytes(w[:plen]))
        es = [b2i(H(pre(w) + m).digest()) % q for w, m in zip(Ws, msgs)]
        privs = np.stack([be(-k * inv(2 * e, q) % q, qlen) for k, e in zip(ks, es)])
        sigs, pubs, st = ref_sign(curve, alg, hname, privs, np.stack([be(k, qlen) for k in ks]), msgs)
        assert (st == 0).all()
        items = {"sig": sigs, "pub": pubs, "msg": objs(msgs), "kind": objs([alg + "_double"] * M),
                 "intended": np.zeros(M, np.int8)}
        vm = [dr.msg() for _ in range(NFILL)]
        vs, vp, st = ref_sign(curve, alg, hname, np.stack([be(dr.scalar(), qlen) for _ in range(NFILL)]),
                              np.stack([be(dr.scalar(), qlen) for _ in range(NFILL)]), vm)
        assert (st == 0).all()
        valid = {"sig": vs, "pub": vp, "msg": objs(vm), "kind": objs(["valid"] * NFILL),
                 "intended": np.zeros(NFILL, np.int8)}
        for cols in (items, valid):
            cols["want"] = ref_verify(curve, alg, hname, cols["sig"], cols["pub"], list(cols["msg"]))
        fam[alg] = {"items": items, "valid": valid, "hash": hname}
    return fam


@functools.lru_cache(None)
def double_smul_family(curve):
    """Raw a*G + b*Y: aG == bY (b = a/d, Y = dG: the doubling branch), aG == -bY and a = b = 0 (infinity).
    want / out: the oracle's status and affine result."""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    dr = Draw(curve, 66000 + cid)
    a = [dr.scalar() for _ in range(2 * M)] + [0] * M
    d = [dr.scalar() for _ in range(3 * M)]
    b = [x * inv(y, q) % q for x, y in zip(a[:M], d)] + [-x * inv(y, q) % q for x, y in zip(a[M:2 * M], d[M:])] + [0] * M
    Ys = smul(curve, d)

    def cols_of(a, b, Ys, kinds, intended):
        ab = np.stack([np.concatenate([be(x, qlen), be(y, qlen)]) for x, y in zip(a, b)])
        out, st = oracle_double_smul(curve, ab, wire(curve, Ys))
        return {"ab": ab, "pub": wire(curve, Ys), "out": out, "want": st, "kind": objs(kinds),
                "intended": np.array(intended, np.int8)}
    items = cols_of(a, b, Ys, ["aG_eq_bY"] * M + ["aG_eq_minus_bY"] * M + ["zero"] * M, [0] * M + [1] * (2 * M))
    valid = cols_of([dr.scalar() for _ in range(NFILL)], [dr.scalar() for _ in range(NFILL)],
                    smul(curve, [dr.scalar() for _ in range(NFILL)]), ["valid"] * NFILL, [0] * NFILL)
    return {"items": items, "valid": valid, "a": a, "b": b, "Y": Ys}


def host_double_smul(curve):
    def run(ab, pk):
        n = ab.shape[0]
        out = np.zeros((n, 2 * ALL_CURVES[curve][1]), np.uint8)
        st = np.zeros(n, np.int8)
        assert hostsim_lib().hostsim_double_smul_batch(ALL_CURVES[curve][0], HOST_W, n, _buf(ab), _buf(pk), _buf(out),
                                                       _buf(st)) == 0
        return out, st
    return run


def host_verify(curve, fn, cols, hlen):
    got = np.full(len(cols["want"]), 7, np.int8)
    assert getattr(hostsim_lib(), fn)(ALL_CURVES[curve][0], HOST_W, len(got), _buf(cols["sig"]), _buf(cols["pub"]),
                                      _buf(cols["dg"]), hlen, _buf(got)) == 0
    return got


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_schnorr_verify_vectors(curve):
    need_reference()
    _, plen, qlen = ALL_CURVES[curve]
    p, q = PRIME[curve], ORDER[curve]
    # ECFSDSA: s*G against (-h)*Y, the two operands of the final addition
    fam = ecfsdsa_family(curve)
    it = fam["items"]
    h = [b2i(d) % q for d in it["dg"]]
    s = [b2i(x[2 * plen:]) for x in it["sig"]]
    Y = [unwire(curve, x) for x in it["pub"]]
    sG, bY = smul(curve, s), smul(curve, [-x for x in h], Y)
    for i, kind in enumerate(it["kind"]):
        assert sG[i] == (bY[i] if kind == "double" else neg(curve, bY[i])), kind
    for cols in (it, fam["valid"]):
        assert (cols["want"] == cols["intended"]).all()
        assert (host_verify(curve, "hostsim_ecfsdsa_verify_batch", cols, fam["hlen"]) == cols["want"]).all()
    # BIP0340: s*G against e*Y' (Y' the key lifted to an even y)
    fam = bip0340_family(curve)
    it = fam["items"]
    for i, kind in enumerate(it["kind"]):
        P = unwire(curve, it["pub"][i])
        e = b2i(it["dg"][i]) % q
        r, s = b2i(it["sig"][i, :plen]), b2i(it["sig"][i, plen:])
        Yl = lift_even(curve, 1, P)[1]
        W, st = dsmul(curve, [s], [-e], [Yl])
        if kind == "infinity":
            assert smul(curve, [s])[0] == smul(curve, [e], [Yl])[0] and st[0] == 1
        else:
            k = fam["ks"][i]
            assert st[0] == 0 and W[0] == smul(curve, [k])[0] and W[0][0] == r and W[0][1] % 2 == 1
    for cols in (it, fam["valid"]):
        assert (cols["want"] == cols["intended"]).all()
        assert (oracle_bip_verify(curve, cols["sig"], cols["pub"], cols["dg"], 32) == cols["want"]).all()
        assert (host_verify(curve, "hostsim_bip0340_verify_batch", cols, 32) == cols["want"]).all()
    # ECSDSA / ECOSDSA: s*G against (-r mod q)*Y, then the reference's verification around the host build
    for alg, fam in ecsdsa_family(curve).items():
        it = fam["items"]
        hl = HASHLIB[fam["hash"]]().digest_size
        e = [-b2i(x[:hl]) % q for x in it["sig"]]
        s = [b2i(x[hl:]) for x in it["sig"]]
        assert smul(curve, s) == smul(curve, e, [unwire(curve, x) for x in it["pub"]])
        for cols in (it, fam["valid"]):
            assert (cols["want"] == cols["intended"]).all()
            got = ecsdsa_verify(curve, fam["hash"], alg == "ECOSDSA", cols["sig"], cols["pub"], list(cols["msg"]),
                                host_double_smul(curve))
            assert (got == cols["want"]).all()
    # raw double-scalar rows
    fam = double_smul_family(curve)
    it = fam["items"]
    aG = smul(curve, [a if a else 1 for a in fam["a"]])
    bY = smul(curve, [b if b else 1 for b in fam["b"]], fam["Y"])
    for i, kind in enumerate(it["kind"]):
        if kind == "aG_eq_bY":
            assert aG[i] == bY[i] and unwire(curve, it["out"][i]) == smul(curve, [2 * fam["a"][i]])[0]
        elif kind == "aG_eq_minus_bY":
            assert aG[i] == neg(curve, bY[i])
        else:
            assert fam["a"][i] == fam["b"][i] == 0
    for cols in (it, fam["valid"]):
        assert (cols["want"] == cols["intended"]).all()
        out, st = host_double_smul(curve)(cols["ab"], cols["pub"])
        assert (st == cols["want"]).all() and (out == cols["out"]).all()


# ------------------------------------------------------------------------------------------ signer restarts


@functools.lru_cache(None)
def ecdsa_sign_family(curve):
    """ECDSA signing on digests of qlen bytes: e = r*d (the explicit restart test) and e = -r*d (s == 0), r = x(kG)
    mod q.  want / sig: the oracle's status and signature."""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    dr = Draw(curve, 67000 + cid)
    ks = [dr.scalar() for _ in range(2 * M)]
    ds = [dr.scalar() for _ in range(2 * M)]
    rs = [W[0] % q for W in smul(curve, ks)]
    es = [(1 if j < M else -1) * r * d % q for j, (r, d) in enumerate(zip(rs, ds))]

    def cols_of(ds, ks, dg, kinds, intended):
        cols = {"priv": np.stack([be(d, qlen) for d in ds]), "nonce": np.stack([be(k, qlen) for k in ks]), "dg": dg,
                "kind": objs(kinds), "intended": np.array(intended, np.int8)}
        cols["sig"], cols["want"] = oracle_sign(curve, cols["priv"], cols["nonce"], dg, qlen)
        return cols
    items = cols_of(ds, ks, np.stack([digest_of_e(curve, e) for e in es]), ["e_eq_rd"] * M + ["s_zero"] * M,
                    [2] * (2 * M))
    valid = cols_of([dr.scalar() for _ in range(NFILL)], [dr.scalar() for _ in range(NFILL)],
                    dr.g.integers(0, 256, size=(NFILL, qlen), dtype=np.uint8), ["valid"] * NFILL, [0] * NFILL)
    return {"items": items, "valid": valid, "r": rs, "e": es, "d": ds, "hlen": qlen}


SIGN_CASES = [(a, h) for a in ("ECSDSA", "ECOSDSA", "ECFSDSA") for h in ("SHA256", "SHA3_256")]


@functools.lru_cache(None)
def schnorr_sign_family(curve, alg, hname):
    """s == 0: d = -k/e with e the scheme's hash of W = kG and the message, reduced mod q.  want / sig: the status and
    signature of the reference's signer with the nonce injected."""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    H = HASHLIB[hname]
    dr = Draw(curve, 68000 + 100 * cid + 10 * [a for a, _ in SIGN_CASES].index(alg) + (hname == "SHA3_256"))
    ks = [dr.scalar() for _ in range(M)]
    Ws = wire(curve, smul(curve, ks))
    msgs = [dr.msg() for _ in range(M)]
    es = [b2i(H((bytes(w) if alg != "ECOSDSA" else bytes(w[:plen])) + m).digest()) % q for w, m in zip(Ws, msgs)]

    def cols_of(ds, ks, msgs, kinds, intended):
        cols = {"priv": np.stack([be(d, qlen) for d in ds]), "nonce": np.stack([be(k, qlen) for k in ks]),
                "msg": objs(msgs), "kind": objs(kinds), "intended": np.array(intended, np.int8)}
        cols["sig"], _, cols["want"] = ref_sign(curve, alg, hname, cols["priv"], cols["nonce"], msgs)
        return cols
    items = cols_of([-k * inv(e, q) % q for k, e in zip(ks, es)], ks, msgs, ["s_zero"] * M, [2] * M)
    valid = cols_of([dr.scalar() for _ in range(NFILL)], [dr.scalar() for _ in range(NFILL)],
                    [dr.msg() for _ in range(NFILL)], ["valid"] * NFILL, [0] * NFILL)
    return {"items": items, "valid": valid, "k": ks, "e": es, "alg": alg, "hash": hname}


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_sign_restart_vectors(curve):
    need_reference()
    q = ORDER[curve]
    fam = ecdsa_sign_family(curve)
    it = fam["items"]
    for i, kind in enumerate(it["kind"]):
        r, d, e = fam["r"][i], fam["d"][i], fam["e"][i]
        assert ecdsa_e(curve, bytes(it["dg"][i])) == e
        assert e == (r * d % q if kind == "e_eq_rd" else -r * d % q)
    for cols in (it, fam["valid"]):
        assert (cols["want"] == cols["intended"]).all()
    assert not it["sig"].any()
    for alg, hname in SIGN_CASES:
        fam = schnorr_sign_family(curve, alg, hname)
        it = fam["items"]
        for i in range(M):
            assert (fam["k"][i] + fam["e"][i] * b2i(it["priv"][i])) % q == 0
        for cols in (it, fam["valid"]):
            assert (cols["want"] == cols["intended"]).all(), (alg, hname)
            sigs, st = hostsim_sign(curve, alg, hname, cols["priv"], cols["nonce"], list(cols["msg"]))
            assert (st == cols["want"]).all() and (sigs == cols["sig"]).all(), (alg, hname)
        assert not it["sig"].any()


# ------------------------------------------------------------------------------------------ on the device

ENGINES = [(c, 8) for c in ALL_CURVES] + [("FRP256V1", 0), ("SECP256R1", 0)]  # 0: the default comb window
_engines = {}


def engine(curve, w):
    import libecc_b200
    if (curve, w) not in _engines:
        _engines[(curve, w)] = libecc_b200.Engine(curve, device=0, comb_window=w)
    return _engines[(curve, w)]


@pytest.fixture
def release_engines():
    """every test gives its engines (tables, stage buffers) back: other test modules keep theirs for the whole run"""
    yield
    import torch
    for eng in _engines.values():
        eng.close()
    _engines.clear()
    torch.cuda.empty_cache()


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def projective(curve, pubs, g):
    """affine keys as X || Y || Z with a random Z != 1 (homogeneous: x = X/Z, y = Y/Z)"""
    p = PRIME[curve]
    out = []
    for row in pubs:
        x, y = unwire(curve, row)
        z = 2 + b2i(g.bytes(80)) % (p - 2)
        out.append(np.concatenate([wire(curve, [(x * z % p, y * z % p)])[0], be(z, ALL_CURVES[curve][1])]))
    return np.stack(out)


@pytest.mark.gpu
@pytest.mark.parametrize("curve,w", ENGINES)
def test_gpu_ecdsa_verify(curve, w, release_engines):
    import torch
    need_reference()
    eng = engine(curve, w)
    g = rng(69000)
    for fam in (ecdsa_family(curve), ecdsa_u0_family(curve)):
        hlen = fam["hlen"]
        for kind in dict.fromkeys(fam["items"]["kind"]):
            for b in batches(fam, kind):
                want = b["want"]
                assert (eng.ecdsa_verify_batch(b["sig"], b["pub"], b["dg"], hlen) == want).all(), kind
                d_v = torch.full((len(want),), 7, dtype=torch.int8, device="cuda")
                eng.ecdsa_verify_batch_dev(cuda(b["sig"]), cuda(b["pub"]), cuda(b["dg"]), hlen, d_v)
                torch.cuda.synchronize()
                assert (d_v.cpu().numpy() == want).all(), kind
                assert (eng.ecdsa_verify_prj_batch(b["sig"], projective(curve, b["pub"], g), b["dg"], hlen)
                        == want).all(), kind
                if "msg" in b:
                    assert (eng.ecdsa_verify_msgs_batch(HNAME[curve], b["sig"], b["pub"], list(b["msg"]))
                            == want).all(), kind


@pytest.mark.gpu
@pytest.mark.parametrize("curve,w", ENGINES)
def test_gpu_schnorr_verify(curve, w, release_engines):
    need_reference()
    eng = engine(curve, w)
    for name, fn in (("ecfsdsa", eng.ecfsdsa_verify_batch), ("bip0340", eng.bip0340_verify_batch)):
        fam = ecfsdsa_family(curve) if name == "ecfsdsa" else bip0340_family(curve)
        for kind in dict.fromkeys(fam["items"]["kind"]):
            for b in batches(fam, kind):
                assert (fn(b["sig"], b["pub"], b["dg"], fam["hlen"]) == b["want"]).all(), (name, kind)
    for alg, fam in ecsdsa_family(curve).items():
        for kind in dict.fromkeys(fam["items"]["kind"]):
            for b in batches(fam, kind):
                got = ecsdsa_verify(curve, fam["hash"], alg == "ECOSDSA", b["sig"], b["pub"], list(b["msg"]),
                                    eng.double_smul_batch)
                assert (got == b["want"]).all(), kind
    fam = double_smul_family(curve)
    for kind in dict.fromkeys(fam["items"]["kind"]):
        for b in batches(fam, kind):
            out, st = eng.double_smul_batch(b["ab"], b["pub"])
            assert (st == b["want"]).all() and (out == b["out"]).all(), kind


@pytest.mark.gpu
@pytest.mark.parametrize("curve,w", ENGINES)
def test_gpu_sign_restarts(curve, w, release_engines):
    import torch
    need_reference()
    from test_gpu_schnorr_sign import sign_dev
    from test_gpu_structured import ref_keygen
    eng = engine(curve, w)
    _, plen, qlen = ALL_CURVES[curve]
    fam = ecdsa_sign_family(curve)
    hlen = fam["hlen"]
    recs = {}
    for kind in dict.fromkeys(fam["items"]["kind"]):
        for b in batches(fam, kind):
            n = len(b["want"])
            sigs, st = eng.ecdsa_sign_batch(b["priv"], b["nonce"], b["dg"], hlen)
            assert (st == b["want"]).all() and (sigs == b["sig"]).all(), kind
            d_s = torch.full((n, 2 * qlen), 0x5A, dtype=torch.uint8, device="cuda")
            d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
            args = [cuda(b["priv"]), cuda(b["nonce"]), cuda(b["dg"])]
            assert eng.lib.eccb200_ecdsa_sign_batch_dev(eng._h, n, *[a.data_ptr() for a in args], hlen, d_s.data_ptr(),
                                                        d_st.data_ptr(), None) == 0
            torch.cuda.synchronize()
            assert (d_st.cpu().numpy() == b["want"]).all() and (d_s.cpu().numpy() == b["sig"]).all(), kind
            for row in b["priv"]:
                if bytes(row) not in recs:
                    rc, prec, _ = ref_keygen(curve, bytes(row))
                    assert rc == 0
                    recs[bytes(row)] = prec
            prec = np.stack([recs[bytes(row)] for row in b["priv"]])
            out, st = eng.ecdsa_sign_structured_batch(prec, prec.shape[1] - 3, b["nonce"], HNAME[curve], b["dg"], hlen)
            assert (st == b["want"]).all() and (out[:, 3:] == b["sig"]).all(), kind
    for alg, hname in SIGN_CASES:
        fam = schnorr_sign_family(curve, alg, hname)
        for b in batches(fam, "s_zero"):
            sigs, st = eng.schnorr_sign_msgs_batch(alg, hname, b["priv"], b["nonce"], list(b["msg"]))
            assert (st == b["want"]).all() and (sigs == b["sig"]).all(), (alg, hname)
            sigs, st = sign_dev(eng, alg, hname, b["priv"], b["nonce"], list(b["msg"]))
            assert (st == b["want"]).all() and (sigs == b["sig"]).all(), (alg, hname)


@pytest.mark.gpu
@pytest.mark.parametrize("curve,alg", [("FRP256V1", "ECFSDSA"), ("SECP521R1", "ECFSDSA"), ("SECP256K1", "BIP0340")])
def test_gpu_msm_batch_with_rare_branches(curve, alg, release_engines):
    """K6 (the whole batch as one multi-scalar multiplication): 2^16 valid signatures that take the rare branches of the
    per-item kernel accept; one forgery among them rejects the batch, and the per-item kernel names it."""
    need_reference()
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    eng = engine(curve, 8)
    dr = Draw(curve, 69100)
    if alg == "ECFSDSA":
        fam = ecfsdsa_family(curve)
        hname, H = fam["hash"], HASHLIB[fam["hash"]]
        ds = [dr.scalar() for _ in range(8)]
        msgs = [dr.msg() for _ in range(8)]
        nonces = np.stack([be(d if j % 2 else q - d, qlen) for j, d in enumerate(ds)])  # nonce point Y and -Y
        sigs, pubs, st = ref_sign(curve, alg, hname, np.stack([be(d, qlen) for d in ds]), nonces, msgs)
        assert (st == 0).all() and (ref_verify(curve, alg, hname, sigs, pubs, msgs) == 0).all()
        Rs = [unwire(curve, s[:2 * plen]) for s in sigs]
        Ys = [unwire(curve, x) for x in pubs]
        assert all(R == (Y if j % 2 else neg(curve, Y)) for j, (R, Y) in enumerate(zip(Rs, Ys)))
        dg = np.stack([np.frombuffer(H(bytes(s[:2 * plen]) + m).digest(), np.uint8) for s, m in zip(sigs, msgs)])
        verify, msm = eng.ecfsdsa_verify_batch, eng.ecfsdsa_verify_msm_batch
        forged = np.flatnonzero(fam["items"]["kind"] == "infinity")[0]
    else:
        fam = bip0340_family(curve)
        ds = [dr.scalar() for _ in range(8)]
        Ps = smul(curve, ds)
        msgs = [dr.msg() for _ in range(8)]
        rows = []
        for d, P, m in zip(ds, Ps, msgs):                         # nonce point Y' (k = d' and k = q - d' sign alike)
            dl, Pl = lift_even(curve, d, P)
            e = b2i(challenge("SHA256", be(P[0], plen), be(P[0], plen), m)) % q
            rows.append((be(P[0], plen), be(dl * (1 + e) % q, qlen)))
        sigs, pubs = pack_sigs(rows), wire(curve, Ps)
        assert (ref_verify(curve, alg, "SHA256", sigs, pubs, msgs) == 0).all()
        dg = np.stack([challenge("SHA256", s[:plen], pk[:plen], m) for s, pk, m in zip(sigs, pubs, msgs)])
        verify, msm = eng.bip0340_verify_batch, eng.bip0340_verify_msm_batch
        forged = np.flatnonzero(fam["items"]["kind"] == "odd_y")[0]
    it, va = fam["items"], fam["valid"]
    ok = it["want"] == 0                                        # the doubling-branch ECFSDSA signatures
    assert ok.any() == (alg == "ECFSDSA")
    S = np.concatenate([it["sig"][ok], sigs, va["sig"]])
    P = np.concatenate([it["pub"][ok], pubs, va["pub"]])
    D = np.concatenate([it["dg"][ok], dg, va["dg"]])
    reps = -(-(1 << 16) // len(S))
    S, P, D = (np.tile(x, (reps, 1))[:1 << 16] for x in (S, P, D))
    hlen = D.shape[1]
    assert msm(S, P, D, hlen)
    j = 40000
    S[j], P[j], D[j] = it["sig"][forged], it["pub"][forged], it["dg"][forged]
    assert not msm(S, P, D, hlen)
    v = verify(S, P, D, hlen)
    assert v[j] == -1 and (np.delete(v, j) == 0).all()
