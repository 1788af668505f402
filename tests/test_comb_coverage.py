"""Every entry of the fixed-base comb table, and the last-digit doubling of the variable-base window.

A comb result reads one table entry per window, so a wrong entry (window i, digit d) corrupts only the scalars whose
digit i is d: about 1 in 2^w of random scalars.  cover() builds, for a curve and a width, a set of scalars below q that
reads every entry a reduced scalar can address, in chunks of at most 2^22:

  - item j in [0, 2^w) takes digit (a_i * j + b_i) mod 2^w in window i < nwin - 1 (a_i odd and seeded, so each window
    sees each digit exactly once, and the windows are decorrelated), and j mod T in the top window, where
    T = (q - 1) >> (w * (nwin - 1)) is the largest top digit of a scalar below q;
  - extras: the top digit T itself under lower parts 0, (q - 1) mod 2^(w * (nwin - 1)) and random values in between,
    0, 1, q - 1, and raw scalars >= q.

CPU: the sets address every (window, digit) pair (fully up to w = 16, on a seeded sample per chunk above), and the host
build of comb_mul agrees with the oracle on the complete sets at w = 4 and 5.  GPU (`-m gpu`): the whole set through
the fixed-base kernel (K1) against the variable-base kernel (K2) on the same scalars with P = G (K2 never reads the
table), bit for bit with the statuses, at the benchmarked widths (bench.DEFAULT_COMB), the default width and the widths
that exercise each way of building the table; a seeded sample and the extras also against the oracle.

window_mul (ec.cuh) recodes k into signed 4-bit digits and adds d*P after every four doublings.  Before the last digit
the accumulator is (k - d)*P, which equals the table point d*P when k = 2d (mod q): add_mixed then takes its P == Q
branch.  recoding_collisions() models the recoding and finds that scalar, q - 2*(q mod 16), exactly when q mod 16 is in
[1, 8].  Each entry point whose window_mul scalar a caller can choose gets crafted items that take that branch, checked
against the oracle or the reference on the CPU (host build) and on the GPU (at lanes 0, 1, 63, 64, 127 of a CTA of
valid items, as a whole CTA, and last in batches of 3*128 +- 1).

The tables here reach 43 GB, so each test closes its engines.  The module name sorts before the GPU modules that keep
their engines for the whole run, so the widest tables are built while the device is still empty."""
import functools

import numpy as np
import pytest

import bench
from common import ALL_CURVES, HASHLEN, ORDER, PRIME, _buf, hostsim_lib, make_signatures, oracle_smul, oracle_verify, \
    rng
from test_bip0340 import oracle_bip_verify
from test_ecdsa_recover_host import host_recover, need_ref, ref_recover, valid_items
from test_ecfsdsa import oracle_fs_verify
from test_rare_branches import HNAME, HOST_W, NFILL, Draw, b2i, batches, be, digest_of_e, host_double_smul, host_verify, \
    lift_even, objs, point_with_x, smul, wire
from test_schnorr import oracle_double_smul

CHUNK = 1 << 22   # items per device call and per host comparison
SAMPLE = 4096     # items of each (curve, width) compared with the oracle, besides the extras
M = 4             # crafted items of each kind per curve

# ------------------------------------------------------------------------------------------ covering scalars


def geometry(curve, w):
    """(nwin, T): the comb's windows, and the largest top-window digit of a scalar below q"""
    q = ORDER[curve]
    nwin = -(-q.bit_length() // w)
    return nwin, (q - 1) >> (w * (nwin - 1))


def multipliers(curve, w):
    """(a, b) of the lower windows: a_i odd, so j -> a_i * j + b_i is a permutation of [0, 2^w)"""
    nwin, _ = geometry(curve, w)
    g = rng(9000 + 100 * ALL_CURVES[curve][0] + w)
    a = 2 * g.integers(0, 1 << (w - 1), size=nwin - 1, dtype=np.uint64) + np.uint64(1)
    b = g.integers(0, 1 << w, size=nwin - 1, dtype=np.uint64)
    return a, b


def nwords(curve):
    return (8 * ALL_CURVES[curve][2] + 63) // 32   # little-endian 32-bit words, one spare


def item_digits(curve, w, j):
    """the comb digits of items j (uint64 array), one column per window"""
    nwin, T = geometry(curve, w)
    a, b = multipliers(curve, w)
    d = np.empty((len(j), nwin), np.uint64)
    d[:, :-1] = (j[:, None] * a + b) & np.uint64((1 << w) - 1)
    d[:, -1] = j % np.uint64(T)
    return d


def pack(curve, w, digits):
    """qlen-byte big-endian scalars from their comb digits"""
    qlen = ALL_CURVES[curve][2]
    nw = nwords(curve)
    words = np.zeros((len(digits), nw), np.uint64)
    for i in range(digits.shape[1]):
        k, s = (w * i) >> 5, (w * i) & 31
        v = digits[:, i] << np.uint64(s)
        words[:, k] |= v & np.uint64(0xFFFFFFFF)
        words[:, k + 1] |= v >> np.uint64(32)
    raw = words.astype("<u4").view(np.uint8)[:, ::-1]
    assert not raw[:, :4 * nw - qlen].any()
    return np.ascontiguousarray(raw[:, 4 * nw - qlen:])


def windows_of(curve, w, sc):
    """the comb digits of scalars (already reduced), one column per window: what comb_mul reads"""
    qlen = ALL_CURVES[curve][2]
    nw = nwords(curve)
    nwin, _ = geometry(curve, w)
    buf = np.zeros((len(sc), 4 * nw), np.uint8)
    buf[:, 4 * nw - qlen:] = sc
    words = np.ascontiguousarray(buf[:, ::-1]).view("<u4").astype(np.uint64)
    out = np.empty((len(sc), nwin), np.uint64)
    for i in range(nwin):
        k, s = (w * i) >> 5, (w * i) & 31
        out[:, i] = ((words[:, k] | (words[:, k + 1] << np.uint64(32))) >> np.uint64(s)) & np.uint64((1 << w) - 1)
    return out


def rows(curve, vals):
    qlen = ALL_CURVES[curve][2]
    return np.frombuffer(b"".join(int(v).to_bytes(qlen, "big") for v in vals), np.uint8).reshape(-1, qlen).copy()


def extra_values(curve, w):
    """the top digit T over lower parts 0, max and random; 0, 1, q - 1; raw scalars >= q (Python integers)"""
    q, qlen = ORDER[curve], ALL_CURVES[curve][2]
    nwin, T = geometry(curve, w)
    sh = w * (nwin - 1)
    lmax = (q - 1) & ((1 << sh) - 1)
    g = rng(9001 + 100 * ALL_CURVES[curve][0] + w)
    lows = [0, lmax] + [b2i(g.bytes(8 * qlen)) % (lmax + 1) for _ in range(14)]
    vals = [(T << sh) | lo for lo in lows] + [0, 1, q - 1]
    top = 1 << (8 * qlen)
    raw = [v + m * q for v in vals[:3] + vals[-3:] for m in (1, 2, 3) if v + m * q < top] + [top - 1]
    return vals + raw


def cover(curve, w, chunk=CHUNK):
    """(first item, scalars) chunks of the covering set, then (None, the extras)"""
    n = 1 << w
    for lo in range(0, n, chunk):
        j = np.arange(lo, min(n, lo + chunk), dtype=np.uint64)
        yield lo, pack(curve, w, item_digits(curve, w, j))
    yield None, rows(curve, extra_values(curve, w))


def below(sc, bound):
    """rows of big-endian scalars that are < bound (same width)"""
    d = sc.astype(np.int16) - bound.astype(np.int16)
    nz = d != 0
    first = nz.argmax(1)
    return nz.any(1) & (d[np.arange(len(d)), first] < 0)


def reduced(curve, sc):
    q = ORDER[curve]
    return rows(curve, [b2i(r) % q for r in sc])


GEN_WIDTHS = list(range(4, 17)) + [18, 20, 22, 24, 26]


@pytest.mark.parametrize("w", GEN_WIDTHS)
@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_cover_addresses_every_entry(curve, w):
    q = ORDER[curve]
    qb = rows(curve, [q])[0]
    nwin, T = geometry(curve, w)
    a, _ = multipliers(curve, w)
    assert (a % 2 == 1).all() and 1 <= T < (1 << w)
    if w <= 16:
        chunks = list(cover(curve, w, chunk=1 << max(4, w - 3)))
        none, extras = chunks.pop()
        assert none is None and [lo for lo, _ in chunks] == list(range(0, 1 << w, 1 << max(4, w - 3)))
    else:
        extras = rows(curve, extra_values(curve, w))
    xv = [b2i(r) for r in extras]
    xr = reduced(curve, extras)
    xd = windows_of(curve, w, xr)
    # the extras: T under lower parts 0 and max, the raw ones >= q and reducing onto scalars below q
    sh = w * (nwin - 1)
    assert xv[0] == T << sh and xv[1] == q - 1 and (xd[:16, -1] == T).all()
    assert all(v < q for v in xv[:19]) and all(v >= q for v in xv[19:])
    if w <= 16:
        seen = np.zeros((nwin, 1 << w), bool)
        for lo, sc in chunks:
            assert len(sc) <= 1 << max(4, w - 3) and below(sc, qb).all()
            d = windows_of(curve, w, sc)
            for i in range(nwin):
                seen[i, d[:, i]] = True
        for i in range(nwin):
            seen[i, xd[:, i]] = True
        assert sum(len(sc) for _, sc in chunks) == 1 << w
        assert seen[:-1, 1:].all(), [(i, np.flatnonzero(~seen[i, 1:])[:4] + 1) for i in range(nwin - 1)
                                     if not seen[i, 1:].all()]
        assert seen[-1, 1:T + 1].all() and not seen[-1, T + 1:].any()
    else:
        # per chunk of the device run: a seeded sample of items has the intended digits and is below q
        g = rng(9002 + w)
        for lo in range(0, 1 << w, CHUNK):
            j = np.unique(np.concatenate([g.integers(lo, lo + CHUNK, 2048, dtype=np.uint64),
                                          np.array([lo, lo + CHUNK - 1], np.uint64)]))
            sc = pack(curve, w, item_digits(curve, w, j))
            assert below(sc, qb).all()
            assert (windows_of(curve, w, sc) == item_digits(curve, w, j)).all()
            assert [b2i(r) for r in sc[:3]] == [sum(int(x) << (w * i) for i, x in enumerate(row))
                                                for row in item_digits(curve, w, j[:3])]


@pytest.mark.parametrize("w", [4, 5])
@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_host_comb_mul_on_the_whole_cover(curve, w):
    """the host build of comb_mul (table from the host build of window_mul) on every entry of the table"""
    sc = np.concatenate([s for _, s in cover(curve, w)])
    want, wst = oracle_smul(curve, sc)
    n = len(sc)
    out = np.zeros_like(want)
    st = np.full(n, 7, np.int8)
    assert hostsim_lib().hostsim_prj_pt_mul_batch(ALL_CURVES[curve][0], w, n, _buf(sc), None, _buf(out), _buf(st)) == 0
    assert (st == wst).all() and (out == want).all(), np.flatnonzero((out != want).any(1) | (st != wst))[:8]


# ------------------------------------------------------------------------------------------ window_mul's recoding


def recode(curve, k):
    """window_mul's digits of k < q: the top digit (0 or 1), then the signed nibbles in [-8, 7], most significant first"""
    nd = (ORDER[curve].bit_length() + 3) // 4
    K = k + int("8" * nd, 16)
    return K >> (4 * nd), [((K >> (4 * i)) & 15) - 8 for i in range(nd - 1, -1, -1)]


def collisions(curve, k):
    """the digit additions of window_mul(k, P) whose operands are equal (+1: add_mixed doubles) or opposite (-1: the
    sum is infinity), as (digits left after this one, d, +-1); the accumulator before each addition is 16 * acc"""
    q = ORDER[curve]
    top, ds = recode(curve, k)
    acc, out = top, []
    for left, d in zip(range(len(ds) - 1, -1, -1), ds):
        acc *= 16
        if d and (acc - d) % q == 0:
            out.append((left, d, +1))
        if d and (acc + d) % q == 0:
            out.append((left, d, -1))
        acc += d
    assert acc == k
    return out


def recoding_collisions(curve):
    """Every scalar k < q for which some digit addition of window_mul meets P == +-Q, by position.  At the digit with
    `left` digits below it, the accumulator is 16*H (H the value of the digits above), and k = 16^left * (16*H + d) +
    low with low in [-8 (16^left - 1) / 15, 7 (16^left - 1) / 15]; every such (H, d, low) with 0 <= k < q is the
    recoding of k.  P == +-Q means 16*H = +-d + t*q, and 0 <= k < q bounds |16*H| by q + 16, so |t| <= 1.
    Returns [(left, d, sign, lowest k, highest k)]."""
    q = ORDER[curve]
    nd = (q.bit_length() + 3) // 4
    found = []
    for left in range(nd):
        p16 = 16 ** left
        lmin, lmax = -8 * (p16 - 1) // 15, 7 * (p16 - 1) // 15
        for d in [x for x in range(-8, 8) if x]:
            for sign in (+1, -1):
                for t in (-1, 0, 1):
                    if (sign * d + t * q) % 16:
                        continue
                    base = p16 * (sign * d + t * q + d)
                    lo, hi = max(0, base + lmin), min(q - 1, base + lmax)
                    if lo <= hi:
                        found.append((left, d, sign, lo, hi))
    return found


DOUBLING = {"SECP256R1": 2, "FRP256V1": 2, "SECP256K1": 2, "SECP192R1": 2, "SECP384R1": 6, "SM2P256V1": 6,
            "BRAINPOOLP256R1": 14, "BRAINPOOLP384R1": 10, "SECP521R1": None, "BRAINPOOLP512R1": None,
            "SECP224R1": None}
DBL_CURVES = [c for c in ALL_CURVES if DOUBLING[c]]


def doubling_scalar(curve):
    q = ORDER[curve]
    m = q % 16
    return q - 2 * m if 1 <= m <= 8 else None


def raw_aliases(curve, k):
    """wire scalars (qlen bytes) other than k that reduce to k"""
    q, qlen = ORDER[curve], ALL_CURVES[curve][2]
    return [k + m * q for m in range(1, 4) if k + m * q < 1 << (8 * qlen)]


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_recoding_model(curve):
    q = ORDER[curve]
    t = doubling_scalar(curve)
    assert sorted(DOUBLING) == sorted(ALL_CURVES)
    assert (q - t if t else None) == DOUBLING[curve]
    found = recoding_collisions(curve)
    assert found == ([(0, -(q % 16), +1, t, t)] if t else []), found
    if t:
        assert collisions(curve, t) == [(0, -(q % 16), +1)]
    g = rng(9003)
    for k in [0, 1, 2, q - 1, q - 2, q - 3] + ([t - 1, t + 1] if t else []) + [b2i(g.bytes(80)) % q for _ in range(64)]:
        if k != t:
            assert collisions(curve, k) == [], k


def test_doubling_scalars_have_no_raw_alias():
    """on the curves with a doubling scalar, 2^(8*qlen) < 2q: no other wire scalar reduces onto it"""
    assert all(raw_aliases(c, doubling_scalar(c)) == [] for c in DBL_CURVES)
    assert len(DBL_CURVES) == 8


# ------------------------------------------------------------------------------------------ the last-digit doubling


def cat_cols(a, b):
    return {k: np.concatenate([a[k], b[k]]) for k in a}


@functools.lru_cache(None)
def families(curve):
    """Per entry point: {"items": crafted items whose window_mul scalar ("v") is the doubling scalar, "valid": valid
    items, "hlen"}; each column set carries the oracle's outputs ("out") and status or verdict ("want")."""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    t = doubling_scalar(curve)
    dr = Draw(curve, 9100 + cid)
    rnd = lambda n: [dr.scalar() for _ in range(n)]
    fam = {}

    def smul_cols(ks, pts, kind):
        sc, pw = rows(curve, ks), wire(curve, pts)
        out, st = oracle_smul(curve, sc, pw)
        return {"sc": sc, "pts": pw, "out": out, "want": st, "kind": objs([kind] * len(ks)),
                "v": np.array([k % q for k in ks], object)}

    # k*P: P random and P = G, the scalar and its raw aliases
    ks = [t] * M + raw_aliases(curve, t)
    fam["prj"] = {"items": smul_cols(ks, (smul(curve, rnd(M - 1) + [1]) * 4)[:len(ks)], "double"),
                  "valid": smul_cols(rnd(NFILL), smul(curve, rnd(NFILL)), "valid")}

    # ECC-CDH: the private key; the shared secret is x(t*P)
    def cdh_cols(ds, peers, kind):
        c = smul_cols(ds, peers, kind)
        c["out"] = c["out"][:, :plen]
        c["want"] = -np.abs(c["want"])          # ecccdh_derive_secret fails on an infinity result
        return c
    fam["cdh"] = {"items": cdh_cols([t] * M, smul(curve, rnd(M)), "double"),
                  "valid": cdh_cols(rnd(NFILL), smul(curve, rnd(NFILL)), "valid")}

    # a*G + b*Y: b, with a random and a = 0
    def dbl_cols(a, b, Ys, kind):
        ab = np.stack([np.concatenate([be(x, qlen), be(y, qlen)]) for x, y in zip(a, b)])
        out, st = oracle_double_smul(curve, ab, wire(curve, Ys))
        return {"ab": ab, "pub": wire(curve, Ys), "out": out, "want": st, "kind": objs([kind] * len(a)),
                "v": np.array(b, object)}
    fam["dbl"] = {"items": dbl_cols(rnd(M - 1) + [0], [t] * M, smul(curve, rnd(M)), "double"),
                  "valid": dbl_cols(rnd(NFILL), rnd(NFILL), smul(curve, rnd(NFILL)), "valid")}

    # ECDSA (digest of qlen bytes): v = r/s = t with s = r/t; e = s*k - r*x makes (r, s) valid for Y = xG, as
    # u*G + v*Y = (e/s + t*x)*G = k*G; the digest of e + 1 must reject
    xs, ks = rnd(M), rnd(M)
    rs = [R[0] % q for R in smul(curve, ks)]
    ss = [r * pow(t, -1, q) % q for r in rs]
    es = [(s * k - r * x) % q for s, k, r, x in zip(ss, ks, rs, xs)]
    sig = np.stack([np.concatenate([be(r, qlen), be(s, qlen)]) for r, s in zip(rs, ss)] * 2)
    items = {"sig": sig, "pub": wire(curve, smul(curve, xs) * 2),
             "dg": np.stack([digest_of_e(curve, e) for e in es] + [digest_of_e(curve, (e + 1) % q) for e in es]),
             "kind": objs(["double"] * M + ["double_bad"] * M), "intended": np.array([0] * M + [-1] * M, np.int8),
             "v": np.array([r * pow(s, -1, q) % q for r, s in zip(rs, ss)] * 2, object)}
    items["want"] = oracle_verify(curve, items["sig"], items["pub"], items["dg"], qlen)
    vs, vp, vdg, vwant = make_signatures(curve, NFILL, tag=9200 + cid, hlen=qlen)
    fam["ecdsa"] = {"items": items, "hlen": qlen,
                    "valid": {"sig": vs, "pub": vp, "dg": vdg, "want": vwant, "kind": objs(["valid"] * NFILL),
                              "intended": np.zeros(NFILL, np.int8), "v": np.zeros(NFILL, object)}}

    # ECFSDSA and BIP0340 in digest form: window_mul's scalar is -h with h the digest mod q, so the digest 2*(q mod 16)
    # gives t.  s = k + h*x (BIP0340: x and k lifted to an even y, r = x(kG)) makes the signature valid; s + 1 rejects.
    def schnorr_cols(scheme, digests, hlen, kind, bad):
        sigs, pubs, vs = [], [], []
        for D in digests:
            x, k = dr.scalar(), dr.scalar()
            P, R = smul(curve, [x, k])
            if scheme == "bip0340":
                x, _ = lift_even(curve, x, P)
                k, R = lift_even(curve, k, R)
                head = be(R[0], plen)
            else:
                head = wire(curve, [R])[0]
            h = D % q
            sigs.append(np.concatenate([head, be((k + h * x + bad) % q, qlen)]))
            pubs.append(P)
            vs.append(-h % q)
        c = {"sig": np.stack(sigs), "pub": wire(curve, pubs), "dg": np.stack([be(D, hlen) for D in digests]),
             "kind": objs([kind] * len(digests)), "intended": np.full(len(digests), -bad, np.int8),
             "v": np.array(vs, object)}
        verify = oracle_fs_verify if scheme == "ecfsdsa" else oracle_bip_verify
        c["want"] = verify(curve, c["sig"], c["pub"], c["dg"], hlen)
        return c
    for scheme in ("ecfsdsa", "bip0340"):
        hlen = 32 if scheme == "bip0340" else HASHLEN[HNAME[curve]]
        crafted = [2 * (q % 16)] * M
        fam[scheme] = {"items": cat_cols(schnorr_cols(scheme, crafted, hlen, "double", 0),
                                         schnorr_cols(scheme, crafted, hlen, "double_bad", 1)),
                       "valid": schnorr_cols(scheme, [b2i(dr.g.bytes(hlen)) for _ in range(NFILL)], hlen, "valid", 0),
                       "hlen": hlen}
    return fam


@functools.lru_cache(None)
def recover_family(curve):
    """ECDSA key recovery (digest of qlen bytes): v = s/r = t with s = t*r, r the x of a curve point below q; the
    reference's __ecdsa_public_key_from_sig gives the keys and statuses"""
    cid, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    t = doubling_scalar(curve)
    dr = Draw(curve, 9400 + cid)
    rs = [point_with_x(curve, 1, min(PRIME[curve], q), dr.g)[0] for _ in range(M)]
    items = {"sig": np.stack([np.concatenate([be(r, qlen), be(t * r % q, qlen)]) for r in rs]),
             "dg": dr.g.integers(0, 256, size=(M, qlen), dtype=np.uint8), "kind": objs(["double"] * M),
             "v": np.array([t] * M, object)}
    vs, vdg, _ = valid_items(curve, NFILL, qlen, 9500 + cid)
    valid = {"sig": vs, "dg": vdg, "kind": objs(["valid"] * NFILL), "v": np.zeros(NFILL, object)}
    for c in (items, valid):
        c["out"], c["want"] = ref_recover(curve, c["sig"], c["dg"], qlen)
    return {"items": items, "valid": valid, "hlen": qlen}


VERIFIERS = {"ecdsa": "hostsim_ecdsa_verify_batch", "ecfsdsa": "hostsim_ecfsdsa_verify_batch",
             "bip0340": "hostsim_bip0340_verify_batch"}


@pytest.mark.parametrize("curve", DBL_CURVES)
def test_host_last_digit_doubling(curve):
    """every crafted item takes the doubling scalar into window_mul, and the host build agrees with the oracle or the
    reference on it and on the valid items"""
    need_ref()
    t = doubling_scalar(curve)
    fam = dict(families(curve), recover=recover_family(curve))
    for name, f in fam.items():
        it = f["items"]
        assert (it["v"] == t).all() and len(it["v"]) >= M, name
        for c in (it, f["valid"]):
            if "intended" in c:
                assert (c["want"] == c["intended"]).all(), (name, c["kind"][c["want"] != c["intended"]])
    assert (fam["prj"]["items"]["want"] == 0).all() and (fam["dbl"]["items"]["want"] == 0).all()
    assert (fam["recover"]["items"]["want"] >= 0).all()
    for c in (fam["prj"]["items"], fam["prj"]["valid"]):
        out, st = np.zeros_like(c["out"]), np.full(len(c["want"]), 7, np.int8)
        assert hostsim_lib().hostsim_prj_pt_mul_batch(ALL_CURVES[curve][0], HOST_W, len(st), _buf(c["sc"]),
                                                      _buf(c["pts"]), _buf(out), _buf(st)) == 0
        assert (st == c["want"]).all() and (out == c["out"]).all()
    for c in (fam["dbl"]["items"], fam["dbl"]["valid"]):
        out, st = host_double_smul(curve)(c["ab"], c["pub"])
        assert (st == c["want"]).all() and (out == c["out"]).all()
    for name, fn in VERIFIERS.items():
        for c in (fam[name]["items"], fam[name]["valid"]):
            assert (host_verify(curve, fn, c, fam[name]["hlen"]) == c["want"]).all(), name
    for c in (fam["recover"]["items"], fam["recover"]["valid"]):
        keys, st = host_recover(curve, c["sig"], c["dg"], fam["recover"]["hlen"])
        assert (st == c["want"]).all() and (keys == c["out"]).all()


# ------------------------------------------------------------------------------------------ on the device

_engines = {}


def engine(curve, w):
    import libecc_b200
    if (curve, w) not in _engines:
        _engines[(curve, w)] = libecc_b200.Engine(curve, device=0, comb_window=w)
    return _engines[(curve, w)]


@pytest.fixture
def release_engines():
    """every test gives its engines (tables of up to 43 GB) back: other test modules keep theirs for the whole run"""
    yield
    import torch
    for eng in _engines.values():
        eng.close()
    _engines.clear()
    torch.cuda.empty_cache()


def table_bytes(curve, w):
    """nwin * 2^w affine entries of two field elements in 32-bit words"""
    return (geometry(curve, w)[0] << w) * 2 * 4 * -(-ALL_CURVES[curve][1] // 4)


COMB_CASES = ([(c, bench.DEFAULT_COMB[c]) for c in ("SECP256R1", "SECP384R1")] + [(c, 0) for c in ALL_CURVES] +
              [(c, w) for w in (4, 7, 16) for c in ALL_CURVES] +
              [("SECP256R1", 18), ("SECP521R1", 18), ("SECP256R1", 24)])


def common_entries(curve, w, sc):
    """the (window, digit) pairs that every one of the (reduced) scalars reads"""
    d = windows_of(curve, w, sc)
    return [(i, int(d[0, i])) for i in range(d.shape[1]) if d[0, i] and (d[:, i] == d[0, i]).all()]


@pytest.mark.gpu
@pytest.mark.parametrize("curve,w", COMB_CASES)
def test_gpu_every_comb_entry(curve, w, release_engines):
    import torch
    _, plen, qlen = ALL_CURVES[curve]
    w = w or (20 if plen > 48 else 22)
    need = table_bytes(curve, w) + (6 << 30)
    free, total = torch.cuda.mem_get_info()
    if need > free:
        pytest.skip(f"the {w}-bit {curve} table needs {need / 2**30:.1f} GiB with the batch buffers; "
                    f"{free / 2**30:.1f} of {total / 2**30:.1f} GiB are free")
    eng = engine(curve, w)
    assert eng.comb_window == w
    G = torch.from_numpy(wire(curve, smul(curve, [1]))[0].copy()).cuda()
    d_g = G.expand(min(CHUNK, 1 << w) + 64, 2 * plen).contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    g = rng(9600 + w)
    nchunks = -(-(1 << w) // CHUNK)
    failing, compared, sampled = [], 0, 0
    for lo, sc in cover(curve, w):
        n = len(sc)
        d_sc = torch.from_numpy(sc).cuda()
        o1 = torch.zeros((n, 2 * plen), dtype=torch.uint8, device="cuda")
        o2 = torch.ones((n, 2 * plen), dtype=torch.uint8, device="cuda")
        s1 = torch.full((n,), 7, dtype=torch.int8, device="cuda")
        s2 = torch.full((n,), 9, dtype=torch.int8, device="cuda")
        eng.prj_pt_mul_batch_dev(d_sc, None, o1, s1, stream)            # K1: the comb table
        eng.prj_pt_mul_batch_dev(d_sc, d_g[:n], o2, s2, stream)         # K2: k*G by the signed window
        bad = torch.nonzero((o1 != o2).any(1) | (s1 != s2)).flatten().cpu().numpy()
        failing.append(sc[bad[:4096]])
        compared += n
        # the oracle on a seeded sample, and on all the extras
        idx = np.arange(n) if lo is None else np.sort(g.choice(n, min(n, -(-SAMPLE // nchunks)), replace=False))
        want, wst = oracle_smul(curve, sc[idx])
        t_idx = torch.from_numpy(idx).cuda()
        got, gst = o1[t_idx].cpu().numpy(), s1[t_idx].cpu().numpy()
        bad = np.flatnonzero((got != want).any(1) | (gst != wst))
        failing.append(sc[idx[bad]])
        sampled += len(idx)
        del d_sc, o1, o2, s1, s2
    failing = np.unique(np.concatenate(failing), axis=0)
    assert compared == (1 << w) + len(extra_values(curve, w)) and sampled >= min(SAMPLE, 1 << w)
    if len(failing):
        # each common pair is probed alone: the scalar d * 2^(w*i) reads entry (i, d) and nothing else
        pairs = common_entries(curve, w, reduced(curve, failing))
        probe = rows(curve, [d << (w * i) for i, d in pairs]) if pairs else rows(curve, [1])
        pout, pst = eng.prj_pt_mul_batch(probe)
        want, wst = oracle_smul(curve, probe)
        named = [pr for pr, o, s, wo, ws in zip(pairs, pout, pst, want, wst) if s != ws or (o != wo).any()]
        pytest.fail(f"{curve} w={w}: {len(failing)} items wrong (K1 against K2 and the oracle); (window, digit) "
                    f"pairs common to all of them: {pairs}; of those, wrong when read alone: {named}")


def dev_verdicts(eng, name, b, hlen):
    if name == "ecdsa":
        return eng.ecdsa_verify_batch(b["sig"], b["pub"], b["dg"], hlen)
    if name == "ecfsdsa":
        return eng.ecfsdsa_verify_batch(b["sig"], b["pub"], b["dg"], hlen)
    return eng.bip0340_verify_batch(b["sig"], b["pub"], b["dg"], hlen)


@pytest.mark.gpu
@pytest.mark.parametrize("curve", DBL_CURVES)
def test_gpu_last_digit_doubling(curve, release_engines):
    """the crafted items of each entry point at lanes 0, 1, 63, 64 and 127 of a CTA of valid items, as a whole CTA and
    last in batches of 383 and 385 items; every item, neighbours included, as the oracle or the reference has it"""
    need_ref()
    eng = engine(curve, 8)
    fam = dict(families(curve), recover=recover_family(curve))
    for name, f in fam.items():
        for kind in dict.fromkeys(f["items"]["kind"]):
            for b in batches(f, kind):
                if name in ("prj", "cdh"):
                    fn = eng.prj_pt_mul_batch if name == "prj" else eng.ecccdh_derive_batch
                    out, st = fn(b["sc"], b["pts"])
                elif name == "dbl":
                    out, st = eng.double_smul_batch(b["ab"], b["pub"])
                elif name == "recover":
                    out, st = eng.ecdsa_recover_batch(b["sig"], b["dg"], f["hlen"])
                else:
                    out, st = None, dev_verdicts(eng, name, b, f["hlen"])
                bad = np.flatnonzero((np.asarray(st) != b["want"]).reshape(len(b["want"]), -1).any(1))
                assert len(bad) == 0, (name, kind, bad[:8], b["kind"][bad[:8]])
                if out is not None:
                    assert (out == b["out"]).all(), (name, kind)
