"""ECKCDSA / ECGDSA / ECRDSA / SM2 signing on the device (eccb200_sign_msgs_batch[_dev]): the reference's known-answer
vectors, parity with the reference's signer under injected nonces (ref_sig_sign_with_randomness_adata), SM2 key errors
at chosen lanes of the CTA-wide inversion, the chunked host pipeline against the device-pointer form, round trips
through the reference's ec_verify, and the argument checks.  Bit-exact: signatures and status bytes."""
import os

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, golden, hx, random_scalars, rng, _buf
from test_sign_msgs_host import ALGS, HASH_IDS, be, pack, ref_sign, ref_verify, workload

pytestmark = pytest.mark.gpu

_engines = {}
COMB_W = 8  # small comb tables and table-building scratch: these engines fit beside the ones other modules keep
NCPU = max(8, os.cpu_count() or 8)


def engine(curve):
    import libecc_b200
    if curve not in _engines:
        _engines[curve] = libecc_b200.Engine(curve, device=0, comb_window=COMB_W)
    return _engines[curve]


@pytest.fixture(autouse=True)
def _release_engines():
    """every test gives its engines (tables, stage buffers) back: other test modules keep theirs for the whole run"""
    yield
    import torch
    for eng in _engines.values():
        eng.close()
    _engines.clear()
    torch.cuda.empty_cache()


def sign_dev(eng, alg, hash_name, privs, nonces, msgs, pubs=None, ids=None):
    import torch
    n = len(msgs)
    blob, off = pack(msgs)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_sigs = torch.zeros((n, eng.sign_sig_len(alg, hash_name)), dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    d_ids = d_ioff = None
    if ids is not None:
        iblob, ioff = pack(ids)
        d_ids, d_ioff = t(iblob), t(ioff.view(np.int64))
    eng.sign_msgs_batch_dev(alg, hash_name, t(privs), t(nonces), t(blob), t(off.view(np.int64)), d_sigs, d_st,
                            d_pubkeys=t(pubs) if pubs is not None else None, d_ids=d_ids, d_id_offsets=d_ioff)
    torch.cuda.synchronize()
    return d_sigs.cpu().numpy(), d_st.cpu().numpy()


def test_kat():
    ran = 0
    for kat in golden("sign_kat.json"):
        if kat["hash"] not in HASH_IDS:
            continue
        curve, alg = kat["curve"], kat["alg"]
        _, plen, qlen = ALL_CURVES[curve]
        eng = engine(curve)
        priv = be(int(kat["priv"], 16), qlen)
        sigs, st = eng.sign_msgs_batch(alg, kat["hash"], priv, hx(kat["nonce"]), [bytes.fromhex(kat["msg"])],
                                       pubkeys=hx(kat["pub"]), ids=[bytes.fromhex(kat["adata"])])
        assert st[0] == 0 and sigs[0].tobytes().hex() == kat["sig"], kat["name"]
        ran += 1
    assert ran == 12


SIZES = (1, 127, 128, 129, 383, 385)
HASHES = ("SHA256", "SHA384", "SHA512", "SHA3_256", "SHA3_512", "SM3")
CASES = [(c, a) for c in ALL_CURVES for a in ALGS]


@pytest.mark.parametrize("curve,alg", CASES)
def test_parity_with_reference(curve, alg):
    """every curve and scheme at every size of SIZES (ragged CTAs), a hash per size, host and device-pointer forms"""
    i = CASES.index((curve, alg))
    eng = engine(curve)
    for j, n in enumerate(SIZES):
        hash_name = HASHES[(i + j) % len(HASHES)]
        if n == 1:  # one valid item (workload puts the edge inputs first)
            privs, nonces, msgs, ids = (a[-1:] for a in workload(curve, alg, 8, 8000 + i))
        else:
            privs, nonces, msgs, ids = workload(curve, alg, n, 8000 + 10 * i + j)
        want, pubs, wst = ref_sign(curve, alg, hash_name, privs, nonces, msgs, ids, nthreads=NCPU)
        got, st = (eng.sign_msgs_batch(alg, hash_name, privs, nonces, msgs, pubkeys=pubs, ids=ids) if (i + j) % 2 == 0
                   else sign_dev(eng, alg, hash_name, privs, nonces, msgs, pubs, ids))
        assert (st == wst).all(), (n, hash_name)
        assert (got == want).all(), (n, hash_name)
        if n > 8:
            assert (st[5:] == 0).all()


@pytest.mark.parametrize("curve,alg,hash_name", [("SECP256R1", "SM2", "SM3"), ("SECP384R1", "ECKCDSA", "SHA384"),
                                                 ("BRAINPOOLP512R1", "ECGDSA", "SHA3_512")])
def test_parity_2_16(curve, alg, hash_name):
    n = 1 << 16
    privs, nonces, msgs, ids = workload(curve, alg, n, 9100)
    ids = [x[:40] for x in ids]
    want, pubs, wst = ref_sign(curve, alg, hash_name, privs, nonces, msgs, ids, nthreads=NCPU)
    got, st = engine(curve).sign_msgs_batch(alg, hash_name, privs, nonces, msgs, pubkeys=pubs, ids=ids)
    assert (st == wst).all() and (got == want).all()
    assert (st[5:] == 0).all()


@pytest.mark.parametrize("curve", ["SM2P256V1", "SECP521R1"])
def test_sm2_errors_at_chosen_lanes(curve):
    """x = q - 1 (ERR) at lanes 0, 1, 63, 64 and 127 of the first CTA and over the whole second CTA: those items stay
    out of the shared inversion of 1 + x, so every other signature is the one of an all-valid batch"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    eng = engine(curve)
    for n in (383, 385):
        g = rng(n)
        privs = random_scalars(curve, n, tag=n + 1)
        nonces = random_scalars(curve, n, tag=n + 2)
        msgs = [g.bytes(int(g.integers(0, 120))) for _ in range(n)]
        ids = [g.bytes(int(g.integers(0, 30))) for _ in range(n)]
        want, pubs, wst = ref_sign(curve, "SM2", "SM3", privs, nonces, msgs, ids, nthreads=NCPU)
        assert (wst == 0).all()
        bad = [0, 1, 63, 64, 127] + list(range(128, 256)) + [n - 1]
        bp = privs.copy()
        for j in bad:
            bp[j] = be(q - 1, qlen)
        for form in ("host", "dev"):
            got, st = (eng.sign_msgs_batch("SM2", "SM3", bp, nonces, msgs, pubkeys=pubs, ids=ids) if form == "host"
                       else sign_dev(eng, "SM2", "SM3", bp, nonces, msgs, pubs, ids))
            keep = np.ones(n, bool)
            keep[bad] = False
            assert (st[bad] == -1).all() and not got[bad].any(), form
            assert (st[keep] == 0).all() and (got[keep] == want[keep]).all(), form


def test_host_pipeline_longer_than_three_chunks():
    """ECCB200_CHUNK_WAVES=1: the chunk is one K1 wave, so 3 * that + 17 items cross at least three chunk boundaries;
    messages of 0..90 bytes and IDs of 0..20 bytes, so both offset arrays cross them at arbitrary bytes"""
    import torch
    import libecc_b200
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 3 * sms * 16 * 128 + 17
    curve, alg, hash_name = "SECP256R1", "SM2", "SM3"
    os.environ["ECCB200_CHUNK_WAVES"] = "1"
    try:
        eng = libecc_b200.Engine(curve, device=0, comb_window=COMB_W)
    finally:
        del os.environ["ECCB200_CHUNK_WAVES"]
    g = rng(4343)
    privs = random_scalars(curve, n, tag=4344)
    nonces = random_scalars(curve, n, tag=4345)
    pubs, pst = eng.prj_pt_mul_batch(privs)
    assert (pst == 0).all()
    lens = g.integers(0, 91, size=n)
    data = g.bytes(int(lens.sum()) + 1)
    cut = np.concatenate([[0], np.cumsum(lens)])
    msgs = [data[cut[j]:cut[j + 1]] for j in range(n)]
    ids = [data[:int(k)] for k in g.integers(0, 21, size=n)]
    got, st = eng.sign_msgs_batch(alg, hash_name, privs, nonces, msgs, pubkeys=pubs, ids=ids)
    dev, dst = sign_dev(eng, alg, hash_name, privs, nonces, msgs, pubs, ids)
    eng.close()
    assert (st == 0).all() and (dst == 0).all()
    assert (got == dev).all()
    idx = np.sort(g.choice(n, 512, replace=False))
    idx[-1] = n - 1
    want, rpubs, wst = ref_sign(curve, alg, hash_name, privs[idx], nonces[idx], [msgs[j] for j in idx],
                                [ids[j] for j in idx], nthreads=NCPU)
    assert (rpubs == pubs[idx]).all()
    assert (wst == 0).all() and (got[idx] == want).all()


@pytest.mark.parametrize("curve,alg,hash_name", [("SECP256R1", a, "SHA256") for a in ALGS] +
                         [("SM2P256V1", "SM2", "SM3"), ("SECP521R1", "ECKCDSA", "SHA512")])
def test_round_trip(curve, alg, hash_name):
    """every OK signature verifies under the reference's ec_verify (SM2: with the ID as adata); a changed message or
    ID does not"""
    n = 4096
    _, plen, qlen = ALL_CURVES[curve]
    g = rng(n + len(alg))
    privs = random_scalars(curve, n, tag=n + 1)
    nonces = random_scalars(curve, n, tag=n + 2)
    msgs = [g.bytes(int(k)) for k in g.integers(0, 80, size=n)]
    ids = [g.bytes(int(k)) for k in g.integers(0, 40, size=n)]
    # the scheme's public key of every item (x^-1*G for ECKCDSA / ECGDSA) from the reference, on 1024 items
    idx = np.sort(g.choice(n, 1024, replace=False))
    _, pubs, wst = ref_sign(curve, alg, hash_name, privs[idx], nonces[idx], [msgs[j] for j in idx],
                            [ids[j] for j in idx], nthreads=NCPU)
    sm = [msgs[j] for j in idx]
    si = [ids[j] for j in idx]
    sigs, st = engine(curve).sign_msgs_batch(alg, hash_name, privs[idx], nonces[idx], sm, pubkeys=pubs, ids=si)
    assert (st == 0).all() and (wst == 0).all()
    assert (ref_verify(curve, alg, hash_name, sigs, pubs, sm, si, nthreads=NCPU) == 0).all()
    sm[5] = sm[5] + b"\x01"
    v = ref_verify(curve, alg, hash_name, sigs, pubs, sm, si, nthreads=NCPU)
    assert v[5] == -1 and (np.delete(v, 5) == 0).all()
    if alg == "SM2":
        si[9] = si[9] + b"\x01"
        sm[5] = sm[5][:-1]
        v = ref_verify(curve, alg, hash_name, sigs, pubs, sm, si, nthreads=NCPU)
        assert v[9] == -1 and (np.delete(v, 9) == 0).all()


def test_api_edges():
    import torch
    import libecc_b200
    curve = "SECP256R1"
    eng = engine(curve)
    lib = libecc_b200.load_library()
    _, plen, qlen = ALL_CURVES[curve]
    n = 4
    privs = random_scalars(curve, n, tag=1)
    nonces = random_scalars(curve, n, tag=2)
    pubs, _ = eng.prj_pt_mul_batch(privs)
    blob, off = pack([b"abc"] * n)
    iblob, ioff = pack([b"id"] * n)
    sigs = np.full((n, 2 * qlen), 0x5A, np.uint8)
    st = np.full(n, 9, np.int8)

    def call(sig_type, hash_type, count, with_pubs=True, with_ids=True, offsets=off, id_offsets=ioff):
        return lib.eccb200_sign_msgs_batch(eng._h, sig_type, hash_type, count, _buf(privs),
                                           _buf(pubs) if with_pubs else None, _buf(nonces), _buf(blob),
                                           _buf(offsets), _buf(iblob) if with_ids else None,
                                           _buf(id_offsets) if with_ids else None, _buf(sigs), _buf(st))

    assert call(8, 11, 0) == 0                    # n = 0: nothing to do, nothing written
    for alg in (0, 1, 3, 4, 5, 9, 10, 20):        # ECDSA and the Schnorr family keep their own entry points
        assert call(alg, 2, n) == -1
    for ht in (0, 1, 9, 10, 12):                  # SHA224 is not hashed on the device
        assert call(6, ht, n) == -1
    assert call(8, 11, n, with_ids=False) == -1   # SM2 without IDs
    assert call(8, 11, n, with_pubs=False) == -1  # SM2 / ECKCDSA without public keys
    assert call(2, 2, n, with_pubs=False) == -1
    bad_off = off.copy()
    bad_off[2] = 0
    assert call(6, 2, n, offsets=bad_off) == -1
    assert call(8, 2, n, id_offsets=bad_off) == -1
    assert (sigs == 0x5A).all() and (st == 9).all()
    assert lib.eccb200_sign_sig_len(eng._h, 2, 4) == 2 * qlen
    assert lib.eccb200_sign_sig_len(eng._h, 2, 5) == 28 + qlen
    assert lib.eccb200_sign_sig_len(eng._h, 8, 11) == 2 * qlen
    assert lib.eccb200_sign_sig_len(eng._h, 3, 2) == -1 and lib.eccb200_sign_sig_len(eng._h, 8, 1) == -1
    # ECGDSA / ECRDSA ignore pubkeys and IDs
    assert call(6, 2, n, with_pubs=False, with_ids=False) == 0 and (st == 0).all()
    # SM3 stays refused by the older entry points
    out = np.zeros((n, 64), np.uint8)
    assert lib.eccb200_hash_batch(eng._h, 11, n, _buf(blob), _buf(off), _buf(out)) == -1
    assert lib.eccb200_schnorr_sign_msgs_batch(eng._h, 3, 11, n, _buf(privs), None, _buf(nonces), _buf(blob),
                                               _buf(off), _buf(sigs), _buf(st)) == -1
    for alg in ALGS.values():                     # and the Schnorr entry point keeps refusing these four schemes
        assert lib.eccb200_schnorr_sign_msgs_batch(eng._h, alg, 2, n, _buf(privs), _buf(pubs), _buf(nonces),
                                                   _buf(blob), _buf(off), _buf(sigs), _buf(st)) == -1
    # _dev: a misaligned buffer is refused before anything runs
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_priv = torch.zeros(n * qlen + 1, dtype=torch.uint8, device="cuda")
    d_priv[1:] = t(privs.reshape(-1))
    d_sigs = torch.full((n, 2 * qlen), 0x5A, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    rc = lib.eccb200_sign_msgs_batch_dev(eng._h, 6, 2, n, d_priv.data_ptr() + 1, None, t(nonces).data_ptr(),
                                         t(blob).data_ptr(), t(off.view(np.int64)).data_ptr(), None, None,
                                         d_sigs.data_ptr(), d_st.data_ptr(), None)
    assert rc == -1 and b"aligned" in lib.eccb200_last_error()
    torch.cuda.synchronize()
    assert (d_sigs == 0x5A).all() and (d_st == 9).all()
    # _dev: an ID over 8191 bytes is an ERR item, its neighbours sign
    ids = [b"", bytes(8192), b"x" * 8191, b"y"]
    want, rp, wst = ref_sign(curve, "SM2", "SM3", privs, nonces, [b"abc"] * n, [ids[0], b"", ids[2], ids[3]])
    got, gst = sign_dev(eng, "SM2", "SM3", privs, nonces, [b"abc"] * n, rp, ids)
    assert list(gst) == [0, -1, 0, 0] and not got[1].any()
    assert (got[[0, 2, 3]] == want[[0, 2, 3]]).all()
