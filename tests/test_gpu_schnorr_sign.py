"""Schnorr-family signing on the device (eccb200_schnorr_sign_msgs_batch[_dev]): the reference's known-answer vectors,
parity with the reference's signer under injected randomness (ref_sig_sign_with_randomness), the chunked host pipeline
against the device-pointer form, a round trip through the device verifiers and the reference's ec_verify, and the
argument checks.  Bit-exact: signatures and status bytes."""
import os

import numpy as np
import pytest

from common import ALL_CURVES, golden, hx, random_scalars, ref_lib, rng, _buf
from test_schnorr_sign_host import ALGS, HASHLIB, pack, ref_sign, workload

pytestmark = pytest.mark.gpu

_engines = {}
COMB_W = 8  # small comb tables and table-building scratch: these engines fit beside the ones other modules keep


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
    torch.cuda.empty_cache()  # the device tensors of the _dev calls go back to the driver, not to torch's cache


def be(v, nbytes):
    return np.frombuffer(int(v).to_bytes(nbytes, "big"), np.uint8)


def sign_dev(eng, alg, hash_name, privs, rand, msgs, pubs=None):
    import torch
    n = len(msgs)
    blob, off = pack(msgs)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_sigs = torch.zeros((n, eng.schnorr_sig_len(alg, hash_name)), dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    d_off = t(off.view(np.int64))
    eng.schnorr_sign_msgs_batch_dev(alg, hash_name, t(privs), t(rand), t(blob), d_off, d_sigs, d_st,
                                    d_pubkeys=t(pubs) if pubs is not None else None)
    torch.cuda.synchronize()
    return d_sigs.cpu().numpy(), d_st.cpu().numpy()


def test_kat():
    ran = 0
    for kat in golden("schnorr_sign_kat.json"):
        if kat["hash"] not in HASHLIB or kat["hash"] == "SHA224":
            continue
        curve, alg = kat["curve"], kat["alg"]
        _, plen, qlen = ALL_CURVES[curve]
        eng = engine(curve)
        priv = be(int(kat["priv"], 16), qlen)
        sigs, st = eng.schnorr_sign_msgs_batch(alg, kat["hash"], priv, hx(kat["randomness"]), [bytes.fromhex(kat["msg"])],
                                               pubkeys=hx(kat["pub"]))
        assert st[0] == 0 and sigs[0].tobytes().hex() == kat["sig"], kat["name"]
        ran += 1
    assert ran == 25


CASES = [(c, a, h) for c in ALL_CURVES for a in ALGS for h in ("SHA512", "SHA3_224")]


@pytest.mark.parametrize("curve,alg,hash_name", CASES)
def test_parity_with_reference(curve, alg, hash_name):
    i = CASES.index((curve, alg, hash_name))
    n = (1, 127, 129, 1000)[i % 4]
    if n == 1:  # one valid item (workload puts the invalid inputs first)
        privs, rand, msgs = (a[-1:] for a in workload(curve, alg, 8, 7000 + i))
    else:
        privs, rand, msgs = workload(curve, alg, n, 7000 + i)
        msgs[8] = b""
        msgs[9] = rng(i).bytes(700)  # several blocks of every hash
    want, pubs, wst = ref_sign(curve, alg, hash_name, privs, rand, msgs)
    eng = engine(curve)
    got, st = (eng.schnorr_sign_msgs_batch(alg, hash_name, privs, rand, msgs, pubkeys=pubs) if i % 2 == 0 else
               sign_dev(eng, alg, hash_name, privs, rand, msgs, pubs))
    assert (st == wst).all()
    assert (got == want).all()
    if n > 8:
        assert (st[:3] == -1).all() and (st[6:] == 0).all()


@pytest.mark.parametrize("curve", ["SECP256K1", "SECP384R1"])
def test_bip0340_key_off_curve(curve):
    _, plen, _ = ALL_CURVES[curve]
    privs, rand, msgs = workload(curve, "BIP0340", 16, 91)
    want, pubs, wst = ref_sign(curve, "BIP0340", "SHA256", privs, rand, msgs)
    pubs[7, plen - 1] ^= 1
    got, st = engine(curve).schnorr_sign_msgs_batch("BIP0340", "SHA256", privs, rand, msgs, pubkeys=pubs)
    assert st[7] == -1 and not got[7].any()
    keep = np.arange(16) != 7
    assert (st[keep] == wst[keep]).all() and (got[keep] == want[keep]).all()


def test_host_pipeline_longer_than_three_chunks():
    """ECCB200_CHUNK_WAVES=1: the chunk is one K1 wave (at most SMs x 16 CTAs x 128 items), so 3 * that + 17 items
    cross at least three chunk boundaries; messages of 0..90 bytes, so the offsets cross them at arbitrary bytes"""
    import torch
    import libecc_b200
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 3 * sms * 16 * 128 + 17
    curve, alg, hash_name = "SECP256R1", "ECSDSA", "SHA256"
    os.environ["ECCB200_CHUNK_WAVES"] = "1"
    try:
        eng = libecc_b200.Engine(curve, device=0, comb_window=COMB_W)
    finally:
        del os.environ["ECCB200_CHUNK_WAVES"]
    g = rng(4242)
    privs = random_scalars(curve, n, tag=4243)
    rand = random_scalars(curve, n, tag=4244)
    lens = g.integers(0, 91, size=n)
    data = g.bytes(int(lens.sum()) + 1)
    cut = np.concatenate([[0], np.cumsum(lens)])
    msgs = [data[cut[j]:cut[j + 1]] for j in range(n)]
    got, st = eng.schnorr_sign_msgs_batch(alg, hash_name, privs, rand, msgs)
    dev, dst = sign_dev(eng, alg, hash_name, privs, rand, msgs)
    eng.close()
    assert (st == 0).all() and (dst == 0).all()
    assert (got == dev).all()
    idx = np.sort(g.choice(n, 512, replace=False))
    idx[-1] = n - 1
    want, _, wst = ref_sign(curve, alg, hash_name, privs[idx], rand[idx], [msgs[j] for j in idx])
    assert (wst == 0).all() and (got[idx] == want).all()


def ref_verify(curve, alg, hash_name, sigs, pubs, msgs):
    n = len(msgs)
    blob, off = pack(msgs)
    v = np.zeros(n, np.int8)
    assert ref_lib().ref_sig_verify_batch(curve.encode(), alg.encode(), hash_name.encode(), n, _buf(sigs), _buf(pubs),
                                          _buf(blob), _buf(off), _buf(v), 8) == 0
    return v


@pytest.mark.parametrize("curve,alg,n", [("SECP256R1", a, 1 << 16) for a in ALGS] +
                         [("SECP256K1", "BIP0340", 1 << 20), ("BRAINPOOLP384R1", "ECFSDSA", 1 << 16)])
def test_round_trip(curve, alg, n):
    eng = engine(curve)
    _, plen, qlen = ALL_CURVES[curve]
    hash_name = "SHA256"
    g = rng(n + len(alg))
    privs = random_scalars(curve, n, tag=n + 1)
    rand = (g.integers(0, 256, size=(n, qlen), dtype=np.uint8) if alg == "BIP0340" else
            random_scalars(curve, n, tag=n + 2))
    msgs = [g.bytes(int(k)) for k in g.integers(0, 80, size=n)]
    pubs, pst = eng.prj_pt_mul_batch(privs)
    assert (pst == 0).all()
    sigs, st = eng.schnorr_sign_msgs_batch(alg, hash_name, privs, rand, msgs, pubkeys=pubs)
    assert (st == 0).all()
    h = HASHLIB[hash_name]
    if alg in ("ECFSDSA", "BIP0340"):
        if alg == "ECFSDSA":
            digest_of = lambda i, m: h(sigs[i, :2 * plen].tobytes() + m).digest()
            verify, msm = eng.ecfsdsa_verify_batch, eng.ecfsdsa_verify_msm_batch
        else:
            ht = h(b"BIP0340/challenge").digest()
            digest_of = lambda i, m: h(ht + ht + sigs[i, :plen].tobytes() + pubs[i, :plen].tobytes() + m).digest()
            verify, msm = eng.bip0340_verify_batch, eng.bip0340_verify_msm_batch
        dg = np.frombuffer(b"".join(digest_of(i, msgs[i]) for i in range(n)), np.uint8).reshape(n, -1)
        assert (verify(sigs, pubs, dg, dg.shape[1]) == 0).all()
        assert msm(sigs, pubs, dg, dg.shape[1])
        j = n // 2  # the digest of a corrupted message
        bad = dg.copy()
        bad[j] = np.frombuffer(digest_of(j, msgs[j] + b"\x01"), np.uint8)
        v = verify(sigs, pubs, bad, dg.shape[1])
        assert v[j] == -1 and (np.delete(v, j) == 0).all()
        assert not msm(sigs, pubs, bad, dg.shape[1])
    idx = np.sort(g.choice(n, 1024, replace=False))
    sm = [msgs[i] for i in idx]
    assert (ref_verify(curve, alg, hash_name, sigs[idx], pubs[idx], sm) == 0).all()
    sm[5] = sm[5] + b"\x01"
    v = ref_verify(curve, alg, hash_name, sigs[idx], pubs[idx], sm)
    assert v[5] == -1 and (np.delete(v, 5) == 0).all()


def test_api_edges():
    import torch
    import libecc_b200
    curve = "SECP256R1"
    eng = engine(curve)
    lib = libecc_b200.load_library()
    _, plen, qlen = ALL_CURVES[curve]
    n = 4
    privs = random_scalars(curve, n, tag=1)
    rand = random_scalars(curve, n, tag=2)
    blob, off = pack([b"abc"] * n)
    sigs = np.full((n, 32 + qlen), 0x5A, np.uint8)
    st = np.full(n, 9, np.int8)

    def call(sig_type, hash_type, count, pubs=None):
        return lib.eccb200_schnorr_sign_msgs_batch(eng._h, sig_type, hash_type, count, _buf(privs),
                                                    _buf(pubs) if pubs is not None else None, _buf(rand), _buf(blob),
                                                    _buf(off), _buf(sigs), _buf(st))

    assert call(3, 2, 0) == 0                     # n = 0: nothing to do, nothing written
    assert call(1, 2, n) == -1                    # ECDSA is not a Schnorr-family scheme
    assert call(3, 1, n) == -1                    # SHA224 is not hashed on the device
    assert call(3, 9, n) == -1
    assert call(20, 2, n) == -1                   # BIP0340 without public keys
    assert (sigs == 0x5A).all() and (st == 9).all()
    bad_off = off.copy()
    bad_off[2] = 0
    assert lib.eccb200_schnorr_sign_msgs_batch(eng._h, 3, 2, n, _buf(privs), None, _buf(rand), _buf(blob),
                                               _buf(bad_off), _buf(sigs), _buf(st)) == -1
    assert (sigs == 0x5A).all() and (st == 9).all()
    # _dev: a misaligned buffer is refused before anything runs
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_priv = torch.zeros(n * qlen + 1, dtype=torch.uint8, device="cuda")
    d_priv[1:] = t(privs.reshape(-1))
    d_sigs = torch.full((n, 32 + qlen), 0x5A, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    rc = lib.eccb200_schnorr_sign_msgs_batch_dev(eng._h, 3, 2, n, d_priv.data_ptr() + 1, None, t(rand).data_ptr(),
                                                 t(blob).data_ptr(), t(off.view(np.int64)).data_ptr(), d_sigs.data_ptr(),
                                                 d_st.data_ptr(), None)
    assert rc == -1 and b"aligned" in lib.eccb200_last_error()
    torch.cuda.synchronize()
    assert (d_sigs == 0x5A).all() and (d_st == 9).all()
