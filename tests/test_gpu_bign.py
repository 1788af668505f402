"""BIGN and DBIGN signing and verification of raw messages on the device (eccb200_bign_sign_msgs_batch[_dev],
eccb200_bign_verify_msgs_batch[_dev]): parity with the reference's signer at ragged sizes on every curve and at 2^16,
ERR items at chosen lanes, the chunked host pipeline against the device-pointer form, round trips through the device
verifier and the reference's ec_verify, the verifier against the reference's verdicts on corrupted signatures, and
the argument checks.  Bit-exact: signatures, status bytes and verdicts."""
import os

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, random_scalars, rng, _buf
from test_bign_host import HASH_IDS, be, corrupted_set, pack, ref_sign, ref_verify, sign_inputs, need_ref

pytestmark = pytest.mark.gpu

_engines = {}
COMB_W = 8  # small comb tables: these engines fit beside the ones other modules keep
SIZES = [1, 2, 31, 127, 128, 129, 385]
HASHES = ["BELT_HASH", "SHA256", "BASH384", "SHA224", "SM3", "BASH512", "SHA3_224", "BASH256", "SHA512"]


def engine(curve):
    import libecc_b200
    if curve not in _engines:
        _engines[curve] = libecc_b200.Engine(curve, device=0, comb_window=COMB_W)
    return _engines[curve]


@pytest.fixture(autouse=True)
def _release_engines():
    yield
    import torch
    for eng in _engines.values():
        eng.close()
    _engines.clear()
    torch.cuda.empty_cache()


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sign_dev(eng, alg, hash_name, privs, msgs, adata, nonces=None):
    import torch
    n = len(msgs)
    blob, off = pack(msgs)
    ab, aoff = pack(adata)
    d_sigs = torch.full((n, eng.bign_sig_len), 0x5A, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    eng.bign_sign_msgs_batch_dev(alg, hash_name, _t(privs), _t(blob), _t(off.view(np.int64)), _t(ab),
                                 _t(aoff.view(np.int64)), d_sigs, d_st,
                                 d_nonces=_t(nonces) if nonces is not None else None)
    torch.cuda.synchronize()
    return d_sigs.cpu().numpy(), d_st.cpu().numpy()


def verify_dev(eng, hash_name, sigs, pubs, msgs, adata):
    import torch
    n = len(msgs)
    blob, off = pack(msgs)
    ab, aoff = pack(adata)
    d_v = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    eng.bign_verify_msgs_batch_dev(hash_name, _t(sigs), _t(pubs), _t(blob), _t(off.view(np.int64)), _t(ab),
                                   _t(aoff.view(np.int64)), d_v)
    torch.cuda.synchronize()
    return d_v.cpu().numpy()


def both_forms(eng, alg, hash_name, privs, msgs, adata, nonces):
    k = nonces if alg == "BIGN" else None
    return {"host": eng.bign_sign_msgs_batch(alg, hash_name, privs, msgs, adata, nonces=k),
            "dev": sign_dev(eng, alg, hash_name, privs, msgs, adata, k)}


@pytest.mark.parametrize("curve", list(ALL_CURVES))
@pytest.mark.parametrize("alg", ["BIGN", "DBIGN"])
def test_parity_with_reference(curve, alg):
    """every curve at every size of SIZES (ragged CTAs), a hash per size, both forms"""
    need_ref()
    i = list(ALL_CURVES).index(curve)
    eng = engine(curve)
    for j, n in enumerate(SIZES):
        hash_name = HASHES[(i + j) % len(HASHES)]
        privs, nonces, msgs, adata = sign_inputs(curve, max(n, 16), 300 + 10 * i + j)
        privs, nonces, msgs, adata = privs[-n:], nonces[-n:], msgs[-n:], adata[-n:]
        want, pubs, wst = ref_sign(curve, alg, hash_name, privs, msgs, adata, nonces)
        assert (wst == 0).all()
        for form, (got, st) in both_forms(eng, alg, hash_name, privs, msgs, adata, nonces).items():
            assert (st == wst).all(), (n, hash_name, form)
            assert (got == want).all(), (n, hash_name, form)


@pytest.mark.parametrize("curve", ["SECP256R1", "BRAINPOOLP256R1"])
@pytest.mark.parametrize("alg", ["BIGN", "DBIGN"])
def test_parity_2_16(curve, alg):
    """2^16 items; on BRAINPOOLP256R1 about a third of DBIGN's rounds fail k < q, so the warps diverge"""
    need_ref()
    n = 1 << 16
    g = rng(310)
    privs = random_scalars(curve, n, tag=311)
    nonces = random_scalars(curve, n, tag=312)
    msgs = [g.bytes(int(g.integers(0, 100))) for _ in range(n)]
    adata = [bytes.fromhex("00090000608648016503040201")] * n
    want, pubs, wst = ref_sign(curve, alg, "BELT_HASH", privs, msgs, adata, nonces)
    eng = engine(curve)
    for form, (got, st) in both_forms(eng, alg, "BELT_HASH", privs, msgs, adata, nonces).items():
        assert (st == wst).all() and (got == want).all(), form
    assert (wst == 0).all()


@pytest.mark.parametrize("curve", ["SECP256R1", "SECP521R1"])
@pytest.mark.parametrize("alg", ["BIGN", "DBIGN"])
def test_err_items_at_chosen_lanes(curve, alg):
    """bad keys, bad nonces and malformed records at lanes 0, 1, 63, 64 and 127 among valid neighbours"""
    need_ref()
    q = ORDER[curve]
    qlen = ALL_CURVES[curve][2]
    n = 200
    privs, nonces, msgs, adata = sign_inputs(curve, n, 320)
    privs[0] = be(0, qlen)
    privs[1] = be(q, qlen)
    nonces[63] = be(q if alg == "BIGN" else 0, qlen)
    adata[64] = b"\x00\x01"
    adata[127] = b"\x00\x03\x00\x03ab"
    want, _, wst = ref_sign(curve, alg, "SHA256", privs, msgs, adata, nonces)
    bad = [0, 1, 64, 127] + ([63] if alg == "BIGN" else [])
    assert (wst[bad] == -1).all() and (np.delete(wst, bad) == 0).all()
    eng = engine(curve)
    for form, (got, st) in both_forms(eng, alg, "SHA256", privs, msgs, adata, nonces).items():
        assert (st == wst).all() and (got == want).all(), form


def test_host_pipeline_longer_than_three_chunks():
    """ECCB200_CHUNK_WAVES=1: 3 * one K1 wave + 17 items cross at least three chunk boundaries, with messages and
    records crossing them at arbitrary bytes; the host forms agree with the device-pointer forms"""
    import torch
    import libecc_b200
    from libecc_b200 import bign_adata
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 3 * sms * 16 * 128 + 17
    curve = "BRAINPOOLP256R1"
    os.environ["ECCB200_CHUNK_WAVES"] = "1"
    try:
        eng = libecc_b200.Engine(curve, device=0, comb_window=COMB_W)
    finally:
        del os.environ["ECCB200_CHUNK_WAVES"]
    g = rng(330)
    privs = random_scalars(curve, n, tag=331)
    lens = g.integers(0, 91, size=n)
    data = g.bytes(int(lens.sum()) + 1)
    cut = np.concatenate([[0], np.cumsum(lens)])
    msgs = [data[cut[j]:cut[j + 1]] for j in range(n)]
    adata = [bign_adata(b"\x06\x09", data[cut[j]:cut[j] + int(lens[j]) // 3]) for j in range(n)]
    got, st = eng.bign_sign_msgs_batch("DBIGN", "BASH256", privs, msgs, adata)
    dev, dst = sign_dev(eng, "DBIGN", "BASH256", privs, msgs, adata)
    assert (st == 0).all() and (dst == 0).all() and (got == dev).all()
    pubs, _ = eng.prj_pt_mul_batch(privs)
    v = eng.bign_verify_msgs_batch("BASH256", got, pubs, msgs, adata)
    vd = verify_dev(eng, "BASH256", got, pubs, msgs, adata)
    eng.close()
    assert (v == 0).all() and (vd == 0).all()
    idx = np.sort(g.choice(n, 256, replace=False))
    idx[-1] = n - 1
    want, _, wst = ref_sign(curve, "DBIGN", "BASH256", privs[idx], [msgs[j] for j in idx], [adata[j] for j in idx])
    assert (wst == 0).all() and (got[idx] == want).all()


@pytest.mark.parametrize("curve,hash_name", [("SECP256R1", "BELT_HASH"), ("SECP384R1", "BASH384"),
                                             ("SECP521R1", "SHA512"), ("BRAINPOOLP256R1", "SHA3_256"),
                                             ("SM2P256V1", "SM3"), ("SECP224R1", "SHA224"),
                                             ("SECP192R1", "BASH224")])
@pytest.mark.parametrize("alg", ["BIGN", "DBIGN"])
def test_round_trip(curve, hash_name, alg):
    """device signer -> device verifier (both forms) -> the reference's ec_verify"""
    need_ref()
    eng = engine(curve)
    privs, nonces, msgs, adata = sign_inputs(curve, 160, 340)
    sigs, st = eng.bign_sign_msgs_batch(alg, hash_name, privs, msgs, adata,
                                        nonces=nonces if alg == "BIGN" else None)
    assert (st == 0).all()
    pubs, pst = eng.prj_pt_mul_batch(privs)
    assert (pst == 0).all()
    assert (eng.bign_verify_msgs_batch(hash_name, sigs, pubs, msgs, adata) == 0).all()
    assert (verify_dev(eng, hash_name, sigs, pubs, msgs, adata) == 0).all()
    assert (ref_verify(curve, hash_name, sigs, pubs, msgs, adata) == 0).all()


@pytest.mark.parametrize("curve,hash_name", [("SECP256R1", "BELT_HASH"), ("SECP521R1", "SHA256"),
                                             ("BRAINPOOLP384R1", "BASH384"), ("SECP192R1", "SHA3_224"),
                                             ("BRAINPOOLP512R1", "BASH512")])
def test_verify_corrupted_vs_reference(curve, hash_name):
    need_ref()
    sigs, pubs, msgs, adata = corrupted_set(curve, hash_name, 350)
    want = ref_verify(curve, hash_name, sigs, pubs, msgs, adata)
    eng = engine(curve)
    assert (eng.bign_verify_msgs_batch(hash_name, sigs, pubs, msgs, adata) == want).all()
    assert (verify_dev(eng, hash_name, sigs, pubs, msgs, adata) == want).all()


def test_api_edges():
    import torch
    import libecc_b200
    curve = "SECP256R1"
    eng = engine(curve)
    lib = libecc_b200.load_library()
    _, plen, qlen = ALL_CURVES[curve]
    sl = qlen // 2 + qlen
    n = 4
    privs = random_scalars(curve, n, tag=1)
    nonces = random_scalars(curve, n, tag=2)
    blob, off = pack([b"abc"] * n)
    ab, aoff = pack([bytes.fromhex("00010000aa")] * n)
    sigs = np.full((n, sl), 0x5A, np.uint8)
    st = np.full(n, 9, np.int8)

    def call(sig_type, hash_type, count, with_nonces=True, offsets=off, adata_offsets=aoff, adata=ab):
        return lib.eccb200_bign_sign_msgs_batch(eng._h, sig_type, hash_type, count, _buf(privs),
                                                _buf(nonces) if with_nonces else None, _buf(blob), _buf(offsets),
                                                _buf(adata) if adata is not None else None, _buf(adata_offsets),
                                                _buf(sigs), _buf(st))

    assert call(19, 16, 0) == 0                     # n = 0: nothing to do, nothing written
    for alg in (0, 1, 2, 8, 14, 17, 20):            # only BIGN (18) and DBIGN (19)
        assert call(alg, 16, n) == -1
    for ht in (0, 9, 10, 12, 13, 15, 21, -1):
        assert call(18, ht, n) == -1 and call(19, ht, n) == -1
    assert call(18, 16, n, with_nonces=False) == -1  # BIGN without nonces
    assert call(19, 16, n, adata=None) == -1
    for bad in ((2, 0), (0, 1)):
        o = off.copy()
        o[bad[0]] = bad[1]
        assert call(18, 16, n, offsets=o) == -1
        a = aoff.copy()
        a[bad[0]] = bad[1]
        assert call(19, 16, n, adata_offsets=a) == -1
    assert (sigs == 0x5A).all() and (st == 9).all()
    # DBIGN ignores the nonces
    assert call(19, 17, n, with_nonces=False) == 0 and (st == 0).all()
    s1 = sigs.copy()
    assert call(19, 17, n) == 0 and (sigs == s1).all()
    # BELT-HASH and BASH stay refused by the older entry points
    out = np.zeros((n, 64), np.uint8)
    for ht in (16, 17, 20):
        assert lib.eccb200_hash_batch(eng._h, ht, n, _buf(blob), _buf(off), _buf(out)) == -1
        assert lib.eccb200_sign_msgs_batch(eng._h, 6, ht, n, _buf(privs), None, _buf(nonces), _buf(blob), _buf(off),
                                           None, None, _buf(sigs), _buf(st)) == -1
        assert lib.eccb200_ecdsa_sign_msgs_batch(eng._h, 14, ht, n, _buf(privs), None, _buf(blob), _buf(off),
                                                 _buf(sigs), _buf(st)) == -1
    # verifier argument checks
    pubs, _ = eng.prj_pt_mul_batch(privs)
    v = np.full(n, 9, np.int8)
    assert lib.eccb200_bign_verify_msgs_batch(eng._h, 16, 0, None, None, None, None, None, None, None) == 0
    assert lib.eccb200_bign_verify_msgs_batch(eng._h, 9, n, _buf(s1), _buf(pubs), _buf(blob), _buf(off), _buf(ab),
                                              _buf(aoff), _buf(v)) == -1
    assert lib.eccb200_bign_verify_msgs_batch(eng._h, 17, n, _buf(s1), None, _buf(blob), _buf(off), _buf(ab),
                                              _buf(aoff), _buf(v)) == -1
    a = aoff.copy()
    a[1] = 0
    a[2] = 0
    a[3] = 0
    a[4] = 0
    a[0] = 1
    assert lib.eccb200_bign_verify_msgs_batch(eng._h, 17, n, _buf(s1), _buf(pubs), _buf(blob), _buf(off), _buf(ab),
                                              _buf(a), _buf(v)) == -1
    assert (v == 9).all()
    assert lib.eccb200_bign_verify_msgs_batch(eng._h, 17, n, _buf(s1), _buf(pubs), _buf(blob), _buf(off), _buf(ab),
                                              _buf(aoff), _buf(v)) == 0 and (v == 0).all()
    # _dev: a misaligned key or signature buffer is refused before anything runs (d_msgs / d_adata may be anywhere)
    d_priv = torch.zeros(n * qlen + 1, dtype=torch.uint8, device="cuda")
    d_priv[1:] = _t(privs.reshape(-1))
    d_sigs = torch.full((n, sl), 0x5A, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    d_blob, d_off, d_ab, d_aoff = _t(blob), _t(off.view(np.int64)), _t(ab), _t(aoff.view(np.int64))
    assert lib.eccb200_bign_sign_msgs_batch_dev(eng._h, 19, 16, n, d_priv.data_ptr() + 1, None, d_blob.data_ptr(),
                                                d_off.data_ptr(), d_ab.data_ptr(), d_aoff.data_ptr(),
                                                d_sigs.data_ptr(), d_st.data_ptr(), None) == -1
    assert b"aligned" in lib.eccb200_last_error()
    assert lib.eccb200_bign_sign_msgs_batch_dev(eng._h, 18, 16, n, _t(privs).data_ptr(), None, d_blob.data_ptr(),
                                                d_off.data_ptr(), d_ab.data_ptr(), d_aoff.data_ptr(),
                                                d_sigs.data_ptr(), d_st.data_ptr(), None) == -1
    torch.cuda.synchronize()
    assert (d_sigs == 0x5A).all() and (d_st == 9).all()
    m1 = torch.zeros(blob.size + 1, dtype=torch.uint8, device="cuda")
    m1[1:] = d_blob
    a1 = torch.zeros(ab.size + 1, dtype=torch.uint8, device="cuda")
    a1[1:] = d_ab
    assert lib.eccb200_bign_sign_msgs_batch_dev(eng._h, 19, 17, n, _t(privs).data_ptr(), None, m1.data_ptr() + 1,
                                                d_off.data_ptr(), a1.data_ptr() + 1, d_aoff.data_ptr(),
                                                d_sigs.data_ptr(), d_st.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert (d_st == 0).all() and (d_sigs.cpu().numpy() == s1).all()
