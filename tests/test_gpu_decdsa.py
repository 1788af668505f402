"""Deterministic ECDSA (RFC 6979 nonces derived on the device) and ECDSA of raw messages (eccb200_decdsa_sign_batch[_dev],
eccb200_ecdsa_sign_msgs_batch[_dev]): the reference's 32 known answers, parity with the reference's DECDSA signer at
ragged sizes and at 2^16, the digest form against the existing signer on Python-derived nonces, invalid keys at chosen
lanes of the CTA-wide inversion, the chunked host pipeline against the device-pointer form, round trips through the
device verifier and the reference's ec_verify, and the argument checks.  Bit-exact: signatures and status bytes."""
import os

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, golden, hx, random_scalars, ref_lib, rng, _buf
from test_decdsa_host import (DIGEST, HASH_IDS, HASHLIB, PY_HASHES, be, pack, py_rfc6979, ref_decdsa,
                              sign_workload)

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


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def digest_dev(eng, hash_name, privs, digests):
    import torch
    n = len(privs)
    d_sigs = torch.full((n, 2 * eng.qlen), 0x5A, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    eng.decdsa_sign_batch_dev(hash_name, _t(privs), _t(digests), d_sigs, d_st)
    torch.cuda.synchronize()
    return d_sigs.cpu().numpy(), d_st.cpu().numpy()


def msgs_dev(eng, alg, hash_name, privs, msgs, nonces=None):
    import torch
    n = len(msgs)
    blob, off = pack(msgs)
    d_sigs = torch.full((n, 2 * eng.qlen), 0x5A, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    eng.ecdsa_sign_msgs_batch_dev(alg, hash_name, _t(privs), _t(blob), _t(off.view(np.int64)), d_sigs, d_st,
                                  d_nonces=_t(nonces) if nonces is not None else None)
    torch.cuda.synchronize()
    return d_sigs.cpu().numpy(), d_st.cpu().numpy()


def all_forms(eng, hash_name, privs, msgs):
    """(sigs, status) of the four DECDSA forms: digest / message entry point, host / device pointers"""
    digests = np.stack([np.frombuffer(HASHLIB[hash_name](m).digest(), np.uint8) for m in msgs]) \
        if hash_name in PY_HASHES else None
    out = {"msgs": eng.ecdsa_sign_msgs_batch("DECDSA", hash_name, privs, msgs),
           "msgs_dev": msgs_dev(eng, "DECDSA", hash_name, privs, msgs)}
    if digests is not None:
        out["digest"] = eng.decdsa_sign_batch(hash_name, privs, digests)
        out["digest_dev"] = digest_dev(eng, hash_name, privs, digests)
    return out


def test_kat():
    """all 32 DECDSA known answers (SHA-224 included) through both entry points in both forms"""
    ran = 0
    for kat in golden("ecdsa_kat.json"):
        if kat["alg"] != "DECDSA":
            continue
        curve, hash_name = kat["curve"], kat["hash"]
        _, _, qlen = ALL_CURVES[curve]
        priv = be(int(kat["priv"], 16), qlen).copy().reshape(1, qlen)
        for form, (sigs, st) in all_forms(engine(curve), hash_name, priv, [bytes.fromhex(kat["msg"])]).items():
            assert st[0] == 0 and sigs[0].tobytes().hex() == kat["sig"], (kat["name"], form)
        ran += 1
    assert ran == 32


SIZES = (1, 127, 128, 129, 383, 385)
HASHES = list(HASH_IDS)


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_parity_with_reference(curve):
    """every curve at every size of SIZES (ragged CTAs), a hash per size, both entry points in both forms"""
    i = list(ALL_CURVES).index(curve)
    eng = engine(curve)
    for j, n in enumerate(SIZES):
        hash_name = HASHES[(i + j) % len(HASHES)]
        if n == 1:  # one valid item (sign_workload puts the edge keys first)
            privs, msgs = sign_workload(curve, 8, 8800 + i)
            privs, msgs = privs[-1:], msgs[-1:]
        else:
            privs, msgs = sign_workload(curve, n, 8800 + 10 * i + j)
        want, _, wst = ref_decdsa(curve, hash_name, privs, msgs, nthreads=NCPU)
        if n > 8:
            assert list(wst[:5]) == [0, 0, 0, -1, -1]
        for form, (got, st) in all_forms(eng, hash_name, privs, msgs).items():
            assert (st == wst).all(), (n, hash_name, form)
            assert (got == want).all(), (n, hash_name, form)


@pytest.mark.parametrize("curve", ["BRAINPOOLP256R1", "SECP256R1"])
def test_parity_2_16(curve):
    """2^16 items: on BRAINPOOLP256R1 a third of the attempts retry, so the warps diverge in the retry loop"""
    n = 1 << 16
    privs, msgs = sign_workload(curve, n, 9200)
    msgs = [m[:64] for m in msgs]
    want, _, wst = ref_decdsa(curve, "SHA256", privs, msgs, nthreads=NCPU)
    eng = engine(curve)
    got, st = eng.ecdsa_sign_msgs_batch("DECDSA", "SHA256", privs, msgs)
    assert (st == wst).all() and (got == want).all()
    digests = np.stack([np.frombuffer(HASHLIB["SHA256"](m).digest(), np.uint8) for m in msgs])
    got, st = digest_dev(eng, "SHA256", privs, digests)
    assert (st == wst).all() and (got == want).all()
    assert (st[5:] == 0).all()


@pytest.mark.parametrize("curve,hash_name", [("SECP256R1", "SHA256"), ("BRAINPOOLP384R1", "SHA224"),
                                             ("SECP521R1", "SHA3_256"), ("SECP192R1", "SHA512")])
def test_digest_form_against_existing_signer(curve, hash_name):
    """decdsa_sign_batch(x, h) == ecdsa_sign_batch(x, k(x, h), h) with k from the Python RFC 6979, crafted digests
    (all-zero, all-0xFF) included"""
    _, _, qlen = ALL_CURVES[curve]
    n = 130
    ds = DIGEST[hash_name]
    privs = random_scalars(curve, n, tag=9300)
    digests = rng(9301).integers(0, 256, size=(n, ds), dtype=np.uint8)
    digests[0] = 0
    digests[1] = 0xFF
    nonces = np.stack([be(py_rfc6979(curve, hash_name, int.from_bytes(privs[i].tobytes(), "big"),
                                     digests[i].tobytes())[0], qlen) for i in range(n)])
    eng = engine(curve)
    want, wst = eng.ecdsa_sign_batch(privs, nonces, digests, ds)
    got, st = eng.decdsa_sign_batch(hash_name, privs, digests)
    assert (wst == 0).all() and (st == 0).all() and (got == want).all()
    got, st = digest_dev(eng, hash_name, privs, digests)
    assert (st == 0).all() and (got == want).all()


@pytest.mark.parametrize("curve", ["SECP256R1", "BRAINPOOLP512R1", "SECP521R1"])
def test_invalid_keys_at_chosen_lanes(curve):
    """keys 0 or q at lanes 0, 1, 63, 64 and 127 of the first CTA, over the whole second CTA and last: those items
    are ERR and stay out of k_ecdsa_sign_finish's shared inversion, so every other signature is unchanged"""
    _, _, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    eng = engine(curve)
    for n in (383, 385):
        g = rng(n + 9400)
        privs = random_scalars(curve, n, tag=n + 9401)
        msgs = [g.bytes(int(g.integers(0, 120))) for _ in range(n)]
        clean = all_forms(eng, "SHA256", privs, msgs)
        bad = [0, 1, 63, 64, 127] + list(range(128, 256)) + [n - 1]
        bp = privs.copy()
        for j, b in enumerate(bad):
            bp[b] = be(0 if j % 2 else q, qlen)
        keep = np.ones(n, bool)
        keep[bad] = False
        for form, (got, st) in all_forms(eng, "SHA256", bp, msgs).items():
            want, wst = clean[form]
            assert (wst == 0).all()
            assert (st[bad] == -1).all() and not got[bad].any(), form
            assert (st[keep] == 0).all() and (got[keep] == want[keep]).all(), form


def test_host_pipeline_longer_than_three_chunks():
    """ECCB200_CHUNK_WAVES=1: the chunk is one K1 wave, so 3 * that + 17 items cross at least three chunk boundaries,
    with messages of 0..90 bytes crossing them at arbitrary bytes"""
    import torch
    import libecc_b200
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 3 * sms * 16 * 128 + 17
    curve = "BRAINPOOLP256R1"
    os.environ["ECCB200_CHUNK_WAVES"] = "1"
    try:
        eng = libecc_b200.Engine(curve, device=0, comb_window=COMB_W)
    finally:
        del os.environ["ECCB200_CHUNK_WAVES"]
    g = rng(9500)
    privs = random_scalars(curve, n, tag=9501)
    lens = g.integers(0, 91, size=n)
    data = g.bytes(int(lens.sum()) + 1)
    cut = np.concatenate([[0], np.cumsum(lens)])
    msgs = [data[cut[j]:cut[j + 1]] for j in range(n)]
    digests = np.stack([np.frombuffer(HASHLIB["SHA3_256"](m).digest(), np.uint8) for m in msgs])
    got, st = eng.ecdsa_sign_msgs_batch("DECDSA", "SHA3_256", privs, msgs)
    got2, st2 = eng.decdsa_sign_batch("SHA3_256", privs, digests)
    dev, dst = msgs_dev(eng, "DECDSA", "SHA3_256", privs, msgs)
    eng.close()
    assert (st == 0).all() and (st2 == 0).all() and (dst == 0).all()
    assert (got == dev).all() and (got2 == dev).all()
    idx = np.sort(g.choice(n, 512, replace=False))
    idx[-1] = n - 1
    want, _, wst = ref_decdsa(curve, "SHA3_256", privs[idx], [msgs[j] for j in idx], nthreads=NCPU)
    assert (wst == 0).all() and (got[idx] == want).all()


@pytest.mark.parametrize("curve,hash_name", [("SECP256R1", "SHA256"), ("SECP384R1", "SHA384"),
                                             ("SECP521R1", "SHA512"), ("BRAINPOOLP256R1", "SHA3_256"),
                                             ("SM2P256V1", "SM3"), ("SECP224R1", "SHA224")])
def test_round_trip(curve, hash_name):
    """DECDSA and ECDSA message signatures verify under the device verifier (hashes 2..8) and the reference's
    ec_verify(…, DECDSA | ECDSA, …); a changed message does not"""
    n = 2048
    g = rng(9600)
    eng = engine(curve)
    privs = random_scalars(curve, n, tag=9601)
    nonces = random_scalars(curve, n, tag=9602)
    pubs, pst = eng.prj_pt_mul_batch(privs)
    assert (pst == 0).all()
    msgs = [g.bytes(int(k)) for k in g.integers(0, 200, size=n)]
    ref = ref_lib()
    for alg, kw in (("DECDSA", {}), ("ECDSA", {"nonces": nonces})):
        sigs, st = eng.ecdsa_sign_msgs_batch(alg, hash_name, privs, msgs, **kw)
        assert (st == 0).all()
        bent = list(msgs)
        bent[5] = bent[5] + b"\x01"
        if hash_name in eng.HASH_IDS:
            blob, off = pack(msgs)
            assert (eng.ecdsa_verify_msgs_batch_raw(hash_name, sigs, pubs, blob, off) == 0).all()
            blob, off = pack(bent)
            v = eng.ecdsa_verify_msgs_batch_raw(hash_name, sigs, pubs, blob, off)
            assert v[5] == -1 and (np.delete(v, 5) == 0).all()
        if ref is None:
            continue
        for m, want5 in ((msgs, 0), (bent, -1)):
            blob, off = pack(m)
            v = np.zeros(n, np.int8)
            assert ref.ref_sig_verify_batch(curve.encode(), alg.encode(), hash_name.encode(), n, _buf(sigs), _buf(pubs),
                                            _buf(blob), _buf(off), _buf(v), NCPU) == 0
            assert v[5] == want5 and (np.delete(v, 5) == 0).all()


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
    digests = rng(3).integers(0, 256, size=(n, 64), dtype=np.uint8)
    blob, off = pack([b"abc"] * n)
    sigs = np.full((n, 2 * qlen), 0x5A, np.uint8)
    st = np.full(n, 9, np.int8)

    def call(sig_type, hash_type, count, with_nonces=True, offsets=off):
        return lib.eccb200_ecdsa_sign_msgs_batch(eng._h, sig_type, hash_type, count, _buf(privs),
                                                 _buf(nonces) if with_nonces else None, _buf(blob), _buf(offsets),
                                                 _buf(sigs), _buf(st))

    assert call(14, 2, 0) == 0                     # n = 0: nothing to do, nothing written
    for alg in (0, 2, 3, 5, 8, 13, 15, 20):         # only ECDSA (1) and DECDSA (14)
        assert call(alg, 2, n) == -1
    for ht in (0, 9, 10, 12, -1):
        assert call(14, ht, n) == -1 and call(1, ht, n) == -1
        assert lib.eccb200_decdsa_sign_batch(eng._h, ht, n, _buf(privs), _buf(digests), _buf(sigs), _buf(st)) == -1
    assert call(1, 2, n, with_nonces=False) == -1   # ECDSA without nonces
    assert call(1, 2, 0, with_nonces=False) == -1
    bad_off = off.copy()
    bad_off[2] = 0
    assert call(14, 2, n, offsets=bad_off) == -1
    bad_off = off.copy()
    bad_off[0] = 1
    assert call(1, 2, n, offsets=bad_off) == -1
    assert (sigs == 0x5A).all() and (st == 9).all()
    # DECDSA ignores the nonces
    assert call(14, 1, n, with_nonces=False) == 0 and (st == 0).all()
    s1 = sigs.copy()
    assert call(14, 1, n) == 0 and (sigs == s1).all()
    # SHA-224 stays refused by the older entry points
    out = np.zeros((n, 64), np.uint8)
    assert lib.eccb200_hash_batch(eng._h, 1, n, _buf(blob), _buf(off), _buf(out)) == -1
    assert lib.eccb200_sign_msgs_batch(eng._h, 6, 1, n, _buf(privs), None, _buf(nonces), _buf(blob), _buf(off), None,
                                       None, _buf(sigs), _buf(st)) == -1
    # _dev: a misaligned buffer is refused before anything runs (d_msgs may be anywhere)
    d_priv = torch.zeros(n * qlen + 1, dtype=torch.uint8, device="cuda")
    d_priv[1:] = _t(privs.reshape(-1))
    d_nonce = torch.zeros(n * qlen + 1, dtype=torch.uint8, device="cuda")
    d_nonce[1:] = _t(nonces.reshape(-1))
    d_sigs = torch.full((n, 2 * qlen), 0x5A, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    d_blob, d_off = _t(blob), _t(off.view(np.int64))
    assert lib.eccb200_decdsa_sign_batch_dev(eng._h, 2, n, d_priv.data_ptr() + 1, _t(digests).data_ptr(),
                                             d_sigs.data_ptr(), d_st.data_ptr(), None) == -1
    assert b"aligned" in lib.eccb200_last_error()
    assert lib.eccb200_ecdsa_sign_msgs_batch_dev(eng._h, 14, 2, n, d_priv.data_ptr() + 1, None, d_blob.data_ptr(),
                                                 d_off.data_ptr(), d_sigs.data_ptr(), d_st.data_ptr(), None) == -1
    assert lib.eccb200_ecdsa_sign_msgs_batch_dev(eng._h, 1, 2, n, _t(privs).data_ptr(), d_nonce.data_ptr() + 1,
                                                 d_blob.data_ptr(), d_off.data_ptr(), d_sigs.data_ptr(),
                                                 d_st.data_ptr(), None) == -1
    assert lib.eccb200_ecdsa_sign_msgs_batch_dev(eng._h, 1, 2, n, _t(privs).data_ptr(), None, d_blob.data_ptr(),
                                                 d_off.data_ptr(), d_sigs.data_ptr(), d_st.data_ptr(), None) == -1
    assert lib.eccb200_ecdsa_sign_msgs_batch_dev(eng._h, 14, 9, n, _t(privs).data_ptr(), None, d_blob.data_ptr(),
                                                 d_off.data_ptr(), d_sigs.data_ptr(), d_st.data_ptr(), None) == -1
    torch.cuda.synchronize()
    assert (d_sigs == 0x5A).all() and (d_st == 9).all()
    # a misaligned d_msgs is fine
    m1 = torch.zeros(blob.size + 1, dtype=torch.uint8, device="cuda")
    m1[1:] = d_blob
    assert lib.eccb200_ecdsa_sign_msgs_batch_dev(eng._h, 14, 1, n, _t(privs).data_ptr(), None, m1.data_ptr() + 1,
                                                 d_off.data_ptr(), d_sigs.data_ptr(), d_st.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert (d_st == 0).all() and (d_sigs.cpu().numpy() == s1).all()
