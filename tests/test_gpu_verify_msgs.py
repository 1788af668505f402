"""ECKCDSA / ECSDSA / ECOSDSA / ECGDSA / ECRDSA / SM2 verification on the device (eccb200_verify_msgs_batch[_dev]): the
reference's known answers, parity of verdicts with the reference's ec_verify on valid and corrupted signatures, round
trips with the device signers at 2^16, rejected items at chosen lanes of the CTA-wide inversion, the crafted vectors of
test_verify_msgs_host, the chunked host pipeline against the device-pointer form, and the argument checks."""
import os

import numpy as np
import pytest

from common import ALL_CURVES, ORDER, hx, random_scalars, rng, _buf
from test_sign_msgs_host import HASH_IDS, be, pack
from test_verify_msgs_host import ALGS, CRAFTED, HASHES, crafted_batch, kat_vectors, ref_verify, rlen, valid_batch

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


def verify_dev(eng, alg, hash_name, sigs, pubs, msgs, ids=None):
    import torch
    n = len(msgs)
    blob, off = pack(msgs)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_v = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    d_ids = d_ioff = None
    if ids is not None:
        iblob, ioff = pack(ids)
        d_ids, d_ioff = t(iblob), t(ioff.view(np.int64))
    eng.verify_msgs_batch_dev(alg, hash_name, t(sigs), t(pubs), t(blob), t(off.view(np.int64)), d_v, d_ids=d_ids,
                              d_id_offsets=d_ioff)
    torch.cuda.synchronize()
    return d_v.cpu().numpy()


def verify(eng, form, alg, hash_name, sigs, pubs, msgs, ids=None):
    if form == "host":
        return eng.verify_msgs_batch(alg, hash_name, sigs, pubs, msgs, ids=ids)
    return verify_dev(eng, alg, hash_name, sigs, pubs, msgs, ids)


def test_kat():
    ran = 0
    for curve, alg, hash_name, sig, pub, msg, adata in kat_vectors():
        if hash_name not in HASH_IDS:
            continue
        eng = engine(curve)
        sigs = np.stack([hx(sig), hx(sig)])
        sigs[1, 0] ^= 0x80
        pubs = np.stack([hx(pub), hx(pub)])
        msgs = [bytes.fromhex(msg)] * 2
        ids = [bytes.fromhex(adata)] * 2 if alg == "SM2" else None
        for form in ("host", "dev"):
            assert list(verify(eng, form, alg, hash_name, sigs, pubs, msgs, ids)) == [0, -1], (curve, alg, form)
        ran += 1
    assert ran == 26


def mix_corruptions(curve, alg, hash_name, sigs, pubs, msgs, ids, tag):
    """a bit of r, of s, of the message or of the key flipped on about one item in three; s = 0 and r = q on a few"""
    _, plen, qlen = ALL_CURVES[curve]
    g = rng(tag)
    rl = rlen(curve, alg, hash_name)
    for i in range(len(msgs)):
        kind = int(g.integers(0, 9))
        if kind == 0:
            sigs[i, int(g.integers(0, rl))] ^= 1 << int(g.integers(0, 8))
        elif kind == 1:
            sigs[i, rl + int(g.integers(0, qlen))] ^= 1 << int(g.integers(0, 8))
        elif kind == 2:
            msgs[i] = msgs[i] + b"\x01"
        elif kind == 3:
            pubs[i, int(g.integers(0, 2 * plen))] ^= 1 << int(g.integers(0, 8))
        elif kind == 4 and i % 4 == 0:
            sigs[i, rl:] = 0
        elif kind == 4 and i % 4 == 1 and rl == qlen:
            sigs[i, :rl] = be(ORDER[curve], qlen)
        elif kind == 4 and alg == "SM2":
            ids[i] = ids[i] + b"\x02"


SIZES = (1, 127, 128, 129, 383, 385)
CASES = [(c, a) for c in ALL_CURVES for a in ALGS]


@pytest.mark.parametrize("curve,alg", CASES)
def test_parity_with_reference(curve, alg):
    """every curve and scheme at every size of SIZES (ragged CTAs), a hash per size, host and device-pointer forms"""
    i = CASES.index((curve, alg))
    eng = engine(curve)
    for j, n in enumerate(SIZES):
        hash_name = HASHES[(i + j) % len(HASHES)]
        tag = 20000 + 10 * i + j
        sigs, pubs, msgs, ids = valid_batch(curve, alg, hash_name, max(n, 3), tag)
        sigs, pubs, msgs = sigs[:n].copy(), pubs[:n].copy(), msgs[:n]
        ids = ids[:n] if ids is not None else None
        if n > 1:
            mix_corruptions(curve, alg, hash_name, sigs, pubs, msgs, ids, tag + 7)
        want = ref_verify(curve, alg, hash_name, sigs, pubs, msgs, ids)
        form = "host" if (i + j) % 2 == 0 else "dev"
        got = verify(eng, form, alg, hash_name, sigs, pubs, msgs, ids)
        assert (got == want).all(), (n, hash_name, form)
        if n > 1:
            assert (want == 0).any() and (want == -1).any()
        else:
            assert want[0] == 0


@pytest.mark.parametrize("curve,alg,hash_name", [("SECP256R1", "ECSDSA", "SHA256"), ("SM2P256V1", "SM2", "SM3"),
                                                 ("SECP384R1", "ECGDSA", "SHA3_384")])
def test_round_trip_2_16(curve, alg, hash_name):
    """2^16 signatures of the device signers all verify, in both forms; one changed message (and for SM2 one changed
    ID) fails exactly that item"""
    n = 1 << 16
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    eng = engine(curve)
    g = rng(31337)
    privs = random_scalars(curve, n, tag=31338)
    nonces = random_scalars(curve, n, tag=31339)
    msgs = [g.bytes(int(k)) for k in g.integers(0, 100, size=n)]
    ids = [g.bytes(int(k)) for k in g.integers(0, 40, size=n)] if alg == "SM2" else None
    if alg == "ECGDSA":  # its public key is x^-1 * G
        kp = np.stack([be(pow(int.from_bytes(x.tobytes(), "big"), -1, q), qlen) for x in privs])
    else:
        kp = privs
    pubs, pst = eng.prj_pt_mul_batch(kp)
    assert (pst == 0).all()
    if alg == "ECSDSA":
        sigs, st = eng.schnorr_sign_msgs_batch(alg, hash_name, privs, nonces, msgs)
    else:
        sigs, st = eng.sign_msgs_batch(alg, hash_name, privs, nonces, msgs, pubkeys=pubs, ids=ids)
    assert (st == 0).all()
    for form in ("host", "dev"):
        assert (verify(eng, form, alg, hash_name, sigs, pubs, msgs, ids) == 0).all(), form
    keep = msgs[40000]
    msgs[40000] = keep + b"\x01"
    v = verify(eng, "host", alg, hash_name, sigs, pubs, msgs, ids)
    assert v[40000] == -1 and (np.delete(v, 40000) == 0).all()
    msgs[40000] = keep
    if alg == "SM2":
        keep = ids[777]
        ids[777] = keep + b"\x01"
        v = verify(eng, "dev", alg, hash_name, sigs, pubs, msgs, ids)
        assert v[777] == -1 and (np.delete(v, 777) == 0).all()
        ids[777] = keep
    idx = np.sort(g.choice(n, 256, replace=False))
    want = ref_verify(curve, alg, hash_name, sigs[idx], pubs[idx], [msgs[j] for j in idx],
                      [ids[j] for j in idx] if ids is not None else None)
    assert (want == 0).all()


@pytest.mark.parametrize("alg", ["ECGDSA", "ECRDSA"])
@pytest.mark.parametrize("curve", ["SECP256R1", "SECP521R1"])
def test_rejected_items_at_chosen_lanes(curve, alg):
    """r = 0, s = 0, r >= q and a key off the curve at lanes 0, 1, 63, 64 and 127 of the first CTA, over the whole
    second CTA and last: those items stay out of the shared inversion, so every other verdict is the one of the
    all-valid batch"""
    _, plen, qlen = ALL_CURVES[curve]
    q = ORDER[curve]
    eng = engine(curve)
    for n in (383, 385):
        hash_name = "SHA256" if n == 383 else "SHA3_512"
        sigs, pubs, msgs, _ = valid_batch(curve, alg, hash_name, n, 30000 + n)
        for form in ("host", "dev"):
            assert (verify(eng, form, alg, hash_name, sigs, pubs, msgs) == 0).all(), form
        bad = [0, 1, 63, 64, 127] + list(range(128, 256)) + [n - 1]
        bs, bp = sigs.copy(), pubs.copy()
        for k, j in enumerate(bad):
            kind = k % 4
            if kind == 0:
                bs[j, :qlen] = 0                               # r = 0
            elif kind == 1:
                bs[j, qlen:] = 0                               # s = 0
            elif kind == 2:
                bs[j, :qlen] = be(q + (j % 3), qlen) if q + 2 < 1 << (8 * qlen) else 0xFF  # r >= q
            else:
                bp[j, 2 * plen - 1] ^= 1                       # key off the curve
        keep = np.ones(n, bool)
        keep[bad] = False
        want = ref_verify(curve, alg, hash_name, bs, bp, msgs)
        assert (want[bad] == -1).all() and (want[keep] == 0).all()
        for form in ("host", "dev"):
            got = verify(eng, form, alg, hash_name, bs, bp, msgs)
            assert (got == want).all(), form


@pytest.mark.parametrize("alg,kind", CRAFTED)
@pytest.mark.parametrize("curve", ["SECP256R1", "FRP256V1", "SECP521R1", "SECP224R1", "SM2P256V1"])
def test_crafted_vectors_on_device(curve, alg, kind):
    """the crafted vectors among valid neighbours (lanes 0, 1, 63, 64, 127 and last of 129 items): rejected by the
    reference and by both forms, the neighbours still verify"""
    hash_name = "SHA256" if curve != "SM2P256V1" else "SM3"
    n = 129
    sigs, pubs, msgs, ids = valid_batch(curve, alg, hash_name, n, 40000 + CRAFTED.index((alg, kind)))
    lanes = [0, 1, 63, 64, 127, 128]
    cs, cp, cm, ci = crafted_batch(curve, alg, hash_name, kind, len(lanes), 41000 + CRAFTED.index((alg, kind)))
    for k, j in enumerate(lanes):
        sigs[j], pubs[j], msgs[j] = cs[k], cp[k], cm[k]
        if ids is not None:
            ids[j] = ci[k]
    want = ref_verify(curve, alg, hash_name, sigs, pubs, msgs, ids)
    keep = np.ones(n, bool)
    keep[lanes] = False
    assert (want[lanes] == -1).all() and (want[keep] == 0).all()
    for form in ("host", "dev"):
        assert (verify(engine(curve), form, alg, hash_name, sigs, pubs, msgs, ids) == want).all(), form


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
    g = rng(5353)
    privs = random_scalars(curve, n, tag=5354)
    nonces = random_scalars(curve, n, tag=5355)
    pubs, pst = eng.prj_pt_mul_batch(privs)
    assert (pst == 0).all()
    lens = g.integers(0, 91, size=n)
    data = g.bytes(int(lens.sum()) + 1)
    cut = np.concatenate([[0], np.cumsum(lens)])
    msgs = [data[cut[j]:cut[j + 1]] for j in range(n)]
    ids = [data[:int(k)] for k in g.integers(0, 21, size=n)]
    sigs, st = eng.sign_msgs_batch(alg, hash_name, privs, nonces, msgs, pubkeys=pubs, ids=ids)
    assert (st == 0).all()
    bad = np.arange(5, n, 9973)
    for j in bad:
        sigs[j, -1] ^= 1
    got = eng.verify_msgs_batch(alg, hash_name, sigs, pubs, msgs, ids=ids)
    dev = verify_dev(eng, alg, hash_name, sigs, pubs, msgs, ids)
    eng.close()
    assert (got == dev).all()
    keep = np.ones(n, bool)
    keep[bad] = False
    assert (got[bad] == -1).all() and (got[keep] == 0).all()
    idx = np.sort(np.concatenate([g.choice(n, 500, replace=False), bad[:11], [n - 1]]))
    want = ref_verify(curve, alg, hash_name, sigs[idx], pubs[idx], [msgs[j] for j in idx], [ids[j] for j in idx])
    assert (want == got[idx]).all()


def test_api_edges():
    import torch
    import libecc_b200
    curve = "SECP256R1"
    eng = engine(curve)
    lib = libecc_b200.load_library()
    _, plen, qlen = ALL_CURVES[curve]
    n = 4
    sigs, pubs, msgs, ids = valid_batch(curve, "SM2", "SM3", n, 50000)
    blob, off = pack(msgs)
    iblob, ioff = pack(ids)
    v = np.full(n, 9, np.int8)

    def call(sig_type, hash_type, count, s=sigs, p=pubs, offsets=off, with_ids=True, id_offsets=ioff, out=v):
        return lib.eccb200_verify_msgs_batch(eng._h, sig_type, hash_type, count, _buf(s) if s is not None else None,
                                             _buf(p) if p is not None else None, _buf(blob),
                                             _buf(offsets) if offsets is not None else None,
                                             _buf(iblob) if with_ids else None,
                                             _buf(id_offsets) if with_ids else None,
                                             _buf(out) if out is not None else None)

    assert call(8, 11, 0) == 0                    # n = 0: nothing to do, nothing written
    for alg in (0, 1, 5, 9, 14, 18, 20):          # ECDSA, ECFSDSA, BIP0340, DECDSA, BIGN: not served here
        assert call(alg, 11, n) == -1
    for ht in (0, 1, 9, 10, 12):
        assert call(8, ht, n) == -1
    assert call(8, 11, n, with_ids=False) == -1   # SM2 without IDs
    assert call(8, 11, n, s=None) == -1 and call(8, 11, n, p=None) == -1 and call(8, 11, n, offsets=None) == -1
    assert call(8, 11, n, out=None) == -1
    bad_off = off.copy()
    bad_off[2] = 0
    assert call(8, 11, n, offsets=bad_off) == -1
    bad_ioff = ioff.copy()
    assert bad_ioff[2] > 0
    bad_ioff[3] = 0
    assert call(8, 11, n, id_offsets=bad_ioff) == -1
    assert (v == 9).all()
    assert call(8, 11, n) == 0 and (v == 0).all()
    assert lib.eccb200_sign_sig_len(eng._h, 3, 2) == -1 and lib.eccb200_sign_sig_len(eng._h, 4, 2) == -1
    # _dev: unsupported schemes and misaligned buffers are refused before anything runs
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_v = torch.full((n,), 9, dtype=torch.int8, device="cuda")
    d_sigs, d_pubs, d_blob, d_off = t(sigs), t(pubs), t(blob), t(off.view(np.int64))
    d_ids, d_ioff = t(iblob), t(ioff.view(np.int64))
    d_mis = torch.zeros(n * 2 * qlen + 16, dtype=torch.uint8, device="cuda")
    d_mis[1:1 + n * 2 * qlen] = d_sigs.reshape(-1)

    def dcall(sig_type, hash_type, s_ptr, p_ptr, with_ids=True):
        return lib.eccb200_verify_msgs_batch_dev(eng._h, sig_type, hash_type, n, s_ptr, p_ptr, d_blob.data_ptr(),
                                                 d_off.data_ptr(), d_ids.data_ptr() if with_ids else None,
                                                 d_ioff.data_ptr() if with_ids else None, d_v.data_ptr(), None)

    for alg in (1, 5, 14, 20):
        assert dcall(alg, 2, d_sigs.data_ptr(), d_pubs.data_ptr()) == -1
    assert dcall(8, 1, d_sigs.data_ptr(), d_pubs.data_ptr()) == -1
    assert dcall(8, 11, d_sigs.data_ptr(), d_pubs.data_ptr(), with_ids=False) == -1
    assert dcall(8, 11, d_mis.data_ptr() + 1, d_pubs.data_ptr()) == -1 and b"aligned" in lib.eccb200_last_error()
    d_pmis = torch.zeros(n * 2 * plen + 16, dtype=torch.uint8, device="cuda")
    d_pmis[8:8 + n * 2 * plen] = d_pubs.reshape(-1)
    assert dcall(8, 11, d_sigs.data_ptr(), d_pmis.data_ptr() + 8) == -1
    torch.cuda.synchronize()
    assert (d_v == 9).all()
    assert dcall(8, 11, d_sigs.data_ptr(), d_pubs.data_ptr()) == 0
    torch.cuda.synchronize()
    assert (d_v == 0).all()
    # an SM2 ID over 8191 bytes makes that item invalid, in both forms; its neighbours verify
    ids2 = list(ids)
    ids2[1] = bytes(8192)
    for form in ("host", "dev"):
        assert list(verify(eng, form, "SM2", "SM3", sigs, pubs, msgs, ids2)) == [0, -1, 0, 0], form
