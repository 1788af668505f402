"""ECDSA public-key recovery on the device (eccb200_ecdsa_recover_batch[_dev]): the reference's known answers, parity
with the reference's __ecdsa_public_key_from_sig on all eleven curves at ragged batch sizes, the crafted kinds (ERR,
Y1 = infinity, Y2 = infinity, both with the doubling branch on the other key) at chosen lanes of a CTA of valid items,
round trips with the device key generation, signer and verifier at 2^16, the chunked host pipeline against the
device-pointer form, and the argument checks.

Every batch is drawn from a per-curve pool of distinct items whose outputs the reference computed once, so any
arrangement of them is checked item by item: the kernel shares three inversions across the 128 threads of a CTA
(r^-1, the window table's Z's and the keys' Z1*Z2), and no item may move its neighbours' keys."""
import os

import numpy as np
import pytest

from common import ALL_CURVES, random_scalars, rng
from test_ecdsa_recover_host import crafted_rows, kat_vectors, parity_batch, ref_recover, valid_items
from test_rare_branches import b2i, be

pytestmark = pytest.mark.gpu

_engines = {}
COMB_W = 8  # small comb tables: these engines fit beside the ones other modules keep
SIZES = (1, 2, 127, 128, 129, 383, 385)
LANES = (0, 1, 63, 64, 127)


def engine(curve):
    import libecc_b200
    if curve not in _engines:
        _engines[curve] = libecc_b200.Engine(curve, device=0, comb_window=COMB_W)
    return _engines[curve]


@pytest.fixture(autouse=True)
def _release_engines():
    """every test gives its engines back: other test modules keep theirs for the whole run"""
    yield
    import torch
    for eng in _engines.values():
        eng.close()
    _engines.clear()
    torch.cuda.empty_cache()


def recover_dev(eng, sigs, digests, hlen):
    import torch
    n = sigs.shape[0]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_keys = torch.full((n, 2, 2 * eng.plen), 0xAA, dtype=torch.uint8, device="cuda")
    d_st = torch.full((n, 2), 9, dtype=torch.int8, device="cuda")
    eng.ecdsa_recover_batch_dev(t(sigs), t(digests), hlen, d_keys, d_st)
    torch.cuda.synchronize()
    return d_keys.cpu().numpy(), d_st.cpu().numpy()


def recover(eng, form, sigs, digests, hlen):
    if form == "host":
        return eng.ecdsa_recover_batch(sigs, digests, hlen)
    return recover_dev(eng, sigs, digests, hlen)


def test_kat():
    for v in kat_vectors():
        curve = v["curve"]
        plen = ALL_CURVES[curve][1]
        sig = np.frombuffer(bytes.fromhex(v["sig"]), np.uint8)[None]
        dg = np.frombuffer(bytes.fromhex(v["digest"]), np.uint8)[None]
        pub = bytes.fromhex(v["pub"])
        half = len(pub) // 2
        pub = be(b2i(pub[:half]), plen).tobytes() + be(b2i(pub[half:]), plen).tobytes()
        want_k, want_s = ref_recover(curve, sig, dg, dg.shape[1])
        for form in ("host", "dev"):
            keys, st = recover(engine(curve), form, sig, dg, dg.shape[1])
            assert (st == want_s).all() and (keys == want_k).all(), (v["name"], form)
            assert pub in (keys[0, 0].tobytes(), keys[0, 1].tobytes()), (v["name"], form)


# ------------------------------------------------------------------------------------------ the per-curve pools

_pools = {}


def pool(curve):
    """(sigs, digests, keys, status, kinds) of distinct items with hlen = qlen: valid signatures, the edge / non-x /
    restart-quirk / r >= p items of the CPU parity batch, and crafted infinity + doubling vectors; kinds names the
    indices of each kind"""
    if curve not in _pools:
        qlen = ALL_CURVES[curve][2]
        tag = 8100 + 10 * ALL_CURVES[curve][0]
        ps, pd = parity_batch(curve, qlen, tag)
        cs, cd, _ = crafted_rows(curve, tag + 5, 8)
        vs, vd, _ = valid_items(curve, 40, qlen, tag + 7)
        sigs, dg = np.concatenate([vs, ps, cs]), np.concatenate([vd, pd, cd])
        keys, st = ref_recover(curve, sigs, dg, qlen)
        nv = len(vs)
        kinds = {
            "valid": [i for i in range(nv) if (st[i] == 0).all()],
            "err": [i for i in range(len(sigs)) if (st[i] == -1).all()],
            "inf1": [i for i in range(len(sigs)) if list(st[i]) == [1, 0]],
            "inf2": [i for i in range(len(sigs)) if list(st[i]) == [0, 1]],
        }
        assert len(kinds["valid"]) == nv and all(len(k) >= 4 for k in kinds.values()), {k: len(v) for k, v in kinds.items()}
        _pools[curve] = (sigs, dg, keys, st, kinds)
    return _pools[curve]


def check(curve, idx, forms=("host", "dev")):
    sigs, dg, keys, st, _ = pool(curve)
    idx = np.asarray(idx)
    qlen = ALL_CURVES[curve][2]
    for form in forms:
        got_k, got_s = recover(engine(curve), form, sigs[idx], dg[idx], qlen)
        bad = np.nonzero((got_s != st[idx]).any(1) | (got_k != keys[idx]).reshape(len(idx), -1).any(1))[0]
        assert len(bad) == 0, (curve, form, len(idx), bad[:10], idx[bad[:10]])


@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_parity_with_reference(curve):
    """every kind of item in random order at every size of SIZES, both forms"""
    npool = len(pool(curve)[0])
    g = rng(8300 + ALL_CURVES[curve][0])
    for n in SIZES:
        idx = np.concatenate([g.permutation(npool) for _ in range(n // npool + 1)])[:n]
        check(curve, idx)


@pytest.mark.parametrize("kind", ["err", "inf1", "inf2"])
@pytest.mark.parametrize("curve", list(ALL_CURVES))
def test_kinds_at_chosen_lanes(curve, kind):
    """the kind at lanes 0, 1, 63, 64 and 127 of the first CTA, as the whole second CTA, and last in batches of 383 and
    385 items, all other items valid"""
    _, _, _, _, kinds = pool(curve)
    valid, special = kinds["valid"], kinds[kind]
    for n in (383, 385):
        idx = np.array([valid[i % len(valid)] for i in range(n)])
        lanes = list(LANES) + list(range(128, 256)) + [n - 1]
        for k, j in enumerate(lanes):
            idx[j] = special[k % len(special)]
        check(curve, idx)


@pytest.mark.parametrize("curve", ["SECP256R1", "SECP256K1", "SECP384R1", "SECP224R1"])
def test_round_trip_2_16(curve):
    """keys from the device key generation, signatures from the device signer: the true key is Y1 or Y2 of every item,
    both keys are finite and both verify on the device; a sample matches the reference"""
    n = 1 << 16
    hlen = 32
    eng = engine(curve)
    privs = random_scalars(curve, n, tag=8501)
    nonces = random_scalars(curve, n, tag=8502)
    dg = rng(8503).integers(0, 256, size=(n, hlen), dtype=np.uint8)
    pubs, pst = eng.prj_pt_mul_batch(privs)
    assert (pst == 0).all()
    sigs, sst = eng.ecdsa_sign_batch(privs, nonces, dg, hlen)
    assert (sst == 0).all()
    keys, st = eng.ecdsa_recover_batch(sigs, dg, hlen)
    dkeys, dst = recover_dev(eng, sigs, dg, hlen)
    assert (st == 0).all() and (dst == st).all() and (dkeys == keys).all()
    assert ((keys[:, 0] == pubs).all(1) | (keys[:, 1] == pubs).all(1)).all()
    for k in range(2):
        assert (eng.ecdsa_verify_batch(sigs, keys[:, k], dg, hlen) == 0).all()
    idx = np.sort(rng(8504).choice(n, 128, replace=False))
    want_k, want_s = ref_recover(curve, sigs[idx], dg[idx], hlen)
    assert (want_s == st[idx]).all() and (want_k == keys[idx]).all()


def test_host_pipeline_longer_than_three_chunks():
    """ECCB200_CHUNK_WAVES=1: the chunk is one wave, so 3 * that + 17 items cross at least three chunk boundaries; the
    host form matches the device-pointer form and the reference on a sample"""
    import torch
    import libecc_b200
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 3 * sms * 16 * 128 + 17
    curve, hlen = "SECP256R1", 48
    os.environ["ECCB200_CHUNK_WAVES"] = "1"
    try:
        eng = libecc_b200.Engine(curve, device=0, comb_window=COMB_W)
    finally:
        del os.environ["ECCB200_CHUNK_WAVES"]
    g = rng(8601)
    sigs = np.concatenate([g.integers(0, 256, size=(n, 1), dtype=np.uint8) & 0x7F,
                           g.integers(0, 256, size=(n, 63), dtype=np.uint8)], axis=1)  # r, s < q: half recover
    dg = g.integers(0, 256, size=(n, hlen), dtype=np.uint8)
    keys, st = eng.ecdsa_recover_batch(sigs, dg, hlen)
    dkeys, dst = recover_dev(eng, sigs, dg, hlen)
    eng.close()
    assert (st == dst).all() and (keys == dkeys).all()
    assert 0.4 < (st[:, 0] == 0).mean() < 0.6
    idx = np.sort(np.concatenate([g.choice(n, 200, replace=False), [0, n - 1]]))
    want_k, want_s = ref_recover(curve, sigs[idx], dg[idx], hlen)
    assert (want_s == st[idx]).all() and (want_k == keys[idx]).all()


def test_api_edges():
    import torch
    import libecc_b200
    curve = "SECP256R1"
    eng = engine(curve)
    lib = libecc_b200.load_library()
    _, plen, qlen = ALL_CURVES[curve]
    sigs, dg, keys, st, kinds = pool(curve)
    idx = kinds["valid"][:4]
    s, d = np.ascontiguousarray(sigs[idx]), np.ascontiguousarray(dg[idx])
    n = len(idx)
    k = np.full((n, 2, 2 * plen), 0xAA, np.uint8)
    o = np.full((n, 2), 9, np.int8)
    ptr = lambda a: a.ctypes.data if a is not None else None

    def call(count, sg=s, di=d, hlen=qlen, kk=k, oo=o):
        return lib.eccb200_ecdsa_recover_batch(eng._h, count, ptr(sg), ptr(di), hlen, ptr(kk), ptr(oo))

    assert call(0) == 0 and call(0, sg=None, di=None, kk=None, oo=None) == 0  # n = 0: nothing to do
    assert call(n, sg=None) == -1 and call(n, di=None) == -1 and call(n, kk=None) == -1 and call(n, oo=None) == -1
    assert call(n, hlen=0) == -1 and call(n, hlen=129) == -1 and b"digest length" in lib.eccb200_last_error()
    assert (k == 0xAA).all() and (o == 9).all()
    assert call(n) == 0 and (o == st[idx]).all() and (k == keys[idx]).all()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_s, d_d = t(s), t(d)
    d_k = torch.full((n, 2, 2 * plen), 0xAA, dtype=torch.uint8, device="cuda")
    d_o = torch.full((n, 2), 9, dtype=torch.int8, device="cuda")
    d_smis = torch.zeros(n * 2 * qlen + 16, dtype=torch.uint8, device="cuda")
    d_smis[8:8 + n * 2 * qlen] = d_s.reshape(-1)
    d_kmis = torch.zeros(n * 4 * plen + 16, dtype=torch.uint8, device="cuda")

    def dcall(count, sp=d_s.data_ptr(), dp=d_d.data_ptr(), hlen=qlen, kp=d_k.data_ptr(), op=d_o.data_ptr()):
        return lib.eccb200_ecdsa_recover_batch_dev(eng._h, count, sp, dp, hlen, kp, op, None)

    assert dcall(0, sp=None, dp=None, kp=None, op=None) == 0
    assert dcall(n, sp=None) == -1 and dcall(n, dp=None) == -1 and dcall(n, kp=None) == -1 and dcall(n, op=None) == -1
    assert dcall(n, hlen=0) == -1 and dcall(n, hlen=129) == -1
    assert dcall(n, sp=d_smis.data_ptr() + 8) == -1 and b"aligned" in lib.eccb200_last_error()
    assert dcall(n, kp=d_kmis.data_ptr() + 4) == -1 and b"aligned" in lib.eccb200_last_error()
    torch.cuda.synchronize()
    assert (d_k == 0xAA).all() and (d_o == 9).all()
    assert dcall(n) == 0
    torch.cuda.synchronize()
    assert (d_o.cpu().numpy() == st[idx]).all() and (d_k.cpu().numpy() == keys[idx]).all()
    # the digest column may sit at any byte (the kernel reads it byte by byte), on every curve
    d_dmis = torch.zeros(n * qlen + 16, dtype=torch.uint8, device="cuda")
    d_dmis[3:3 + n * qlen] = d_d.reshape(-1)
    d_o.fill_(9)
    assert dcall(n, dp=d_dmis.data_ptr() + 3) == 0
    torch.cuda.synchronize()
    assert (d_o.cpu().numpy() == st[idx]).all()
    # with Python's wrappers
    with pytest.raises(ValueError):
        eng.ecdsa_recover_batch(s[:, :-1], d, qlen)
