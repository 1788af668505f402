"""Schnorr-family signing rate on one GPU (DESIGN.md §9): 2^20 signatures per scheme of 32-byte messages, ECSDSA /
ECOSDSA / ECFSDSA on SECP256R1 and BIP0340 on SECP256K1, SHA-256.  Device-resident rate: CUDA events around
eccb200_schnorr_sign_msgs_batch_dev after a warm-up of the same shape; end-to-end rate: host clock around the
host-pointer entry point on packed messages (copies included); eccb200_ecdsa_sign_batch_dev at the same size for
comparison.  Every timed output is checked against the host-pointer form, and a seeded sample against the unmodified
reference's signer.
Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import libecc_b200  # noqa: E402
from common import ALL_CURVES, random_scalars, rng  # noqa: E402
from test_schnorr_sign_host import ref_sign  # noqa: E402

N = 1 << 20
REPS = 3
dev = torch.device("cuda:0")
stream = torch.cuda.current_stream().cuda_stream
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()
print(f"GPU: {smi[0] if smi else torch.cuda.get_device_name(0)}")


def timed(fn):
    for _ in range(REPS):  # warm-up of the same shape
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS


for alg, curve in (("ECSDSA", "SECP256R1"), ("ECOSDSA", "SECP256R1"), ("ECFSDSA", "SECP256R1"), ("BIP0340", "SECP256K1")):
    _, plen, qlen = ALL_CURVES[curve]
    eng = libecc_b200.Engine(curve)
    g = rng(11)
    privs = random_scalars(curve, N, tag=12)
    rand = random_scalars(curve, N, tag=13)
    blob = g.integers(0, 256, size=32 * N, dtype=np.uint8)
    msgs = [blob[32 * i:32 * i + 32].tobytes() for i in range(N)]
    pubs, _ = eng.prj_pt_mul_batch(privs)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_x, d_r, d_p, d_m = t(privs), t(rand), t(pubs), t(blob)
    d_off = t((np.arange(N + 1, dtype=np.int64) * 32))
    sl = eng.schnorr_sig_len(alg, "SHA256")
    d_sig = torch.zeros((N, sl), dtype=torch.uint8, device=dev)
    d_st = torch.zeros(N, dtype=torch.int8, device=dev)
    ms = timed(lambda: eng.schnorr_sign_msgs_batch_dev(alg, "SHA256", d_x, d_r, d_m, d_off, d_sig, d_st, d_pubkeys=d_p,
                                                       stream_handle=stream))
    off = np.arange(N + 1, dtype=np.uint64) * 32
    sigs = np.zeros((N, sl), np.uint8)
    st = np.zeros(N, np.int8)

    def host_call():  # the host-pointer entry point on packed messages: copies, kernels, synchronisation
        assert eng.lib.eccb200_schnorr_sign_msgs_batch(
            eng._h, eng.SCHNORR_ALGS[alg], eng.HASH_IDS["SHA256"], N, privs.ctypes.data, pubs.ctypes.data,
            rand.ctypes.data, blob.ctypes.data, off.ctypes.data, sigs.ctypes.data, st.ctypes.data) == 0
    host_call()  # warm-up
    t0 = time.perf_counter()
    for _ in range(REPS):
        host_call()
    e2e = (time.perf_counter() - t0) / REPS
    api_sigs, api_st = eng.schnorr_sign_msgs_batch(alg, "SHA256", privs, rand, msgs, pubkeys=pubs)
    assert (api_sigs == sigs).all() and (api_st == st).all()
    assert (st == 0).all() and (d_st.cpu().numpy() == 0).all() and (d_sig.cpu().numpy() == sigs).all()
    idx = np.sort(rng(14).choice(N, 256, replace=False))
    want, _, wst = ref_sign(curve, alg, "SHA256", privs[idx], rand[idx], [msgs[i] for i in idx])
    assert (wst == 0).all() and (sigs[idx] == want).all()
    print(f"{curve} {alg} sign, SHA-256, 32-byte messages: device-resident {N / ms / 1e3:.2f} M/s ({ms:.2f} ms per 2^20), "
          f"end-to-end {N / e2e / 1e6:.2f} M/s; outputs match the host-pointer form and a sample of the reference")
    if alg == "ECSDSA":
        dg = t(g.integers(0, 256, size=(N, 32), dtype=np.uint8))
        d_es = torch.zeros((N, 2 * qlen), dtype=torch.uint8, device=dev)

        def ecdsa():
            assert eng.lib.eccb200_ecdsa_sign_batch_dev(eng._h, N, d_x.data_ptr(), d_r.data_ptr(), dg.data_ptr(), 32,
                                                        d_es.data_ptr(), d_st.data_ptr(), stream) == 0
        ms = timed(ecdsa)
        assert (d_st.cpu().numpy() == 0).all()
        print(f"{curve} ECDSA sign (pre-hashed digests), same size: device-resident {N / ms / 1e3:.2f} M/s "
              f"({ms:.2f} ms per 2^20)")
    eng.close()
