"""ECKCDSA / ECGDSA / ECRDSA / SM2 signing rate on one GPU (DESIGN.md §9): 2^20 signatures per scheme of 32-byte
messages, ECKCDSA / ECGDSA / ECRDSA on SECP256R1 with SHA-256 and SM2 on SM2P256V1 with SM3 and a 16-byte ID.
Device-resident rate: CUDA events around eccb200_sign_msgs_batch_dev after a warm-up of the same shape; end-to-end
rate: host clock around the host-pointer entry point on packed messages (copies included).  Every timed output is
checked against the host-pointer form, and a seeded sample against the unmodified reference's signer.
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
from common import random_scalars, rng  # noqa: E402
from test_sign_msgs_host import ref_sign  # noqa: E402

N = 1 << 20
REPS = 3
ID = b"1234567812345678"
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


for alg, curve, hash_name in (("ECKCDSA", "SECP256R1", "SHA256"), ("ECGDSA", "SECP256R1", "SHA256"),
                              ("ECRDSA", "SECP256R1", "SHA256"), ("SM2", "SM2P256V1", "SM3")):
    eng = libecc_b200.Engine(curve)
    g = rng(21)
    privs = random_scalars(curve, N, tag=22)
    nonces = random_scalars(curve, N, tag=23)
    blob = g.integers(0, 256, size=32 * N, dtype=np.uint8)
    msgs = [blob[32 * i:32 * i + 32].tobytes() for i in range(N)]
    ids = [ID] * N
    # the scheme's public key: x*G for SM2; ECKCDSA's is x^-1*G, but the signer takes whatever key it is given, so x*G
    # stands in for the timing and the reference's own key is used for the sample below
    pubs, _ = eng.prj_pt_mul_batch(privs)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    id_blob = np.frombuffer(ID * N, np.uint8)
    d_x, d_k, d_p, d_m, d_id = t(privs), t(nonces), t(pubs), t(blob), t(id_blob)
    d_off = t(np.arange(N + 1, dtype=np.int64) * 32)
    d_ioff = t(np.arange(N + 1, dtype=np.int64) * len(ID))
    sl = eng.sign_sig_len(alg, hash_name)
    d_sig = torch.zeros((N, sl), dtype=torch.uint8, device=dev)
    d_st = torch.zeros(N, dtype=torch.int8, device=dev)
    ms = timed(lambda: eng.sign_msgs_batch_dev(alg, hash_name, d_x, d_k, d_m, d_off, d_sig, d_st, d_pubkeys=d_p,
                                               d_ids=d_id, d_id_offsets=d_ioff, stream_handle=stream))
    off = np.arange(N + 1, dtype=np.uint64) * 32
    ioff = np.arange(N + 1, dtype=np.uint64) * len(ID)
    sigs = np.zeros((N, sl), np.uint8)
    st = np.zeros(N, np.int8)

    def host_call():  # the host-pointer entry point on packed messages: copies, kernels, synchronisation
        assert eng.lib.eccb200_sign_msgs_batch(
            eng._h, eng.SIGN_ALGS[alg], eng.SIGN_HASH_IDS[hash_name], N, privs.ctypes.data, pubs.ctypes.data,
            nonces.ctypes.data, blob.ctypes.data, off.ctypes.data, id_blob.ctypes.data, ioff.ctypes.data,
            sigs.ctypes.data, st.ctypes.data) == 0
    host_call()  # warm-up
    t0 = time.perf_counter()
    for _ in range(REPS):
        host_call()
    e2e = (time.perf_counter() - t0) / REPS
    api_sigs, api_st = eng.sign_msgs_batch(alg, hash_name, privs, nonces, msgs, pubkeys=pubs, ids=ids)
    assert (api_sigs == sigs).all() and (api_st == st).all()
    assert (st == 0).all() and (d_st.cpu().numpy() == 0).all() and (d_sig.cpu().numpy() == sigs).all()
    idx = np.sort(rng(24).choice(N, 256, replace=False))
    want, rpubs, wst = ref_sign(curve, alg, hash_name, privs[idx], nonces[idx], [msgs[i] for i in idx],
                                [ids[i] for i in idx])
    got, gst = eng.sign_msgs_batch(alg, hash_name, privs[idx], nonces[idx], [msgs[i] for i in idx], pubkeys=rpubs,
                                   ids=[ids[i] for i in idx])
    assert (wst == 0).all() and (gst == 0).all() and (got == want).all()
    if alg != "ECKCDSA":  # the key enters only ECKCDSA's z and SM2's Z; SM2's is x*G
        assert (sigs[idx] == want).all()
    print(f"{curve} {alg} sign, {hash_name}, 32-byte messages: device-resident {N / ms / 1e3:.2f} M/s "
          f"({ms:.2f} ms per 2^20), end-to-end {N / e2e / 1e6:.2f} M/s; outputs match the host-pointer form and a "
          f"sample of the reference")
    eng.close()
