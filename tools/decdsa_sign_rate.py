"""Deterministic ECDSA (RFC 6979) signing rate on one GPU (DESIGN.md §9): 2^20 signatures of 32-byte messages per
configuration, in one run, device-resident:
  - eccb200_ecdsa_sign_batch_dev (caller's nonces, digests given), the baseline;
  - eccb200_decdsa_sign_batch_dev (nonces derived on the device, digests given);
  - eccb200_ecdsa_sign_msgs_batch_dev with ECDSA and with DECDSA (messages hashed on the device);
on SECP256R1 / SHA-256, BRAINPOOLP256R1 / SHA-256 (retry divergence), SECP384R1 / SHA-384 and SECP521R1 / SHA-512;
plus the end-to-end host-pointer DECDSA message form (copies included, host clock).  CUDA events around each call
after a warm-up of the same shape.  Every DECDSA output is checked against the host-pointer digest form and a seeded
sample against the unmodified reference's DECDSA signer.  Prints the card's name and power limit with the numbers."""
import hashlib
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
from test_decdsa_host import ref_decdsa  # noqa: E402

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


for curve, hash_name in (("SECP256R1", "SHA256"), ("BRAINPOOLP256R1", "SHA256"), ("SECP384R1", "SHA384"),
                         ("SECP521R1", "SHA512")):
    eng = libecc_b200.Engine(curve)
    g = rng(31)
    privs = random_scalars(curve, N, tag=32)
    nonces = random_scalars(curve, N, tag=33)
    blob = g.integers(0, 256, size=32 * N, dtype=np.uint8)
    msgs = [blob[32 * i:32 * i + 32].tobytes() for i in range(N)]
    hf = getattr(hashlib, hash_name.lower())
    digests = np.frombuffer(b"".join(hf(m).digest() for m in msgs), np.uint8).reshape(N, -1)
    hl = digests.shape[1]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_x, d_k, d_h, d_m = t(privs), t(nonces), t(digests), t(blob)
    d_off = t(np.arange(N + 1, dtype=np.int64) * 32)
    d_sig = torch.zeros((N, 2 * eng.qlen), dtype=torch.uint8, device=dev)
    d_st = torch.zeros(N, dtype=torch.int8, device=dev)
    rates = {}

    def ecdsa_digest():
        assert eng.lib.eccb200_ecdsa_sign_batch_dev(eng._h, N, d_x.data_ptr(), d_k.data_ptr(), d_h.data_ptr(), hl,
                                                    d_sig.data_ptr(), d_st.data_ptr(), stream) == 0
    rates["ECDSA digests"] = timed(ecdsa_digest)
    rates["ECDSA messages"] = timed(lambda: eng.ecdsa_sign_msgs_batch_dev("ECDSA", hash_name, d_x, d_m, d_off, d_sig,
                                                                          d_st, d_nonces=d_k, stream_handle=stream))
    assert (d_st.cpu().numpy() == 0).all()
    rates["DECDSA messages"] = timed(lambda: eng.ecdsa_sign_msgs_batch_dev("DECDSA", hash_name, d_x, d_m, d_off, d_sig,
                                                                           d_st, stream_handle=stream))
    msg_sigs = d_sig.cpu().numpy()
    rates["DECDSA digests"] = timed(lambda: eng.decdsa_sign_batch_dev(hash_name, d_x, d_h, d_sig, d_st,
                                                                      stream_handle=stream))
    dev_sigs, dev_st = d_sig.cpu().numpy(), d_st.cpu().numpy()
    off = np.arange(N + 1, dtype=np.uint64) * 32
    sigs = np.zeros((N, 2 * eng.qlen), np.uint8)
    st = np.zeros(N, np.int8)

    def host_call():  # the host-pointer DECDSA message form on packed messages: copies, kernels, synchronisation
        assert eng.lib.eccb200_ecdsa_sign_msgs_batch(eng._h, 14, eng.DECDSA_HASH_IDS[hash_name], N, privs.ctypes.data,
                                                     None, blob.ctypes.data, off.ctypes.data, sigs.ctypes.data,
                                                     st.ctypes.data) == 0
    host_call()  # warm-up
    t0 = time.perf_counter()
    for _ in range(REPS):
        host_call()
    e2e = (time.perf_counter() - t0) / REPS
    hsigs, hst = eng.decdsa_sign_batch(hash_name, privs, digests)
    assert (hst == 0).all() and (dev_st == 0).all() and (st == 0).all()
    assert (dev_sigs == hsigs).all() and (msg_sigs == hsigs).all() and (sigs == hsigs).all()
    idx = np.sort(rng(34).choice(N, 256, replace=False))
    want, _, wst = ref_decdsa(curve, hash_name, privs[idx], [msgs[i] for i in idx])
    assert (wst == 0).all() and (hsigs[idx] == want).all()
    base = rates["ECDSA digests"]
    print(f"{curve} {hash_name}, 32-byte messages, device-resident: " +
          ", ".join(f"{k} {N / v / 1e3:.2f} M/s ({v:.2f} ms, {base / v:.2f}x)" for k, v in rates.items()) +
          f"; end-to-end DECDSA messages {N / e2e / 1e6:.2f} M/s; outputs match the host-pointer digest form and a "
          f"sample of the reference")
    eng.close()
