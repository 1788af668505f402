"""ECDSA public-key recovery rate on one GPU (DESIGN.md §9): 2^20 valid signatures on 32-byte digests, made by the
device key generation and signer, on SECP256R1, SECP256K1, SECP384R1 and SECP224R1.  Device-resident rate: CUDA events
around eccb200_ecdsa_recover_batch_dev after a warm-up of the same shape; end-to-end rate: host clock around the
host-pointer entry point (copies included).  In the same run, eccb200_ecdsa_verify_batch_dev on the same signatures,
digests and true keys: recovery costs one verification's elliptic-curve work plus one addition and the square root.
Every output is checked (both keys finite, the true key among them, both forms agree) and a seeded sample against the
unmodified reference's __ecdsa_public_key_from_sig.  Prints the card's name and power limit with the numbers.  Curve
names on the command line restrict the run to those curves."""
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
from common import rng  # noqa: E402
from test_ecdsa_recover_host import ref_recover  # noqa: E402

N = 1 << 20
REPS = 3
HLEN = 32
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


def scalars(eng, tag):
    """N scalars in [1, q-1]: the top bit cleared (q > 2^(8*qlen - 1) on the four curves) and the low bit set"""
    raw = rng(tag).integers(0, 256, size=(N, eng.qlen), dtype=np.uint8)
    raw[:, 0] &= 0x7F
    raw[:, -1] |= 1
    return raw


for curve in ("SECP256R1", "SECP256K1", "SECP384R1", "SECP224R1"):
    if len(sys.argv) > 1 and curve not in sys.argv[1:]:
        continue
    eng = libecc_b200.Engine(curve)
    privs, nonces = scalars(eng, 41), scalars(eng, 42)
    dg = rng(43).integers(0, 256, size=(N, HLEN), dtype=np.uint8)
    pubs, pst = eng.prj_pt_mul_batch(privs)
    sigs, sst = eng.ecdsa_sign_batch(privs, nonces, dg, HLEN)
    assert (pst == 0).all() and (sst == 0).all()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_s, d_d, d_p = t(sigs), t(dg), t(pubs)
    d_k = torch.zeros((N, 2, 2 * eng.plen), dtype=torch.uint8, device=dev)
    d_st = torch.full((N, 2), 9, dtype=torch.int8, device=dev)
    d_v = torch.full((N,), 9, dtype=torch.int8, device=dev)
    ms = timed(lambda: eng.ecdsa_recover_batch_dev(d_s, d_d, HLEN, d_k, d_st, stream_handle=stream))
    ms_v = timed(lambda: eng.ecdsa_verify_batch_dev(d_s, d_p, d_d, HLEN, d_v, stream_handle=stream))
    keys, st = eng.ecdsa_recover_batch(sigs, dg, HLEN)  # warm-up of the host form
    t0 = time.perf_counter()
    for _ in range(REPS):
        keys, st = eng.ecdsa_recover_batch(sigs, dg, HLEN)
    e2e = (time.perf_counter() - t0) / REPS
    assert (st == 0).all() and (d_st.cpu().numpy() == 0).all() and (d_k.cpu().numpy() == keys).all()
    assert (d_v.cpu().numpy() == 0).all()
    assert ((keys[:, 0] == pubs).all(1) | (keys[:, 1] == pubs).all(1)).all()
    idx = np.sort(rng(44).choice(N, 64, replace=False))
    want_k, want_s = ref_recover(curve, sigs[idx], dg[idx], HLEN)
    assert (want_s == st[idx]).all() and (want_k == keys[idx]).all()
    print(f"{curve} ECDSA recovery, 32-byte digests: device-resident {N / ms / 1e3:.2f} M/s ({ms:.2f} ms per 2^20), "
          f"end-to-end {N / e2e / 1e6:.2f} M/s; ECDSA verification of the same signatures device-resident "
          f"{N / ms_v / 1e3:.2f} M/s ({ms_v:.2f} ms); recovery / verification = {ms_v / ms:.2f}; all keys checked, "
          f"the reference agrees on a sample")
    eng.close()
