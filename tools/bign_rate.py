"""BIGN / DBIGN signing and BIGN verification rates on one GPU (DESIGN.md §9): 2^20 items of 32-byte messages per
configuration, in one run, device-resident, with a 13-byte adata record (a 9-byte OID):
  - eccb200_ecdsa_sign_batch_dev (caller's nonces, digests given) and the bare double-scalar kernel
    (eccb200_double_smul_batch_dev), the baselines;
  - eccb200_bign_sign_msgs_batch_dev with BIGN (caller's nonces) and DBIGN (nonces derived on the device);
  - eccb200_bign_verify_msgs_batch_dev on the BIGN signatures;
on SECP256R1 with BELT-HASH and with SHA-256, and BRAINPOOLP256R1 with BELT-HASH (DBIGN's k >= q rounds).  CUDA
events around each call after a warm-up of the same shape.  The signatures must verify, and a seeded sample must equal
the unmodified reference's signatures.  Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import libecc_b200  # noqa: E402
from common import random_scalars, rng  # noqa: E402
from test_bign_host import ref_sign  # noqa: E402

N = 1 << 20
REPS = 3
dev = torch.device("cuda:0")
stream = torch.cuda.current_stream().cuda_stream
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()
print(f"GPU: {smi[0] if smi else torch.cuda.get_device_name(0)}")
ADATA = libecc_b200.bign_adata(bytes.fromhex("608648016503040201"))


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


for curve, hash_name in (("SECP256R1", "BELT_HASH"), ("SECP256R1", "SHA256"), ("BRAINPOOLP256R1", "BELT_HASH")):
    eng = libecc_b200.Engine(curve)
    g = rng(41)
    privs = random_scalars(curve, N, tag=42)
    nonces = random_scalars(curve, N, tag=43)
    blob = g.integers(0, 256, size=32 * N, dtype=np.uint8)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_x, d_k, d_m = t(privs), t(nonces), t(blob)
    d_off = t(np.arange(N + 1, dtype=np.int64) * 32)
    d_ad = t(np.frombuffer(ADATA * N, np.uint8).copy())
    d_adoff = t(np.arange(N + 1, dtype=np.int64) * len(ADATA))
    d_sig = torch.zeros((N, eng.bign_sig_len), dtype=torch.uint8, device=dev)
    d_st = torch.zeros(N, dtype=torch.int8, device=dev)
    pubs, pst = eng.prj_pt_mul_batch(privs)
    assert (pst == 0).all()
    d_pub = t(pubs)
    rates = {}
    d_dig = t(g.integers(0, 256, size=(N, 32), dtype=np.uint8))
    d_esig = torch.zeros((N, 2 * eng.qlen), dtype=torch.uint8, device=dev)
    d_ab = torch.cat([d_k, d_x], dim=1).contiguous()
    d_w = torch.zeros((N, 2 * eng.plen), dtype=torch.uint8, device=dev)

    def ecdsa_digest():
        assert eng.lib.eccb200_ecdsa_sign_batch_dev(eng._h, N, d_x.data_ptr(), d_k.data_ptr(), d_dig.data_ptr(), 32,
                                                    d_esig.data_ptr(), d_st.data_ptr(), stream) == 0

    def double_smul():
        assert eng.lib.eccb200_double_smul_batch_dev(eng._h, N, d_ab.data_ptr(), d_pub.data_ptr(), d_w.data_ptr(),
                                                     d_st.data_ptr(), stream) == 0
    rates["ECDSA sign (digests)"] = timed(ecdsa_digest)
    rates["double-scalar kernel"] = timed(double_smul)
    rates["DBIGN sign"] = timed(lambda: eng.bign_sign_msgs_batch_dev("DBIGN", hash_name, d_x, d_m, d_off, d_ad, d_adoff,
                                                                      d_sig, d_st, stream_handle=stream))
    assert (d_st.cpu().numpy() == 0).all()
    dsigs = d_sig.cpu().numpy()
    rates["BIGN sign"] = timed(lambda: eng.bign_sign_msgs_batch_dev("BIGN", hash_name, d_x, d_m, d_off, d_ad, d_adoff,
                                                                     d_sig, d_st, d_nonces=d_k, stream_handle=stream))
    assert (d_st.cpu().numpy() == 0).all()
    bsigs = d_sig.cpu().numpy()
    d_v = torch.zeros(N, dtype=torch.int8, device=dev)
    rates["BIGN verify"] = timed(lambda: eng.bign_verify_msgs_batch_dev(hash_name, d_sig, d_pub, d_m, d_off, d_ad,
                                                                         d_adoff, d_v, stream_handle=stream))
    assert (d_v.cpu().numpy() == 0).all()
    idx = np.sort(rng(44).choice(N, 256, replace=False))
    msgs = [blob[32 * i:32 * i + 32].tobytes() for i in idx]
    for alg, got in (("BIGN", bsigs), ("DBIGN", dsigs)):
        want, _, wst = ref_sign(curve, alg, hash_name, privs[idx], msgs, [ADATA] * len(idx), nonces[idx])
        assert (wst == 0).all() and (got[idx] == want).all(), alg
    print(f"{curve} {hash_name}, 32-byte messages, device-resident, 2^20 items: " +
          ", ".join(f"{k} {N / v / 1e3:.1f} M/s ({v:.2f} ms)" for k, v in rates.items()) +
          "; signatures verify and a sample equals the reference")
    eng.close()
