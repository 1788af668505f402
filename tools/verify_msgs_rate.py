"""ECKCDSA / ECSDSA / ECOSDSA / ECGDSA / ECRDSA / SM2 verification rate on one GPU (DESIGN.md §9): 2^20 valid signatures
per scheme of 32-byte messages, made by the device signers, the first five on SECP256R1 with SHA-256 and SM2 on
SM2P256V1 with SM3 and a 16-byte ID.  Device-resident rate: CUDA events around eccb200_verify_msgs_batch_dev after a
warm-up of the same shape; end-to-end rate: host clock around the host-pointer entry point on packed messages (copies
included).  The bare double-scalar launch (eccb200_double_smul_batch_dev) on the same n and curve shows what the prep
and finish kernels add to the elliptic-curve work.  Every verdict is checked (all valid, both forms agree), and a
seeded sample against the unmodified reference's ec_verify.  Prints the card's name and power limit with the numbers.
Scheme names on the command line (e.g. `ECGDSA SM2`) restrict the run to those schemes."""
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
from common import ORDER, random_scalars, rng  # noqa: E402
from test_verify_msgs_host import ref_verify  # noqa: E402

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


CONFIGS = (("ECKCDSA", "SECP256R1", "SHA256"), ("ECSDSA", "SECP256R1", "SHA256"), ("ECOSDSA", "SECP256R1", "SHA256"),
           ("ECGDSA", "SECP256R1", "SHA256"), ("ECRDSA", "SECP256R1", "SHA256"), ("SM2", "SM2P256V1", "SM3"))
bare = {}
for alg, curve, hash_name in CONFIGS:
    if len(sys.argv) > 1 and alg not in sys.argv[1:]:
        continue
    eng = libecc_b200.Engine(curve)
    q = ORDER[curve]
    g = rng(31)
    privs = random_scalars(curve, N, tag=32)
    nonces = random_scalars(curve, N, tag=33)
    blob = g.integers(0, 256, size=32 * N, dtype=np.uint8)
    msgs = [blob[32 * i:32 * i + 32].tobytes() for i in range(N)]
    ids = [ID] * N
    if alg in ("ECKCDSA", "ECGDSA"):  # the public key of these two is x^-1 * G
        kp = np.stack([np.frombuffer(pow(int.from_bytes(x.tobytes(), "big"), -1, q).to_bytes(eng.qlen, "big"),
                                     np.uint8) for x in privs])
    else:
        kp = privs
    pubs, pst = eng.prj_pt_mul_batch(kp)
    assert (pst == 0).all()
    if alg in ("ECSDSA", "ECOSDSA"):
        sigs, st = eng.schnorr_sign_msgs_batch(alg, hash_name, privs, nonces, msgs)
    else:
        sigs, st = eng.sign_msgs_batch(alg, hash_name, privs, nonces, msgs, pubkeys=pubs, ids=ids)
    assert (st == 0).all()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    id_blob = np.frombuffer(ID * N, np.uint8).copy()
    d_s, d_p, d_m, d_id = t(sigs), t(pubs), t(blob), t(id_blob)
    d_off = t(np.arange(N + 1, dtype=np.int64) * 32)
    d_ioff = t(np.arange(N + 1, dtype=np.int64) * len(ID))
    d_v = torch.full((N,), 9, dtype=torch.int8, device=dev)
    ms = timed(lambda: eng.verify_msgs_batch_dev(alg, hash_name, d_s, d_p, d_m, d_off, d_v, d_ids=d_id,
                                                 d_id_offsets=d_ioff, stream_handle=stream))
    if curve not in bare:  # the double-scalar kernel alone on the same n: a || b and the keys already on the device
        ab = np.concatenate([random_scalars(curve, N, tag=34), random_scalars(curve, N, tag=35)], axis=1)
        d_ab, d_w = t(ab), torch.zeros((N, 2 * eng.plen), dtype=torch.uint8, device=dev)
        d_st = torch.zeros(N, dtype=torch.int8, device=dev)
        bare[curve] = timed(lambda: eng.lib.eccb200_double_smul_batch_dev(
            eng._h, N, d_ab.data_ptr(), d_p.data_ptr(), d_w.data_ptr(), d_st.data_ptr(), stream))
        assert (d_st.cpu().numpy() == 0).all()
    off = np.arange(N + 1, dtype=np.uint64) * 32
    ioff = np.arange(N + 1, dtype=np.uint64) * len(ID)
    v = np.full(N, 9, np.int8)

    def host_call():  # the host-pointer entry point on packed messages: copies, kernels, synchronisation
        assert eng.lib.eccb200_verify_msgs_batch(
            eng._h, eng.VERIFY_ALGS[alg], eng.SIGN_HASH_IDS[hash_name], N, sigs.ctypes.data, pubs.ctypes.data,
            blob.ctypes.data, off.ctypes.data, id_blob.ctypes.data, ioff.ctypes.data, v.ctypes.data) == 0
    host_call()  # warm-up
    t0 = time.perf_counter()
    for _ in range(REPS):
        host_call()
    e2e = (time.perf_counter() - t0) / REPS
    assert (v == 0).all() and (d_v.cpu().numpy() == 0).all()
    assert (eng.verify_msgs_batch(alg, hash_name, sigs, pubs, msgs, ids=ids) == 0).all()
    idx = np.sort(rng(36).choice(N, 256, replace=False))
    want = ref_verify(curve, alg, hash_name, sigs[idx], pubs[idx], [msgs[i] for i in idx],
                      [ids[i] for i in idx] if alg == "SM2" else None)
    assert (want == 0).all()
    print(f"{curve} {alg} verify, {hash_name}, 32-byte messages: device-resident {N / ms / 1e3:.2f} M/s "
          f"({ms:.2f} ms per 2^20), end-to-end {N / e2e / 1e6:.2f} M/s; bare double-scalar kernel "
          f"{N / bare[curve] / 1e3:.2f} M/s ({bare[curve]:.2f} ms); all verdicts valid, the reference agrees on a "
          f"sample")
    eng.close()
