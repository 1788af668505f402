"""libecc_b200 — ctypes binding of the C ABI in include/libecc_b200.h (used by tests/ and bench.py).

The product is the shared library ``libecc_b200/libecc_b200.so`` (hand-written sm_90a CUDA behind a C ABI that
mirrors libecc's prj_pt_mul / ECDSA-verify entry points).  This module only loads it and marshals buffers; it
contains no arithmetic and has no CPU fallback: if the library is missing or no H100 is visible, it raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ECCB200_LIB", os.path.join(_HERE, "libecc_b200.so"))

CURVE_IDS = {"FRP256V1": 1, "SECP256R1": 4, "SECP384R1": 5,   # libecc ec_curve_type (src/lib_ecc_types.h:147-)
             "BRAINPOOLP256R1": 8, "BRAINPOOLP384R1": 12, "SECP256K1": 19, "SECP521R1": 6,
             "SM2P256V1": 17, "BRAINPOOLP512R1": 9, "SECP224R1": 3, "SECP192R1": 2}

# Every symbol include/libecc_b200.h and include/libecc_b200_dropin.h declare (tests check they are exported).
ABI_SYMBOLS = [
    "eccb200_ctx_create", "eccb200_ctx_destroy", "eccb200_curve_sizes", "eccb200_curve_name",
    "eccb200_prj_pt_mul_batch", "eccb200_prj_pt_mul_batch_dev", "eccb200_ecdsa_verify_batch",
    "eccb200_ecdsa_verify_batch_dev", "eccb200_fp_mul_monty_batch", "eccb200_comb_window",
    "eccb200_kernel_launches", "eccb200_last_error", "eccb200_ecdsa_uv_batch",
    "eccb200_profile_enable", "eccb200_profile_read", "eccb200_imad_peak", "eccb200_prj_pt_unique_batch",
    "eccb200_host_alloc", "eccb200_host_alloc_input", "eccb200_host_free", "eccb200_ecdsa_sign_batch", "eccb200_ecdsa_sign_batch_dev",
    "eccb200_ecccdh_derive_batch", "eccb200_ecccdh_derive_batch_dev", "eccb200_fp_mul_chain_bench", "eccb200_hash_batch", "eccb200_ecdsa_verify_msgs_batch",
    "eccb200_structured_pub_key_import_batch", "eccb200_structured_pub_key_export_batch",
    "eccb200_structured_key_pair_batch", "eccb200_ecdsa_verify_structured_batch", "eccb200_ecdsa_sign_structured_batch",
    "eccb200_ecfsdsa_verify_batch", "eccb200_ecfsdsa_verify_batch_dev",
    "eccb200_ecfsdsa_verify_msm_batch", "eccb200_ecfsdsa_verify_msm_batch_dev",
    "eccb200_bip0340_verify_msm_batch", "eccb200_bip0340_verify_msm_batch_dev",
    "eccb200_prj_pt_mul_batch_dev_gather", "eccb200_ipc_alloc", "eccb200_ipc_open", "eccb200_ipc_close",
    "eccb200_ipc_free", "eccb200_flag_wait", "eccb200_flag_signal",
    "eccb200_multi_create", "eccb200_multi_destroy", "eccb200_multi_device_count", "eccb200_multi_ctx",
    "eccb200_multi_prj_pt_mul_batch", "eccb200_multi_ecdsa_verify_batch",
    "eccb200_ecdsa_verify_msgs_batch_dev", "eccb200_copy_to_host", "eccb200_ecdsa_verify_keystate_batch",
    "eccb200_fp_addsub_batch", "eccb200_ecdsa_verify_prj_batch", "eccb200_bip0340_verify_batch",
    "eccb200_bip0340_verify_batch_dev", "eccb200_push_results", "eccb200_bind_thread_near_device",
    "eccb200_pipeline_chunk_bounds", "eccb200_double_smul_batch", "eccb200_double_smul_batch_dev",
    "eccb200_schnorr_sign_msgs_batch", "eccb200_schnorr_sign_msgs_batch_dev", "eccb200_sign_msgs_batch",
    "eccb200_sign_msgs_batch_dev", "eccb200_sign_sig_len", "eccb200_verify_msgs_batch", "eccb200_verify_msgs_batch_dev",
    "eccb200_ecdsa_recover_batch", "eccb200_ecdsa_recover_batch_dev",
    "eccb200_decdsa_sign_batch", "eccb200_decdsa_sign_batch_dev", "eccb200_ecdsa_sign_msgs_batch",
    "eccb200_ecdsa_sign_msgs_batch_dev", "eccb200_bign_sign_msgs_batch", "eccb200_bign_sign_msgs_batch_dev",
    "eccb200_bign_verify_msgs_batch", "eccb200_bign_verify_msgs_batch_dev",
]

_lib = None


class EccB200Error(RuntimeError):
    pass


def load_library() -> ctypes.CDLL:
    """Load libecc_b200.so (fails loudly when it has not been built: there is no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EccB200Error(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = ctypes.CDLL(LIB_PATH)
    u8p, i8p, u32 = ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32
    lib.eccb200_ctx_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.eccb200_ctx_create.restype = ctypes.c_int
    lib.eccb200_ctx_destroy.argtypes = [ctypes.c_void_p]
    lib.eccb200_ctx_destroy.restype = None
    lib.eccb200_curve_sizes.argtypes = [ctypes.c_int, ctypes.POINTER(u32), ctypes.POINTER(u32)]
    lib.eccb200_curve_name.argtypes = [ctypes.c_int]
    lib.eccb200_curve_name.restype = ctypes.c_char_p
    lib.eccb200_prj_pt_mul_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, i8p]
    lib.eccb200_prj_pt_mul_batch_dev.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, i8p, ctypes.c_void_p]
    lib.eccb200_ecdsa_verify_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, u32, i8p]
    lib.eccb200_ecdsa_verify_batch_dev.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, u32, i8p, ctypes.c_void_p]
    lib.eccb200_fp_mul_monty_batch.argtypes = [ctypes.c_void_p, ctypes.c_int, u32, u8p, u8p, u8p]
    lib.eccb200_prj_pt_unique_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, i8p]
    lib.eccb200_ecdsa_uv_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u32, u8p]
    lib.eccb200_profile_enable.argtypes = [ctypes.c_void_p, ctypes.c_int]
    lib.eccb200_profile_read.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float), ctypes.c_int]
    lib.eccb200_ecdsa_sign_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, u32, u8p, i8p]
    lib.eccb200_ecdsa_sign_batch_dev.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, u32, u8p, i8p, ctypes.c_void_p]
    lib.eccb200_ecccdh_derive_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, i8p]
    lib.eccb200_ecccdh_derive_batch_dev.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, i8p, ctypes.c_void_p]
    lib.eccb200_fp_mul_chain_bench.argtypes = [ctypes.c_void_p, ctypes.c_int, u32, u8p, u8p, u8p, ctypes.c_int,
                                               ctypes.POINTER(ctypes.c_float)]
    lib.eccb200_hash_batch.argtypes = [ctypes.c_void_p, ctypes.c_int, u32, u8p, u8p, u8p]
    lib.eccb200_ecdsa_verify_msgs_batch.argtypes = [ctypes.c_void_p, ctypes.c_int, u32, u8p, u8p, u8p, u8p, i8p]
    lib.eccb200_structured_pub_key_import_batch.argtypes = [ctypes.c_void_p, u32, u8p, ctypes.c_int, u8p, i8p]
    lib.eccb200_structured_pub_key_export_batch.argtypes = [ctypes.c_void_p, u32, u8p, ctypes.c_int, u8p]
    lib.eccb200_structured_key_pair_batch.argtypes = [ctypes.c_void_p, u32, u8p, u32, ctypes.c_int, u8p, i8p]
    lib.eccb200_ecdsa_verify_structured_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, ctypes.c_int, ctypes.c_int,
                                                          u8p, u32, i8p]
    lib.eccb200_ecdsa_sign_structured_batch.argtypes = [ctypes.c_void_p, u32, u8p, u32, ctypes.c_int, ctypes.c_int,
                                                        u8p, u8p, u32, u8p, i8p]
    lib.eccb200_ecfsdsa_verify_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, u32, i8p]
    lib.eccb200_ecfsdsa_verify_batch_dev.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, u32, i8p, ctypes.c_void_p]
    lib.eccb200_ecfsdsa_verify_msm_batch.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, u32, u8p,
                                                     ctypes.POINTER(ctypes.c_int)]
    lib.eccb200_ecfsdsa_verify_msm_batch_dev.argtypes = [ctypes.c_void_p, u32, u8p, u8p, u8p, u32, u8p,
                                                         ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]
    lib.eccb200_bip0340_verify_msm_batch.argtypes = lib.eccb200_ecfsdsa_verify_msm_batch.argtypes
    lib.eccb200_bip0340_verify_msm_batch_dev.argtypes = lib.eccb200_ecfsdsa_verify_msm_batch_dev.argtypes
    vp, u64 = ctypes.c_void_p, ctypes.c_uint64
    lib.eccb200_prj_pt_mul_batch_dev_gather.argtypes = [vp, u32, u8p, u8p, u8p, i8p, ctypes.c_int, vp, vp, vp, u32,
                                                        vp, ctypes.c_int, u32, vp]
    lib.eccb200_push_results.argtypes = [vp, ctypes.c_int, vp, vp, ctypes.c_size_t, vp, u32, vp, ctypes.c_int, u32, vp]
    lib.eccb200_ipc_alloc.argtypes = [vp, ctypes.c_size_t, ctypes.POINTER(vp), vp]
    lib.eccb200_ipc_open.argtypes = [vp, vp, ctypes.POINTER(vp)]
    lib.eccb200_ipc_close.argtypes = [vp, vp]
    lib.eccb200_ipc_free.argtypes = [vp, vp]
    lib.eccb200_flag_wait.argtypes = [vp, vp, ctypes.c_int, u32, vp]
    lib.eccb200_flag_signal.argtypes = [vp, vp, ctypes.c_int, u32, vp]
    lib.eccb200_multi_create.argtypes = [ctypes.POINTER(vp), ctypes.c_int, vp, ctypes.c_int, ctypes.c_int]
    lib.eccb200_multi_destroy.argtypes = [vp]
    lib.eccb200_multi_destroy.restype = None
    lib.eccb200_multi_device_count.argtypes = [vp]
    lib.eccb200_multi_ctx.argtypes = [vp, ctypes.c_int]
    lib.eccb200_multi_ctx.restype = vp
    lib.eccb200_multi_prj_pt_mul_batch.argtypes = [vp, u64, u8p, u8p, u8p, i8p]
    lib.eccb200_multi_ecdsa_verify_batch.argtypes = [vp, u64, u8p, u8p, u8p, u32, i8p]
    lib.eccb200_ecdsa_verify_msgs_batch_dev.argtypes = [vp, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, i8p, vp]
    lib.eccb200_schnorr_sign_msgs_batch.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, u8p, vp, u8p,
                                                    i8p]
    lib.eccb200_schnorr_sign_msgs_batch_dev.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, u8p, vp,
                                                        u8p, i8p, vp]
    lib.eccb200_sign_msgs_batch.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, u8p, vp, u8p, vp, u8p,
                                            i8p]
    lib.eccb200_sign_msgs_batch_dev.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, u8p, vp, u8p, vp,
                                                u8p, i8p, vp]
    lib.eccb200_sign_sig_len.argtypes = [vp, ctypes.c_int, ctypes.c_int]
    lib.eccb200_verify_msgs_batch.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, vp, i8p]
    lib.eccb200_verify_msgs_batch_dev.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, vp, i8p,
                                                  vp]
    lib.eccb200_copy_to_host.argtypes = [vp, vp, vp, ctypes.c_size_t]
    lib.eccb200_bind_thread_near_device.argtypes = [ctypes.c_int]
    lib.eccb200_pipeline_chunk_bounds.argtypes = [u32, u32, u32, u32, ctypes.c_int, vp, ctypes.c_int]
    lib.eccb200_fp_addsub_batch.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p]
    lib.eccb200_ecdsa_verify_prj_batch.argtypes = [vp, u32, u8p, u8p, u8p, u32, i8p]
    lib.eccb200_bip0340_verify_batch.argtypes = [vp, u32, u8p, u8p, u8p, u32, i8p]
    lib.eccb200_double_smul_batch.argtypes = [vp, u32, u8p, u8p, u8p, i8p]
    lib.eccb200_double_smul_batch_dev.argtypes = [vp, u32, u8p, u8p, u8p, i8p, vp]
    lib.eccb200_bip0340_verify_batch_dev.argtypes = [vp, u32, u8p, u8p, u8p, u32, i8p, vp]
    lib.eccb200_ecdsa_verify_keystate_batch.argtypes = [vp, u32, u8p, u8p, i8p, u8p, u32, i8p]
    lib.eccb200_ecdsa_recover_batch.argtypes = [vp, u32, u8p, u8p, u32, u8p, i8p]
    lib.eccb200_ecdsa_recover_batch_dev.argtypes = [vp, u32, u8p, u8p, u32, u8p, i8p, vp]
    lib.eccb200_decdsa_sign_batch.argtypes = [vp, ctypes.c_int, u32, u8p, u8p, u8p, i8p]
    lib.eccb200_decdsa_sign_batch_dev.argtypes = [vp, ctypes.c_int, u32, u8p, u8p, u8p, i8p, vp]
    lib.eccb200_ecdsa_sign_msgs_batch.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, i8p]
    lib.eccb200_ecdsa_sign_msgs_batch_dev.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, i8p,
                                                      vp]
    lib.eccb200_bign_sign_msgs_batch.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, vp, u8p,
                                                 i8p]
    lib.eccb200_bign_sign_msgs_batch_dev.argtypes = [vp, ctypes.c_int, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, vp,
                                                     u8p, i8p, vp]
    lib.eccb200_bign_verify_msgs_batch.argtypes = [vp, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, vp, i8p]
    lib.eccb200_bign_verify_msgs_batch_dev.argtypes = [vp, ctypes.c_int, u32, u8p, u8p, u8p, vp, u8p, vp, i8p, vp]
    lib.eccb200_host_alloc.argtypes = [ctypes.c_size_t]
    lib.eccb200_host_alloc.restype = ctypes.c_void_p
    lib.eccb200_host_alloc_input.argtypes = [ctypes.c_size_t]
    lib.eccb200_host_alloc_input.restype = ctypes.c_void_p
    lib.eccb200_host_free.argtypes = [ctypes.c_void_p]
    lib.eccb200_host_free.restype = None
    lib.eccb200_comb_window.argtypes = [ctypes.c_void_p]
    lib.eccb200_kernel_launches.argtypes = [ctypes.c_void_p]
    lib.eccb200_kernel_launches.restype = ctypes.c_uint64
    lib.eccb200_last_error.restype = ctypes.c_char_p
    _lib = lib
    return lib


def curve_sizes(curve: str) -> Tuple[int, int]:
    lib = load_library()
    plen, qlen = ctypes.c_uint32(), ctypes.c_uint32()
    if lib.eccb200_curve_sizes(CURVE_IDS[curve], ctypes.byref(plen), ctypes.byref(qlen)):
        raise EccB200Error("unknown curve")
    return plen.value, qlen.value


def _as_u8(a, nbytes: Optional[int] = None) -> np.ndarray:
    arr = np.frombuffer(a, dtype=np.uint8) if isinstance(a, (bytes, bytearray, memoryview)) else np.asarray(a)
    arr = np.ascontiguousarray(arr.reshape(-1).view(np.uint8))
    if nbytes is not None and arr.size != nbytes:
        raise ValueError(f"expected {nbytes} bytes, got {arr.size}")
    return arr


def bign_adata(oid: bytes, t: bytes = b"") -> bytes:
    """The BIGN / DBIGN adata record of the reference (bign_set_adata): oid_len and t_len as 2-byte big-endian
    integers, then the hash OID (DER content bytes), then t (DBIGN's additional nonce data)."""
    if len(oid) + len(t) + 4 > 0xFFFF:
        raise ValueError("BIGN adata longer than 65535 bytes")
    return len(oid).to_bytes(2, "big") + len(t).to_bytes(2, "big") + bytes(oid) + bytes(t)


def pinned_empty(shape, dtype=np.uint8, write_combined: bool = False) -> np.ndarray:
    """numpy array backed by page-locked memory from eccb200_host_alloc (freed with the array);
    write_combined=True uses eccb200_host_alloc_input (for input buffers the host only writes)."""
    lib = load_library()
    shape = (shape,) if isinstance(shape, int) else tuple(shape)
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = (lib.eccb200_host_alloc_input if write_combined else lib.eccb200_host_alloc)(max(nbytes, 1))
    if not p:
        raise EccB200Error("eccb200_host_alloc failed")
    buf = (ctypes.c_uint8 * max(nbytes, 1)).from_address(p)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    class _Owner:
        def __del__(self, p=p, lib=lib):
            lib.eccb200_host_free(p)
    _PIN_OWNERS[id(buf)] = (buf, _Owner())
    return arr


_PIN_OWNERS = {}


class Engine:
    """One engine context = one curve on one GPU (eccb200_ctx)."""

    def __init__(self, curve: str, device: int = 0, comb_window: int = 0):
        self.lib = load_library()
        self.curve = curve
        self.curve_id = CURVE_IDS[curve]
        self.plen, self.qlen = curve_sizes(curve)
        self.device = device
        h = ctypes.c_void_p()
        if self.lib.eccb200_ctx_create(ctypes.byref(h), self.curve_id, device, comb_window):
            raise EccB200Error("eccb200_ctx_create: " + self.lib.eccb200_last_error().decode())
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self.lib.eccb200_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc:
            raise EccB200Error(f"{what}: " + self.lib.eccb200_last_error().decode())

    @property
    def comb_window(self) -> int:
        return self.lib.eccb200_comb_window(self._h)

    @property
    def kernel_launches(self) -> int:
        return int(self.lib.eccb200_kernel_launches(self._h))

    def profile_enable(self, on: bool = True):
        self._check(self.lib.eccb200_profile_enable(self._h, int(on)), "eccb200_profile_enable")

    def profile_read(self):
        """Durations (ms) of the kernels of the last device-pointer call (waits for them)."""
        buf = (ctypes.c_float * 4)()
        k = self.lib.eccb200_profile_read(self._h, buf, 4)
        if k < 0:
            raise EccB200Error("eccb200_profile_read: " + self.lib.eccb200_last_error().decode())
        return [float(buf[i]) for i in range(k)]

    # ---- host-buffer API (H2D / D2H inside the call) -------------------------------------------------------
    def prj_pt_mul_batch(self, scalars, points=None, out=None, status=None) -> Tuple[np.ndarray, np.ndarray]:
        """scalars: n*qlen big-endian bytes; points: n*2*plen affine bytes or None (=G).
        Returns (out[n, 2*plen] uint8, status[n] int8); pass `out` / `status` to reuse (e.g. pinned) buffers."""
        sc = _as_u8(scalars)
        n = sc.size // self.qlen
        if sc.size != n * self.qlen:
            raise ValueError("scalars length is not a multiple of qlen")
        pt = _as_u8(points, n * 2 * self.plen) if points is not None else None
        if out is None:
            out = np.zeros((n, 2 * self.plen), dtype=np.uint8)
        if status is None:
            status = np.zeros(n, dtype=np.int8)
        assert out.nbytes == n * 2 * self.plen and status.nbytes == n and out.flags.c_contiguous
        self._check(self.lib.eccb200_prj_pt_mul_batch(
            self._h, n, sc.ctypes.data, pt.ctypes.data if pt is not None else None,
            out.ctypes.data, status.ctypes.data), "eccb200_prj_pt_mul_batch")
        return out, status

    def ecdsa_verify_batch(self, sigs, pubkeys, digests, hlen: int, verdict=None) -> np.ndarray:
        sg = _as_u8(sigs)
        n = sg.size // (2 * self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        dg = _as_u8(digests, n * hlen)
        if verdict is None:
            verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_verify_batch(
            self._h, n, sg.ctypes.data, pk.ctypes.data, dg.ctypes.data, hlen, verdict.ctypes.data),
            "eccb200_ecdsa_verify_batch")
        return verdict

    def ecdsa_recover_batch(self, sigs, digests, hlen: int) -> Tuple[np.ndarray, np.ndarray]:
        """ECDSA public-key recovery: sigs [n][2*qlen] = r || s, digests [n][hlen].  Returns (keys[n, 2, 2*plen] uint8:
        affine Y1 then Y2, status[n, 2] int8: OK / INFINITY per key, ERR for both where the reference returns -1)."""
        sg = _as_u8(sigs)
        n = sg.size // (2 * self.qlen)
        if sg.size != n * 2 * self.qlen:
            raise ValueError("sigs length is not a multiple of 2*qlen")
        dg = _as_u8(digests, n * hlen)
        keys = np.zeros((n, 2, 2 * self.plen), dtype=np.uint8)
        status = np.zeros((n, 2), dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_recover_batch(self._h, n, sg.ctypes.data, dg.ctypes.data, hlen,
                                                         keys.ctypes.data, status.ctypes.data),
                    "eccb200_ecdsa_recover_batch")
        return keys, status

    def ecdsa_verify_prj_batch(self, sigs, prj_pubkeys, digests, hlen: int) -> np.ndarray:
        """Public keys as X || Y || Z (homogeneous projective, 3*plen bytes each)."""
        sg = _as_u8(sigs)
        n = sg.size // (2 * self.qlen)
        pk = _as_u8(prj_pubkeys, n * 3 * self.plen)
        dg = _as_u8(digests, n * hlen)
        verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_verify_prj_batch(self._h, n, sg.ctypes.data, pk.ctypes.data, dg.ctypes.data,
                                                            hlen, verdict.ctypes.data), "eccb200_ecdsa_verify_prj_batch")
        return verdict

    def ecdsa_sign_batch(self, privkeys, nonces, digests, hlen: int, out=None, status=None) -> Tuple[np.ndarray, np.ndarray]:
        d = _as_u8(privkeys)
        n = d.size // self.qlen
        k = _as_u8(nonces, n * self.qlen)
        dg = _as_u8(digests, n * hlen)
        sigs = out if out is not None else np.zeros((n, 2 * self.qlen), dtype=np.uint8)
        status = status if status is not None else np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_sign_batch(self._h, n, d.ctypes.data, k.ctypes.data, dg.ctypes.data, hlen,
                                                      sigs.ctypes.data, status.ctypes.data), "eccb200_ecdsa_sign_batch")
        return sigs, status

    def ecccdh_derive_batch(self, privkeys, peer_pubkeys, out=None, status=None) -> Tuple[np.ndarray, np.ndarray]:
        d = _as_u8(privkeys)
        n = d.size // self.qlen
        pk = _as_u8(peer_pubkeys, n * 2 * self.plen)
        shared = out if out is not None else np.zeros((n, self.plen), dtype=np.uint8)
        status = status if status is not None else np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecccdh_derive_batch(self._h, n, d.ctypes.data, pk.ctypes.data,
                                                         shared.ctypes.data, status.ctypes.data),
                    "eccb200_ecccdh_derive_batch")
        return shared, status

    HASH_IDS = {"SHA256": 2, "SHA384": 3, "SHA512": 4, "SHA3_224": 5, "SHA3_256": 6, "SHA3_384": 7,
                "SHA3_512": 8}                            # libecc hash_alg_type values hashed on the device
    REF_HASH_IDS = {"SHA224": 1, "SHA256": 2, "SHA384": 3, "SHA512": 4, "SHA3_224": 5, "SHA3_256": 6, "SHA3_384": 7,
                    "SHA3_512": 8}                        # header byte of structured signatures (lib_ecc_types.h:82-)
    HASH_LEN = {"SHA256": 32, "SHA384": 48, "SHA512": 64, "SHA3_224": 28, "SHA3_256": 32, "SHA3_384": 48, "SHA3_512": 64}

    @staticmethod
    def _pack_msgs(msgs):
        off = np.zeros(len(msgs) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(m) for m in msgs])
        blob = np.frombuffer(b"".join(bytes(m) for m in msgs) or b"\0", dtype=np.uint8).copy()
        return blob, off

    def hash_batch(self, hash_name: str, msgs) -> np.ndarray:
        blob, off = self._pack_msgs(msgs)
        out = np.zeros((len(msgs), self.HASH_LEN[hash_name]), dtype=np.uint8)
        self._check(self.lib.eccb200_hash_batch(self._h, self.HASH_IDS[hash_name], len(msgs), blob.ctypes.data,
                                                off.ctypes.data, out.ctypes.data), "eccb200_hash_batch")
        return out

    def hash_batch_raw(self, hash_name: str, blob, offsets) -> np.ndarray:
        """Messages already packed: blob uint8, offsets uint64[n + 1]."""
        blob = _as_u8(blob)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = off.size - 1
        out = np.zeros((n, self.HASH_LEN[hash_name]), dtype=np.uint8)
        self._check(self.lib.eccb200_hash_batch(self._h, self.HASH_IDS[hash_name], n, blob.ctypes.data,
                                                off.ctypes.data, out.ctypes.data), "eccb200_hash_batch")
        return out

    def ecdsa_verify_msgs_batch_raw(self, hash_name: str, sigs, pubkeys, blob, offsets, verdict=None) -> np.ndarray:
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = off.size - 1
        sg = _as_u8(sigs, n * 2 * self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        blob = _as_u8(blob)
        if verdict is None:
            verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_verify_msgs_batch(self._h, self.HASH_IDS[hash_name], n, sg.ctypes.data,
                                                             pk.ctypes.data, blob.ctypes.data, off.ctypes.data,
                                                             verdict.ctypes.data), "eccb200_ecdsa_verify_msgs_batch")
        return verdict

    def ecdsa_verify_msgs_batch_dev(self, hash_name: str, d_sigs, d_pubkeys, d_msgs, d_offsets, d_digests, d_verdict,
                                    stream_handle: int = 0):
        n = d_sigs.numel() // (2 * self.qlen)
        self._check(self.lib.eccb200_ecdsa_verify_msgs_batch_dev(
            self._h, self.HASH_IDS[hash_name], n, d_sigs.data_ptr(), d_pubkeys.data_ptr(), d_msgs.data_ptr(),
            d_offsets.data_ptr(), d_digests.data_ptr(), d_verdict.data_ptr(), ctypes.c_void_p(stream_handle)),
            "eccb200_ecdsa_verify_msgs_batch_dev")

    SCHNORR_ALGS = {"ECSDSA": 3, "ECOSDSA": 4, "ECFSDSA": 5, "BIP0340": 20}  # libecc ec_alg_type values

    def schnorr_sig_len(self, alg: str, hash_name: str) -> int:
        return {"ECFSDSA": 2 * self.plen + self.qlen, "BIP0340": self.plen + self.qlen}.get(
            alg, self.HASH_LEN[hash_name] + self.qlen)

    def schnorr_sign_msgs_batch(self, alg: str, hash_name: str, privkeys, randomness, msgs,
                                pubkeys=None) -> Tuple[np.ndarray, np.ndarray]:
        """ECSDSA / ECOSDSA / ECFSDSA / BIP0340 signatures of raw messages, hashed on the device.  randomness[i] is what
        the reference's rand callback would return: the nonce k (qlen bytes) or, for BIP0340, the auxiliary value a.
        pubkeys (n*2*plen affine) are required for BIP0340 only.  Returns (sigs[n, siglen], status[n]):
        0 OK, -1 ERR, 2 RETRY (see include/libecc_b200.h)."""
        n = len(msgs)
        d = _as_u8(privkeys, n * self.qlen)
        r = _as_u8(randomness, n * self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen) if pubkeys is not None else None
        blob, off = self._pack_msgs(msgs)
        sigs = np.zeros((n, self.schnorr_sig_len(alg, hash_name)), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_schnorr_sign_msgs_batch(
            self._h, self.SCHNORR_ALGS[alg], self.HASH_IDS[hash_name], n, d.ctypes.data,
            pk.ctypes.data if pk is not None else None, r.ctypes.data, blob.ctypes.data, off.ctypes.data,
            sigs.ctypes.data, status.ctypes.data), "eccb200_schnorr_sign_msgs_batch")
        return sigs, status

    def schnorr_sign_msgs_batch_dev(self, alg: str, hash_name: str, d_privkeys, d_randomness, d_msgs, d_offsets,
                                    d_sigs, d_status, d_pubkeys=None, stream_handle: int = 0):
        """Device-tensor form (asynchronous on `stream_handle`); d_offsets: n + 1 uint64 entries, not re-checked."""
        n = d_privkeys.numel() // self.qlen
        self._check(self.lib.eccb200_schnorr_sign_msgs_batch_dev(
            self._h, self.SCHNORR_ALGS[alg], self.HASH_IDS[hash_name], n, d_privkeys.data_ptr(),
            d_pubkeys.data_ptr() if d_pubkeys is not None else None, d_randomness.data_ptr(), d_msgs.data_ptr(),
            d_offsets.data_ptr(), d_sigs.data_ptr(), d_status.data_ptr(), ctypes.c_void_p(stream_handle)),
            "eccb200_schnorr_sign_msgs_batch_dev")

    SIGN_ALGS = {"ECKCDSA": 2, "ECGDSA": 6, "ECRDSA": 7, "SM2": 8}  # libecc ec_alg_type values
    SIGN_HASH_IDS = dict(HASH_IDS, SM3=11)  # the message signers also hash with SM3

    def sign_sig_len(self, alg: str, hash_name: str) -> int:
        n = self.lib.eccb200_sign_sig_len(self._h, self.SIGN_ALGS[alg], self.SIGN_HASH_IDS[hash_name])
        self._check(0 if n > 0 else -1, "eccb200_sign_sig_len")
        return n

    def sign_msgs_batch(self, alg: str, hash_name: str, privkeys, nonces, msgs, pubkeys=None,
                        ids=None) -> Tuple[np.ndarray, np.ndarray]:
        """ECKCDSA / ECGDSA / ECRDSA / SM2 signatures of raw messages, hashed on the device (hash_name may be "SM3").
        nonces[i] is the k the reference's rand callback would return (qlen bytes).  pubkeys (n*2*plen affine) are
        required for ECKCDSA and SM2, ids (a list of byte strings, the SM2 user IDs) for SM2.  Returns
        (sigs[n, siglen], status[n]): 0 OK, -1 ERR, 2 RETRY (see include/libecc_b200.h)."""
        n = len(msgs)
        d = _as_u8(privkeys, n * self.qlen)
        k = _as_u8(nonces, n * self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen) if pubkeys is not None else None
        blob, off = self._pack_msgs(msgs)
        id_blob, id_off = self._pack_msgs(ids) if ids is not None else (None, None)
        sigs = np.zeros((n, self.sign_sig_len(alg, hash_name)), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_sign_msgs_batch(
            self._h, self.SIGN_ALGS[alg], self.SIGN_HASH_IDS[hash_name], n, d.ctypes.data,
            pk.ctypes.data if pk is not None else None, k.ctypes.data, blob.ctypes.data, off.ctypes.data,
            id_blob.ctypes.data if id_blob is not None else None, id_off.ctypes.data if id_off is not None else None,
            sigs.ctypes.data, status.ctypes.data), "eccb200_sign_msgs_batch")
        return sigs, status

    def sign_msgs_batch_dev(self, alg: str, hash_name: str, d_privkeys, d_nonces, d_msgs, d_offsets, d_sigs, d_status,
                            d_pubkeys=None, d_ids=None, d_id_offsets=None, stream_handle: int = 0):
        """Device-tensor form (asynchronous on `stream_handle`); d_offsets / d_id_offsets: n + 1 uint64 entries, not
        re-checked."""
        n = d_privkeys.numel() // self.qlen
        ptr = lambda t: t.data_ptr() if t is not None else None
        self._check(self.lib.eccb200_sign_msgs_batch_dev(
            self._h, self.SIGN_ALGS[alg], self.SIGN_HASH_IDS[hash_name], n, d_privkeys.data_ptr(), ptr(d_pubkeys),
            d_nonces.data_ptr(), d_msgs.data_ptr(), d_offsets.data_ptr(), ptr(d_ids), ptr(d_id_offsets),
            d_sigs.data_ptr(), d_status.data_ptr(), ctypes.c_void_p(stream_handle)), "eccb200_sign_msgs_batch_dev")

    ECDSA_ALGS = {"ECDSA": 1, "DECDSA": 14}  # libecc ec_alg_type values
    DECDSA_HASH_IDS = dict(SIGN_HASH_IDS, SHA224=1)  # the deterministic / message ECDSA signers also take SHA-224
    DECDSA_HASH_LEN = dict(HASH_LEN, SHA224=28, SM3=32)

    def decdsa_sign_batch(self, hash_name: str, privkeys, digests) -> Tuple[np.ndarray, np.ndarray]:
        """Deterministic ECDSA (RFC 6979 nonces derived on the device) of digests[n, digest size of hash_name].
        Returns (sigs[n, 2*qlen], status[n]): 0 OK, -1 ERR, 2 RETRY (see include/libecc_b200.h)."""
        hl = self.DECDSA_HASH_LEN[hash_name]
        d = _as_u8(privkeys)
        n = d.size // self.qlen
        dg = _as_u8(digests, n * hl)
        sigs = np.zeros((n, 2 * self.qlen), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_decdsa_sign_batch(self._h, self.DECDSA_HASH_IDS[hash_name], n, d.ctypes.data,
                                                       dg.ctypes.data, sigs.ctypes.data, status.ctypes.data),
                    "eccb200_decdsa_sign_batch")
        return sigs, status

    def decdsa_sign_batch_dev(self, hash_name: str, d_privkeys, d_digests, d_sigs, d_status, stream_handle: int = 0):
        """Device-tensor form (asynchronous on `stream_handle`)."""
        n = d_privkeys.numel() // self.qlen
        self._check(self.lib.eccb200_decdsa_sign_batch_dev(
            self._h, self.DECDSA_HASH_IDS[hash_name], n, d_privkeys.data_ptr(), d_digests.data_ptr(), d_sigs.data_ptr(),
            d_status.data_ptr(), ctypes.c_void_p(stream_handle)), "eccb200_decdsa_sign_batch_dev")

    def ecdsa_sign_msgs_batch(self, alg: str, hash_name: str, privkeys, msgs, nonces=None) -> Tuple[np.ndarray, np.ndarray]:
        """ECDSA (the caller's nonces, qlen bytes each) or DECDSA (RFC 6979 nonces, `nonces` ignored) signatures of raw
        messages, hashed on the device.  Returns (sigs[n, 2*qlen], status[n]): 0 OK, -1 ERR, 2 RETRY."""
        n = len(msgs)
        d = _as_u8(privkeys, n * self.qlen)
        k = _as_u8(nonces, n * self.qlen) if nonces is not None else None
        blob, off = self._pack_msgs(msgs)
        sigs = np.zeros((n, 2 * self.qlen), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_sign_msgs_batch(
            self._h, self.ECDSA_ALGS[alg], self.DECDSA_HASH_IDS[hash_name], n, d.ctypes.data,
            k.ctypes.data if k is not None else None, blob.ctypes.data, off.ctypes.data, sigs.ctypes.data,
            status.ctypes.data), "eccb200_ecdsa_sign_msgs_batch")
        return sigs, status

    def ecdsa_sign_msgs_batch_dev(self, alg: str, hash_name: str, d_privkeys, d_msgs, d_offsets, d_sigs, d_status,
                                  d_nonces=None, stream_handle: int = 0):
        """Device-tensor form (asynchronous on `stream_handle`); d_offsets: n + 1 uint64 entries, not re-checked."""
        n = d_privkeys.numel() // self.qlen
        self._check(self.lib.eccb200_ecdsa_sign_msgs_batch_dev(
            self._h, self.ECDSA_ALGS[alg], self.DECDSA_HASH_IDS[hash_name], n, d_privkeys.data_ptr(),
            d_nonces.data_ptr() if d_nonces is not None else None, d_msgs.data_ptr(), d_offsets.data_ptr(),
            d_sigs.data_ptr(), d_status.data_ptr(), ctypes.c_void_p(stream_handle)), "eccb200_ecdsa_sign_msgs_batch_dev")

    BIGN_ALGS = {"BIGN": 18, "DBIGN": 19}  # libecc ec_alg_type values
    # the BIGN signers and verifier also take BELT-HASH and BASH (hash_alg_type 16..20)
    BIGN_HASH_IDS = dict(DECDSA_HASH_IDS, BELT_HASH=16, BASH224=17, BASH256=18, BASH384=19, BASH512=20)
    BIGN_HASH_LEN = dict(DECDSA_HASH_LEN, BELT_HASH=32, BASH224=28, BASH256=32, BASH384=48, BASH512=64)

    @property
    def bign_sig_len(self) -> int:
        """Bytes of a BIGN / DBIGN signature s0 || s1: qlen / 2 + qlen."""
        return self.qlen // 2 + self.qlen

    def bign_sign_msgs_batch(self, alg: str, hash_name: str, privkeys, msgs, adata,
                             nonces=None) -> Tuple[np.ndarray, np.ndarray]:
        """BIGN (the caller's nonces, qlen bytes each) or DBIGN (deterministic nonces, `nonces` ignored) signatures of
        raw messages, hashed on the device; adata[i] is item i's record (bign_adata).  Returns (sigs[n, bign_sig_len],
        status[n]): 0 OK, -1 ERR (see include/libecc_b200.h)."""
        n = len(msgs)
        d = _as_u8(privkeys, n * self.qlen)
        k = _as_u8(nonces, n * self.qlen) if nonces is not None else None
        blob, off = self._pack_msgs(msgs)
        ad_blob, ad_off = self._pack_msgs(adata)
        sigs = np.zeros((n, self.bign_sig_len), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_bign_sign_msgs_batch(
            self._h, self.BIGN_ALGS[alg], self.BIGN_HASH_IDS[hash_name], n, d.ctypes.data,
            k.ctypes.data if k is not None else None, blob.ctypes.data, off.ctypes.data, ad_blob.ctypes.data,
            ad_off.ctypes.data, sigs.ctypes.data, status.ctypes.data), "eccb200_bign_sign_msgs_batch")
        return sigs, status

    def bign_sign_msgs_batch_dev(self, alg: str, hash_name: str, d_privkeys, d_msgs, d_offsets, d_adata,
                                 d_adata_offsets, d_sigs, d_status, d_nonces=None, stream_handle: int = 0):
        """Device-tensor form (asynchronous on `stream_handle`); offsets: n + 1 uint64 entries, not re-checked."""
        n = d_privkeys.numel() // self.qlen
        self._check(self.lib.eccb200_bign_sign_msgs_batch_dev(
            self._h, self.BIGN_ALGS[alg], self.BIGN_HASH_IDS[hash_name], n, d_privkeys.data_ptr(),
            d_nonces.data_ptr() if d_nonces is not None else None, d_msgs.data_ptr(), d_offsets.data_ptr(),
            d_adata.data_ptr(), d_adata_offsets.data_ptr(), d_sigs.data_ptr(), d_status.data_ptr(),
            ctypes.c_void_p(stream_handle)), "eccb200_bign_sign_msgs_batch_dev")

    def bign_verify_msgs_batch(self, hash_name: str, sigs, pubkeys, msgs, adata) -> np.ndarray:
        """BIGN / DBIGN verification of raw messages: verdict[n], 0 valid, -1 invalid."""
        n = len(msgs)
        sg = _as_u8(sigs, n * self.bign_sig_len)
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        blob, off = self._pack_msgs(msgs)
        ad_blob, ad_off = self._pack_msgs(adata)
        verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_bign_verify_msgs_batch(
            self._h, self.BIGN_HASH_IDS[hash_name], n, sg.ctypes.data, pk.ctypes.data, blob.ctypes.data,
            off.ctypes.data, ad_blob.ctypes.data, ad_off.ctypes.data, verdict.ctypes.data),
            "eccb200_bign_verify_msgs_batch")
        return verdict

    def bign_verify_msgs_batch_dev(self, hash_name: str, d_sigs, d_pubkeys, d_msgs, d_offsets, d_adata,
                                   d_adata_offsets, d_verdict, stream_handle: int = 0):
        """Device-tensor form (asynchronous on `stream_handle`)."""
        n = d_verdict.numel()
        self._check(self.lib.eccb200_bign_verify_msgs_batch_dev(
            self._h, self.BIGN_HASH_IDS[hash_name], n, d_sigs.data_ptr(), d_pubkeys.data_ptr(), d_msgs.data_ptr(),
            d_offsets.data_ptr(), d_adata.data_ptr(), d_adata_offsets.data_ptr(), d_verdict.data_ptr(),
            ctypes.c_void_p(stream_handle)), "eccb200_bign_verify_msgs_batch_dev")

    VERIFY_ALGS = {"ECKCDSA": 2, "ECSDSA": 3, "ECOSDSA": 4, "ECGDSA": 6, "ECRDSA": 7, "SM2": 8}  # ec_alg_type values

    def verify_sig_len(self, alg: str, hash_name: str) -> int:
        """signature length of verify_msgs_batch: hsize + qlen (ECSDSA, ECOSDSA), min(hsize, qlen) + qlen (ECKCDSA),
        2*qlen (ECGDSA, ECRDSA, SM2)"""
        if alg not in self.VERIFY_ALGS:
            raise KeyError(alg)
        hs = dict(self.HASH_LEN, SM3=32)[hash_name]
        return {"ECSDSA": hs, "ECOSDSA": hs, "ECKCDSA": min(hs, self.qlen)}.get(alg, self.qlen) + self.qlen

    def verify_msgs_batch(self, alg: str, hash_name: str, sigs, pubkeys, msgs, ids=None) -> np.ndarray:
        """ECKCDSA / ECSDSA / ECOSDSA / ECGDSA / ECRDSA / SM2 verification of raw messages, hashed on the device
        (hash_name may be "SM3").  sigs: n * verify_sig_len bytes, pubkeys: n * 2*plen affine, ids (a list of byte
        strings, the SM2 user IDs) required for SM2.  Returns verdict[n]: 0 valid, -1 invalid."""
        n = len(msgs)
        sg = _as_u8(sigs, n * self.verify_sig_len(alg, hash_name))
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        blob, off = self._pack_msgs(msgs)
        id_blob, id_off = self._pack_msgs(ids) if ids is not None else (None, None)
        verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_verify_msgs_batch(
            self._h, self.VERIFY_ALGS[alg], self.SIGN_HASH_IDS[hash_name], n, sg.ctypes.data, pk.ctypes.data,
            blob.ctypes.data, off.ctypes.data, id_blob.ctypes.data if id_blob is not None else None,
            id_off.ctypes.data if id_off is not None else None, verdict.ctypes.data), "eccb200_verify_msgs_batch")
        return verdict

    def verify_msgs_batch_dev(self, alg: str, hash_name: str, d_sigs, d_pubkeys, d_msgs, d_offsets, d_verdict,
                              d_ids=None, d_id_offsets=None, stream_handle: int = 0):
        """Device-tensor form (asynchronous on `stream_handle`); n = d_verdict.numel(); d_offsets / d_id_offsets:
        n + 1 uint64 entries, not re-checked."""
        n = d_verdict.numel()
        ptr = lambda t: t.data_ptr() if t is not None else None
        self._check(self.lib.eccb200_verify_msgs_batch_dev(
            self._h, self.VERIFY_ALGS[alg], self.SIGN_HASH_IDS[hash_name], n, d_sigs.data_ptr(), d_pubkeys.data_ptr(),
            d_msgs.data_ptr(), d_offsets.data_ptr(), ptr(d_ids), ptr(d_id_offsets), d_verdict.data_ptr(),
            ctypes.c_void_p(stream_handle)), "eccb200_verify_msgs_batch_dev")

    def copy_to_host(self, d_ptr: int, nbytes: int) -> np.ndarray:
        out = np.empty(nbytes, dtype=np.uint8)
        self._check(self.lib.eccb200_copy_to_host(self._h, out.ctypes.data, ctypes.c_void_p(d_ptr), nbytes),
                    "eccb200_copy_to_host")
        return out

    def ecdsa_verify_msgs_batch(self, hash_name: str, sigs, pubkeys, msgs) -> np.ndarray:
        n = len(msgs)
        sg = _as_u8(sigs, n * 2 * self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        blob, off = self._pack_msgs(msgs)
        verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_verify_msgs_batch(self._h, self.HASH_IDS[hash_name], n, sg.ctypes.data,
                                                             pk.ctypes.data, blob.ctypes.data, off.ctypes.data,
                                                             verdict.ctypes.data), "eccb200_ecdsa_verify_msgs_batch")
        return verdict

    def ecfsdsa_verify_batch(self, sigs, pubkeys, digests, hlen: int) -> np.ndarray:
        """digests[i] = H(r_i || m_i); sigs [n][2*plen + qlen]."""
        sg = _as_u8(sigs)
        n = sg.size // (2 * self.plen + self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        dg = _as_u8(digests, n * hlen)
        verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecfsdsa_verify_batch(self._h, n, sg.ctypes.data, pk.ctypes.data, dg.ctypes.data,
                                                          hlen, verdict.ctypes.data), "eccb200_ecfsdsa_verify_batch")
        return verdict

    def _schnorr_msm(self, fn_name: str, siglen: int, sigs, pubkeys, digests, hlen: int, seed: Optional[bytes]) -> bool:
        sg = _as_u8(sigs)
        n = sg.size // siglen
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        dg = _as_u8(digests, n * hlen)
        ok = ctypes.c_int(0)
        sd = None
        if seed is not None:
            if len(seed) != 32:
                raise ValueError("seed must be 32 bytes")
            sd = ctypes.cast(ctypes.create_string_buffer(bytes(seed), 32), ctypes.c_void_p)
        self._check(getattr(self.lib, fn_name)(self._h, n, sg.ctypes.data, pk.ctypes.data, dg.ctypes.data, hlen, sd,
                                               ctypes.byref(ok)), fn_name)
        return ok.value == 1

    def ecfsdsa_verify_msm_batch(self, sigs, pubkeys, digests, hlen: int, seed: Optional[bytes] = None) -> bool:
        """The whole batch as ONE multi-scalar multiplication (the reference's verify_batch form): True iff every
        signature verifies.  seed: 32 bytes (None: from the OS)."""
        return self._schnorr_msm("eccb200_ecfsdsa_verify_msm_batch", 2 * self.plen + self.qlen, sigs, pubkeys, digests,
                                 hlen, seed)

    def bip0340_verify_msm_batch(self, sigs, pubkeys, digests, hlen: int, seed: Optional[bytes] = None) -> bool:
        """BIP0340 in the same form (sigs [n][plen + qlen] = r || s, digests = tagged challenge hashes)."""
        return self._schnorr_msm("eccb200_bip0340_verify_msm_batch", self.plen + self.qlen, sigs, pubkeys, digests, hlen,
                                 seed)

    def ecfsdsa_verify_msm_batch_dev(self, n: int, d_sigs: int, d_pubkeys: int, d_digests: int, hlen: int,
                                     seed: Optional[bytes] = None, stream: int = 0) -> bool:
        ok = ctypes.c_int(0)
        sd = ctypes.cast(ctypes.create_string_buffer(bytes(seed), 32), ctypes.c_void_p) if seed is not None else None
        self._check(self.lib.eccb200_ecfsdsa_verify_msm_batch_dev(self._h, n, ctypes.c_void_p(d_sigs),
                                                                  ctypes.c_void_p(d_pubkeys), ctypes.c_void_p(d_digests),
                                                                  hlen, sd, ctypes.byref(ok), ctypes.c_void_p(stream)),
                    "eccb200_ecfsdsa_verify_msm_batch_dev")
        return ok.value == 1

    def double_smul_batch(self, ab, pubkeys) -> Tuple[np.ndarray, np.ndarray]:
        """W_i = a_i*G + b_i*Y_i (affine); ab [n][2*qlen] = a || b."""
        sc = _as_u8(ab)
        n = sc.size // (2 * self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        out = np.zeros((n, 2 * self.plen), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_double_smul_batch(self._h, n, sc.ctypes.data, pk.ctypes.data, out.ctypes.data,
                                                       status.ctypes.data), "eccb200_double_smul_batch")
        return out, status

    def bip0340_verify_batch(self, sigs, pubkeys, digests, hlen: int) -> np.ndarray:
        """sigs [n][plen + qlen] = r || s; digests[i] = tagged hash of r_i || x(Y_i) || m_i."""
        sg = _as_u8(sigs)
        n = sg.size // (self.plen + self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        dg = _as_u8(digests, n * hlen)
        verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_bip0340_verify_batch(self._h, n, sg.ctypes.data, pk.ctypes.data, dg.ctypes.data,
                                                          hlen, verdict.ctypes.data), "eccb200_bip0340_verify_batch")
        return verdict

    # ---- the reference's structured key / signature records (include/libecc_b200.h)
    def structured_pub_key_import_batch(self, records, alg: int = 1) -> Tuple[np.ndarray, np.ndarray]:
        rec = _as_u8(records)
        n = rec.size // (3 + 3 * self.plen)
        out = np.zeros((n, 2 * self.plen), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_structured_pub_key_import_batch(self._h, n, rec.ctypes.data, alg, out.ctypes.data,
                                                                     status.ctypes.data),
                    "eccb200_structured_pub_key_import_batch")
        return out, status

    def structured_pub_key_export_batch(self, pubkeys, alg: int = 1) -> np.ndarray:
        pk = _as_u8(pubkeys)
        n = pk.size // (2 * self.plen)
        out = np.zeros((n, 3 + 3 * self.plen), dtype=np.uint8)
        self._check(self.lib.eccb200_structured_pub_key_export_batch(self._h, n, pk.ctypes.data, alg, out.ctypes.data),
                    "eccb200_structured_pub_key_export_batch")
        return out

    def structured_key_pair_batch(self, priv_records, priv_len: int, alg: int = 1) -> Tuple[np.ndarray, np.ndarray]:
        rec = _as_u8(priv_records)
        n = rec.size // (3 + priv_len)
        out = np.zeros((n, 3 + 3 * self.plen), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_structured_key_pair_batch(self._h, n, rec.ctypes.data, priv_len, alg,
                                                               out.ctypes.data, status.ctypes.data),
                    "eccb200_structured_key_pair_batch")
        return out, status

    def ecdsa_verify_structured_batch(self, sig_records, pub_records, hash_name: str, digests, hlen: int,
                                      alg: int = 1) -> np.ndarray:
        sr = _as_u8(sig_records)
        n = sr.size // (3 + 2 * self.qlen)
        pr = _as_u8(pub_records, n * (3 + 3 * self.plen))
        dg = _as_u8(digests, n * hlen)
        verdict = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_verify_structured_batch(self._h, n, sr.ctypes.data, pr.ctypes.data, alg,
                                                                   self.REF_HASH_IDS[hash_name], dg.ctypes.data, hlen,
                                                                   verdict.ctypes.data),
                    "eccb200_ecdsa_verify_structured_batch")
        return verdict

    def ecdsa_sign_structured_batch(self, priv_records, priv_len: int, nonces, hash_name: str, digests, hlen: int,
                                    alg: int = 1) -> Tuple[np.ndarray, np.ndarray]:
        rec = _as_u8(priv_records)
        n = rec.size // (3 + priv_len)
        k = _as_u8(nonces, n * self.qlen)
        dg = _as_u8(digests, n * hlen)
        out = np.zeros((n, 3 + 2 * self.qlen), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_ecdsa_sign_structured_batch(self._h, n, rec.ctypes.data, priv_len, alg,
                                                                 self.REF_HASH_IDS[hash_name], k.ctypes.data,
                                                                 dg.ctypes.data, hlen, out.ctypes.data,
                                                                 status.ctypes.data),
                    "eccb200_ecdsa_sign_structured_batch")
        return out, status

    def prj_pt_unique_batch(self, prj_points) -> Tuple[np.ndarray, np.ndarray]:
        pp = _as_u8(prj_points)
        n = pp.size // (3 * self.plen)
        out = np.zeros((n, 2 * self.plen), dtype=np.uint8)
        status = np.zeros(n, dtype=np.int8)
        self._check(self.lib.eccb200_prj_pt_unique_batch(self._h, n, pp.ctypes.data, out.ctypes.data,
                                                         status.ctypes.data), "eccb200_prj_pt_unique_batch")
        return out, status

    def ecdsa_uv_batch(self, sigs, digests, hlen: int) -> np.ndarray:
        sg = _as_u8(sigs)
        n = sg.size // (2 * self.qlen)
        dg = _as_u8(digests, n * hlen)
        out = np.zeros((n, 2 * self.qlen), dtype=np.uint8)
        self._check(self.lib.eccb200_ecdsa_uv_batch(self._h, n, sg.ctypes.data, dg.ctypes.data, hlen,
                                                    out.ctypes.data), "eccb200_ecdsa_uv_batch")
        return out

    def fp_mul_chain_bench(self, a, b, iters: int, striped: bool):
        x = _as_u8(a)
        n = x.size // self.plen
        y = _as_u8(b, n * self.plen)
        out = np.zeros((n, self.plen), dtype=np.uint8)
        ms = ctypes.c_float()
        self._check(self.lib.eccb200_fp_mul_chain_bench(self._h, int(striped), n, x.ctypes.data, y.ctypes.data,
                                                        out.ctypes.data, iters, ctypes.byref(ms)),
                    "eccb200_fp_mul_chain_bench")
        return out, float(ms.value)

    def fp_mul_monty_batch(self, a, b, which: int = 0) -> np.ndarray:
        x = _as_u8(a)
        n = x.size // self.plen
        y = _as_u8(b, n * self.plen)
        out = np.zeros((n, self.plen), dtype=np.uint8)
        self._check(self.lib.eccb200_fp_mul_monty_batch(self._h, which, n, x.ctypes.data, y.ctypes.data,
                                                        out.ctypes.data), "eccb200_fp_mul_monty_batch")
        return out

    def fp_addsub_batch(self, a, b, op: int, which: int = 0) -> np.ndarray:
        """op 0 = a + b, 1 = a - b, 2 = a * a * R^-1 (mod p for which = 0, mod q for 1)."""
        x = _as_u8(a)
        n = x.size // self.plen
        y = _as_u8(b, n * self.plen)
        out = np.zeros((n, self.plen), dtype=np.uint8)
        self._check(self.lib.eccb200_fp_addsub_batch(self._h, which, op, n, x.ctypes.data, y.ctypes.data,
                                                     out.ctypes.data), "eccb200_fp_addsub_batch")
        return out

    # ---- device-buffer API (torch uint8/int8 CUDA tensors; asynchronous on torch's current stream) ---------
    def prj_pt_mul_batch_dev(self, d_scalars, d_points, d_out, d_status, stream_handle: int = 0):
        n = d_scalars.numel() // self.qlen
        self._check(self.lib.eccb200_prj_pt_mul_batch_dev(
            self._h, n, d_scalars.data_ptr(), d_points.data_ptr() if d_points is not None else None,
            d_out.data_ptr(), d_status.data_ptr(), ctypes.c_void_p(stream_handle)), "eccb200_prj_pt_mul_batch_dev")

    def prj_pt_mul_batch_dev_gather(self, n: int, p_scalars: int, p_points, p_out: int, p_status: int, dst_out, dst_status,
                                    dst_flag, flag_value: int, p_wait_flags, wait_count: int, wait_value: int,
                                    stream_handle: int = 0):
        """Raw-pointer form (ints): see eccb200_prj_pt_mul_batch_dev_gather in include/libecc_b200.h."""
        k = len(dst_out)
        arr = lambda xs: (ctypes.c_void_p * max(k, 1))(*[ctypes.c_void_p(x) for x in xs])
        a_out, a_st, a_fl = arr(dst_out), arr(dst_status), arr(dst_flag)
        self._check(self.lib.eccb200_prj_pt_mul_batch_dev_gather(
            self._h, n, p_scalars, p_points, p_out, p_status, k, a_out, a_st, a_fl, flag_value & 0xFFFFFFFF,
            p_wait_flags, wait_count, wait_value & 0xFFFFFFFF, ctypes.c_void_p(stream_handle)),
            "eccb200_prj_pt_mul_batch_dev_gather")

    def push_results(self, dst_ptrs, p_src: int, nbytes: int, dst_flags, flag_value: int, p_wait_flags, wait_count: int,
                     wait_value: int, stream_handle: int = 0):
        k = len(dst_ptrs)
        a_dst = (ctypes.c_void_p * k)(*[ctypes.c_void_p(x) for x in dst_ptrs])
        a_fl = (ctypes.c_void_p * k)(*[ctypes.c_void_p(x) for x in dst_flags])
        self._check(self.lib.eccb200_push_results(self._h, k, a_dst, ctypes.c_void_p(p_src), nbytes, a_fl,
                                                  flag_value & 0xFFFFFFFF, p_wait_flags, wait_count,
                                                  wait_value & 0xFFFFFFFF, ctypes.c_void_p(stream_handle)),
                    "eccb200_push_results")

    def ipc_alloc(self, nbytes: int):
        p = ctypes.c_void_p()
        h = (ctypes.c_uint8 * 64)()
        self._check(self.lib.eccb200_ipc_alloc(self._h, nbytes, ctypes.byref(p), h), "eccb200_ipc_alloc")
        return int(p.value), bytes(h)

    def ipc_open(self, handle: bytes) -> int:
        p = ctypes.c_void_p()
        h = (ctypes.c_uint8 * 64)(*handle)
        self._check(self.lib.eccb200_ipc_open(self._h, h, ctypes.byref(p)), "eccb200_ipc_open")
        return int(p.value)

    def ipc_close(self, ptr: int):
        self._check(self.lib.eccb200_ipc_close(self._h, ctypes.c_void_p(ptr)), "eccb200_ipc_close")

    def ipc_free(self, ptr: int):
        self._check(self.lib.eccb200_ipc_free(self._h, ctypes.c_void_p(ptr)), "eccb200_ipc_free")

    def flag_wait(self, p_flags: int, count: int, value: int, stream_handle: int = 0):
        self._check(self.lib.eccb200_flag_wait(self._h, ctypes.c_void_p(p_flags), count, value & 0xFFFFFFFF,
                                               ctypes.c_void_p(stream_handle)), "eccb200_flag_wait")

    def flag_signal(self, flag_ptrs, value: int, stream_handle: int = 0):
        a = (ctypes.c_void_p * len(flag_ptrs))(*[ctypes.c_void_p(x) for x in flag_ptrs])
        self._check(self.lib.eccb200_flag_signal(self._h, a, len(flag_ptrs), value & 0xFFFFFFFF,
                                                 ctypes.c_void_p(stream_handle)), "eccb200_flag_signal")

    def prj_pt_mul_batch_dev_raw(self, n: int, p_scalars: int, p_points, p_out: int, p_status: int, stream_handle: int = 0):
        """eccb200_prj_pt_mul_batch_dev on raw device addresses (ints)."""
        self._check(self.lib.eccb200_prj_pt_mul_batch_dev(self._h, n, p_scalars, p_points, p_out, p_status,
                                                          ctypes.c_void_p(stream_handle)), "eccb200_prj_pt_mul_batch_dev")

    def ecdsa_verify_batch_dev(self, d_sigs, d_pubkeys, d_digests, hlen: int, d_verdict, stream_handle: int = 0):
        n = d_sigs.numel() // (2 * self.qlen)
        self._check(self.lib.eccb200_ecdsa_verify_batch_dev(
            self._h, n, d_sigs.data_ptr(), d_pubkeys.data_ptr(), d_digests.data_ptr(), hlen,
            d_verdict.data_ptr(), ctypes.c_void_p(stream_handle)), "eccb200_ecdsa_verify_batch_dev")

    def ecdsa_recover_batch_dev(self, d_sigs, d_digests, hlen: int, d_keys, d_status, stream_handle: int = 0):
        """d_sigs [n][2*qlen], d_digests [n][hlen] -> d_keys [n][2][2*plen], d_status [n][2] (CUDA tensors)."""
        n = d_sigs.numel() // (2 * self.qlen)
        self._check(self.lib.eccb200_ecdsa_recover_batch_dev(
            self._h, n, d_sigs.data_ptr(), d_digests.data_ptr(), hlen, d_keys.data_ptr(), d_status.data_ptr(),
            ctypes.c_void_p(stream_handle)), "eccb200_ecdsa_recover_batch_dev")


class MultiEngine:
    """One curve on several GPUs of ONE process (eccb200_multi): host-pointer batches are sharded internally."""

    def __init__(self, curve: str, devices=None, comb_window: int = 0):
        self.lib = load_library()
        self.curve = curve
        self.plen, self.qlen = curve_sizes(curve)
        h = ctypes.c_void_p()
        arr = (ctypes.c_int * len(devices))(*devices) if devices else None
        if self.lib.eccb200_multi_create(ctypes.byref(h), CURVE_IDS[curve], arr, len(devices) if devices else 0,
                                         comb_window):
            raise EccB200Error("eccb200_multi_create: " + self.lib.eccb200_last_error().decode())
        self._h = h

    @property
    def device_count(self) -> int:
        return self.lib.eccb200_multi_device_count(self._h)

    def close(self):
        if getattr(self, "_h", None):
            self.lib.eccb200_multi_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def prj_pt_mul_batch(self, scalars, points=None, out=None, status=None):
        sc = _as_u8(scalars)
        n = sc.size // self.qlen
        pt = _as_u8(points, n * 2 * self.plen) if points is not None else None
        if out is None:
            out = np.zeros((n, 2 * self.plen), dtype=np.uint8)
        if status is None:
            status = np.zeros(n, dtype=np.int8)
        if self.lib.eccb200_multi_prj_pt_mul_batch(self._h, n, sc.ctypes.data, pt.ctypes.data if pt is not None else None,
                                                   out.ctypes.data, status.ctypes.data):
            raise EccB200Error("eccb200_multi_prj_pt_mul_batch: " + self.lib.eccb200_last_error().decode())
        return out, status

    def ecdsa_verify_batch(self, sigs, pubkeys, digests, hlen: int, verdict=None):
        sg = _as_u8(sigs)
        n = sg.size // (2 * self.qlen)
        pk = _as_u8(pubkeys, n * 2 * self.plen)
        dg = _as_u8(digests, n * hlen)
        if verdict is None:
            verdict = np.zeros(n, dtype=np.int8)
        if self.lib.eccb200_multi_ecdsa_verify_batch(self._h, n, sg.ctypes.data, pk.ctypes.data, dg.ctypes.data, hlen,
                                                     verdict.ctypes.data):
            raise EccB200Error("eccb200_multi_ecdsa_verify_batch: " + self.lib.eccb200_last_error().decode())
        return verdict
