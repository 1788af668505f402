/*
 * libecc_b200.h — C ABI of the H100-native batched scalar-multiplication / ECDSA-verification engine.
 *
 * This is the drop-in boundary for the hot path of ANSSI-FR/libecc (SURVEY.md §8b).  The reference has no FFI:
 * its boundary is the C symbol + struct ABI of libec.a / libsign.a.  Two layers are exported:
 *
 *  (1) this header: a flat, struct-free batch API on libecc's WIRE FORMATS (big-endian byte strings exactly as
 *      produced by nn_export_to_buf  src/nn/nn.c:511  and  prj_pt_export_to_aff_buf  src/curves/prj_pt.c:600).
 *      Each entry point names the reference function it replaces.
 *  (2) libecc_b200_dropin.h: the reference's own entry points (prj_pt_mul, prj_pt_mul_blind, and the ECDSA
 *      verify_batch slot) on the reference's own structs, implemented on top of (1).
 *
 * Conventions kept from the reference: int return, 0 = success, -1 = error (src/utils/utils.h:137-143); the caller
 * owns every buffer; nothing is retained after return; callable from any thread (one context may be used by one
 * thread at a time; create one context per thread or guard it).  All arithmetic runs on the GPU; if no CUDA device
 * or the wrong architecture is present every call fails with -1 (there is NO CPU fallback).
 */
#ifndef LIBECC_B200_H
#define LIBECC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Curve identifiers = the reference's ec_curve_type values (src/lib_ecc_types.h:147-). */
#define ECCB200_FRP256V1 1
#define ECCB200_SECP256R1 4
#define ECCB200_SECP384R1 5
/* additional short-Weierstrass curves served by the same kernels (generic-a / a = 0 doubling, generic reduction) */
#define ECCB200_BRAINPOOLP256R1 8
#define ECCB200_BRAINPOOLP384R1 12
#define ECCB200_SECP256K1 19
#define ECCB200_SECP521R1 6
#define ECCB200_SM2P256V1 17
#define ECCB200_BRAINPOOLP512R1 9
#define ECCB200_SECP224R1 3
#define ECCB200_SECP192R1 2

/* Per-item status codes written by the batch calls. */
#define ECCB200_OK 0        /* finite result / valid signature                                          */
#define ECCB200_INFINITY 1  /* result is the point at infinity (prj_pt_iszero), output bytes are zero    */
#define ECCB200_ERR (-1)    /* what the reference reports with ret = -1 (bad point, r/s range, bad sig)  */
#define ECCB200_RETRY 2     /* signing only: the reference would restart with a fresh nonce (r = 0, s = 0, ...) */

typedef struct eccb200_ctx eccb200_ctx;

/*
 * Create an engine context for one curve on one device: uploads the curve constants and builds the fixed-base
 * comb table T[i][d] = d * 2^(w*i) * G on the GPU.  Replaces import_params (src/curves/ec_params.c:24) as the
 * place where per-curve state is derived.  comb_window: bits per fixed-base window: 4..16, or an even value in
 * 18..26 (table of ceil(qbits/w) * 2^w * 2*plen bytes, built from a half-width table: 3.2 GiB at 22 bits and
 * 40 GiB at 26 bits for a 256-bit curve); 0 = default.
 */
int eccb200_ctx_create(eccb200_ctx **ctx, int curve_id, int device, int comb_window);
void eccb200_ctx_destroy(eccb200_ctx *ctx);

/* ceil(bitlen(p)/8) and ceil(bitlen(q)/8) for a curve id; -1 if unknown. */
int eccb200_curve_sizes(int curve_id, uint32_t *plen, uint32_t *qlen);
/* Reference curve name ("SECP256R1", ...) for an id, or NULL. */
const char *eccb200_curve_name(int curve_id);

/*
 * Batched prj_pt_mul + prj_pt_unique + prj_pt_export_to_aff_buf
 *   (src/curves/prj_pt.c:1759 prj_pt_mul; :241 prj_pt_unique; :600 prj_pt_export_to_aff_buf).
 *   scalars : n * qlen bytes, big-endian, any value in [0, 2^(8*qlen)) (reduced mod q like the reference's ladder)
 *   points  : n * 2*plen bytes affine big-endian x||y, or NULL for the curve generator G (params->ec_gen)
 *   out     : n * 2*plen bytes affine big-endian x||y (zero for non-OK items)
 *   status  : n bytes, ECCB200_OK / ECCB200_INFINITY / ECCB200_ERR (point not on curve or coordinate >= p:
 *             the reference fails prj_pt_import_from_aff_buf :541-545 / prj_pt_mul :1767)
 * Host-pointer version: blocking, includes the host<->device copies (pipelined over three streams in chunks of whole
 * kernel waves that ramp up from one wave and down to one wave, see eccb200_pipeline_chunk_bounds).  Page-locked caller buffers (eccb200_host_alloc, cudaHostAlloc, cudaHostRegister) are DMA'd directly;
 * pageable ones are staged through the context's own pinned buffers at the cost of one memcpy each way.
 */
int eccb200_prj_pt_mul_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *scalars, const uint8_t *points,
			     uint8_t *out, int8_t *status);

/*
 * Same, on device-resident buffers, enqueued on `stream` (a cudaStream_t; NULL = default stream); asynchronous.
 * Rules for every *_dev entry point:
 *  - a context is used by one host thread at a time; its *_dev calls may name different streams, but they share one
 *    set of scratch buffers, so the library chains them on the device (each call's kernels wait for the previous
 *    call's) — use one context per stream to overlap calls;
 *  - on the 256-, 384- and 512-bit curves the scalar / point / signature / key / output buffers must be 16-byte
 *    aligned (the kernels use 16-byte vector accesses); a misaligned pointer is refused with -1, never dereferenced.
 */
int eccb200_prj_pt_mul_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_scalars, const uint8_t *d_points,
				 uint8_t *d_out, int8_t *d_status, void *stream);

/*
 * Multi-GPU, one process per GPU (SURVEY.md §8e "final result gather"): the normalisation kernel of a batch stores
 * every result not only into d_out / d_status but also straight into up to 8 destination buffers on PEER GPUs —
 * buffers allocated with eccb200_ipc_alloc in the peer's process and mapped here with eccb200_ipc_open — so the
 * gather travels over NVLink as ordinary stores of the kernel that produces the bytes, and no collective kernel
 * competes with the arithmetic for the SMs.  dst_out[j] / dst_status[j] point at THIS rank's slot of destination j
 * (same [n][2*plen] / [n] layout as d_out / d_status).  When the last thread block has stored its results the kernel
 * publishes flag_value to *dst_flag[j] (system-scope release); the destination waits for it with eccb200_flag_wait.
 * Flow control: if wait_count > 0 the normalisation kernel (not the scalar multiplication before it) first waits
 * until d_wait_flags[i] >= wait_value for all i < wait_count — the destinations' "buffer released" acknowledgements
 * (eccb200_flag_signal), flags in this GPU's memory.
 * n must be > 0.  Flags are 32-bit counters compared modulo 2^32.
 */
int eccb200_prj_pt_mul_batch_dev_gather(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_scalars,
					const uint8_t *d_points, uint8_t *d_out, int8_t *d_status, int n_dst,
					uint8_t *const *dst_out, int8_t *const *dst_status, uint32_t *const *dst_flag,
					uint32_t flag_value, const uint32_t *d_wait_flags, int wait_count,
					uint32_t wait_value, void *stream);
/* Copy-engine form of the same gather: DMA `bytes` from d_src to up to 8 peer-mapped destinations on `stream` (NVLink,
 * no SM involved), after the destinations' acknowledgements (d_wait_flags, in this GPU's memory) if wait_count > 0,
 * then publish flag_value to *dst_flag[j].  Used pipelined: the push of step s overlaps the kernels of step s + 1. */
int eccb200_push_results(eccb200_ctx *ctx, int n_dst, void *const *dst, const void *d_src, size_t bytes,
			 uint32_t *const *dst_flag, uint32_t flag_value, const uint32_t *d_wait_flags, int wait_count,
			 uint32_t wait_value, void *stream);
/* Device memory that other processes on the box can map: cudaMalloc + cudaIpcGetMemHandle (zero-filled).  The
 * 64-byte handle is passed to the peers by any means (bench.py: torch.distributed); they map it with
 * eccb200_ipc_open (peer access over NVLink is enabled on first use) and unmap it with eccb200_ipc_close. */
int eccb200_ipc_alloc(eccb200_ctx *ctx, size_t bytes, void **d_ptr, uint8_t handle[64]);
int eccb200_ipc_open(eccb200_ctx *ctx, const uint8_t handle[64], void **d_ptr);
int eccb200_ipc_close(eccb200_ctx *ctx, void *d_ptr);
int eccb200_ipc_free(eccb200_ctx *ctx, void *d_ptr);
/* Stream-ordered flag operations of the gather: wait until d_flags[i] >= value for all i < count (flags in this
 * GPU's memory); publish value to count (<= 8) flags, typically peer-mapped, after everything enqueued before. */
int eccb200_flag_wait(eccb200_ctx *ctx, const uint32_t *d_flags, int count, uint32_t value, void *stream);
int eccb200_flag_signal(eccb200_ctx *ctx, uint32_t *const *d_flags, int count, uint32_t value, void *stream);

/*
 * Multi-GPU, ONE process (SURVEY.md §8b "multi-GPU fan-out is internal"): a context set over several devices
 * (devices == NULL or n_devices <= 0: every visible device); the batch calls below shard [0, n) into contiguous
 * ranges, one per device, run each shard through that device's host-pointer pipeline on its own host thread, and
 * every device DMAs its results straight into the caller's arrays — there is no gather step.  Same argument
 * meaning, status codes and error behaviour as the single-device calls; n is 64-bit.
 */
typedef struct eccb200_multi eccb200_multi;
int eccb200_multi_create(eccb200_multi **m, int curve_id, const int *devices, int n_devices, int comb_window);
void eccb200_multi_destroy(eccb200_multi *m);
int eccb200_multi_device_count(const eccb200_multi *m);
eccb200_ctx *eccb200_multi_ctx(eccb200_multi *m, int index); /* the per-device context (owned by m) */
int eccb200_multi_prj_pt_mul_batch(eccb200_multi *m, uint64_t n, const uint8_t *scalars, const uint8_t *points,
				   uint8_t *out, int8_t *status);
int eccb200_multi_ecdsa_verify_batch(eccb200_multi *m, uint64_t n, const uint8_t *sigs, const uint8_t *pubkeys,
				     const uint8_t *digests, uint32_t hlen, int8_t *verdict);

/*
 * Batched prj_pt_unique + prj_pt_export_to_aff_buf (src/curves/prj_pt.c:241, :600) on the reference's homogeneous
 * projective wire format (X||Y||Z big-endian, 3*plen bytes, prj_pt_export_to_buf :562): one simultaneous inversion
 * per GPU thread instead of one fp_inv per point.  Points are validated like prj_pt_import_from_buf (:462-500).
 *   status: ECCB200_OK / ECCB200_INFINITY (Z == 0; the reference's prj_pt_unique errors on it) / ECCB200_ERR.
 */
int eccb200_prj_pt_unique_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *prj_points, uint8_t *out_aff,
				int8_t *status);

/*
 * Batched ECDSA verification on pre-hashed messages: replaces, per signature, __ecdsa_verify_init's checks
 * (src/sig/ecdsa_common.c:645-658) and __ecdsa_verify_finalize steps 3-10 (:760-810); hashing (step 2) stays on
 * the host in the reference's src/hash.  This is what fills the ECDSA verify_batch slot the reference leaves
 * unsupported (src/sig/sig_algs_internal.h:294).
 *   sigs    : n * 2*qlen bytes r||s;  pubkeys : n * 2*plen bytes affine x||y;  digests : n * hlen bytes
 *   verdict : n bytes, ECCB200_OK (valid) / ECCB200_ERR (invalid, or any error such as key not on curve)
 */
int eccb200_ecdsa_verify_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
			       const uint8_t *digests, uint32_t hlen, int8_t *verdict);
int eccb200_ecdsa_verify_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
				   const uint8_t *d_digests, uint32_t hlen, int8_t *d_verdict, void *stream);
/* The same with a per-key state column: 0 = affine key in pubkeys[i]; 1 = the key is the point at infinity
 * (pubkeys[i] ignored) — the reference's ec_verify accepts such an ec_pub_key and computes W' = u*G
 * (src/curves/prj_pt.c:1767-1775 gives v*infinity = infinity); -1 = rejected key.  For callers that hold
 * reference structs (the drop-in layer). */
/* The same with the public keys in the reference's homogeneous projective form X || Y || Z (3*plen bytes each: what an
 * ec_pub_key's y holds, Z != 1 in general): key import (prj_pt_import_from_buf's checks, src/curves/prj_pt.c:462-500)
 * and the batched prj_pt_unique run on the device in front of the verification kernel, chunk by chunk. */
int eccb200_ecdsa_verify_prj_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *prj_pubkeys,
				   const uint8_t *digests, uint32_t hlen, int8_t *verdict);
int eccb200_ecdsa_verify_keystate_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
					const int8_t *key_state, const uint8_t *digests, uint32_t hlen,
					int8_t *verdict);

/*
 * Batched ECDSA public-key recovery on pre-hashed messages: __ecdsa_public_key_from_sig per item
 * (src/sig/ecdsa_common.c:867-1011, behind ecdsa_public_key_from_sig src/sig/ecdsa.c:73 and
 * decdsa_public_key_from_sig src/sig/decdsa.c; the key type changes nothing in the computation).
 *   sigs    : n * 2*qlen bytes r||s;  digests : n * hlen bytes, hlen 1..128 (e as for verification, :942-950)
 *   keys    : n * 2 * 2*plen bytes, affine Y1 = v*R1 + u*G then Y2 = v*R2 + u*G (:992-999) with R1 = (r, sqrt1),
 *             R2 = (r, -sqrt1), sqrt1 the first root of the reference's fp_sqrt (src/fp/fp_sqrt.c),
 *             u = -e/r and v = s/r mod q (:981-990); a key is zero unless its status is OK
 *   status  : n * 2 bytes, one per key: ECCB200_OK / ECCB200_INFINITY (the reference returns that key as the point at
 *             infinity without complaint); both ECCB200_ERR where the reference returns -1: r or s outside [1, q-1]
 *             (:900-912), r >= p (fp_set_nn, :958; possible on FRP256V1 only), or r^3 + ar + b not a square (:959)
 * Only x = r is tried.  The reference's restart (:914-931, :960-971) first tries r + 2q, never r + q, and can not succeed
 * on the curves of this library (cofactor 1, so q > p/2: r + 2q >= p, which fp_set_nn refuses, src/fp/fp.c:213).  So a
 * signature whose nonce point had x >= q gives ECCB200_ERR, or keys from x = r when that happens to be an x coordinate,
 * exactly as the reference does; never the keys of x = r + q.  One kernel launch per chunk: one ECDSA verification's
 * elliptic-curve work plus one point addition per item.  The _dev form runs on `stream`; on the 256-, 384- and 512-bit
 * curves d_sigs and d_keys must be 16-byte aligned.
 */
int eccb200_ecdsa_recover_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *digests, uint32_t hlen,
				uint8_t *keys, int8_t *status);
int eccb200_ecdsa_recover_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_digests,
				    uint32_t hlen, uint8_t *d_keys, int8_t *d_status, void *stream);

/*
 * Batched ECDSA signing on pre-hashed messages with caller-supplied nonces: replaces, per signature,
 * __ecdsa_sign_finalize steps 3-11 (src/sig/ecdsa_common.c:403-560): k*G (:479), prj_pt_unique (:481), r = x mod q,
 * s = k^-1 (e + r*d) mod q (:537-540).  The nonce comes from the caller exactly as the reference's signing context
 * takes it from its `rand` callback (src/sig/sig_algs_internal.h:158; eccb200_decdsa_sign_batch below derives RFC 6979
 * nonces on the device instead).  Key generation is eccb200_prj_pt_mul_batch with points == NULL (src/sig/ec_key.c, d*G).
 *   privkeys, nonces : n * qlen bytes each, values in [1, q-1] (else ECCB200_ERR);  digests : n * hlen bytes
 *   sigs : n * 2*qlen bytes r||s (zero unless status is OK);  status : ECCB200_OK / ECCB200_RETRY / ECCB200_ERR
 * NOTE: like every entry point of this library this is a throughput path, NOT a constant-time one.
 */
int eccb200_ecdsa_sign_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *privkeys, const uint8_t *nonces,
			     const uint8_t *digests, uint32_t hlen, uint8_t *sigs, int8_t *status);
int eccb200_ecdsa_sign_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_privkeys, const uint8_t *d_nonces,
				 const uint8_t *d_digests, uint32_t hlen, uint8_t *d_sigs, int8_t *d_status,
				 void *stream);

/*
 * Batched deterministic ECDSA (DECDSA) on pre-hashed messages: per item the nonce of RFC 6979 §3.2 exactly as the
 * reference derives it (__ecdsa_rfc6979_nonce, src/sig/ecdsa_common.c:48-169), with HMAC over hash_type as hmac_init /
 * hmac_update / hmac_finalize of src/hash/hmac.c compute it, then the signature of eccb200_ecdsa_sign_batch with that
 * nonce and hlen = the digest size.  One kernel derives k (one item per thread, the k >= q retry loop in the thread),
 * then the comb, the batched normalisation and the ECDSA finish kernel run as for eccb200_ecdsa_sign_batch.
 *   privkeys : n * qlen bytes, x in [1, q-1] (else ECCB200_ERR, and no HMAC work for that item)
 *   digests  : n * digest_size(hash_type) bytes, digest i = H(m_i)
 *   hash_type: 1 (SHA224), 2 .. 8 (SHA256, SHA384, SHA512, SHA3_224 .. SHA3_512) or 11 (SM3)
 *   sigs     : n * 2*qlen bytes r||s, zero unless status is OK
 *   status   : ECCB200_OK; ECCB200_ERR for x outside [1, q-1] or a derived k of 0 (the reference checks k >= q only,
 *              :149-150, and would fail later on the point at infinity); ECCB200_RETRY where __ecdsa_sign_finalize would
 *              `goto restart` (r == 0 :490-494, e == r*x :514-518, s == 0 :546-550).  The reference does not end those
 *              cases with a new signature: on r == 0 it derives the same k again and never returns; on the other two it
 *              derives a k from an all-zero digest, because the digest was wiped at :497.  This entry point does neither
 *              and reports RETRY; no honest or crafted input is known to reach these cases.
 * An unsupported hash_type returns -1 (eccb200_last_error) and writes nothing.  SHA-224 is accepted by the four
 * deterministic / message ECDSA signers only.  The _dev form follows the rules of every *_dev entry point (one scratch
 * set per context, calls chained across streams; 16-byte alignment of the privkey and signature buffers on the
 * 256/384/512-bit curves).
 * NOTE: like every entry point of this library this is a throughput path, NOT a constant-time one.
 */
#define ECCB200_ALG_ECDSA 1
#define ECCB200_ALG_DECDSA 14
#define ECCB200_HASH_SHA224 1
int eccb200_decdsa_sign_batch(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *privkeys,
			      const uint8_t *digests, uint8_t *sigs, int8_t *status);
int eccb200_decdsa_sign_batch_dev(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *d_privkeys,
				  const uint8_t *d_digests, uint8_t *d_sigs, int8_t *d_status, void *stream);

/*
 * ECDSA (sig_type ECCB200_ALG_ECDSA, the caller's nonces) or DECDSA (ECCB200_ALG_DECDSA, RFC 6979 nonces; nonces
 * ignored, may be NULL) of raw messages, hashed on the device: the whole of ec_sign(…, ECDSA | DECDSA, hash_type, NULL,
 * 0) per item.  The nonce kernel hashes each message (and derives k for DECDSA), then the chain of
 * eccb200_ecdsa_sign_batch signs the digest.
 *   privkeys, nonces : n * qlen bytes each (nonces: ECDSA only), values in [1, q-1] (else ECCB200_ERR)
 *   msgs / offsets : message i is msgs[offsets[i] .. offsets[i+1]), offsets has n + 1 entries, starts at 0 and never
 *                decreases (checked here; the _dev form does not re-check it)
 *   hash_type, sigs, status : as eccb200_decdsa_sign_batch (for ECDSA, RETRY means what it means for
 *                eccb200_ecdsa_sign_batch: a fresh nonce would succeed)
 * Any other sig_type, an unsupported hash_type, or ECDSA without nonces returns -1 (eccb200_last_error) and writes
 * nothing.  The _dev form: 16-byte alignment of the privkey, nonce and signature buffers on the 256/384/512-bit curves,
 * not of d_msgs.
 */
int eccb200_ecdsa_sign_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *privkeys,
				  const uint8_t *nonces, const uint8_t *msgs, const uint64_t *offsets, uint8_t *sigs,
				  int8_t *status);
int eccb200_ecdsa_sign_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
				      const uint8_t *d_privkeys, const uint8_t *d_nonces, const uint8_t *d_msgs,
				      const uint64_t *d_offsets, uint8_t *d_sigs, int8_t *d_status, void *stream);

/*
 * BIGN (sig_type ECCB200_ALG_BIGN, the caller's nonces) or DBIGN (ECCB200_ALG_DBIGN, deterministic nonces; nonces
 * ignored, may be NULL) signatures of raw messages, hashed on the device: ec_sign(…, BIGN | DBIGN, hash_type, adata,
 * adata_len) per item (__bign_sign_finalize, src/sig/bign_common.c:468-722), with l = qlen / 2:
 *   H = hash(m); W = k*G affine; s0 = the first min(l, 32) bytes of BELT-HASH(oid || the first 2l bytes of LE(W_x) ||
 *   H), zero-padded to l bytes (on SECP521R1, l = 33 and s0[32] = 0); s1 = (k - h - (s0 + 2^(8l)) * x) mod q with
 *   h = OS2I(reverse(H)) mod q and s0 read little-endian.  There is no restart case: s1 = 0 is emitted.
 * DBIGN derives k as __bign_determinitic_nonce (:200-342) does: belt-block rounds keyed by BELT-HASH(oid || the first
 * 2l bytes of LE(x) || t) over H zero-padded to n = max(2, hlen / 16) blocks, at least 2n rounds, until 0 < k < q.
 *   privkeys, nonces : n * qlen bytes each (nonces: BIGN only), big-endian, values in [1, q-1] (else ECCB200_ERR)
 *   msgs / offsets   : message i is msgs[offsets[i] .. offsets[i+1]), offsets has n + 1 entries
 *   adata / adata_offsets : item i's record adata[adata_offsets[i] .. adata_offsets[i+1]), the reference's layout
 *                (bign_set_adata, :149-183): oid_len (2 bytes, big-endian) || t_len (2 bytes, big-endian) || oid || t,
 *                trailing bytes allowed.  Empty, shorter than 4 bytes, oid_len + t_len > len - 4 or longer than 65535
 *                bytes (the reference's adata_len is a u16; :97-147) is ECCB200_ERR.  The OID is not checked against
 *                the hash; t is used by DBIGN only.
 *   hash_type        : 1 (SHA224), 2 .. 8 (SHA256 .. SHA3_512), 11 (SM3), 16 (BELT_HASH) or 17 .. 20 (BASH224 ..
 *                BASH512).  16 .. 20 are accepted by the four BIGN entry points only.
 *   sigs             : n * (l + qlen) bytes s0 || LE(s1) (36, 42, 48, 72, 96 or 99 bytes per item), zero unless OK
 *   status           : ECCB200_OK or ECCB200_ERR (x or the BIGN nonce outside [1, q-1], or a malformed record)
 * An unsupported sig_type or hash_type, BIGN without nonces, a NULL buffer, or (host form) offsets or adata_offsets
 * that do not start at 0 or that decrease return -1 (eccb200_last_error) and write nothing; n = 0 returns 0.  The
 * _dev form keeps its scratch (k, digests) in the context, grown on demand, does not re-check the offsets, and needs
 * 16-byte alignment of the privkey, nonce and signature buffers on the 256/384/512-bit curves, not of d_msgs or
 * d_adata.
 * NOTE: like every entry point of this library this is a throughput path, NOT a constant-time one.
 */
#define ECCB200_ALG_BIGN 18
#define ECCB200_ALG_DBIGN 19
#define ECCB200_HASH_BELT_HASH 16
int eccb200_bign_sign_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *privkeys,
				 const uint8_t *nonces, const uint8_t *msgs, const uint64_t *offsets, const uint8_t *adata,
				 const uint64_t *adata_offsets, uint8_t *sigs, int8_t *status);
int eccb200_bign_sign_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
				     const uint8_t *d_privkeys, const uint8_t *d_nonces, const uint8_t *d_msgs,
				     const uint64_t *d_offsets, const uint8_t *d_adata, const uint64_t *d_adata_offsets,
				     uint8_t *d_sigs, int8_t *d_status, void *stream);

/*
 * BIGN / DBIGN verification of raw messages (both schemes verify alike): ec_verify(…, BIGN, hash_type, adata,
 * adata_len) per item (__bign_verify_init / __bign_verify_finalize, src/sig/bign_common.c:742-993).  Reject s1 >= q;
 * W' = ((s1 + h) mod q)*G + (s0 + 2^(8l))*Y; reject W' at infinity; accept iff s0 equals the first l bytes of
 * BELT-HASH(oid || the first 2l bytes of LE(W'_x) || H), zero-padded as in signing.  One kernel checks the record and
 * s1, hashes the message and prepares the scalars, the double-scalar kernel of eccb200_verify_msgs_batch computes W',
 * and one kernel runs the BELT-HASH test.
 *   sigs : n * (l + qlen) bytes;  pubkeys : n * 2*plen affine keys;  msgs, adata, hash_type : as the signer
 *   verdict : 0 valid, -1 invalid (a malformed record, s1 >= q, a key off the curve, or a failed test)
 * Argument errors as the signer.  The _dev form: 16-byte alignment of the signature and key buffers on the
 * 256/384/512-bit curves.
 */
int eccb200_bign_verify_msgs_batch(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *sigs,
				   const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *offsets,
				   const uint8_t *adata, const uint64_t *adata_offsets, int8_t *verdict);
int eccb200_bign_verify_msgs_batch_dev(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *d_sigs,
				       const uint8_t *d_pubkeys, const uint8_t *d_msgs, const uint64_t *d_offsets,
				       const uint8_t *d_adata, const uint64_t *d_adata_offsets, int8_t *d_verdict,
				       void *stream);

/*
 * Batched ECC-CDH shared-secret derivation: ecccdh_derive_secret (src/ecdh/ecccdh.c:167-233) per item — peer key
 * import with on-curve check (src/sig/ec_key.c:181-214), prj_pt_mul(d, Q) (:209), reject infinity (:216-217),
 * export of the affine x coordinate (:220-224).
 *   privkeys : n * qlen;  peer_pubkeys : n * 2*plen affine;  shared : n * plen (x coordinate);  status OK / ERR
 */
int eccb200_ecccdh_derive_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *privkeys, const uint8_t *peer_pubkeys,
				uint8_t *shared, int8_t *status);
int eccb200_ecccdh_derive_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_privkeys,
				    const uint8_t *d_peer_pubkeys, uint8_t *d_shared, int8_t *d_status, void *stream);

/*
 * Hashing of short messages on the device (SHA-256 / SHA-384 / SHA-512 and SHA3-224 / 256 / 384 / 512; hash_type =
 * the reference's hash_alg_type value: 2, 3, 4 and 5 .. 8 — src/lib_ecc_types.h:82-).  Replaces hfunc_scattered of the matching hash_mapping
 * (src/hash/hash_algs.h:232-241; sha256_scattered src/hash/sha256.c:201) for a batch: message i is
 * msgs[offsets[i] .. offsets[i+1]), offsets has n+1 entries, digests is [n][digest_size].
 */
int eccb200_hash_batch(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *msgs, const uint64_t *offsets,
		       uint8_t *digests);

/* ECDSA verification of raw messages: eccb200_hash_batch + eccb200_ecdsa_verify_batch fused on the device, i.e. the
 * whole of ec_verify(…, ECDSA, hash_type, NULL, 0) (src/sig/sig_algs.c:655) per item. */
int eccb200_ecdsa_verify_msgs_batch(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *sigs,
				    const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *offsets,
				    int8_t *verdict);

/* Same on device-resident buffers (d_offsets: n + 1 entries starting at 0, non-decreasing; d_digests: [n][digest_size]
 * scratch), hash kernel + verification kernel enqueued on `stream`; asynchronous. */
int eccb200_ecdsa_verify_msgs_batch_dev(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *d_sigs,
					const uint8_t *d_pubkeys, const uint8_t *d_msgs, const uint64_t *d_offsets,
					uint8_t *d_digests, int8_t *d_verdict, void *stream);
/*
 * Batched Schnorr-family signing of raw messages, hashed on the device.  The hash these schemes sign covers the point
 * W = k*G, so it runs after the scalar multiplication: k*G (comb), batched normalisation, then one kernel per item that
 * hashes W with the message and computes s = k + e*x mod q, with e the WHOLE digest reduced mod q:
 *   ECCB200_ALG_ECSDSA  r = H(W_x || W_y || m), e = OS2I(r) mod q;  sig r || s, hsize + qlen bytes
 *   ECCB200_ALG_ECOSDSA r = H(W_x || m), e = OS2I(r) mod q;         sig r || s, hsize + qlen bytes
 *                       (__ecsdsa_sign_init / _finalize, src/sig/ecsdsa_common.c:141-399)
 *   ECCB200_ALG_ECFSDSA e = H(W_x || W_y || m) mod q;               sig W_x || W_y || s, 2*plen + qlen bytes
 *                       (src/sig/ecfsdsa.c:120-356)
 *   ECCB200_ALG_BIP0340 k = H_nonce(t || P_x || m) mod q with t = x' XOR H_aux(a), e = H_challenge(R_x || P_x || m)
 *                       mod q, x and k negated when y(P) resp. y(R) is odd;  sig R_x || s, plen + qlen bytes
 *                       (_bip0340_sign, src/sig/bip0340.c:45-101, 161-371)
 *   privkeys   : n * qlen bytes, x in [1, q-1] (else ECCB200_ERR)
 *   randomness : n * qlen bytes, what the reference's `rand` callback would return (_ec_sign, src/sig/sig_algs.c:473):
 *                the nonce k in [1, q-1] (else ECCB200_ERR) for ECSDSA / ECOSDSA / ECFSDSA, the auxiliary value a
 *                (drawn below 2^(8*qlen), src/sig/bip0340.c:248-254) for BIP0340
 *   pubkeys    : n * 2*plen affine, BIP0340 only (NULL allowed otherwise): P_x and the parity of P_y are taken from it
 *                as the reference takes them from the key pair, without checking P = x*G; off the curve: ECCB200_ERR
 *   msgs / offsets : message i is msgs[offsets[i] .. offsets[i+1]), offsets has n + 1 entries, starts at 0 and never
 *                decreases (checked here; the _dev form does not re-check it)
 *   hash_type  : 2 .. 8 (SHA256, SHA384, SHA512, SHA3_224 .. SHA3_512)
 *   sigs       : [n][siglen], zero unless status is OK
 *   status     : ECCB200_OK / ECCB200_ERR / ECCB200_RETRY (the reference would fail or restart and fresh randomness
 *                would succeed: e == 0 or s == 0 for ECSDSA / ECOSDSA, s == 0 for ECFSDSA, a derived k == 0 for BIP0340)
 * An unsupported sig_type or hash_type returns -1 (eccb200_last_error).  The _dev form follows the rules of every
 * *_dev entry point (one scratch set per context, calls chained across streams; 16-byte alignment of the privkey,
 * pubkey, randomness and signature buffers on the 256/384/512-bit curves, not of d_msgs).
 * NOTE: like every entry point of this library this is a throughput path, NOT a constant-time one.
 */
#define ECCB200_ALG_ECSDSA 3
#define ECCB200_ALG_ECOSDSA 4
#define ECCB200_ALG_ECFSDSA 5
#define ECCB200_ALG_BIP0340 20
int eccb200_schnorr_sign_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
				    const uint8_t *privkeys, const uint8_t *pubkeys, const uint8_t *randomness,
				    const uint8_t *msgs, const uint64_t *offsets, uint8_t *sigs, int8_t *status);
int eccb200_schnorr_sign_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
					const uint8_t *d_privkeys, const uint8_t *d_pubkeys,
					const uint8_t *d_randomness, const uint8_t *d_msgs,
					const uint64_t *d_offsets, uint8_t *d_sigs, int8_t *d_status, void *stream);

/*
 * Batched ECKCDSA / ECGDSA / ECRDSA / SM2 signing of raw messages, hashed on the device: k*G (comb), batched
 * normalisation, then one kernel that hashes and computes r and s per item.  W = k*G affine, x the private scalar, k
 * the caller's nonce (what the reference's `rand` callback would return), each scheme as the reference's default build:
 *   ECCB200_ALG_ECKCDSA h = H(z || m), z the first block-size bytes of Y_x || Y_y (zero-padded or cut);
 *                       r = H(W_x); both keep their rightmost r_len = min(hsize, qlen) bytes; e = OS2I(r XOR h) mod q;
 *                       s = x*(k - e) mod q;  sig r || s, r_len + qlen bytes    (src/sig/eckcdsa.c:202-471)
 *   ECCB200_ALG_ECGDSA  e = -(leftmost bitlen(q) bits of H(m)) mod q, r = W_x mod q, s = x*(k*r + e) mod q;
 *                       sig r || s, 2*qlen bytes                                 (src/sig/ecgdsa.c:181-347)
 *   ECCB200_ALG_ECRDSA  e = OS2I(byte-reversed H(m)) mod q, 0 replaced by 1, r = W_x mod q, s = r*x + k*e mod q;
 *                       sig r || s, 2*qlen bytes                                 (src/sig/ecrdsa.c:196-346)
 *   ECCB200_ALG_SM2     Z = H(ENTL || ID || a || b || G_x || G_y || Y_x || Y_y), e = OS2I(H(Z || m)),
 *                       r = (e + W_x) mod q, s = (1 + x)^-1 * (k - r*x) mod q;  sig r || s, 2*qlen bytes
 *                       (src/sig/sm2.c:136-455; like the reference, no restart on r + k == q)
 *   privkeys   : n * qlen bytes, x in [1, q-1], for SM2 in [1, q-2] (else ECCB200_ERR)
 *   pubkeys    : n * 2*plen affine, ECKCDSA and SM2 only (ignored otherwise): Y enters z / Z as given, without a check
 *                against x; off the curve: ECCB200_ERR
 *   nonces     : n * qlen bytes, k in [1, q-1] (else ECCB200_ERR)
 *   msgs / offsets : message i is msgs[offsets[i] .. offsets[i+1]), offsets has n + 1 entries, starts at 0 and never
 *                decreases (checked here; the _dev form does not re-check it)
 *   ids / id_offsets : SM2 only (ignored otherwise), the same layout: item i's ID is ids[id_offsets[i] ..
 *                id_offsets[i+1]), at most 8191 bytes (SM2_MAX_ID_LEN; checked here, an ECCB200_ERR item in the _dev
 *                form); an empty ID is valid
 *   hash_type  : 2 .. 8 (SHA256, SHA384, SHA512, SHA3_224 .. SHA3_512) or 11 (SM3); only these two entry points take SM3
 *   sigs       : [n][eccb200_sign_sig_len], zero unless status is OK
 *   status     : ECCB200_OK / ECCB200_ERR / ECCB200_RETRY (the reference would restart and a fresh nonce would succeed:
 *                r == 0 for ECGDSA / ECRDSA / SM2, s == 0 for all four)
 * Any other sig_type (the Schnorr family and ECDSA have their own entry points), any other hash_type, or SM2 without
 * ids, or ECKCDSA / SM2 without pubkeys, returns -1 (eccb200_last_error) and writes nothing.  The _dev form follows the
 * rules of every *_dev entry point (one scratch set per context, calls chained across streams; 16-byte alignment of
 * the privkey, pubkey, nonce and signature buffers on the 256/384/512-bit curves, not of d_msgs or d_ids).
 * NOTE: like every entry point of this library this is a throughput path, NOT a constant-time one.
 */
#define ECCB200_ALG_ECKCDSA 2
#define ECCB200_ALG_ECGDSA 6
#define ECCB200_ALG_ECRDSA 7
#define ECCB200_ALG_SM2 8
#define ECCB200_HASH_SM3 11
int eccb200_sign_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *privkeys,
			    const uint8_t *pubkeys, const uint8_t *nonces, const uint8_t *msgs, const uint64_t *offsets,
			    const uint8_t *ids, const uint64_t *id_offsets, uint8_t *sigs, int8_t *status);
int eccb200_sign_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *d_privkeys,
				const uint8_t *d_pubkeys, const uint8_t *d_nonces, const uint8_t *d_msgs,
				const uint64_t *d_offsets, const uint8_t *d_ids, const uint64_t *d_id_offsets,
				uint8_t *d_sigs, int8_t *d_status, void *stream);
/* Signature length in bytes of eccb200_sign_msgs_batch on this context's curve, or -1 (unsupported sig_type / hash). */
int eccb200_sign_sig_len(eccb200_ctx *ctx, int sig_type, int hash_type);

/*
 * Batched ECKCDSA / ECSDSA / ECOSDSA / ECGDSA / ECRDSA / SM2 verification of raw messages, hashed on the device: one
 * kernel for the signature checks, the hash and the mod-q scalars a, b; the double-scalar kernel W' = a*G + b*Y (as
 * eccb200_double_smul_batch); one kernel for the acceptance test.  Y is the public key, each scheme as the reference's
 * default build (ec_verify with the SM2 ID as ancillary data):
 *   ECCB200_ALG_ECSDSA / _ECOSDSA  sig r || s, hsize + qlen bytes; s in ]0, q[, e = -(OS2I(r) mod q) != 0; a = s, b = e;
 *                       accept iff H(W'_x || W'_y || m) (ECOSDSA: H(W'_x || m)) == r   (src/sig/ecsdsa_common.c:425-609)
 *   ECCB200_ALG_ECKCDSA sig r || s, min(hsize, qlen) + qlen bytes; s in ]0, q[, z the first block-size bytes of
 *                       Y_x || Y_y (zero-padded or cut), e = OS2I(r XOR rightmost(H(z || m))) mod q; a = e, b = s;
 *                       accept iff the rightmost r_len bytes of H(W'_x) == r            (src/sig/eckcdsa.c:543-832)
 *   ECCB200_ALG_ECGDSA  sig r || s, 2*qlen bytes; r, s in ]0, q[, e = leftmost bitlen(q) bits of H(m); a = r^-1 e,
 *                       b = r^-1 s; accept iff W'_x mod q == r                           (src/sig/ecgdsa.c:413-600)
 *   ECCB200_ALG_ECRDSA  sig r || s, 2*qlen bytes; r, s in ]0, q[, h = OS2I(byte-reversed H(m)) mod q, 0 replaced by 1;
 *                       a = h^-1 s, b = -h^-1 r; accept iff W'_x mod q == r (not the ISO 14888-3 variant, which
 *                       hashes without the byte reversal)                                (src/sig/ecrdsa.c:417-600)
 *   ECCB200_ALG_SM2     sig r || s, 2*qlen bytes; r, s in ]0, q[, t = r + s mod q != 0; a = s, b = t; accept iff
 *                       (OS2I(H(Z || m)) + W'_x) mod q == r, Z as in eccb200_sign_msgs_batch  (src/sig/sm2.c:518-700)
 *   W' at infinity is invalid in every scheme.
 *   sigs       : [n][siglen] with the lengths above (eccb200_sign_sig_len gives them for ECKCDSA / ECGDSA / ECRDSA /
 *                SM2 only)
 *   pubkeys    : n * 2*plen affine, every scheme; a key off the curve makes that item invalid
 *   msgs / offsets, ids / id_offsets : as eccb200_sign_msgs_batch (the offsets are checked in the host form only); ids
 *                are required for SM2 and ignored otherwise; an SM2 ID longer than 8191 bytes makes that item invalid
 *                (the reference's sm2_compute_Z fails on it), in both forms
 *   hash_type  : 2 .. 8 or 11 (SM3), for all six schemes
 *   verdict    : per item 0 (valid) or -1 (invalid, or any error such as a key off the curve)
 * Any other sig_type (ECDSA, ECFSDSA and BIP0340 have their own entry points), any other hash_type, or SM2 without ids
 * returns -1 (eccb200_last_error) and writes nothing.  The _dev form follows the rules of every *_dev entry point (one
 * scratch set per context, calls chained across streams; 16-byte alignment of d_sigs and d_pubkeys on the
 * 256/384/512-bit curves, not of d_msgs or d_ids).
 * NOTE: like every entry point of this library this is a throughput path, NOT a constant-time one.
 */
int eccb200_verify_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *sigs,
			      const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *offsets, const uint8_t *ids,
			      const uint64_t *id_offsets, int8_t *verdict);
int eccb200_verify_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *d_sigs,
				  const uint8_t *d_pubkeys, const uint8_t *d_msgs, const uint64_t *d_offsets,
				  const uint8_t *d_ids, const uint64_t *d_id_offsets, int8_t *d_verdict, void *stream);

/* cudaMemcpy device -> host (for callers that do not link the CUDA runtime). */
int eccb200_copy_to_host(eccb200_ctx *ctx, void *host_dst, const void *d_src, size_t bytes);

/*
 * ECFSDSA verification (SURVEY.md §8f.4: the Schnorr-type scheme for which the reference ships a verify_batch,
 * src/sig/ecfsdsa.c:711-1074), per item like ec_verify(…, ECFSDSA, …) (src/sig/ecfsdsa.c:416-610):
 * sigs [n][2*plen + qlen] = r || s with r = W_x || W_y, digests[i] = H(r_i || m_i) (the whole digest is
 * reduced mod q, whatever its length), pubkeys as for ECDSA.  verdict 0 / -1.  The same comb + signed-window kernel as ECDSA, without
 * the inversion mod q.
 */
int eccb200_ecfsdsa_verify_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
				 const uint8_t *digests, uint32_t hlen, int8_t *verdict);
int eccb200_ecfsdsa_verify_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
				     const uint8_t *d_digests, uint32_t hlen, int8_t *d_verdict, void *stream);

/*
 * ECFSDSA batch verification in the form the reference's verify_batch slot computes it (_ecfsdsa_verify_batch,
 * src/sig/ecfsdsa.c:814-1055): ONE random linear combination for the whole batch,
 *        (sum a_i s_i) G  +  sum a_i (-W_i)  +  sum (-a_i e_i) Y_i  ==  point at infinity,
 * where the reference feeds its 2n+1 terms to the Bos-Coster heap (src/sig/sig_algs.c:1052) and this library runs them as
 * a multi-scalar multiplication with the bucket method on the device (K6, libecc_b200/csrc/msm.cuh): ~26 mixed additions
 * per signature instead of a full double-scalar multiplication.  Inputs as eccb200_ecfsdsa_verify_batch.
 *   *all_valid = 1 iff every item is well formed (W_i and Y_i on the curve, s_i < q - the checks of the reference's loop,
 *                :881-921, :941, :983) and the combination vanishes; 0 otherwise (an empty batch: 0, as :740).  Like the
 *                reference's function this says nothing about WHICH signature is bad - eccb200_ecfsdsa_verify_batch does -
 *                and a batch holding a forgery passes with probability 2^-128 (the coefficients a_i are 128 bits of a
 *                ChaCha20 stream keyed by `seed`).
 *   seed       : 32 bytes the signers cannot predict; NULL draws them from the operating system (getrandom).  A fixed
 *                seed makes the call reproducible (tests).
 * Returns 0 when the verification ran (whatever the verdict), -1 on an error (eccb200_last_error).
 */
int eccb200_ecfsdsa_verify_msm_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
				     const uint8_t *digests, uint32_t hlen, const uint8_t *seed, int *all_valid);
int eccb200_ecfsdsa_verify_msm_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
					 const uint8_t *d_digests, uint32_t hlen, const uint8_t *seed, int *all_valid,
					 void *stream);

/*
 * The same for BIP0340 (the reference's _bip0340_verify_batch, src/sig/bip0340.c:1040-1290): inputs as
 * eccb200_bip0340_verify_batch (sigs [n][plen + qlen] = r || s, digests = the tagged challenge hashes).  The points R_i are
 * lifted from r_i on the device (even y, src/sig/bip0340.c:1188-1196: one exponentiation per signature, p = 3 mod 4) and the
 * keys taken at their even-y representative; a batch with an r_i that is no x coordinate of the curve is rejected, as
 * aff_pt_y_from_x fails in the reference.  -1 on SECP224R1 (p = 1 mod 4: use eccb200_bip0340_verify_batch).
 */
int eccb200_bip0340_verify_msm_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
				     const uint8_t *digests, uint32_t hlen, const uint8_t *seed, int *all_valid);
int eccb200_bip0340_verify_msm_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
					 const uint8_t *d_digests, uint32_t hlen, const uint8_t *seed, int *all_valid,
					 void *stream);

/*
 * Batched double-scalar multiplication W_i = a_i*G + b_i*Y_i with affine results: the sequence prj_pt_mul, prj_pt_mul,
 * prj_pt_add, prj_pt_unique that every Schnorr-type verification of the reference runs before it hashes the recomputed
 * point (ECSDSA / ECOSDSA src/sig/ecsdsa_common.c:493-497, ECKCDSA, ...), as ONE kernel launch per batch: comb for G,
 * signed window for Y, shared inversions.  The hashing of W' stays with the caller (src/hash).
 *   ab      : n * 2*qlen bytes a || b, any values (reduced mod q like the reference's ladder)
 *   pubkeys : n * 2*plen bytes affine x || y;  out : n * 2*plen bytes affine W (zero unless status is OK)
 *   status  : ECCB200_OK / ECCB200_INFINITY (prj_pt_unique would fail) / ECCB200_ERR (key not on the curve)
 */
int eccb200_double_smul_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *ab, const uint8_t *pubkeys, uint8_t *out,
			      int8_t *status);
int eccb200_double_smul_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_ab, const uint8_t *d_pubkeys,
				  uint8_t *d_out, int8_t *d_status, void *stream);

/*
 * BIP0340 (Schnorr over x-only keys) verification, per item like ec_verify(…, BIP0340, …)
 * (src/sig/bip0340.c:383-577): sigs [n][plen + qlen] = r || s with r a field element < p and s < q; pubkeys affine
 * x || y as for ECDSA (the kernel lifts the key to its even-y representative, :540-545); digests[i] = the tagged hash
 * H(H("BIP0340/challenge") || H("BIP0340/challenge") || r_i || x(Y_i) || m_i) computed by the host with src/hash (the
 * whole digest is reduced mod q).  The same comb + signed-window kernel as ECDSA (SCHEME = 2), plus one shared
 * inversion for the affine W' (the scheme tests the parity of y(W')).  verdict 0 / -1.
 */
int eccb200_bip0340_verify_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
				 const uint8_t *digests, uint32_t hlen, int8_t *verdict);
int eccb200_bip0340_verify_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
				     const uint8_t *d_digests, uint32_t hlen, int8_t *d_verdict, void *stream);

/*
 * The reference's structured key / signature records (SURVEY.md §8f.2), batched.  `alg` is the reference's
 * ec_alg_type (ECDSA = 1, DECDSA = 14; src/lib_ecc_types.h:22-), `hash_type` its hash_alg_type; the third header byte
 * is the context's curve id.
 *   structured public key   [0][alg][curve] X || Y || Z   3 + 3*plen bytes  (src/sig/ec_key.c:451-497)
 *   structured private key  [1][alg][curve] x             3 + priv_len bytes, priv_len >= qlen
 *                                                          (src/sig/ec_key.c:358-408; EC_PRIV_KEY_EXPORT_SIZE
 *                                                          src/sig/ec_key.h:75-83 is 64 or 66 in the default build)
 *   structured signature    [alg][hash][curve] r || s     3 + 2*qlen bytes  (src/sig/sig_algs.c:742-790)
 */
#define ECCB200_ALG_ECDSA 1
#define ECCB200_ALG_DECDSA 14

/* ec_structured_pub_key_import_from_buf (src/sig/ec_key.c:410-449) -> affine keys [n][2*plen] for the verify entry
 * points.  status: 0 ok, 1 the key is the point at infinity (the reference accepts that import), -1 rejected (header,
 * coordinate >= p, not on the curve: prj_pt_import_from_buf src/curves/prj_pt.c:462-500). */
int eccb200_structured_pub_key_import_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *records, int alg,
					    uint8_t *pubkeys, int8_t *status);

/* ec_structured_pub_key_export_to_buf (src/sig/ec_key.c:451-497) of affine keys; Z is written as 1. */
int eccb200_structured_pub_key_export_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *pubkeys, int alg,
					    uint8_t *records);

/* ec_structured_key_pair_import_from_priv_key_buf (src/sig/ec_key.c:499-545: header check, x < q
 * src/sig/ecdsa_common.c:188, Y = x*G :193) followed by the structured export of the public half.
 * status: 0 ok, 1 x = 0 (Y at infinity), -1 rejected. */
int eccb200_structured_key_pair_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *priv_records, uint32_t priv_len,
				      int alg, uint8_t *pub_records, int8_t *status);

/* ec_structured_sig_import_from_buf (src/sig/sig_algs.c:702-740) + ec_structured_pub_key_import_from_buf +
 * ec_verify on pre-hashed messages, per item; verdict 0 / -1 like eccb200_ecdsa_verify_batch. */
int eccb200_ecdsa_verify_structured_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sig_records,
					  const uint8_t *pub_records, int alg, int hash_type, const uint8_t *digests,
					  uint32_t hlen, int8_t *verdict);

/* eccb200_ecdsa_sign_batch on structured private keys, producing structured signatures
 * (ec_structured_sig_export_to_buf src/sig/sig_algs.c:742-790). */
int eccb200_ecdsa_sign_structured_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *priv_records, uint32_t priv_len,
					int alg, int hash_type, const uint8_t *nonces, const uint8_t *digests,
					uint32_t hlen, uint8_t *sig_records, int8_t *status);

/* The chunking rule of the host-pointer pipeline as a pure function (no GPU needed; unit-tested on the CPU): chunk
 * boundaries 0 = b[0] < ... < b[k] = n for a batch of n items, given the items of one kernel wave, the equal-chunk size,
 * the capacity of the stage buffers and whether the ramp-up / ramp-down shaping applies (fixed-base pipelines).  Writes
 * at most cap boundaries, returns their number (k + 1). */
int eccb200_pipeline_chunk_bounds(uint32_t n, uint32_t wave_items, uint32_t equal_chunk_items, uint32_t capacity_items,
				  int shaped, uint32_t *bounds, int cap);

/* Binds the calling host thread to the CPUs local to `device` (its PCI device's local_cpulist): page-locked memory
 * the thread allocates afterwards and the copies it performs stay on the GPU's NUMA node.  Returns the number of CPUs
 * bound to, 0 if nothing was changed, -1 on error.  The multi-device calls do this for their worker threads. */
int eccb200_bind_thread_near_device(int device);

/* Page-locked host memory for the host-pointer entry points (wrappers of cudaHostAlloc / cudaFreeHost so that a C
 * caller need not link the CUDA runtime).  NULL on failure. */
void *eccb200_host_alloc(size_t bytes);
void *eccb200_host_alloc_input(size_t bytes); /* write-combined: for buffers the host only writes (batch inputs) */
void eccb200_host_free(void *p);

/* Field-level entry point used by the arithmetic unit tests (pattern: src/arithmetic_tests FP_MUL_MONTY):
 * out[i] = a[i]*b[i]*R^-1 mod p (which = 0) or mod q (which = 1), R = 2^(8*plen); inputs must be < modulus. */
int eccb200_fp_mul_monty_batch(eccb200_ctx *ctx, int which, uint32_t n, const uint8_t *a, const uint8_t *b,
			       uint8_t *out);

/* The same pattern for FP_ADD / FP_SUB / FP_SQR_MONTY (src/fp/fp_montgomery.c:26,35,53): op 0 = a + b, 1 = a - b,
 * 2 = a*a*R^-1 (b ignored), mod p (which = 0) or mod q (1). */
int eccb200_fp_addsub_batch(eccb200_ctx *ctx, int which, int op, uint32_t n, const uint8_t *a, const uint8_t *b,
			    uint8_t *out);

/* Mod-q scalar preparation of ECDSA verification alone (nn_modinv / nn_mod_mul on the order q,
 * src/sig/ecdsa_common.c:777-791): out[i] = u || v, u = e*s^-1 mod q, v = r*s^-1 mod q, 2*qlen bytes big-endian.
 * s must be in [1, q-1].  Unit-test entry point. */
int eccb200_ecdsa_uv_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *digests, uint32_t hlen,
			   uint8_t *out);

/* Per-kernel device timing of the device-pointer entry points (CUDA events recorded on the caller's stream around
 * each kernel).  eccb200_profile_read waits for the timed calls issued since the previous read (up to 64), sums their
 * durations per kernel position and returns how many values (ms) it wrote:
 * prj_pt_mul_batch_dev -> [scalar-mult kernel, batched normalisation]; ecdsa_verify_batch_dev -> [verify kernel]. */
int eccb200_profile_enable(eccb200_ctx *ctx, int on);
int eccb200_profile_read(eccb200_ctx *ctx, float *ms, int cap);

/* Layout experiment behind DESIGN.md §3: `iters` dependent Montgomery products per element with the production
 * one-thread-per-element multiplier (striped = 0) or with the words of an element striped over 8 lanes and
 * __shfl_sync carries (striped = 1; 256-bit curves).  Results are identical; *ms is the kernel time. */
int eccb200_fp_mul_chain_bench(eccb200_ctx *ctx, int striped, uint32_t n, const uint8_t *a, const uint8_t *b,
			       uint8_t *out, int iters, float *ms);

/* imad_peak micro-benchmark: measured 32x32+64 integer multiply-add throughput of the device (IMAD32 per second) —
 * the denominator of the roofline for this integer-MAD-bound path (SURVEY.md §8d) — and the same figure per clock
 * per SM at the device's nominal maximum SM clock. */
int eccb200_imad_peak(int device, double *imad32_per_s, double *imad_per_clk_per_sm);

/* Introspection for bench.py / tests. */
int eccb200_comb_window(const eccb200_ctx *ctx);
uint64_t eccb200_kernel_launches(const eccb200_ctx *ctx);  /* kernels launched by this context so far */
const char *eccb200_last_error(void);                      /* thread-local message for the last -1 */

#ifdef __cplusplus
}
#endif
#endif
