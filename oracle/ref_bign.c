/*
 * oracle/ref_bign.c — the reference's BIGN / DBIGN signer with injected BIGN nonces and per-item adata records, its
 * ec_verify for BIGN, and its BELT block cipher, BELT-HASH and BASH hashes, as flat batch wrappers.
 *
 * TEST INFRASTRUCTURE ONLY.  Compiled against the reference's headers and linked to oracle/_ref/libecc_ref.so (the
 * unmodified reference, oracle/Makefile) into oracle/_ref/libecc_ref_bign.so by oracle/ref_bign.mk.  It contains no
 * arithmetic of its own: every signature, verdict and digest comes from the reference.  Only tests/ and tools/ load it.
 *
 * Reference entry points used (paths relative to /root/reference/src):
 *   _ec_sign, ec_verify, ec_get_sig_len  sig/sig_algs.c     ec_key_pair_import_from_priv_key_buf  sig/ec_key.c
 *   ec_pub_key_export_to_aff_buf, ec_pub_key_import_from_aff_buf  sig/ec_key.c
 *   belt_init, belt_encrypt, belt_hash   hash/belt-hash.c   get_hash_by_name, hfunc_scattered    hash/hash_algs.c
 */
#include "libsig.h"
#include "hash/belt-hash.h"
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
	ec_params params;
	u32 plen, qlen;
} curve_t;

typedef struct {
	const curve_t *c;
	ec_alg_type alg;
	hash_alg_type ht;
	u32 siglen;
	uint32_t lo, hi;
	const uint8_t *privkeys, *nonces, *sigs, *pubkeys, *msgs, *adata;
	const uint64_t *off, *adata_off;
	uint8_t *sigs_out, *pubkeys_out;
	int8_t *out;
} job_t;

static int load_curve(curve_t *c, const char *name)
{
	const ec_str_params *sp = NULL;
	size_t l = strlen(name);
	if (l > 250) return -1;
	if (ec_get_curve_params_by_name((const u8 *)name, (u8)(l + 1), &sp) || sp == NULL) return -1;
	if (import_params(&c->params, sp)) return -1;
	c->plen = (u32)BYTECEIL(c->params.ec_fp.p_bitlen);
	c->qlen = (u32)BYTECEIL(c->params.ec_gen_order_bitlen);
	return 0;
}

/* BIGN's `rand` callback returns item i's nonce; 0 and values >= q are refused (the signature then fails). */
static __thread const uint8_t *tl_nonce;
static __thread uint32_t tl_nonce_len;

static int nonce_from_item(nn_t out, nn_src_t bound)
{
	int cmp = 0, iszero = 0;
	if (nn_init_from_buf(out, tl_nonce, (u16)tl_nonce_len) || nn_cmp(out, bound, &cmp) || nn_iszero(out, &iszero))
		return -1;
	return (cmp >= 0 || iszero) ? -1 : 0;
}

static void *sign_worker(void *arg)
{
	job_t *j = (job_t *)arg;
	const curve_t *c = j->c;
	for (uint32_t i = j->lo; i < j->hi; i++) {
		ec_key_pair kp;
		nn x;
		int cmp = 0, iszero = 1;
		const uint8_t *xb = j->privkeys + (size_t)i * c->qlen;
		uint8_t *sig = j->sigs_out + (size_t)i * j->siglen;
		const uint64_t adlen = j->adata_off[i + 1] - j->adata_off[i];
		memset(sig, 0, j->siglen);
		memset(j->pubkeys_out + (size_t)i * 2 * c->plen, 0, 2 * c->plen);
		j->out[i] = -1;
		if (nn_init_from_buf(&x, xb, (u16)c->qlen) || nn_iszero(&x, &iszero) ||
		    nn_cmp(&x, &c->params.ec_gen_order, &cmp) || iszero || cmp >= 0)
			continue;
		if (ec_key_pair_import_from_priv_key_buf(&kp, &c->params, xb, (u8)c->qlen, j->alg) ||
		    ec_pub_key_export_to_aff_buf(&kp.pub_key, j->pubkeys_out + (size_t)i * 2 * c->plen, (u8)(2 * c->plen)))
			continue;
		if (adlen > 0xffff) continue; /* not expressible: the reference's adata_len is a u16 */
		tl_nonce = j->nonces ? j->nonces + (size_t)i * c->qlen : xb;
		tl_nonce_len = c->qlen;
		if (_ec_sign(sig, (u8)j->siglen, &kp, j->msgs + j->off[i], (u32)(j->off[i + 1] - j->off[i]), nonce_from_item,
			     j->alg, j->ht, j->adata + j->adata_off[i], (u16)adlen)) {
			memset(sig, 0, j->siglen);
			continue;
		}
		j->out[i] = 0;
	}
	return NULL;
}

static void *verify_worker(void *arg)
{
	job_t *j = (job_t *)arg;
	const curve_t *c = j->c;
	for (uint32_t i = j->lo; i < j->hi; i++) {
		ec_pub_key pk;
		const uint64_t adlen = j->adata_off[i + 1] - j->adata_off[i];
		j->out[i] = -1;
		if (adlen > 0xffff ||
		    ec_pub_key_import_from_aff_buf(&pk, &c->params, j->pubkeys + (size_t)i * 2 * c->plen, (u8)(2 * c->plen),
						   j->alg))
			continue;
		if (ec_verify(j->sigs + (size_t)i * j->siglen, (u8)j->siglen, &pk, j->msgs + j->off[i],
			      (u32)(j->off[i + 1] - j->off[i]), j->alg, j->ht, j->adata + j->adata_off[i], (u16)adlen))
			continue;
		j->out[i] = 0;
	}
	return NULL;
}

static int run(job_t *p, uint32_t n, int nthreads, void *(*fn)(void *))
{
	if (nthreads < 1) nthreads = 1;
	if ((uint32_t)nthreads > n) nthreads = n ? (int)n : 1;
	pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
	job_t *jobs = (job_t *)calloc((size_t)nthreads, sizeof(job_t));
	for (int t = 0; t < nthreads; t++) {
		jobs[t] = *p;
		jobs[t].lo = (uint32_t)(((uint64_t)n * (uint64_t)t) / (uint64_t)nthreads);
		jobs[t].hi = (uint32_t)(((uint64_t)n * (uint64_t)(t + 1)) / (uint64_t)nthreads);
		pthread_create(&th[t], NULL, fn, &jobs[t]);
	}
	for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
	free(th);
	free(jobs);
	return 0;
}

static int setup(job_t *p, curve_t *c, const char *curve, int dbign, const char *hash)
{
	const hash_mapping *hm = NULL;
	u8 sl = 0;
	memset(p, 0, sizeof(*p));
	if (load_curve(c, curve) || get_hash_by_name(hash, &hm) || hm == NULL) return -1;
	p->alg = dbign ? DBIGN : BIGN;
	p->ht = hm->type;
	if (ec_get_sig_len(&c->params, p->alg, p->ht, &sl)) return -1;
	p->c = c;
	p->siglen = sl;
	return 0;
}

/*
 * Sign message i (msgs[off[i] .. off[i+1])) with private key i under BIGN (dbign = 0; nonces[i], qlen bytes, through
 * the rand callback) or DBIGN (dbign = 1; nonces ignored: _dbign_sign_init sets rand to NULL) and the reference's hash
 * `hash`, with item i's adata record adata[adata_off[i] .. adata_off[i+1]).  Keys outside [1, q-1] are refused before
 * the reference sees them.  pubkeys_out[i] = x*G, affine.  status[i]: 0 signed, -1 refused.
 */
int ref_bign_sign(const char *curve, int dbign, const char *hash, uint32_t n, const uint8_t *privkeys,
		  const uint8_t *nonces, const uint8_t *msgs, const uint64_t *off, const uint8_t *adata,
		  const uint64_t *adata_off, uint8_t *sigs_out, uint8_t *pubkeys_out, int8_t *status, int nthreads)
{
	curve_t c;
	job_t p;
	if (setup(&p, &c, curve, dbign, hash)) return -1;
	p.privkeys = privkeys;
	p.nonces = dbign ? NULL : nonces;
	p.msgs = msgs;
	p.off = off;
	p.adata = adata;
	p.adata_off = adata_off;
	p.sigs_out = sigs_out;
	p.pubkeys_out = pubkeys_out;
	p.out = status;
	return run(&p, n, nthreads, sign_worker);
}

/* ec_verify (BIGN) of signature i over message i with item i's adata record under the affine key i.  verdict[i]: 0
 * valid, -1 invalid or key refused. */
int ref_bign_verify(const char *curve, const char *hash, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
		    const uint8_t *msgs, const uint64_t *off, const uint8_t *adata, const uint64_t *adata_off,
		    int8_t *verdict, int nthreads)
{
	curve_t c;
	job_t p;
	if (setup(&p, &c, curve, 0, hash)) return -1;
	p.sigs = sigs;
	p.pubkeys = pubkeys;
	p.msgs = msgs;
	p.off = off;
	p.adata = adata;
	p.adata_off = adata_off;
	p.out = verdict;
	return run(&p, n, nthreads, verify_worker);
}

/* belt-block encryption of n 16-byte blocks, block i under the 32-byte key i */
int ref_belt_encrypt(uint32_t n, const uint8_t *keys, const uint8_t *in, uint8_t *out)
{
	for (uint32_t i = 0; i < n; i++) {
		u8 ks[BELT_KEY_SCHED_LEN];
		if (belt_init(keys + (size_t)i * 32, 32, ks)) return -1;
		belt_encrypt(in + (size_t)i * 16, out + (size_t)i * 16, ks);
	}
	return 0;
}

/* the reference's hash `hash` (e.g. "BELT_HASH", "BASH256") of one message; digest size or -1 */
int ref_bign_hash(const char *hash, const uint8_t *msg, uint32_t len, uint8_t *out)
{
	const hash_mapping *hm = NULL;
	const u8 *inputs[2] = { msg, NULL };
	const u32 ilens[2] = { len, 0 };
	if (get_hash_by_name(hash, &hm) || hm == NULL) return -1;
	if (hm->hfunc_scattered(inputs, ilens, out)) return -1;
	return hm->digest_size;
}
