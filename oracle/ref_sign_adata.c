/*
 * oracle/ref_sign_adata.c — the reference's ECKCDSA / ECGDSA / ECRDSA / SM2 signer with injected nonces and per-item
 * ancillary data (the SM2 user ID), and ec_verify with the same ancillary data, as flat batch wrappers.  The
 * Schnorr-family counterpart without ancillary data is oracle/ref_sign_rand.c.
 *
 * TEST INFRASTRUCTURE ONLY.  Compiled against the reference's headers and linked to oracle/_ref/libecc_ref.so (the
 * unmodified reference, oracle/Makefile) into oracle/_ref/libecc_ref_sign_adata.so by oracle/ref_sign_adata.mk.  It
 * contains no arithmetic of its own: every signature and verdict comes from the reference's _ec_sign / ec_verify.
 * Only tests/ and tools/ load it.
 *
 * Reference entry points used (paths relative to /root/reference/src):
 *   ec_get_curve_params_by_name  curves/curves.c:25      import_params                      curves/ec_params.c:24
 *   ec_key_pair_import_from_priv_key_buf sig/ec_key.c:289  ec_pub_key_export_to_aff_buf     sig/ec_key.c
 *   _ec_sign                     sig/sig_algs.c:473      ec_get_sig_len                     sig/sig_algs.c
 *   get_hash_by_name             hash/hash_algs.c        ec_verify, ec_pub_key_import_from_aff_buf sig/sig_algs.c, sig/ec_key.c
 */
#include "libsig.h"
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
	const uint8_t *privkeys, *randomness, *msgs, *adata;
	const uint64_t *off, *adata_off;
	uint8_t *sigs_out, *pubkeys_out;
	int8_t *status;
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

static int alg_by_name(const char *name, ec_alg_type *alg)
{
	static const struct { const char *n; ec_alg_type a; } tab[] = {
		{ "ECKCDSA", ECKCDSA }, { "ECGDSA", ECGDSA }, { "ECRDSA", ECRDSA }, { "SM2", SM2 },
	};
	for (unsigned i = 0; i < sizeof(tab) / sizeof(tab[0]); i++)
		if (!strcmp(name, tab[i].n)) {
			*alg = tab[i].a;
			return 0;
		}
	return -1;
}

/* The `rand` callback returns item i's nonce randomness[i] (qlen bytes), the way the reference's self tests inject
 * them (tests/ec_self_tests_core.h).  It keeps the rand contract: it fails for 0 and for a value >= its bound q.  A
 * second call for the same signature is one of the four schemes' "goto restart" cases: it fails, so that the
 * signature fails instead of looping on the same nonce. */
static __thread const uint8_t *tl_rand;
static __thread uint32_t tl_rand_len;
static __thread int tl_rand_refused;
static __thread int tl_rand_calls;

static int rand_from_item(nn_t out, nn_src_t bound)
{
	int cmp = 0;
	if (tl_rand_calls++) return -1;
	if (nn_init_from_buf(out, tl_rand, (u16)tl_rand_len) || nn_cmp(out, bound, &cmp)) return -1;
	if (cmp >= 0) {
		tl_rand_refused = 1;
		return -1;
	}
	return 0;
}

static int rand_nonzero_from_item(nn_t out, nn_src_t bound)
{
	int iszero = 0;
	if (rand_from_item(out, bound)) return -1;
	if (nn_iszero(out, &iszero) || iszero) {
		tl_rand_refused = 1;
		return -1;
	}
	return 0;
}

static void *worker(void *arg)
{
	job_t *j = (job_t *)arg;
	const curve_t *c = j->c;
	for (uint32_t i = j->lo; i < j->hi; i++) {
		ec_key_pair kp;
		nn x;
		int cmp = 0, iszero = 1;
		const uint8_t *xb = j->privkeys + (size_t)i * c->qlen;
		uint8_t *sig = j->sigs_out + (size_t)i * j->siglen;
		memset(sig, 0, j->siglen);
		memset(j->pubkeys_out + (size_t)i * 2 * c->plen, 0, 2 * c->plen);
		j->status[i] = -1;
		if (nn_init_from_buf(&x, xb, (u16)c->qlen) || nn_iszero(&x, &iszero) ||
		    nn_cmp(&x, &c->params.ec_gen_order, &cmp) || iszero || cmp >= 0)
			continue;
		if (ec_key_pair_import_from_priv_key_buf(&kp, &c->params, xb, (u8)c->qlen, j->alg) ||
		    ec_pub_key_export_to_aff_buf(&kp.pub_key, j->pubkeys_out + (size_t)i * 2 * c->plen, (u8)(2 * c->plen)))
			continue;
		tl_rand = j->randomness + (size_t)i * c->qlen;
		tl_rand_len = c->qlen;
		tl_rand_refused = 0;
		tl_rand_calls = 0;
		/* SM2 needs an ID (sm2_compute_Z refuses NULL): the empty one when the caller gives none */
		const u8 *ad = j->adata ? j->adata + j->adata_off[i] : (j->alg == SM2 ? (const u8 *)"" : NULL);
		const u16 adlen = j->adata ? (u16)(j->adata_off[i + 1] - j->adata_off[i]) : 0;
		if (_ec_sign(sig, (u8)j->siglen, &kp, j->msgs + j->off[i], (u32)(j->off[i + 1] - j->off[i]),
			     rand_nonzero_from_item, j->alg, j->ht, ad, adlen)) {
			memset(sig, 0, j->siglen);
			j->status[i] = tl_rand_refused ? -1 : 2;
			continue;
		}
		j->status[i] = 0;
	}
	return NULL;
}

/*
 * Sign message i (msgs[off[i] .. off[i+1])) with private key i under alg ("ECKCDSA", "ECGDSA", "ECRDSA", "SM2") and
 * hash (the reference's hash name), the reference's rand callback returning randomness[i], and item i's ancillary
 * data adata[adata_off[i] .. adata_off[i+1]) (adata == NULL: none; SM2 then signs with the empty ID).  Keys outside
 * [1, q-1] are refused before the reference sees them (the reference's SM2 key pair also refuses q-1).
 * pubkeys_out[i] = the scheme's public key, affine (x*G, or x^-1*G for ECKCDSA and ECGDSA).  status[i]: 0 signed;
 * -1 key refused or nonce refused; 2 the reference failed on valid inputs, i.e. one of its "restart with a fresh
 * nonce" cases (r == 0, s == 0).
 */
int ref_sig_sign_with_randomness_adata(const char *curve, const char *alg_name, const char *hash, uint32_t n,
				       const uint8_t *privkeys, const uint8_t *randomness, const uint8_t *msgs,
				       const uint64_t *off, const uint8_t *adata, const uint64_t *adata_off,
				       uint8_t *sigs_out, uint8_t *pubkeys_out, int8_t *status, int nthreads)
{
	curve_t c;
	job_t p;
	const hash_mapping *hm = NULL;
	u8 sl = 0;
	memset(&p, 0, sizeof(p));
	if (load_curve(&c, curve) || alg_by_name(alg_name, &p.alg)) return -1;
	if (get_hash_by_name(hash, &hm) || hm == NULL) return -1;
	p.ht = hm->type;
	if (ec_get_sig_len(&c.params, p.alg, p.ht, &sl)) return -1;
	p.c = &c;
	p.siglen = sl;
	p.privkeys = privkeys;
	p.randomness = randomness;
	p.msgs = msgs;
	p.off = off;
	p.adata = adata;
	p.adata_off = adata_off;
	p.sigs_out = sigs_out;
	p.pubkeys_out = pubkeys_out;
	p.status = status;
	if (nthreads < 1) nthreads = 1;
	if ((uint32_t)nthreads > n) nthreads = n ? (int)n : 1;
	pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
	job_t *jobs = (job_t *)calloc((size_t)nthreads, sizeof(job_t));
	for (int t = 0; t < nthreads; t++) {
		jobs[t] = p;
		jobs[t].lo = (uint32_t)(((uint64_t)n * (uint64_t)t) / (uint64_t)nthreads);
		jobs[t].hi = (uint32_t)(((uint64_t)n * (uint64_t)(t + 1)) / (uint64_t)nthreads);
		pthread_create(&th[t], NULL, worker, &jobs[t]);
	}
	for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
	free(th);
	free(jobs);
	return 0;
}

typedef struct {
	const curve_t *c;
	ec_alg_type alg;
	hash_alg_type ht;
	u32 siglen;
	uint32_t lo, hi;
	const uint8_t *sigs, *pubkeys, *msgs, *adata;
	const uint64_t *off, *adata_off;
	int8_t *verdict;
} verify_job_t;

static void *verify_worker(void *arg)
{
	verify_job_t *j = (verify_job_t *)arg;
	const curve_t *c = j->c;
	for (uint32_t i = j->lo; i < j->hi; i++) {
		ec_pub_key pk;
		j->verdict[i] = -1;
		if (ec_pub_key_import_from_aff_buf(&pk, &c->params, j->pubkeys + (size_t)i * 2 * c->plen,
						   (u8)(2 * c->plen), j->alg))
			continue;
		const u8 *ad = j->adata ? j->adata + j->adata_off[i] : NULL;
		const u16 adlen = j->adata ? (u16)(j->adata_off[i + 1] - j->adata_off[i]) : 0;
		if (ec_verify(j->sigs + (size_t)i * j->siglen, (u8)j->siglen, &pk, j->msgs + j->off[i],
			      (u32)(j->off[i + 1] - j->off[i]), j->alg, j->ht, ad, adlen))
			continue;
		j->verdict[i] = 0;
	}
	return NULL;
}

/* ec_verify of signature i over message i with item i's ancillary data adata[adata_off[i] .. adata_off[i+1]) (the
 * SM2 ID) under the affine public key i.  verdict[i]: 0 valid, -1 invalid or key refused. */
int ref_sig_verify_adata_batch(const char *curve, const char *alg_name, const char *hash, uint32_t n,
			       const uint8_t *sigs, const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *off,
			       const uint8_t *adata, const uint64_t *adata_off, int8_t *verdict, int nthreads)
{
	curve_t c;
	verify_job_t p;
	const hash_mapping *hm = NULL;
	u8 sl = 0;
	memset(&p, 0, sizeof(p));
	if (load_curve(&c, curve) || alg_by_name(alg_name, &p.alg)) return -1;
	if (get_hash_by_name(hash, &hm) || hm == NULL) return -1;
	p.ht = hm->type;
	if (ec_get_sig_len(&c.params, p.alg, p.ht, &sl)) return -1;
	p.c = &c;
	p.siglen = sl;
	p.sigs = sigs;
	p.pubkeys = pubkeys;
	p.msgs = msgs;
	p.off = off;
	p.adata = adata;
	p.adata_off = adata_off;
	p.verdict = verdict;
	if (nthreads < 1) nthreads = 1;
	if ((uint32_t)nthreads > n) nthreads = n ? (int)n : 1;
	pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
	verify_job_t *jobs = (verify_job_t *)calloc((size_t)nthreads, sizeof(verify_job_t));
	for (int t = 0; t < nthreads; t++) {
		jobs[t] = p;
		jobs[t].lo = (uint32_t)(((uint64_t)n * (uint64_t)t) / (uint64_t)nthreads);
		jobs[t].hi = (uint32_t)(((uint64_t)n * (uint64_t)(t + 1)) / (uint64_t)nthreads);
		pthread_create(&th[t], NULL, verify_worker, &jobs[t]);
	}
	for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
	free(th);
	free(jobs);
	return 0;
}
