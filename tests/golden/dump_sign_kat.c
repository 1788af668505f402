/*
 * tests/golden/dump_sign_kat.c — extracts the reference's own ECKCDSA / ECGDSA / ECRDSA / SM2 signing vectors on the
 * engine's eleven curves, with the nonce their harness injects (bound q) and the ancillary data (the SM2 user ID), into
 * tests/golden/sign_kat.json.  The reference's ECRDSA vectors all lie on GOST curves, so none is extracted.  Run where
 * the reference's sources exist; the fixture (not this program's inputs) is committed:
 *
 *   make -C oracle ref
 *   gcc -O0 -std=gnu11 -w -DWITH_STDLIB -I/root/reference/src tests/golden/dump_sign_kat.c \
 *       -o oracle/_ref/dump_sign_kat -Loracle/_ref -lecc_ref -Wl,-rpath,"$PWD/oracle/_ref"
 *   oracle/_ref/dump_sign_kat tests/golden
 *
 * It #includes the reference's test-vector header in place (nothing is copied into the repo) and links
 * oracle/_ref/libecc_ref.so.  Source (relative to /root/reference/src): tests/ec_self_tests_core.h
 * ec_fixed_vector_tests[] (:4915).
 */
#include "libsig.h"
#include "tests/ec_self_tests_core.h"
#include <stdio.h>
#include <string.h>

static void hex(FILE *f, const char *key, const u8 *b, unsigned int len, int last)
{
	fprintf(f, "\"%s\": \"", key);
	for (unsigned int i = 0; i < len; i++) fprintf(f, "%02x", b[i]);
	fprintf(f, "\"%s", last ? "" : ", ");
}

static const char *curve_name(const ec_str_params *sp)
{
	return (const char *)sp->name->buf;
}

static int wanted_curve(const ec_str_params *sp)
{
	const char *n = curve_name(sp);
	return !strcmp(n, "SECP256R1") || !strcmp(n, "SECP384R1") || !strcmp(n, "FRP256V1") ||
	       !strcmp(n, "BRAINPOOLP256R1") || !strcmp(n, "BRAINPOOLP384R1") || !strcmp(n, "SECP256K1") ||
	       !strcmp(n, "SECP521R1") || !strcmp(n, "SM2P256V1") || !strcmp(n, "BRAINPOOLP512R1") ||
	       !strcmp(n, "SECP224R1") || !strcmp(n, "SECP192R1");
}

static const char *hash_name(hash_alg_type t)
{
	const hash_mapping *hm = NULL;
	if (get_hash_by_type(t, &hm) || !hm) return "?";
	return hm->name;
}

static void jstr(FILE *f, const char *key, const char *s, int last)
{
	fprintf(f, "\"%s\": \"", key);
	for (; s && *s; s++) {
		if (*s == '"' || *s == '\\') fputc('\\', f);
		if ((unsigned char)*s >= 0x20) fputc(*s, f);
	}
	fprintf(f, "\"%s", last ? "" : ", ");
}

int main(int argc, char **argv)
{
	const char *dir = (argc > 1) ? argv[1] : ".";
	char path[512];
	FILE *f;
	int first = 1;

	snprintf(path, sizeof(path), "%s/sign_kat.json", dir);
	f = fopen(path, "w");
	if (!f) return 1;
	fprintf(f, "[\n");
	for (unsigned int i = 0; i < sizeof(ec_fixed_vector_tests) / sizeof(ec_fixed_vector_tests[0]); i++) {
		const ec_test_case *t = ec_fixed_vector_tests[i];
		ec_params params;
		ec_key_pair kp;
		u8 pub[2 * 66], rbuf[66], plen, qlen;
		nn r, bound;
		const char *alg;
		if (!t) continue;
		if (t->sig_type == ECKCDSA) alg = "ECKCDSA";
		else if (t->sig_type == ECGDSA) alg = "ECGDSA";
		else if (t->sig_type == ECRDSA) alg = "ECRDSA";
		else if (t->sig_type == SM2) alg = "SM2";
		else continue;
		/* the scheme is checked first: entries of other schemes may carry no curve at all */
		if (!wanted_curve(t->ec_str_p) || !t->nn_random) continue;
		if (import_params(&params, t->ec_str_p)) return 1;
		plen = (u8)BYTECEIL(params.ec_fp.p_bitlen);
		qlen = (u8)BYTECEIL(params.ec_gen_order_bitlen);
		if (ec_key_pair_import_from_priv_key_buf(&kp, &params, t->priv_key, t->priv_key_len, t->sig_type)) return 1;
		if (ec_pub_key_export_to_aff_buf(&kp.pub_key, pub, (u8)(2 * plen))) return 1;
		if (nn_copy(&bound, &params.ec_gen_order)) return 1;
		if (t->nn_random(&r, &bound) || nn_export_to_buf(rbuf, qlen, &r)) return 1;
		fprintf(f, "%s {", first ? "" : ",\n");
		first = 0;
		jstr(f, "name", t->name, 0);
		jstr(f, "curve", curve_name(t->ec_str_p), 0);
		jstr(f, "alg", alg, 0);
		jstr(f, "hash", hash_name(t->hash_type), 0);
		hex(f, "priv", t->priv_key, t->priv_key_len, 0);
		hex(f, "pub", pub, (unsigned int)(2 * plen), 0);
		hex(f, "msg", (const u8 *)t->msg, t->msglen, 0);
		hex(f, "nonce", rbuf, qlen, 0);
		hex(f, "adata", t->adata ? t->adata : (const u8 *)"", t->adata ? t->adata_len : 0, 0);
		hex(f, "sig", t->exp_sig, t->exp_siglen, 1);
		fprintf(f, "}");
	}
	fprintf(f, "\n]\n");
	fclose(f);
	return 0;
}
