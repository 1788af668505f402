/*
 * tests/golden/dump_bign_kat.c — extracts the reference's own BIGN and DBIGN signing vectors (all on the STB curves
 * bign256v1 / bign384v1 / bign512v1, which the engine does not have) into tests/golden/bign_kat.json, with each
 * vector's curve parameters, the nonce its harness injects (BIGN only; DBIGN derives it), and the adata record.  Run
 * where the reference's sources exist; the fixture (not this program's inputs) is committed:
 *
 *   make -C oracle ref
 *   gcc -O0 -std=gnu11 -w -DWITH_STDLIB -I/root/reference/src tests/golden/dump_bign_kat.c \
 *       -o oracle/_ref/dump_bign_kat -Loracle/_ref -lecc_ref -Wl,-rpath,"$PWD/oracle/_ref"
 *   oracle/_ref/dump_bign_kat tests/golden
 *
 * It #includes the reference's test-vector header in place (nothing is copied into the repo) and links
 * oracle/_ref/libecc_ref.so.  Source (relative to /root/reference/src): tests/ec_self_tests_core.h
 * ec_fixed_vector_tests[], with the vectors of tests/bign_test_vectors.h and tests/dbign_test_vectors.h.
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

	snprintf(path, sizeof(path), "%s/bign_kat.json", dir);
	f = fopen(path, "w");
	if (!f) return 1;
	fprintf(f, "[\n");
	for (unsigned int i = 0; i < sizeof(ec_fixed_vector_tests) / sizeof(ec_fixed_vector_tests[0]); i++) {
		const ec_test_case *t = ec_fixed_vector_tests[i];
		ec_params params;
		u8 buf[2 * 66], plen, qlen;
		nn r, bound;
		const hash_mapping *hm = NULL;
		if (!t || (t->sig_type != BIGN && t->sig_type != DBIGN)) continue;
		if (import_params(&params, t->ec_str_p)) return 1;
		plen = (u8)BYTECEIL(params.ec_fp.p_bitlen);
		qlen = (u8)BYTECEIL(params.ec_gen_order_bitlen);
		if (get_hash_by_type(t->hash_type, &hm) || !hm) return 1;
		fprintf(f, "%s {", first ? "" : ",\n");
		first = 0;
		jstr(f, "name", t->name, 0);
		jstr(f, "alg", t->sig_type == BIGN ? "BIGN" : "DBIGN", 0);
		jstr(f, "curve", (const char *)t->ec_str_p->name->buf, 0);
		if (nn_export_to_buf(buf, plen, &params.ec_fp.p)) return 1;
		hex(f, "p", buf, plen, 0);
		if (fp_export_to_buf(buf, plen, &params.ec_curve.a)) return 1;
		hex(f, "a", buf, plen, 0);
		if (fp_export_to_buf(buf, plen, &params.ec_curve.b)) return 1;
		hex(f, "b", buf, plen, 0);
		if (prj_pt_export_to_aff_buf(&params.ec_gen, buf, 2 * plen)) return 1;
		hex(f, "g", buf, 2 * plen, 0);
		if (nn_export_to_buf(buf, qlen, &params.ec_gen_order)) return 1;
		hex(f, "q", buf, qlen, 0);
		jstr(f, "hash", hm->name, 0);
		hex(f, "priv", t->priv_key, t->priv_key_len, 0);
		if (t->sig_type == BIGN && t->nn_random) {
			if (nn_copy(&bound, &params.ec_gen_order) || t->nn_random(&r, &bound) || nn_export_to_buf(buf, qlen, &r))
				return 1;
			hex(f, "nonce", buf, qlen, 0);
		} else {
			hex(f, "nonce", buf, 0, 0);
		}
		hex(f, "msg", (const u8 *)t->msg, t->msglen, 0);
		hex(f, "adata", t->adata ? t->adata : (const u8 *)"", t->adata ? t->adata_len : 0, 0);
		hex(f, "sig", t->exp_sig, t->exp_siglen, 1);
		fprintf(f, "}");
	}
	fprintf(f, "\n]\n");
	fclose(f);
	return 0;
}
