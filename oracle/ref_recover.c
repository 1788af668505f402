/*
 * oracle/ref_recover.c — the reference's ECDSA public-key recovery (__ecdsa_public_key_from_sig) and its y-from-x
 * lift (aff_pt_y_from_x) as flat batch wrappers.
 *
 * TEST INFRASTRUCTURE ONLY.  Compiled against the reference's headers and linked to oracle/_ref/libecc_ref.so (the
 * unmodified reference, oracle/Makefile) into oracle/_ref/libecc_ref_recover.so by oracle/ref_recover.mk.  It contains
 * no arithmetic of its own: every key and root comes from the reference.  Only tests/ and tools/ load it.
 *
 * Reference entry points used (paths relative to /root/reference/src):
 *   __ecdsa_public_key_from_sig  sig/ecdsa_common.c:867     aff_pt_y_from_x           curves/aff_pt.c:102
 *   prj_pt_iszero                curves/prj_pt.c:107        prj_pt_export_to_aff_buf  curves/prj_pt.h:73
 *   ec_get_curve_params_by_name  curves/curves.c:25         import_params             curves/ec_params.c:24
 *   fp_import_from_buf / fp_export_to_buf                    fp/fp.h:95-96
 */
#include "libsig.h"
#include <stdint.h>
#include <string.h>

typedef struct {
	ec_params params;
	u32 plen, qlen;
} curve_t;

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

/*
 * Per item: __ecdsa_public_key_from_sig on sig[i] = r || s (2*qlen bytes) and digest[i] (hlen bytes).
 *   keys   [n][2][2*plen]: affine Y1 then Y2 (zero unless the status is 0)
 *   status [n][2]: 0 finite, 1 the point at infinity (prj_pt_iszero), -1 both when the reference returns -1
 * Returns -1 for an unknown curve or hlen outside 1..255, else 0.
 */
int ref_ecdsa_recover_batch(const char *curve_name, uint32_t n, const uint8_t *sigs, const uint8_t *digests,
			    uint32_t hlen, uint8_t *keys, int8_t *status)
{
	curve_t c;
	if (load_curve(&c, curve_name) || hlen == 0 || hlen > 255) return -1;
	const u32 siglen = 2 * c.qlen, klen = 2 * c.plen;
	for (uint32_t i = 0; i < n; i++) {
		ec_pub_key pub[2];
		uint8_t *out = keys + (size_t)i * 2 * klen;
		memset(out, 0, 2 * klen);
		status[2 * i] = status[2 * i + 1] = -1;
		if (__ecdsa_public_key_from_sig(&pub[0], &pub[1], &c.params, sigs + (size_t)i * siglen, (u8)siglen,
						digests + (size_t)i * hlen, (u8)hlen, ECDSA))
			continue;
		for (int k = 0; k < 2; k++) {
			int iszero = 0;
			if (prj_pt_iszero(&pub[k].y, &iszero)) {
				status[2 * i + k] = -1;
			} else if (iszero) {
				status[2 * i + k] = 1;
			} else {
				status[2 * i + k] = prj_pt_export_to_aff_buf(&pub[k].y, out + k * klen, klen) ? -1 : 0;
			}
		}
	}
	return 0;
}

/*
 * Per item: x[i] (plen bytes, imported with fp_import_from_buf, so x < p) -> aff_pt_y_from_x's two outputs.
 *   y1, y2 [n][plen] (zero unless ok), ok [n]: 0 when x^3 + ax + b is a square, -1 otherwise or for x >= p
 */
int ref_y_from_x(const char *curve_name, uint32_t n, const uint8_t *xs, uint8_t *y1, uint8_t *y2, int8_t *ok)
{
	curve_t c;
	if (load_curve(&c, curve_name)) return -1;
	for (uint32_t i = 0; i < n; i++) {
		fp x, a, b;
		uint8_t *o1 = y1 + (size_t)i * c.plen, *o2 = y2 + (size_t)i * c.plen;
		memset(o1, 0, c.plen);
		memset(o2, 0, c.plen);
		ok[i] = -1;
		if (fp_init(&x, &c.params.ec_fp) || fp_init(&a, &c.params.ec_fp) || fp_init(&b, &c.params.ec_fp)) continue;
		if (fp_import_from_buf(&x, xs + (size_t)i * c.plen, (u16)c.plen)) continue;
		if (aff_pt_y_from_x(&a, &b, &x, &c.params.ec_curve)) continue;
		if (fp_export_to_buf(o1, (u16)c.plen, &a) || fp_export_to_buf(o2, (u16)c.plen, &b)) continue;
		ok[i] = 0;
	}
	return 0;
}
