/*
 * tests/hostsim/bign.cpp — TEST-ONLY host build of the BIGN / DBIGN signer and verifier: belt.cuh, bash.cuh and the
 * BIGN cores of ec.cuh compiled by g++, on top of the rest of the host build (hostsim.cpp).  Built into
 * tests/hostsim/_build/libecc_hostsim_bign.so by tests/test_bign_host.py, the way decdsa.cpp is; never loaded by
 * libecc_b200/.
 */
#include "hostsim.cpp"

template <int N>
static uint32_t det_nonce_n(const uint8_t *q_be, int qbits, const uint8_t *theta, const uint8_t *h, int hlen,
			    uint8_t *k_be)
{
	const int qlen = (qbits + 7) / 8;
	Fe<N> q, k;
	load_be<N>(q, q_be, qlen);
	const uint32_t rounds = bign_det_nonce<N>(k, theta, h, hlen, q, qbits, kBeltH);
	store_be<N>(k_be, k, qlen);
	return rounds;
}

extern "C" {

/* belt-block of n blocks, block i under the 32-byte key i */
int hostsim_belt_encrypt(uint32_t n, const uint8_t *keys, const uint8_t *in, uint8_t *out)
{
	for (uint32_t i = 0; i < n; i++) {
		uint32_t k[8], x[4];
		belt_load_block(k, keys + (size_t)i * 32);
		belt_load_block(k + 4, keys + (size_t)i * 32 + 16);
		belt_load_block(x, in + (size_t)i * 16);
		belt_block(x, k, kBeltH);
		belt_store_block(out + (size_t)i * 16, x);
	}
	return 0;
}

/* any BIGN message hash (bign_hash_src) of one contiguous message; digest size or -1 */
int hostsim_bign_hash(int hash_type, const uint8_t *msg, uint64_t len, uint8_t *out)
{
	const int ds = bign_hash_digest_size(hash_type);
	if (!ds) return -1;
	bign_hash_src(hash_type, ByteSpan{ msg }, len, out, kBeltH);
	return ds;
}

/* the S-box as the device code sees it */
void hostsim_belt_sbox(uint8_t *out) { memcpy(out, kBeltH, 256); }

/* bign_det_nonce for any group order q (qlen big-endian bytes, qbits bits; the STB curves too): k (qlen bytes,
 * big-endian) and the number of rounds, or -1 for an unsupported size */
int hostsim_bign_det_nonce(const uint8_t *q_be, int qbits, const uint8_t *theta, const uint8_t *h, int hlen,
			   uint8_t *k_be)
{
	switch ((qbits + 31) / 32) {
	case 6: return (int)det_nonce_n<6>(q_be, qbits, theta, h, hlen, k_be);
	case 7: return (int)det_nonce_n<7>(q_be, qbits, theta, h, hlen, k_be);
	case 8: return (int)det_nonce_n<8>(q_be, qbits, theta, h, hlen, k_be);
	case 12: return (int)det_nonce_n<12>(q_be, qbits, theta, h, hlen, k_be);
	case 16: return (int)det_nonce_n<16>(q_be, qbits, theta, h, hlen, k_be);
	case 17: return (int)det_nonce_n<17>(q_be, qbits, theta, h, hlen, k_be);
	default: return -1;
	}
}

/* BELT-HASH(oid || first 2l bytes of LE(x) || t) for an l of the caller's choice (x_le: 2l bytes) */
int hostsim_bign_theta(const uint8_t *oid, uint32_t oid_len, const uint8_t *x_le, uint32_t two_l, const uint8_t *t,
		       uint32_t t_len, uint8_t *theta)
{
	belt_hash_src(Seg3{ oid, oid_len, x_le, two_l, t }, (uint64_t)oid_len + two_l + t_len, theta, kBeltH);
	return 0;
}

/*
 * Same contract as eccb200_bign_sign_msgs_batch (sig_type 18 takes nonces, 19 derives them), item by item with the
 * kernels' building blocks: the hash and the nonce of k_bign_nonce, the comb (w = comb window), the normalisation and
 * bign_sign_core.  The offsets are trusted.
 */
int hostsim_bign_sign(int curve_id, int w, int sig_type, int hash_type, uint32_t n, const uint8_t *privkeys,
		      const uint8_t *nonces, const uint8_t *msgs, const uint64_t *off, const uint8_t *ad,
		      const uint64_t *ad_off, uint8_t *sigs, int8_t *status)
{
	const int ds = bign_hash_digest_size(hash_type);
	if (!ds || (sig_type != SIG_BIGN && sig_type != SIG_DBIGN) || (sig_type == SIG_BIGN && !nonces)) return -1;
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		typedef Field<typename C::Fq> Fq;
		constexpr int N = C::N, QL = C::QLEN, SL = C::QLEN / 2 + C::QLEN;
		const std::vector<uint32_t> &tab = table_for<C>(w);
		for (uint32_t i = 0; i < n; i++) {
			uint8_t h[64];
			bign_hash_src(hash_type, ByteSpan{ msgs + off[i] }, off[i + 1] - off[i], h, kBeltH);
			const uint8_t *rec = ad + ad_off[i];
			const uint64_t adlen = ad_off[i + 1] - ad_off[i];
			Fe<N> x, k;
			load_be<N>(x, privkeys + (size_t)i * QL, QL);
			Fq::set_zero(k);
			if (sig_type == SIG_DBIGN) {
				uint32_t oid_len, t_len;
				if (!Fq::is_zero(x) && !Fq::geq_mod(x) && bign_adata_parse(rec, adlen, oid_len, t_len)) {
					uint8_t theta[32];
					Fe<N> q;
					bign_theta<C>(theta, rec + 4, oid_len, rec + 4 + oid_len, t_len, x, kBeltH);
					bign_order<C>(q);
					bign_det_nonce<N>(k, theta, h, ds, q, C::QBITS, kBeltH);
				}
			} else {
				load_be<N>(k, nonces + (size_t)i * QL, QL);
			}
			Jac<C> W;
			comb_mul<C>(W, k, tab.data(), w);
			uint8_t Wb[2 * 66];
			jac_to_wire<C>(W, Wb);
			status[i] = (int8_t)bign_sign_core<C>(sigs + (size_t)i * SL, Wb, x, k, h, ds, rec, adlen, kBeltH);
		}
		return 0;
	});
}

/* Same contract as eccb200_bign_verify_msgs_batch, item by item: bign_verify_prep_core, W' = a*G + b*Y as
 * hostsim_verify_msgs computes it (comb window w), then the s0 test of k_bign_verify_finish. */
int hostsim_bign_verify(int curve_id, int w, int hash_type, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
			const uint8_t *msgs, const uint64_t *off, const uint8_t *ad, const uint64_t *ad_off,
			int8_t *verdict)
{
	const int ds = bign_hash_digest_size(hash_type);
	if (!ds) return -1;
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		constexpr int N = C::N, L = C::QLEN / 2, SL = C::QLEN / 2 + C::QLEN;
		const std::vector<uint32_t> &tab = table_for<C>(w);
		for (uint32_t i = 0; i < n; i++) {
			const uint8_t *sig = sigs + (size_t)i * SL, *pk = pubkeys + (size_t)i * 2 * C::PLEN;
			const uint8_t *rec = ad + ad_off[i];
			const uint64_t adlen = ad_off[i + 1] - ad_off[i];
			uint8_t h[64];
			bign_hash_src(hash_type, ByteSpan{ msgs + off[i] }, off[i + 1] - off[i], h, kBeltH);
			Fe<N> a, b;
			bign_verify_prep_core<C>(a, b, sig, h, ds, rec, adlen);
			verdict[i] = -1;
			Aff<C> Y;
			if (!load_point<C>(Y, pk)) continue;
			Jac<C> aG, W;
			comb_mul<C>(aG, a, tab.data(), w);
			window_mul<C>(W, b, Y, &aG, ThreadInverter<C>());
			uint8_t Wb[2 * 66];
			if (jac_to_wire<C>(W, Wb)) continue; /* infinity, also every item the prep refused (a = b = 0) */
			uint32_t oid_len, t_len;
			if (!bign_adata_parse(rec, adlen, oid_len, t_len)) continue;
			uint8_t s0[L];
			bign_s0<C>(s0, rec + 4, oid_len, Wb, h, ds, kBeltH);
			if (!memcmp(s0, sig, L)) verdict[i] = 0;
		}
		return 0;
	});
}

} /* extern "C" */
