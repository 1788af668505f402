/*
 * tests/hostsim/decdsa.cpp — TEST-ONLY host build of the deterministic / raw-message ECDSA signer: SHA-224, HMAC and
 * the RFC 6979 nonce of hmac.cuh / ec.cuh compiled by g++, and the whole signer (nonce kernel, comb, finish) on top of
 * the rest of the host build (hostsim.cpp).  Built into tests/hostsim/_build/libecc_hostsim_decdsa.so by
 * tests/test_decdsa_host.py, the way schnorr_sign.cpp is; never loaded by libecc_b200/.
 */
#include "hostsim.cpp"

extern "C" {
/* any of the nine hashes of the deterministic signer (1..8, 11) of one contiguous message; digest size or -1 */
int hostsim_decdsa_hash(int hash_type, const uint8_t *msg, uint64_t len, uint8_t *out)
{
	if (!decdsa_hash_digest_size(hash_type)) return -1;
	decdsa_hash_src(hash_type, ByteSpan{ msg }, len, out);
	return decdsa_hash_digest_size(hash_type);
}

/* HMAC_key(msg) with hmac_src; a key longer than the block size is hashed first, as hash/hmac.c:45-56 does (the
 * device never needs that branch: RFC 6979 keys are digest-sized).  Digest size or -1. */
int hostsim_hmac(int hash_type, const uint8_t *key, uint32_t klen, const uint8_t *msg, uint64_t mlen, uint8_t *out)
{
	if (!decdsa_hash_digest_size(hash_type)) return -1;
	uint8_t hk[64];
	if (klen > (uint32_t)decdsa_hash_block_size(hash_type)) {
		decdsa_hash_src(hash_type, ByteSpan{ key }, klen, hk);
		key = hk;
		klen = (uint32_t)decdsa_hash_digest_size(hash_type);
	}
	hmac_src(hash_type, key, klen, ByteSpan{ msg }, mlen, out);
	return decdsa_hash_digest_size(hash_type);
}

/* k[i] = the RFC 6979 nonce of privkeys[i] and digests[i] (rfc6979_nonce) and retries[i] its k >= q retries; k = 0
 * and retries = -1 where x is outside [1, q-1], as the nonce kernel leaves it */
int hostsim_rfc6979_nonce(int curve_id, int hash_type, uint32_t n, const uint8_t *privkeys, const uint8_t *digests,
			  uint8_t *k_out, int32_t *retries)
{
	const int ds = decdsa_hash_digest_size(hash_type);
	if (!ds) return -1;
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		typedef Field<typename C::Fq> Fq;
		constexpr int N = C::N;
		for (uint32_t i = 0; i < n; i++) {
			Fe<N> x, k;
			load_be<N>(x, privkeys + (size_t)i * C::QLEN, C::QLEN);
			Fq::set_zero(k);
			retries[i] = -1;
			if (!Fq::is_zero(x) && !Fq::geq_mod(x))
				retries[i] = rfc6979_nonce<C>(k, hash_type, x, digests + (size_t)i * ds, (uint32_t)ds);
			store_be<N>(k_out + (size_t)i * C::QLEN, k, C::QLEN);
		}
		return 0;
	});
}

/*
 * Same contract as eccb200_decdsa_sign_batch (msgs == nullptr: digests given) and eccb200_ecdsa_sign_msgs_batch
 * (msgs / off given; sig_type 1 takes nonces, 14 derives them), item by item with the kernels' building blocks: the
 * hash and rfc6979_nonce of k_ecdsa_nonce, the comb (w = comb window), the normalisation, and k_ecdsa_sign_finish's
 * arithmetic with one Field::inv per item instead of the CTA-wide inversion.  The offsets are trusted.
 */
int hostsim_ecdsa_det_sign(int curve_id, int w, int sig_type, int hash_type, uint32_t n, const uint8_t *privkeys,
			   const uint8_t *nonces, const uint8_t *digests, const uint8_t *msgs, const uint64_t *off,
			   uint8_t *sigs, int8_t *status)
{
	const int ds = decdsa_hash_digest_size(hash_type);
	if (!ds || (sig_type != 1 && sig_type != 14) || (sig_type == 1 && !nonces)) return -1;
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		typedef Field<typename C::Fq> Fq;
		constexpr int N = C::N, QL = C::QLEN;
		const std::vector<uint32_t> &tab = table_for<C>(w);
		for (uint32_t i = 0; i < n; i++) {
			uint8_t h[64];
			if (msgs) decdsa_hash_src(hash_type, ByteSpan{ msgs + off[i] }, off[i + 1] - off[i], h);
			else memcpy(h, digests + (size_t)i * ds, (size_t)ds);
			Fe<N> x, k, r, s, zero;
			Fq::set_zero(zero);
			load_be<N>(x, privkeys + (size_t)i * QL, QL);
			const bool x_ok = !Fq::is_zero(x) && !Fq::geq_mod(x);
			if (sig_type == 14) {
				Fq::set_zero(k);
				if (x_ok) rfc6979_nonce<C>(k, hash_type, x, h, (uint32_t)ds);
			} else {
				load_be<N>(k, nonces + (size_t)i * QL, QL);
			}
			const bool k_ok = !Fq::is_zero(k) && !Fq::geq_mod(k);
			int st = -1;
			r = zero;
			s = zero;
			if (k_ok) {
				Jac<C> W;
				comb_mul<C>(W, k, tab.data(), w);
				uint8_t Wb[2 * 66];
				jac_to_wire<C>(W, Wb);
				Fe<N> ev, km, kinv, xm, t;
				load_be<N>(r, Wb, C::PLEN);
				scalar_reduce<C>(r);                        /* r = W_x mod q          */
				digest_to_scalar<C>(ev, h, (uint32_t)ds);
				Fq::to_mont(km, k);
				Fq::inv(kinv, km);                          /* k^-1 in Montgomery form */
				Fq::to_mont(xm, x);
				Fq::mul(t, r, xm);                          /* x*r mod q              */
				bool restart = Fq::is_zero(r) || Fq::eq(t, ev);
				Fq::add(t, t, ev);
				Fq::mul(s, t, kinv);                        /* s = k^-1 (e + x*r)     */
				restart = restart || Fq::is_zero(s);
				st = x_ok ? (restart ? 2 : 0) : -1;
			}
			if (st != 0) {
				r = zero;
				s = zero;
			}
			store_be<N>(sigs + (size_t)i * 2 * QL, r, QL);
			store_be<N>(sigs + (size_t)i * 2 * QL + QL, s, QL);
			status[i] = (int8_t)st;
		}
		return 0;
	});
}

} /* extern "C" */
