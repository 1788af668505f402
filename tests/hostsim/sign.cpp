/*
 * tests/hostsim/sign.cpp — TEST-ONLY host build of the ECKCDSA / ECGDSA / ECRDSA / SM2 message signer: SM3, the
 * three-segment byte source, SM2's Z, the comb and the scheme core of ec.cuh / sm3.cuh compiled by g++ on top of the
 * rest of the host build (hostsim.cpp).  Built into tests/hostsim/_build/libecc_hostsim_sign.so by
 * tests/test_sign_msgs_host.py, the way schnorr_sign.cpp is; never loaded by libecc_b200/.
 */
#include "hostsim.cpp"

extern "C" {
/* H(pre || mid || post) over the three-segment source with any hash of the message signers (2..8, 11); returns the
 * digest size or -1 */
int hostsim_msg_hash_seg3(int hash_type, const uint8_t *pre, uint32_t npre, const uint8_t *mid, uint64_t nmid,
			  const uint8_t *post, uint64_t npost, uint8_t *out)
{
	if (!msg_hash_digest_size(hash_type)) return -1;
	msg_hash_seg3(hash_type, Seg3{ pre, npre, mid, nmid, post }, (uint64_t)npre + nmid + npost, out);
	return msg_hash_digest_size(hash_type);
}

/* SM3 of one contiguous message */
int hostsim_sm3(const uint8_t *msg, uint64_t len, uint8_t *out)
{
	sm3_src(ByteSpan{ msg }, len, out);
	return 32;
}

/* Same contract as eccb200_sign_msgs_batch, item by item with the kernels' building blocks: the comb (w = comb
 * window), the normalisation, (1 + x)^-1 for SM2 (one Field::inv per item instead of the CTA-wide one) and the scheme
 * core (msgs_sign_core).  The offsets are trusted. */
int hostsim_sign_msgs(int sig_type, int hash_type, int curve_id, int w, uint32_t n, const uint8_t *privkeys,
		      const uint8_t *pubkeys, const uint8_t *nonces, const uint8_t *msgs, const uint64_t *off,
		      const uint8_t *ids, const uint64_t *id_off, uint8_t *sigs, int8_t *status)
{
	if (!msg_hash_digest_size(hash_type)) return -1;
	if (sig_type != SIG_ECKCDSA && sig_type != SIG_ECGDSA && sig_type != SIG_ECRDSA && sig_type != SIG_SM2) return -1;
	const bool sm2 = sig_type == SIG_SM2, with_key = sm2 || sig_type == SIG_ECKCDSA;
	if ((with_key && !pubkeys) || (sm2 && (!ids || !id_off))) return -1;
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		typedef Field<typename C::Fq> Fq;
		constexpr int N = C::N;
		const std::vector<uint32_t> &tab = table_for<C>(w);
		const int siglen = msgs_sig_len<C>(sig_type, msg_hash_digest_size(hash_type));
		for (uint32_t i = 0; i < n; i++) {
			Fe<N> x, k, kr, ix;
			load_be<N>(x, privkeys + (size_t)i * C::QLEN, C::QLEN);
			load_be<N>(k, nonces + (size_t)i * C::QLEN, C::QLEN);
			const uint8_t *pk = with_key ? pubkeys + (size_t)i * 2 * C::PLEN : nullptr;
			bool key_ok = true;
			if (with_key) {
				Aff<C> P;
				key_ok = load_point<C>(P, pk);
			}
			Fq::set_zero(ix);
			if (sm2 && msgs_key_in_range<C>(SIG_SM2, x)) {
				Fe<N> u;
				sm2_one_plus_x<C>(u, x);
				Fq::inv(ix, u);
			}
			kr = k;
			scalar_reduce<C>(kr);
			Jac<C> W;
			comb_mul<C>(W, kr, tab.data(), w);
			uint8_t Wb[2 * 66];
			jac_to_wire<C>(W, Wb);
			const uint64_t idlen = sm2 ? id_off[i + 1] - id_off[i] : 0;
			status[i] = (int8_t)msgs_sign_core<C>(sigs + (size_t)i * siglen, sig_type, hash_type, Wb, x, k,
							      msgs + off[i], off[i + 1] - off[i], pk, key_ok,
							      sm2 ? ids + id_off[i] : nullptr,
							      idlen > kSm2MaxIdLen ? kSm2MaxIdLen + 1 : (uint32_t)idlen, ix);
		}
		return 0;
	});
}

} /* extern "C" */
