/*
 * tests/hostsim/schnorr_sign.cpp — TEST-ONLY host build of the Schnorr-family signer (ECSDSA, ECOSDSA, ECFSDSA,
 * BIP0340): the segmented hash, the BIP0340 tag digests and nonce, the comb and the scheme core of ec.cuh / sha2.cuh
 * compiled by g++ on top of the rest of the host build (hostsim.cpp).  Built into
 * tests/hostsim/_build/libecc_hostsim_schnorr.so by tests/test_schnorr_sign_host.py; never loaded by libecc_b200/.
 */
#include "hostsim.cpp"

extern "C" {
/* the segmented hash of the Schnorr-family signers: H(pre || msg), hash_type 2..8; returns the digest size or -1 */
int hostsim_hash_segments(int hash_type, const uint8_t *pre, uint32_t npre, const uint8_t *msg, uint64_t nmsg,
			  uint8_t *out)
{
	if (!sha2_digest_size(hash_type) || npre > (uint32_t)kSchnorrMaxPrefix) return -1;
	hash_segments(hash_type, pre, npre, msg, nmsg, out);
	return sha2_digest_size(hash_type);
}

/* H(tag) of the BIP0340 tags 0 aux, 1 nonce, 2 challenge */
int hostsim_bip0340_tag_hash(int hash_type, int tag, uint8_t *out)
{
	if (!sha2_digest_size(hash_type) || tag < 0 || tag > 2) return -1;
	bip0340_tag_hash(hash_type, tag, out);
	return sha2_digest_size(hash_type);
}

/* Same contract as eccb200_schnorr_sign_msgs_batch, with the kernels' building blocks item by item: the BIP0340 nonce
 * (bip0340_nonce), the comb (w = comb window), the normalisation, the scheme core (schnorr_sign_core) */
int hostsim_schnorr_sign(int sig_type, int hash_type, int curve_id, int w, uint32_t n, const uint8_t *privkeys,
			 const uint8_t *pubkeys, const uint8_t *randomness, const uint8_t *msgs, const uint64_t *off,
			 uint8_t *sigs, int8_t *status)
{
	if (!sha2_digest_size(hash_type)) return -1;
	if (sig_type != SIG_ECSDSA && sig_type != SIG_ECOSDSA && sig_type != SIG_ECFSDSA && sig_type != SIG_BIP0340) return -1;
	const bool bip = sig_type == SIG_BIP0340;
	if (bip && !pubkeys) return -1;
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		typedef Field<typename C::Fq> Fq;
		constexpr int N = C::N;
		const std::vector<uint32_t> &tab = table_for<C>(w);
		const int siglen = schnorr_sig_len<C>(sig_type, sha2_digest_size(hash_type));
		uint8_t tags[3][64];
		for (int t = 0; t < 3; t++) bip0340_tag_hash(hash_type, t, tags[t]);
		for (uint32_t i = 0; i < n; i++) {
			Fe<N> x, k, kr;
			const uint8_t *pk = bip ? pubkeys + (size_t)i * 2 * C::PLEN : nullptr;
			const uint8_t *m = msgs + off[i];
			const uint64_t mlen = off[i + 1] - off[i];
			load_be<N>(x, privkeys + (size_t)i * C::QLEN, C::QLEN);
			bool key_ok = true;
			if (bip) {
				Aff<C> P;
				key_ok = load_point<C>(P, pk);
				Fq::set_zero(k);
				if (key_ok && !Fq::is_zero(x) && !Fq::geq_mod(x))
					bip0340_nonce<C>(k, hash_type, x, pk, randomness + (size_t)i * C::QLEN, m, mlen, tags[0],
							 tags[1]);
			} else {
				load_be<N>(k, randomness + (size_t)i * C::QLEN, C::QLEN);
			}
			kr = k;
			scalar_reduce<C>(kr);
			Jac<C> W;
			comb_mul<C>(W, kr, tab.data(), w);
			uint8_t Wb[2 * 66];
			jac_to_wire<C>(W, Wb);
			status[i] = (int8_t)schnorr_sign_core<C>(sigs + (size_t)i * siglen, sig_type, hash_type, Wb, x, k, m, mlen,
								 pk, key_ok, tags[2]);
		}
		return 0;
	});
}


} /* extern "C" */
