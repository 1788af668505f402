/*
 * tests/hostsim/verify_msgs.cpp — TEST-ONLY host build of the ECKCDSA / ECSDSA / ECOSDSA / ECGDSA / ECRDSA / SM2
 * message verifier: the scheme cores of ec.cuh (msgs_verify_prep_core, msgs_verify_scale, msgs_verify_accept), the comb
 * and the signed window compiled by g++ on top of the host build of the signer (sign.cpp).  Built into
 * tests/hostsim/_build/libecc_hostsim_verify_msgs.so by tests/test_verify_msgs_host.py; never loaded by libecc_b200/.
 */
#include "sign.cpp"

extern "C" {

/* Same contract as eccb200_verify_msgs_batch, item by item with the kernels' building blocks: the prep core, one
 * Field::inv per item for ECGDSA / ECRDSA instead of the CTA-wide inversion, W' = a*G + b*Y as
 * hostsim_double_smul_batch computes it (comb window w), then the acceptance test.  The offsets are trusted. */
int hostsim_verify_msgs(int sig_type, int hash_type, int curve_id, int w, uint32_t n, const uint8_t *sigs,
			const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *off, const uint8_t *ids,
			const uint64_t *id_off, int8_t *verdict)
{
	if (!msg_hash_digest_size(hash_type)) return -1;
	if (sig_type != SIG_ECKCDSA && sig_type != SIG_ECSDSA && sig_type != SIG_ECOSDSA && sig_type != SIG_ECGDSA &&
	    sig_type != SIG_ECRDSA && sig_type != SIG_SM2)
		return -1;
	const bool sm2 = sig_type == SIG_SM2;
	if (sm2 && (!ids || !id_off)) return -1;
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		typedef Field<typename C::Fq> Fq;
		constexpr int N = C::N;
		const std::vector<uint32_t> &tab = table_for<C>(w);
		const int siglen = msgs_verify_sig_len<C>(sig_type, msg_hash_digest_size(hash_type));
		for (uint32_t i = 0; i < n; i++) {
			const uint8_t *sig = sigs + (size_t)i * siglen, *pk = pubkeys + (size_t)i * 2 * C::PLEN;
			const uint64_t idlen = sm2 ? id_off[i + 1] - id_off[i] : 0;
			const uint32_t idl = idlen > kSm2MaxIdLen ? kSm2MaxIdLen + 1 : (uint32_t)idlen;
			Fe<N> a, b, den;
			const bool ok = msgs_verify_prep_core<C>(sig_type, hash_type, sig, pk, msgs + off[i], off[i + 1] - off[i],
								 idl, a, b, den);
			if (ok && msgs_verify_inverts(sig_type)) {
				Fe<N> dm, inv;
				Fq::to_mont(dm, den);
				Fq::inv(inv, dm);
				msgs_verify_scale<C>(a, b, inv);
			}
			verdict[i] = -1;
			Aff<C> Y;
			if (!load_point<C>(Y, pk)) continue;
			Jac<C> aG, W;
			comb_mul<C>(aG, a, tab.data(), w);
			window_mul<C>(W, b, Y, &aG, ThreadInverter<C>());
			uint8_t Wb[2 * 66];
			if (jac_to_wire<C>(W, Wb)) continue; /* infinity, also every item the prep refused (a = b = 0) */
			if (msgs_verify_accept<C>(sig_type, hash_type, sig, Wb, pk, msgs + off[i], off[i + 1] - off[i],
						  sm2 ? ids + id_off[i] : nullptr, idl))
				verdict[i] = 0;
		}
		return 0;
	});
}

} /* extern "C" */
