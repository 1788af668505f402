/*
 * tests/hostsim/ecdsa_recover.cpp — TEST-ONLY host build of the ECDSA public-key recovery: the cores of ec.cuh
 * (ecdsa_recover_core: range checks, Field::sqrt, u and v, comb + signed window, the final additions) compiled by g++
 * on top of the host build of the device arithmetic (hostsim.cpp), with one inversion per item (ThreadInverter) where
 * the kernel shares them across its CTA.  Built into tests/hostsim/_build/libecc_hostsim_recover.so by
 * tests/test_ecdsa_recover_host.py; never loaded by libecc_b200/.
 */
#include "hostsim.cpp"

extern "C" {

/* Same contract as eccb200_ecdsa_recover_batch: keys [n][2][2*plen] (zero unless OK), status [n][2] 0 / 1 / -1. */
int hostsim_ecdsa_recover(int curve_id, int w, uint32_t n, const uint8_t *sigs, const uint8_t *digests, uint32_t hlen,
			  uint8_t *keys, int8_t *status)
{
	if (hlen == 0 || hlen > 128) return -1;
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		constexpr int N = C::N;
		const std::vector<uint32_t> &tab = table_for<C>(w);
		for (uint32_t i = 0; i < n; i++) {
			Fe<N> r, s, e;
			load_be<N>(r, sigs + (size_t)i * 2 * C::QLEN, C::QLEN);
			load_be<N>(s, sigs + (size_t)i * 2 * C::QLEN + C::QLEN, C::QLEN);
			digest_to_scalar<C>(e, digests + (size_t)i * hlen, hlen);
			uint8_t *out = keys + (size_t)i * 4 * C::PLEN;
			memset(out, 0, 4 * C::PLEN);
			Jac<C> Y1, Y2;
			if (!ecdsa_recover_core<C>(Y1, Y2, r, s, e, tab.data(), w)) {
				status[2 * i] = status[2 * i + 1] = -1;
				continue;
			}
			status[2 * i] = (int8_t)jac_to_wire<C>(Y1, out);
			status[2 * i + 1] = (int8_t)jac_to_wire<C>(Y2, out + 2 * C::PLEN);
		}
		return 0;
	});
}

/* x [n][plen] (< p) -> the two roots of x^3 + ax + b in the reference's order (y2 = p - y1), ok 0 / -1, and the trips
 * through the Tonelli-Shanks loop (0 on the curves with p = 3 mod 4). */
int hostsim_y_from_x(int curve_id, uint32_t n, const uint8_t *xs, uint8_t *y1, uint8_t *y2, int8_t *ok, int32_t *loops)
{
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		typedef Field<typename C::Fp> F;
		constexpr int N = C::N;
		for (uint32_t i = 0; i < n; i++) {
			Fe<N> x, ym, yn, t;
			load_be<N>(x, xs + (size_t)i * C::PLEN, C::PLEN);
			memset(y1 + (size_t)i * C::PLEN, 0, C::PLEN);
			memset(y2 + (size_t)i * C::PLEN, 0, C::PLEN);
			ok[i] = -1;
			loops[i] = 0;
			if (F::geq_mod(x)) continue;
			Aff<C> R;
			int lp = 0;
			const bool sq = ecdsa_recover_point<C>(R, x, &lp);
			loops[i] = lp;
			if (!sq) continue;
			F::from_mont(ym, R.y);
			F::neg(t, R.y);
			F::from_mont(yn, t);
			store_be<N>(y1 + (size_t)i * C::PLEN, ym, C::PLEN);
			store_be<N>(y2 + (size_t)i * C::PLEN, yn, C::PLEN);
			ok[i] = 0;
		}
		return 0;
	});
}

} /* extern "C" */
