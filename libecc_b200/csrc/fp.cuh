/*
 * fp.cuh — prime-field arithmetic for the device (replaces the reference's src/nn + src/fp on the hot path).
 *
 * Reference counterparts (paths relative to /root/reference/src):
 *   Field<F>::mul   fp_mul_monty  fp/fp_montgomery.c:44 -> nn_mul_redc1 nn/nn_mul_redc1.c:124-218 (CIOS)
 *   Field<F>::sqr   fp_sqr_monty  fp/fp_montgomery.c:53
 *   Field<F>::add   fp_add_monty  fp/fp_montgomery.c:26 -> nn_mod_add nn/nn_add.c:337
 *   Field<F>::sub   fp_sub_monty  fp/fp_montgomery.c:35 -> nn_mod_sub nn/nn_add.c:398
 *   Field<F>::inv   fp_inv        fp/fp_mul.c:51 -> nn_modinv_fermat_redc nn/nn_modinv.c:538
 *   to_mont/from_mont  fp_redcify / fp_unredcify  fp/fp_mul_redc1.c:62,79
 *
 * Representation: an element is N 32-bit little-endian words held in registers (N = 8 for 256-bit, 12 for
 * 384-bit), always fully reduced (< m), in Montgomery form with R = 2^(32N) — the same R as the reference's
 * 64-bit-limb R = 2^(64n), so Montgomery-form values are bit-identical to the reference's.
 * One thread owns whole elements; there is no cross-lane traffic in the arithmetic (DESIGN.md §3 records the
 * measurement behind that choice).
 *
 * The modulus is a compile-time constant of the field tag F (curve_constants.inc), so the compiler folds the
 * special words of the NIST primes (0, 1, 0xffffffff, M0 == 1) out of the reduction.
 *
 * Two multiplier back ends produce bit-identical results:
 *   - portable C++ (this file): CIOS over 32x32->64 products; also compiles for the host so that the unit tests
 *     in tests/hostsim can check the algorithms without a GPU (test-only; the product never runs on the host);
 *   - PTX (fp_ptx.cuh, device only): IMAD.WIDE carry chains, the default on the device (-DECC_NO_PTX selects the portable one).
 */
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__)
#define ECC_HD __host__ __device__ __forceinline__
#define ECC_D __device__ __forceinline__
#define ECC_NOINLINE __host__ __device__ __noinline__
#else
#define ECC_HD inline
#define ECC_D inline
#define ECC_NOINLINE __attribute__((noinline))
#endif

#define ECC_CONST_ARRAY(NAME, CNT, ...)                      \
	static constexpr ECC_HD uint32_t NAME(int i)          \
	{                                                     \
		constexpr uint32_t v[CNT] = { __VA_ARGS__ }; \
		return v[i];                                  \
	}

namespace eccb200 {

#include "curve_constants.inc"

template <int N> struct Fe {
	uint32_t w[N];
};

#if defined(ECC_COUNT_MULS)
/* host-only instrumentation (tests/hostsim): counts field multiplications, the M_impl of SURVEY.md §8d */
extern thread_local unsigned long long g_fe_mul_count;
#define ECC_COUNT_MUL() (++g_fe_mul_count)
#else
#define ECC_COUNT_MUL() ((void)0)
#endif

template <class F> struct FieldPortable {
	static constexpr int N = F::N;
	typedef Fe<N> E;

	/* r = a*b*R^-1 mod m.  32-bit-word CIOS: same recurrence as nn_mul_redc1.c:175-205 with WORD_BITS = 32. */
	static ECC_HD void mul(E &r, const E &a, const E &b)
	{
		uint32_t t[N + 2];
		ECC_COUNT_MUL();
#pragma unroll
		for (int i = 0; i < N + 2; i++) t[i] = 0;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t c = 0;
#pragma unroll
			for (int j = 0; j < N; j++) {
				uint64_t s = (uint64_t)a.w[j] * b.w[i] + t[j] + c;
				t[j] = (uint32_t)s;
				c = s >> 32;
			}
			uint64_t s = (uint64_t)t[N] + c;
			t[N] = (uint32_t)s;
			t[N + 1] = (uint32_t)(s >> 32);
			uint32_t m = t[0] * F::M0;
			c = ((uint64_t)m * F::P(0) + t[0]) >> 32;
#pragma unroll
			for (int j = 1; j < N; j++) {
				uint64_t s2 = (uint64_t)m * F::P(j) + t[j] + c;
				t[j - 1] = (uint32_t)s2;
				c = s2 >> 32;
			}
			s = (uint64_t)t[N] + c;
			t[N - 1] = (uint32_t)s;
			t[N] = t[N + 1] + (uint32_t)(s >> 32);
		}
		/* t < 2m: conditional subtraction (nn_mul_redc1.c:210-211) */
		uint32_t d[N];
		uint64_t bw = 0;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t s = (uint64_t)t[i] - F::P(i) - bw;
			d[i] = (uint32_t)s;
			bw = (s >> 32) & 1;
		}
		bool ge = (t[N] != 0) || (bw == 0);
#pragma unroll
		for (int i = 0; i < N; i++) r.w[i] = ge ? d[i] : t[i];
	}

	static ECC_HD void sqr(E &r, const E &a) { mul(r, a, a); }

	static ECC_HD void add(E &r, const E &a, const E &b)
	{
		uint32_t s[N], d[N];
		uint64_t c = 0, bw = 0;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t t = (uint64_t)a.w[i] + b.w[i] + c;
			s[i] = (uint32_t)t;
			c = t >> 32;
		}
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t t = (uint64_t)s[i] - F::P(i) - bw;
			d[i] = (uint32_t)t;
			bw = (t >> 32) & 1;
		}
		bool ge = (c != 0) || (bw == 0);
#pragma unroll
		for (int i = 0; i < N; i++) r.w[i] = ge ? d[i] : s[i];
	}

	static ECC_HD void sub(E &r, const E &a, const E &b)
	{
		uint32_t d[N];
		uint64_t bw = 0, c = 0;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t t = (uint64_t)a.w[i] - b.w[i] - bw;
			d[i] = (uint32_t)t;
			bw = (t >> 32) & 1;
		}
		uint32_t mask = (uint32_t)0 - (uint32_t)bw;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t t = (uint64_t)d[i] + (F::P(i) & mask) + c;
			r.w[i] = (uint32_t)t;
			c = t >> 32;
		}
	}
};

} // namespace eccb200

#if defined(__CUDA_ARCH__) && !defined(ECC_NO_PTX)
#include "fp_ptx.cuh"
#endif

namespace eccb200 {

#if defined(__CUDA_ARCH__) && !defined(ECC_NO_PTX)
template <class F> struct FieldCore : FieldPtx<F> {};
#else
template <class F> struct FieldCore : FieldPortable<F> {};
#endif

template <class F> struct Field : FieldCore<F> {
	static constexpr int N = F::N;
	typedef Fe<N> E;
	typedef FieldCore<F> Core;
	using Core::add;
	using Core::mul;
	using Core::sqr;
	using Core::sub;

	/* An out-of-line copy of the product for kernels that otherwise inline it (K1): calling it for some of the
	 * products of the loop body keeps the body inside the instruction cache (ECC_K1_OOL_MULS, ec.cuh). */
#if defined(__CUDA_ARCH__) && !defined(ECC_NO_PTX)
	static __device__ __noinline__ E mul_ool_fn(E a, E b) { return Core::mul_fn(a, b); }
	static __device__ __forceinline__ void mul_ool(E &r, const E &a, const E &b) { r = mul_ool_fn(a, b); }
#else
	static ECC_HD void mul_ool(E &r, const E &a, const E &b) { Core::mul(r, a, b); }
#endif

	static ECC_HD void set_zero(E &r)
	{
#pragma unroll
		for (int i = 0; i < N; i++) r.w[i] = 0;
	}
	static ECC_HD void set_one(E &r) /* 1 in Montgomery form */
	{
#pragma unroll
		for (int i = 0; i < N; i++) r.w[i] = F::ONE(i);
	}
	static ECC_HD bool is_zero(const E &a)
	{
		uint32_t acc = 0;
#pragma unroll
		for (int i = 0; i < N; i++) acc |= a.w[i];
		return acc == 0;
	}
	static ECC_HD bool eq(const E &a, const E &b)
	{
		uint32_t acc = 0;
#pragma unroll
		for (int i = 0; i < N; i++) acc |= a.w[i] ^ b.w[i];
		return acc == 0;
	}
	/* a >= m ? (raw integer comparison; used to validate wire inputs) */
	static ECC_HD bool geq_mod(const E &a)
	{
		uint64_t bw = 0;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t t = (uint64_t)a.w[i] - F::P(i) - bw;
			bw = (t >> 32) & 1;
		}
		return bw == 0;
	}
	/* r = a - m if a >= m else a  (raw integers < 2^(32N)) */
	static ECC_HD void cond_sub_mod(E &r, const E &a)
	{
		uint32_t d[N];
		uint64_t bw = 0;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t t = (uint64_t)a.w[i] - F::P(i) - bw;
			d[i] = (uint32_t)t;
			bw = (t >> 32) & 1;
		}
#pragma unroll
		for (int i = 0; i < N; i++) r.w[i] = bw ? a.w[i] : d[i];
	}
	static ECC_HD void neg(E &r, const E &a)
	{
		E z;
		set_zero(z);
		sub(r, z, a);
	}
	static ECC_HD void dbl(E &r, const E &a) { add(r, a, a); }
	static ECC_HD void to_mont(E &r, const E &a)
	{
		E rr;
#pragma unroll
		for (int i = 0; i < N; i++) rr.w[i] = F::RR(i);
		mul(r, a, rr);
	}
	static ECC_HD void from_mont(E &r, const E &a)
	{
		E one;
#pragma unroll
		for (int i = 0; i < N; i++) one.w[i] = (i == 0) ? 1u : 0u;
		mul(r, a, one);
	}
	static ECC_HD void cmov(E &r, const E &a, bool take)
	{
#pragma unroll
		for (int i = 0; i < N; i++) r.w[i] = take ? a.w[i] : r.w[i];
	}

	/*
	 * r = a^-1 (Montgomery in, Montgomery out; a == 0 gives 0) — the inversion every caller uses (fp_inv, fp/fp_mul.c:51;
	 * nn_modinv, nn/nn_modinv.c for the scalars).  Bernstein-Yang "safegcd" division steps instead of a Fermat power:
	 * the inversion is always ONE serial chain per CTA (cta_inverse_128) or per thread, so what matters is its latency,
	 * and ~750 division steps on 30-bit limbs are several times shorter than ~330 dependent field products.
	 *
	 *   state  f = m, g = x (the plain integer held in `a`), d = 0, e = 1, eta = -1, with the invariants
	 *          d*x == f and e*x == g (mod m);
	 *   step   (eta, f, g) -> (-eta-1, g, (g-f)/2) if eta < 0 and g odd, else (eta-1, f, (g + (g odd)*f)/2)
	 *          [Bernstein-Yang 2019, "Fast constant-time gcd computation and modular inversion", divstep with delta = -eta];
	 *   batch  30 steps are run on the low words only and summarised in a 2x2 integer matrix t with
	 *          2^30 (f', g') = t (f, g); the full-width f, g and (mod m) d, e are then updated with t in one pass each;
	 *   bound  g reaches 0 within floor((49 BITS + 57) / 17) steps for BITS >= 46 (their Theorem 11.2); the loop leaves
	 *          as soon as g == 0 and never runs more than that many steps;
	 *   end    f = +-1, so x^-1 = f*d; two extra products turn (aR)^-1 into the Montgomery form a^-1 R.
	 * Values are kept in L signed limbs of 30 bits (all but the top one in [0, 2^30)); d and e stay in (-2m, m).
	 * Should the bound ever be violated (it is a theorem; the check costs nothing) the Fermat power is used instead.
	 */
	static constexpr int GCD_L = (F::BITS + 2 + 29) / 30;
	static constexpr int GCD_BATCHES = ((49 * F::BITS + 57) / 17 + 29) / 30;
	struct GcdMat {
		int32_t u, v, q, r;
	};
	/* 30 division steps on the low 32 bits of f and g; returns the new eta */
	static ECC_HD int32_t gcd_divsteps_30(int32_t eta, uint32_t f, uint32_t g, GcdMat &t)
	{
		uint32_t u = 1, v = 0, q = 0, r = 1; /* two's complement arithmetic on unsigned words (no signed overflow) */
#pragma unroll 1
		for (int i = 0; i < 30; i++) {
			uint32_t c1 = (uint32_t)(eta >> 31); /* all ones iff eta < 0 */
			const uint32_t c2 = 0u - (g & 1u);   /* all ones iff g is odd */
			const uint32_t x = (f ^ c1) - c1, y = (u ^ c1) - c1, z = (v ^ c1) - c1; /* (-f, -u, -v) iff eta < 0 */
			g += x & c2;
			q += y & c2;
			r += z & c2;
			c1 &= c2; /* swap iff eta < 0 and g odd */
			eta = (int32_t)(((uint32_t)eta ^ c1) - (c1 + 1u));
			f += g & c1;
			u += q & c1;
			v += r & c1;
			g >>= 1;
			u <<= 1;
			v <<= 1;
		}
		t.u = (int32_t)u;
		t.v = (int32_t)v;
		t.q = (int32_t)q;
		t.r = (int32_t)r;
		return eta;
	}
	static ECC_HD void inv(E &r, const E &a)
	{
		constexpr int L = GCD_L;
		constexpr int32_t M30 = (int32_t)((1u << 30) - 1u);
		constexpr uint32_t MINV30 = (0u - F::M0) & (uint32_t)M30; /* m^-1 mod 2^30 (M0 is -m^-1 mod 2^32) */
		int32_t mod[L], f[L], g[L], d[L], e[L];
		/* 32-bit words -> 30-bit limbs */
#pragma unroll
		for (int i = 0; i < L; i++) {
			const int bit = 30 * i, w = bit >> 5, sh = bit & 31;
			uint32_t lo_m = (w < N) ? F::P(w < N ? w : 0) : 0u, hi_m = (w + 1 < N) ? F::P(w + 1 < N ? w + 1 : 0) : 0u;
			uint32_t lo_a = (w < N) ? a.w[w < N ? w : 0] : 0u, hi_a = (w + 1 < N) ? a.w[w + 1 < N ? w + 1 : 0] : 0u;
			uint32_t vm = sh ? ((lo_m >> sh) | (hi_m << (32 - sh))) : lo_m;
			uint32_t va = sh ? ((lo_a >> sh) | (hi_a << (32 - sh))) : lo_a;
			mod[i] = (int32_t)(vm & (uint32_t)M30);
			f[i] = mod[i];
			g[i] = (int32_t)(va & (uint32_t)M30);
			d[i] = 0;
			e[i] = 0;
		}
		e[0] = 1;
		int32_t eta = -1;
		uint32_t g_nonzero = 1;
#pragma unroll 1
		for (int it = 0; it < GCD_BATCHES && g_nonzero; it++) {
			GcdMat t;
			eta = gcd_divsteps_30(eta, (uint32_t)f[0] | ((uint32_t)f[1] << 30), (uint32_t)g[0] | ((uint32_t)g[1] << 30), t);
			const int64_t u = t.u, v = t.v, q = t.q, rr = t.r;
			{ /* (d, e) <- t (d, e) / 2^30 mod m, staying in (-2m, m) */
				const int32_t sd = d[L - 1] >> 31, se = e[L - 1] >> 31;
				int32_t md = (t.u & sd) + (t.v & se), me = (t.q & sd) + (t.r & se);
				int64_t cd = u * d[0] + v * e[0], ce = q * d[0] + rr * e[0];
				md -= (int32_t)((MINV30 * (uint32_t)cd + (uint32_t)md) & (uint32_t)M30);
				me -= (int32_t)((MINV30 * (uint32_t)ce + (uint32_t)me) & (uint32_t)M30);
				cd += (int64_t)mod[0] * md;
				ce += (int64_t)mod[0] * me;
				cd >>= 30; /* the low 30 bits are zero by the choice of md, me */
				ce >>= 30;
#pragma unroll
				for (int i = 1; i < L; i++) {
					cd += u * d[i] + v * e[i] + (int64_t)mod[i] * md;
					ce += q * d[i] + rr * e[i] + (int64_t)mod[i] * me;
					d[i - 1] = (int32_t)cd & M30;
					e[i - 1] = (int32_t)ce & M30;
					cd >>= 30;
					ce >>= 30;
				}
				d[L - 1] = (int32_t)cd;
				e[L - 1] = (int32_t)ce;
			}
			{ /* (f, g) <- t (f, g) / 2^30, exact */
				int64_t cf = u * f[0] + v * g[0], cg = q * f[0] + rr * g[0];
				cf >>= 30;
				cg >>= 30;
				uint32_t acc = 0;
#pragma unroll
				for (int i = 1; i < L; i++) {
					cf += u * f[i] + v * g[i];
					cg += q * f[i] + rr * g[i];
					f[i - 1] = (int32_t)cf & M30;
					g[i - 1] = (int32_t)cg & M30;
					acc |= (uint32_t)g[i - 1];
					cf >>= 30;
					cg >>= 30;
				}
				f[L - 1] = (int32_t)cf;
				g[L - 1] = (int32_t)cg;
				g_nonzero = acc | (uint32_t)g[L - 1];
			}
		}
		if (g_nonzero) { /* unreachable by the step bound; keeps the result right no matter what */
			inv_fermat(r, a);
			return;
		}
		/* x^-1 = f * d with f = +-1 (f = m only for x = 0, where d = 0): negate d if f < 0, then bring it into [0, m) */
		{
			const int32_t sf = f[L - 1] >> 31;
			int32_t carry = 0;
#pragma unroll
			for (int i = 0; i < L; i++) { /* d <- (d ^ sf) - sf, limb-wise with carries */
				int32_t vv = (d[i] ^ sf) - sf + carry;
				if (i < L - 1) {
					carry = vv >> 30;
					vv &= M30;
				}
				d[i] = vv;
			}
			/* (d ^ sf) on the lower limbs complements 30-bit fields: (x ^ -1) - (-1) = -x holds limb-wise because the
			 * arithmetic shift of the carry propagates the borrow */
#pragma unroll 1
			for (int rep = 0; rep < 2; rep++) { /* d in (-2m, 2m) -> add m while negative (at most twice) */
				const int32_t neg = d[L - 1] >> 31;
				carry = 0;
#pragma unroll
				for (int i = 0; i < L; i++) {
					int32_t vv = d[i] + (mod[i] & neg) + carry;
					if (i < L - 1) {
						carry = vv >> 30;
						vv &= M30;
					}
					d[i] = vv;
				}
			}
			{ /* and subtract m once if d >= m (d in [0, 2m) after a negation of a value in (-m, 0]... (-2m, m)) */
				int32_t tmp[L];
				carry = 0;
#pragma unroll
				for (int i = 0; i < L; i++) {
					int32_t vv = d[i] - mod[i] + carry;
					if (i < L - 1) {
						carry = vv >> 30;
						vv &= M30;
					}
					tmp[i] = vv;
				}
				const int32_t keep = tmp[L - 1] >> 31; /* negative: d < m, keep d */
#pragma unroll
				for (int i = 0; i < L; i++) d[i] = (d[i] & keep) | (tmp[i] & ~keep);
			}
		}
		/* 30-bit limbs -> 32-bit words: (aR)^-1 as a plain integer in [0, m) */
		E xi;
#pragma unroll
		for (int w = 0; w < N; w++) {
			const int bit = 32 * w, i = bit / 30, sh = bit % 30;
			uint64_t lo = (i < L) ? (uint64_t)(uint32_t)d[i < L ? i : 0] : 0u;
			uint64_t mid = (i + 1 < L) ? (uint64_t)(uint32_t)d[i + 1 < L ? i + 1 : 0] : 0u;
			uint64_t hi = (i + 2 < L) ? (uint64_t)(uint32_t)d[i + 2 < L ? i + 2 : 0] : 0u;
			/* bits [sh, sh + 32) of lo | mid << 30 | hi << 60 */
			uint64_t v = (lo >> sh) | (mid << (30 - sh));
			if (sh > 28) v |= hi << (60 - sh);
			xi.w[w] = (uint32_t)v;
		}
		/* (aR)^-1 -> a^-1 R: multiply by R^3 (two Montgomery products: RR*RR = R^3, then xi*R^3 = a^-1 R) */
		E rr2, r3;
#pragma unroll
		for (int i = 0; i < N; i++) rr2.w[i] = F::RR(i);
		mul(r3, rr2, rr2);
		mul(r, xi, r3);
	}

	/*
	 * r = a^(m-2) (Montgomery in, Montgomery out): Fermat inversion, 4-bit fixed window over the constant exponent
	 * (fp_inv, fp/fp_mul.c:51 -> nn_mod_pow_redc, nn/nn_mod_pow.c:39 is a bit-by-bit ladder; same result).
	 * a == 0 gives 0.  Kept as the cross-check of inv() in the tests and as its unreachable fall-back.
	 */
	static ECC_HD void inv_fermat(E &r, const E &a)
	{
		E tbl[16];
		set_one(tbl[0]);
		tbl[1] = a;
#pragma unroll 1
		for (int i = 2; i < 16; i++) mul(tbl[i], tbl[i - 1], a);
		E acc;
		set_one(acc);
#pragma unroll 1
		for (int wi = N - 1; wi >= 0; wi--) {
			uint32_t ew = pm2_word(wi);
#pragma unroll 1
			for (int nb = 7; nb >= 0; nb--) {
#pragma unroll 1
				for (int q = 0; q < 4; q++) sqr(acc, acc);
				uint32_t d = (ew >> (4 * nb)) & 15u;
				mul(acc, acc, tbl[d]);
			}
		}
		r = acc;
	}

	/*
	 * r = a^((m+1)/4) (Montgomery in, Montgomery out): for a prime m = 3 mod 4 this is a square root of a whenever a
	 * is a square; returns r^2 == a.  4-bit fixed window over the constant exponent (m >> 2) + 1.  The reference's
	 * fp_sqrt (fp/fp_sqrt.c, Tonelli-Shanks) returns the same pair {r, m - r}; callers pick by parity.
	 */
	static ECC_HD bool sqrt_3mod4(E &r, const E &a)
	{
		uint32_t ex[N];
		uint64_t cy = 1;
#pragma unroll
		for (int i = 0; i < N; i++) {
			const uint32_t hi = i + 1 < N ? F::P(i + 1 < N ? i + 1 : 0) : 0u;
			const uint64_t t = (uint64_t)((F::P(i) >> 2) | (hi << 30)) + cy;
			ex[i] = (uint32_t)t;
			cy = t >> 32;
		}
		E tbl[16];
		set_one(tbl[0]);
		tbl[1] = a;
#pragma unroll 1
		for (int i = 2; i < 16; i++) mul(tbl[i], tbl[i - 1], a);
		E acc;
		set_one(acc);
#pragma unroll 1
		for (int wi = N - 1; wi >= 0; wi--) {
			uint32_t ew = 0;
#pragma unroll
			for (int k = 0; k < N; k++) ew = (k == wi) ? ex[k] : ew;
#pragma unroll 1
			for (int nb = 7; nb >= 0; nb--) {
#pragma unroll 1
				for (int q = 0; q < 4; q++) sqr(acc, acc);
				mul(acc, acc, tbl[(ew >> (4 * nb)) & 15u]);
			}
		}
		r = acc;
		E chk;
		sqr(chk, acc);
		return eq(chk, a);
	}

	/*
	 * r = the root of a that the reference's fp_sqrt returns FIRST (fp/fp_sqrt.c; the second is m - r), when a is
	 * a square; returns whether it is.  Montgomery in, Montgomery out; a == 0 gives 0 (:153-160).  Fp tags only.
	 *   m = 3 mod 4 (SQRT_S == 1): a^((m+1)/4), the reference's shortcut (:184-193), by sqrt_3mod4;
	 *   otherwise: Tonelli-Shanks restated step by step (:194-253) with the reference's constants, m - 1 = Q * 2^S and
	 *   c = z^Q for z its smallest non-residue counting up from 0 (tools/gen_curve_constants.py).  Which root comes out
	 *   depends on every factor the loop multiplies in, so the loop makes the reference's choices, not just any.
	 * `loops` (optional) receives the number of trips through the main loop.  Not constant time, like the reference.
	 */
	static ECC_HD bool sqrt(E &r, const E &a, int *loops = nullptr)
	{
		if (loops) *loops = 0;
		if (F::SQRT_S == 1) return sqrt_3mod4(r, a);
		if (is_zero(a)) {
			set_zero(r);
			return true;
		}
		E x, t, c, b, tmp, one;
		pow_sqrt_qh(x, a); /* a^((Q-1)/2) */
		mul(r, x, a);      /* r = a^((Q+1)/2) (:201-203) */
		mul(t, r, x);      /* t = a^Q (:204) */
		set_one(one);
		/* Legendre symbol (:162-166): a^((m-1)/2) = t^(2^(S-1)) must be 1 */
		tmp = t;
#pragma unroll 1
		for (int k = 0; k < F::SQRT_S - 1; k++) sqr(tmp, tmp);
		if (!eq(tmp, one)) return false;
#pragma unroll
		for (int i = 0; i < N; i++) c.w[i] = F::SQRT_C(i);
		int m = F::SQRT_S;
#pragma unroll 1
		while (!eq(t, one)) { /* (:209-253) */
			int i = 1;
			sqr(tmp, t);
#pragma unroll 1
			while (!eq(tmp, one) && i < m) { /* lowest i in (0, m) with t^(2^i) == 1; exists because a is a square */
				sqr(tmp, tmp);
				i++;
			}
			b = c; /* b = c^(2^(m-i-1)) */
#pragma unroll 1
			for (int k = 0; k < m - i - 1; k++) sqr(b, b);
			mul(r, r, b);
			sqr(c, b);
			mul(t, t, c);
			m = i;
			if (loops) ++*loops;
		}
		return true;
	}

      private:
	/* r = a^((Q-1)/2) for the Tonelli-Shanks constant SQRT_QH: 4-bit fixed window, as in sqrt_3mod4 */
	static ECC_HD void pow_sqrt_qh(E &r, const E &a)
	{
		E tbl[16];
		set_one(tbl[0]);
		tbl[1] = a;
#pragma unroll 1
		for (int i = 2; i < 16; i++) mul(tbl[i], tbl[i - 1], a);
		E acc;
		set_one(acc);
#pragma unroll 1
		for (int wi = N - 1; wi >= 0; wi--) {
			uint32_t ew = 0;
#pragma unroll
			for (int k = 0; k < N; k++) ew = (k == wi) ? F::SQRT_QH(k) : ew;
#pragma unroll 1
			for (int nb = 7; nb >= 0; nb--) {
#pragma unroll 1
				for (int q = 0; q < 4; q++) sqr(acc, acc);
				mul(acc, acc, tbl[(ew >> (4 * nb)) & 15u]);
			}
		}
		r = acc;
	}

	static ECC_HD uint32_t pm2_word(int i)
	{
		uint32_t v = 0;
#pragma unroll
		for (int k = 0; k < N; k++) v = (k == i) ? F::PM2(k) : v;
		return v;
	}
};

} // namespace eccb200
