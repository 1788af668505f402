/*
 * ec.cuh — short-Weierstrass group law on the device (replaces the reference's src/curves/prj_pt.c hot path).
 *
 * The reference computes prj_pt_mul with a masked Montgomery ladder over the Renes-Costello-Batina complete
 * addition in homogeneous projective coordinates (curves/prj_pt.c:971-1071, :1569-1720): 513 complete additions
 * = 8 724 field multiplications per 256-bit scalar.  Its result is only defined up to the projective class (the
 * input is blinded with a random lambda, :1266-1291), i.e. by the affine point.  The device is therefore free
 * to use a different algorithm as long as the affine output / infinity flag / error code agree:
 *
 *   - Jacobian coordinates (X/Z^2, Y/Z^3), a = -3 doubling (dbl-2001-b, 3M+5S), general add (12M+4S) and mixed
 *     add with an affine operand (8M+3S);
 *   - every exceptional case of the incomplete formulas is handled explicitly (P = inf, Q = inf, P = Q -> double,
 *     P = -Q -> inf), so the result is the group-law result for ALL inputs, like the reference's complete formulas;
 *   - fixed base (k*G): comb over a precomputed affine table T[i][d] = d * 2^(w*i) * G, one mixed add per
 *     window, no doublings (K1);
 *   - variable base (k*P): signed 4-bit fixed window, 8-entry Jacobian table per thread (K2).
 *
 * The three curves of BASELINE.json have a = p - 3 (curves/known/ec_params_secp256r1.h:78-83, ..._frp256v1.h:84-89,
 * ..._secp384r1.h) and use the a = -3 doubling; the additional curves (Brainpool P256r1 / P384r1: generic a,
 * secp256k1: a = 0) select their doubling through Curve::A_KIND (tools/gen_curve_constants.py).
 */
#pragma once
#include "fp.cuh"
#include "sha2.cuh"
#include "sm3.cuh"
#include "hmac.cuh"
#include "belt.cuh"
#include "bash.cuh"

namespace eccb200 {

template <class C> struct Jac {
	Fe<C::N> X, Y, Z; /* Z == 0 <=> point at infinity (prj_pt_iszero, curves/prj_pt.c:107) */
};

template <class C> struct Aff {
	Fe<C::N> x, y; /* Montgomery form */
};

template <class C> struct EC {
	static constexpr int N = C::N;
	typedef Field<typename C::Fp> F;
	typedef Fe<N> E;
	typedef Jac<C> J;
	typedef Aff<C> A;

	static ECC_HD void set_inf(J &p)
	{
		F::set_one(p.X);
		F::set_one(p.Y);
		F::set_zero(p.Z);
	}
	static ECC_HD bool is_inf(const J &p) { return F::is_zero(p.Z); }

	static ECC_HD void from_affine(J &p, const A &a)
	{
		p.X = a.x;
		p.Y = a.y;
		F::set_one(p.Z);
	}

	static ECC_HD void load_a(E &r)
	{
#pragma unroll
		for (int i = 0; i < N; i++) r.w[i] = C::A_MONT(i);
	}

	/* u = x^3 + a x + b (Montgomery form): the right-hand side of the curve equation */
	static ECC_HD void curve_rhs(E &u, const E &x)
	{
		E t, b;
		F::sqr(t, x);
		F::mul(u, t, x);      /* x^3 */
		if (C::A_KIND == 0) {
			F::add(t, x, x);
			F::add(t, t, x);  /* 3x */
			F::sub(u, u, t);
		} else if (C::A_KIND == 2) {
			E am;
			load_a(am);
			F::mul(t, am, x);
			F::add(u, u, t);
		}
#pragma unroll
		for (int i = 0; i < N; i++) b.w[i] = C::B_MONT(i);
		F::add(u, u, b);
	}

	/* y^2 == x^3 + a x + b (all Montgomery form); affine form of prj_pt_is_on_curve (curves/prj_pt.c:144-190) */
	static ECC_HD bool on_curve(const A &a)
	{
		E t, u;
		curve_rhs(u, a.x);
		F::sqr(t, a.y);
		return F::eq(t, u);
	}

	/* Out-of-line copy of dbl for the exceptional (P == Q) branches of the additions: keeps the rarely taken
	 * path from being inlined into every hot loop. */
	static ECC_NOINLINE void dbl_slow(J &r, const J &p) { dbl(r, p); }

	/* Jacobian doubling, r may alias p, inf -> inf (Z3 = 0).  Three formulas selected at compile time by the curve:
	 * a = -3 (dbl-2001-b, 3M + 5S: the three curves of BASELINE.json), a = 0 (dbl-2009-l, 2M + 5S: secp256k1) and
	 * generic a (dbl-2007-bl, 2M + 8S: Brainpool). */
	static ECC_HD void dbl(J &r, const J &p)
	{
		if (C::A_KIND == 1) {
			E a_, b_, c_, d_, e_, f_, t;
			F::sqr(a_, p.X);
			F::sqr(b_, p.Y);
			F::sqr(c_, b_);
			F::add(t, p.X, b_);
			F::sqr(d_, t);
			F::sub(d_, d_, a_);
			F::sub(d_, d_, c_);
			F::add(d_, d_, d_);      /* D = 2((X+B)^2 - A - C) */
			F::add(e_, a_, a_);
			F::add(e_, e_, a_);      /* E = 3A */
			F::sqr(f_, e_);
			F::mul(t, p.Y, p.Z);
			F::add(r.Z, t, t);       /* Z3 = 2YZ */
			F::sub(f_, f_, d_);
			F::sub(r.X, f_, d_);     /* X3 = F - 2D */
			F::sub(t, d_, r.X);
			F::mul(f_, e_, t);
			F::add(c_, c_, c_);
			F::add(c_, c_, c_);
			F::add(c_, c_, c_);      /* 8C */
			F::sub(r.Y, f_, c_);
			return;
		}
		if (C::A_KIND == 2) {
			E xx, yy, yyyy, zz, s_, m_, t, am;
			F::sqr(xx, p.X);
			F::sqr(yy, p.Y);
			F::sqr(yyyy, yy);
			F::sqr(zz, p.Z);
			F::add(t, p.X, yy);
			F::sqr(s_, t);
			F::sub(s_, s_, xx);
			F::sub(s_, s_, yyyy);
			F::add(s_, s_, s_);      /* S = 2((X+YY)^2 - XX - YYYY) */
			F::add(t, p.Y, p.Z);
			F::sqr(r.Z, t);
			F::sub(r.Z, r.Z, yy);
			F::sub(r.Z, r.Z, zz);    /* Z3 = (Y+Z)^2 - YY - ZZ */
			F::sqr(t, zz);
			load_a(am);
			F::mul(m_, am, t);       /* a ZZ^2 */
			F::add(t, xx, xx);
			F::add(t, t, xx);
			F::add(m_, m_, t);       /* M = 3XX + a ZZ^2 */
			F::sqr(t, m_);
			F::sub(t, t, s_);
			F::sub(r.X, t, s_);      /* X3 = M^2 - 2S */
			F::sub(t, s_, r.X);
			F::mul(s_, m_, t);
			F::add(yyyy, yyyy, yyyy);
			F::add(yyyy, yyyy, yyyy);
			F::add(yyyy, yyyy, yyyy); /* 8 YYYY */
			F::sub(r.Y, s_, yyyy);
			return;
		}
		E delta, gamma, beta, alpha, t0, t1;
		F::sqr(delta, p.Z);
		F::sqr(gamma, p.Y);
		F::mul(beta, p.X, gamma);
		F::sub(t0, p.X, delta);
		F::add(t1, p.X, delta);
		F::mul(alpha, t0, t1);
		F::add(t0, alpha, alpha);
		F::add(alpha, t0, alpha); /* 3 (X-delta)(X+delta) */
		F::add(t1, p.Y, p.Z);
		F::sqr(t0, t1);
		F::sub(t0, t0, gamma);
		F::sub(r.Z, t0, delta);   /* Z3 = (Y+Z)^2 - gamma - delta */
		F::add(t0, beta, beta);
		F::add(t0, t0, t0);       /* 4 beta */
		F::add(t1, t0, t0);       /* 8 beta */
		F::sqr(r.X, alpha);
		F::sub(r.X, r.X, t1);     /* X3 = alpha^2 - 8 beta */
		F::sub(t0, t0, r.X);
		F::mul(t1, alpha, t0);
		F::sqr(t0, gamma);
		F::add(t0, t0, t0);
		F::add(t0, t0, t0);
		F::add(t0, t0, t0);       /* 8 gamma^2 */
		F::sub(r.Y, t1, t0);
	}

	/*
	 * r = p + q, q affine (Z2 = 1): 8M + 3S.  Exceptional cases resolved explicitly so that the result equals the
	 * group law for every input, matching what prj_pt_add's complete formulas give (curves/prj_pt.c:1204).
	 */
	static ECC_HD void add_mixed(J &r, const J &p, const A &q)
	{
		E z1z1, u2, s2, h, rr, hh, hhh, v, t;
		F::sqr(z1z1, p.Z);
		F::mul(u2, q.x, z1z1);
		F::mul(t, q.y, p.Z);
		F::mul(s2, t, z1z1);
		F::sub(h, u2, p.X);
		F::sub(rr, s2, p.Y);
		bool p_inf = F::is_zero(p.Z);
		bool h0 = F::is_zero(h);
		if (p_inf) {
			from_affine(r, q);
			return;
		}
		if (h0) {
			if (F::is_zero(rr)) {
				J qq;
				from_affine(qq, q);
				dbl_slow(r, qq);
			} else {
				set_inf(r);
			}
			return;
		}
		F::sqr(hh, h);
		F::mul(hhh, h, hh);
		F::mul(v, p.X, hh);
		E x3, y3, z3;
		F::sqr(x3, rr);
		F::sub(x3, x3, hhh);
		F::sub(x3, x3, v);
		F::sub(x3, x3, v);
		F::sub(t, v, x3);
		F::mul(y3, rr, t);
		F::mul(t, p.Y, hhh);
		F::sub(y3, y3, t);
		F::mul(z3, p.Z, h);
		r.X = x3;
		r.Y = y3;
		r.Z = z3;
	}

	/* r = p + q, both Jacobian (add-1998-cmo-2): 12M + 4S, exceptional cases resolved explicitly. */
	static ECC_HD void add_full(J &r, const J &p, const J &q)
	{
		E z1z1, z2z2, u1, u2, s1, s2, h, rr, hh, hhh, v, t;
		F::sqr(z1z1, p.Z);
		F::sqr(z2z2, q.Z);
		F::mul(u1, p.X, z2z2);
		F::mul(u2, q.X, z1z1);
		F::mul(t, p.Y, q.Z);
		F::mul(s1, t, z2z2);
		F::mul(t, q.Y, p.Z);
		F::mul(s2, t, z1z1);
		F::sub(h, u2, u1);
		F::sub(rr, s2, s1);
		bool p_inf = F::is_zero(p.Z), q_inf = F::is_zero(q.Z);
		if (p_inf) {
			r = q;
			return;
		}
		if (q_inf) {
			r = p;
			return;
		}
		if (F::is_zero(h)) {
			if (F::is_zero(rr)) {
				J pp = p;
				dbl_slow(r, pp);
			} else {
				set_inf(r);
			}
			return;
		}
		F::sqr(hh, h);
		F::mul(hhh, h, hh);
		F::mul(v, u1, hh);
		E x3, y3, z3;
		F::sqr(x3, rr);
		F::sub(x3, x3, hhh);
		F::sub(x3, x3, v);
		F::sub(x3, x3, v);
		F::sub(t, v, x3);
		F::mul(y3, rr, t);
		F::mul(t, s1, hhh);
		F::sub(y3, y3, t);
		F::mul(t, p.Z, q.Z);
		F::mul(z3, t, h);
		r.X = x3;
		r.Y = y3;
		r.Z = z3;
	}

	/* out-of-line copy of add_full for code that adds up many points outside the hot loops (bucket reduction of the
	 * multi-scalar multiplication): one body per kernel instead of one per call site */
	static ECC_NOINLINE void add_full_ool(J &r, const J &p, const J &q) { add_full(r, p, q); }

	static ECC_HD void neg(J &r, const J &p)
	{
		r.X = p.X;
		r.Z = p.Z;
		F::neg(r.Y, p.Y);
	}

	/*
	 * Extended Jacobian ("XYZZ") accumulator of the fixed-base comb: x = X/ZZ, y = Y/ZZZ with ZZ^3 == ZZZ^2;
	 * ZZ == 0 <=> point at infinity.  Mixed addition madd-2008-s: 8M + 2S (one squaring less than the Jacobian
	 * mixed addition, because Z^2 and Z^3 are carried instead of recomputed).  Exceptional cases as in add_mixed.
	 */
	struct XZ {
		E X, Y, ZZ, ZZZ;
	};
	static ECC_HD void xz_set_inf(XZ &p)
	{
		F::set_one(p.X);
		F::set_one(p.Y);
		F::set_zero(p.ZZ);
		F::set_zero(p.ZZZ);
	}
	static ECC_HD void xz_from_affine(XZ &p, const A &a)
	{
		p.X = a.x;
		p.Y = a.y;
		F::set_one(p.ZZ);
		F::set_one(p.ZZZ);
	}
	/* rarely taken P == Q branch of xz_add_mixed: 2Q through the Jacobian doubling, then ZZ = Z^2, ZZZ = Z^3 */
	static ECC_NOINLINE void xz_dbl_affine_slow(XZ &r, const A &q)
	{
		J qq, d;
		from_affine(qq, q);
		dbl(d, qq);
		r.X = d.X;
		r.Y = d.Y;
		F::sqr(r.ZZ, d.Z);
		F::mul(r.ZZZ, r.ZZ, d.Z);
	}
	/* the i-th of the eight products of xz_add_mixed: the first ECC_K1_OOL_MULS of them call the out-of-line copy when
	 * the translation unit inlines the multiplier (K1), see Field::mul_ool */
#ifndef ECC_K1_OOL_MULS
#define ECC_K1_OOL_MULS 0
#endif
	template <int I> static ECC_HD void xz_mul(E &r, const E &a, const E &b)
	{
#if defined(ECC_INLINE_MUL)
		if (I < ECC_K1_OOL_MULS) {
			F::mul_ool(r, a, b);
			return;
		}
#endif
		F::mul(r, a, b);
	}
	static ECC_HD void xz_add_mixed(XZ &r, const XZ &p, const A &q)
	{
		E u2, s2, pp_, rr, ppp, qv, t;
		if (F::is_zero(p.ZZ)) { /* first non-zero window of the comb */
			xz_from_affine(r, q);
			return;
		}
		xz_mul<0>(u2, q.x, p.ZZ);
		xz_mul<1>(s2, q.y, p.ZZZ);
		F::sub(pp_, u2, p.X); /* P */
		F::sub(rr, s2, p.Y);  /* R */
		if (F::is_zero(pp_)) {
			if (F::is_zero(rr)) xz_dbl_affine_slow(r, q);
			else xz_set_inf(r);
			return;
		}
		E x3, y3;
		F::sqr(t, pp_);        /* PP */
		xz_mul<2>(ppp, pp_, t);   /* PPP */
		xz_mul<3>(qv, p.X, t);    /* Q = X1 * PP */
		E zz3;
		xz_mul<4>(zz3, p.ZZ, t);  /* ZZ3 = ZZ1 * PP */
		F::sqr(x3, rr);
		F::sub(x3, x3, ppp);
		F::sub(x3, x3, qv);
		F::sub(x3, x3, qv);    /* X3 = R^2 - PPP - 2Q */
		F::sub(t, qv, x3);
		xz_mul<5>(y3, rr, t);
		xz_mul<6>(t, p.Y, ppp);
		F::sub(y3, y3, t);     /* Y3 = R (Q - X3) - Y1 PPP */
		xz_mul<7>(t, p.ZZZ, ppp); /* ZZZ3 = ZZZ1 * PPP */
		r.ZZZ = t;
		r.ZZ = zz3;
		r.X = x3;
		r.Y = y3;
	}
	/* XYZZ -> Jacobian with Z' = ZZ: x = X ZZ / ZZ^2, y = Y ZZZ / ZZ^3 (ZZ^3 == ZZZ^2).  2M. */
	static ECC_HD void xz_to_jac(J &r, const XZ &p)
	{
		F::mul(r.X, p.X, p.ZZ);
		F::mul(r.Y, p.Y, p.ZZZ);
		r.Z = p.ZZ;
	}
};

/* ---------------------------------------------------------------------------------------------- wire format */

/* len big-endian bytes (libecc wire format, nn_init_from_buf nn/nn.c:479) -> N little-endian 32-bit words; portable
 * byte-wise form for the host build of the tests (the kernels use load_wire / store_wire of kernels.cuh) */
template <int N> ECC_HD void load_be(Fe<N> &r, const uint8_t *buf, int len = 4 * N)
{
	for (int i = 0; i < N; i++) r.w[i] = 0;
	for (int j = 0; j < len && j < 4 * N; j++) r.w[j >> 2] |= (uint32_t)buf[len - 1 - j] << (8 * (j & 3));
}

/* nn_export_to_buf (nn/nn.c:511) */
template <int N> ECC_HD void store_be(uint8_t *buf, const Fe<N> &a, int len = 4 * N)
{
	for (int j = 0; j < len; j++) buf[len - 1 - j] = (j < 4 * N) ? (uint8_t)(a.w[j >> 2] >> (8 * (j & 3))) : 0;
}

/* ---------------------------------------------------------------------------------------------- scalars */

/* Reduce a raw wire scalar (QLEN bytes, so < 2^(8*QLEN)) modulo q: the reference's ladder yields (k mod q)*P for any
 * k (curves/prj_pt.c:1591-1619).  Shifted conditional subtractions of q << sh, sh = 8*QLEN - bitlen(q) .. 0: a single
 * step for the 256/384-bit curves (2^(8*QLEN) < 2q), eight for the 521-bit one (66-byte scalars, q < 2^521). */
template <class C> ECC_HD void scalar_reduce(Fe<C::N> &k)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N;
	constexpr int SH = 8 * C::QLEN - C::QBITS;
	static_assert(SH >= 0 && SH < 32 && C::QBITS + SH <= 32 * N, "scalar_reduce: q << SH must fit N words");
#pragma unroll
	for (int sh = SH; sh > 0; sh--) {
		uint32_t d[N];
		uint64_t bw = 0;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint32_t lo = (i > 0) ? C::Fq::P(i - 1) : 0u;
			uint32_t qs = (C::Fq::P(i) << sh) | (lo >> (32 - sh)); /* word i of q << sh */
			uint64_t t = (uint64_t)k.w[i] - qs - bw;
			d[i] = (uint32_t)t;
			bw = (t >> 32) & 1;
		}
#pragma unroll
		for (int i = 0; i < N; i++) k.w[i] = bw ? k.w[i] : d[i];
	}
	for (int it = 0; it < 2; it++) Fq::cond_sub_mod(k, k);
}

/* 64-bit funnel shifts on word pairs (static register indices only: the scalar walks through the window loop by
 * being shifted, never by dynamic indexing — see DESIGN.md §8, "nvcc stack-colouring hazard"). */
ECC_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, int sh) /* low word of ((hi:lo) >> sh), 0 <= sh < 32 */
{
#if defined(__CUDA_ARCH__)
	return __funnelshift_r(lo, hi, sh);
#else
	return (uint32_t)((((uint64_t)hi << 32) | lo) >> sh);
#endif
}
ECC_HD uint32_t funnel_l(uint32_t lo, uint32_t hi, int sh) /* high word of ((hi:lo) << sh), 0 <= sh < 32 */
{
#if defined(__CUDA_ARCH__)
	return __funnelshift_l(lo, hi, sh);
#else
	return (uint32_t)(((((uint64_t)hi << 32) | lo) << sh) >> 32);
#endif
}

/* k >>= w (0 < w < 32) */
template <int N> ECC_HD void shift_right(Fe<N> &k, int w)
{
#pragma unroll
	for (int j = 0; j < N - 1; j++) k.w[j] = funnel_r(k.w[j], k.w[j + 1], w);
	k.w[N - 1] >>= w;
}

/*
 * Fixed-base comb: acc = sum_i T[i][digit_i(k)],  T[i][d] = d * 2^(w*i) * G  (affine, Montgomery form, entry
 * (i << w) + d; d == 0 unused), 4 <= w <= 26.  One mixed addition per non-zero window, no doublings.  k must be < q.
 * For k < q the accumulator before window i is (k mod 2^(w*i))*G with 0 <= k mod 2^(w*i) < 2^(w*i) <= d*2^(w*i) < q,
 * so the add never meets P = +-Q; add_mixed resolves those cases anyway.
 */
template <class C> ECC_HD void load_table_entry(Aff<C> &t, const uint32_t *__restrict__ table, size_t e)
{
	constexpr int N = C::N;
	const uint32_t *base = table + e * (2 * N);
#if defined(__CUDA_ARCH__)
	if (N % 4 == 0) {
		const uint4 *src = reinterpret_cast<const uint4 *>(base);
#pragma unroll
		for (int j = 0; j < N / 4; j++) {
			uint4 v = __ldg(src + j);
			t.x.w[4 * j] = v.x;
			t.x.w[4 * j + 1] = v.y;
			t.x.w[4 * j + 2] = v.z;
			t.x.w[4 * j + 3] = v.w;
		}
#pragma unroll
		for (int j = 0; j < N / 4; j++) {
			uint4 v = __ldg(src + N / 4 + j);
			t.y.w[4 * j] = v.x;
			t.y.w[4 * j + 1] = v.y;
			t.y.w[4 * j + 2] = v.z;
			t.y.w[4 * j + 3] = v.w;
		}
	} else { /* N even: 8-byte loads */
		const uint2 *src = reinterpret_cast<const uint2 *>(base);
#pragma unroll
		for (int j = 0; j < N / 2; j++) {
			uint2 v = __ldg(src + j);
			t.x.w[2 * j] = v.x;
			t.x.w[2 * j + 1] = v.y;
		}
#pragma unroll
		for (int j = 0; j < N / 2; j++) {
			uint2 v = __ldg(src + N / 2 + j);
			t.y.w[2 * j] = v.x;
			t.y.w[2 * j + 1] = v.y;
		}
	}
#else
	for (int j = 0; j < N; j++) {
		t.x.w[j] = base[j];
		t.y.w[j] = base[N + j];
	}
#endif
}

template <class C> ECC_HD void comb_mul(Jac<C> &out, const Fe<C::N> &k, const uint32_t *__restrict__ table, int w)
{
	typedef EC<C> G;
	constexpr int N = C::N;
	typename G::XZ acc; /* extended Jacobian accumulator: 8M + 2S per window (xz_add_mixed) */
	G::xz_set_inf(acc);
	const int nwin = (C::QBITS + w - 1) / w;
	const uint32_t mask = (1u << w) - 1u;
	Fe<N> kk = k; /* consumed w bits at a time from the least significant end */
#pragma unroll 1
	for (int i = 0; i < nwin; i++) {
		uint32_t d = kk.w[0] & mask;
		shift_right<N>(kk, w);
#if defined(__CUDA_ARCH__) && defined(ECC_COMB_PREFETCH)
		/* the NEXT window's entry is requested into L2 while this window's addition runs: the gathers are random
		 * accesses into a table of tens of GB, i.e. DRAM latency on the critical path of every window otherwise */
		if (i + 1 < nwin) {
			const uint32_t nd = kk.w[0] & mask;
			const uint32_t *nxt = table + (((size_t)(i + 1) << w) + nd) * (2 * N);
			asm volatile("prefetch.global.L2 [%0];" ::"l"(nxt));
			if ((2 * N * 4) % 128 != 0 && (2 * N * 4) > 64) asm volatile("prefetch.global.L2 [%0];" ::"l"(nxt + 2 * N - 1));
		}
#endif
		if (d != 0) {
			Aff<C> t;
			load_table_entry<C>(t, table, ((size_t)i << w) + d);
			typename G::XZ r;
			G::xz_add_mixed(r, acc, t);
			acc = r;
		}
	}
	G::xz_to_jac(out, acc); /* (X ZZ, Y ZZZ, ZZ): the Jacobian form K4 / the verification tail expect */
}

/* One field inversion for the calling thread alone: the inverter of the host build of the tests and of the one-off
 * table construction.  K2 / K3 pass an inverter that shares ONE inversion among the 128 threads of the CTA
 * (cta_inverse_128, kernels.cuh); an inverter of that kind must be called by every thread of the CTA. */
template <class C> struct ThreadInverter {
	ECC_HD void operator()(Fe<C::N> &r, const Fe<C::N> &a) const { Field<typename C::Fp>::inv(r, a); }
};

/*
 * Variable base: acc = k*P (+ addend), P affine and on the curve, k < q.  Signed 4-bit fixed window:
 * K' = k + 0x88..8 (one 8 per nibble); digit_i = nibble_i(K') - 8 in [-8, 7], plus a top digit = the carry out.
 * Table tbl[j] = (j+1)*P, j = 0..7, built with 7 mixed additions and then made AFFINE with one inversion
 * (Montgomery's trick over the seven Z's, and the addend's): every window addition is a mixed one (8M + 3S instead of
 * 12M + 4S), for ~50 products of conversion plus the thread's share of the inverter.  None of the multiples is the
 * point at infinity (the group order is a prime > 8).  The optional addend (uG of an ECDSA verification,
 * sig/ecdsa_common.c:796) is converted by the same inversion and added by one extra trip through the loop body, so the
 * kernel holds a single inlined copy of the addition.
 */
template <class C, class Inv>
ECC_HD void window_mul(Jac<C> &acc, const Fe<C::N> &k, const Aff<C> &P, const Jac<C> *addend, const Inv &invert)
{
	typedef EC<C> G;
	typedef Field<typename C::Fp> F;
	constexpr int N = C::N;
	Jac<C> tbl[8]; /* after the conversion only X, Y are meaningful (affine) */
	G::from_affine(tbl[0], P);
#pragma unroll 1
	for (int j = 1; j < 8; j++) G::add_mixed(tbl[j], tbl[j - 1], P); /* j == 1 takes the P == Q (doubling) branch */

	/* simultaneous inversion of Z(2P) .. Z(8P) and of the addend's Z */
	const bool have_add = addend != nullptr && !G::is_inf(*addend);
	Aff<C> add_aff;
	{
		Fe<N> pre[7]; /* pre[j] = Z(2P) * ... * Z((j+2)P) */
		pre[0] = tbl[1].Z;
#pragma unroll 1
		for (int j = 2; j < 8; j++) F::mul(pre[j - 1], pre[j - 2], tbl[j].Z);
		Fe<N> tot = pre[6], inv, zi, zi2, zi3, t;
		if (have_add) F::mul(tot, pre[6], addend->Z);
		invert(inv, tot);
		if (have_add) {
			F::mul(zi, inv, pre[6]);
			F::mul(t, inv, addend->Z);
			inv = t;
			F::sqr(zi2, zi);
			F::mul(zi3, zi2, zi);
			F::mul(add_aff.x, addend->X, zi2);
			F::mul(add_aff.y, addend->Y, zi3);
		}
#pragma unroll 1
		for (int j = 7; j >= 1; j--) {
			if (j > 1) {
				F::mul(zi, inv, pre[j - 2]);
				F::mul(t, inv, tbl[j].Z);
				inv = t;
			} else {
				zi = inv;
			}
			F::sqr(zi2, zi);
			F::mul(zi3, zi2, zi);
			F::mul(t, tbl[j].X, zi2);
			tbl[j].X = t;
			F::mul(t, tbl[j].Y, zi3);
			tbl[j].Y = t;
		}
	}

	/* K' = k + 0x88..8 over the ND = ceil(bitlen(q)/4) nibbles a reduced scalar occupies; the carry lands in
	 * nibble ND (0 or 1).  K' is then moved to the top of the N words so that nibbles leave from the MSB end. */
	constexpr int ND = (C::QBITS + 3) / 4;
	constexpr int PAD = 32 * N - 4 * ND; /* unused high bits: 0 for 256/384-bit, 52 for the 521-bit curve */
	uint32_t kk[N];
	uint64_t c = 0;
#pragma unroll
	for (int i = 0; i < N; i++) {
		const int nib = ND - 8 * i; /* nibbles of this word below ND */
		const uint32_t eights = nib >= 8 ? 0x88888888u : (nib <= 0 ? 0u : (0x88888888u >> (4 * (8 - nib))));
		uint64_t s = (uint64_t)k.w[i] + eights + c;
		kk[i] = (uint32_t)s;
		c = s >> 32;
	}
	if (PAD > 0) {
		constexpr int WS = PAD / 32, BS = PAD % 32;
		constexpr int TW = (4 * ND) / 32 < N ? (4 * ND) / 32 : 0; /* (index clamp only for the dead PAD == 0 case) */
		c = (kk[TW] >> ((4 * ND) % 32)) & 1u; /* top digit */
#pragma unroll
		for (int j = N - 1; j >= 0; j--) {
			uint32_t hi = (j - WS >= 0) ? kk[j - WS] : 0u;
			uint32_t lo = (j - WS - 1 >= 0) ? kk[j - WS - 1] : 0u;
			kk[j] = BS ? funnel_l(lo, hi, BS) : hi;
		}
	}
	G::set_inf(acc);
	if (c) G::from_affine(acc, P); /* top digit (weight 16^ND) is 0 or 1 */
#pragma unroll 1
	for (int di = ND - 1; di >= -1; di--) {
		Aff<C> e;
		Jac<C> t;
		bool have;
		if (di >= 0) {
#pragma unroll 1
			for (int q = 0; q < 4; q++) G::dbl(acc, acc);
			int d = (int)(kk[N - 1] >> 28) - 8; /* most significant nibble, then K' <<= 4 */
#pragma unroll
			for (int j = N - 1; j > 0; j--) kk[j] = funnel_l(kk[j - 1], kk[j], 4);
			kk[0] <<= 4;
			int ad = d < 0 ? -d : d;
			have = d != 0;
			const Jac<C> &te = tbl[(ad - 1) & 7];
			e.x = te.X;
			e.y = te.Y;
			if (d < 0) F::neg(e.y, e.y);
		} else {
			have = have_add;
			if (have) e = add_aff;
		}
		if (have) {
			G::add_mixed(t, acc, e);
			acc = t;
		}
	}
}

template <class C>
ECC_HD void window_mul(Jac<C> &acc, const Fe<C::N> &k, const Aff<C> &P, const Jac<C> *addend = nullptr)
{
	window_mul<C>(acc, k, P, addend, ThreadInverter<C>());
}

/* ---------------------------------------------------------------------------------------------- ECDSA */

/*
 * e = leftmost min(8*hlen, bitlen(q)) bits of the digest as an integer, reduced mod q:
 * steps 3-4 of __ecdsa_verify_finalize (sig/ecdsa_common.c:760-777).  Byte loads: hlen is arbitrary.
 */
template <class C> ECC_HD void digest_to_scalar(Fe<C::N> &e, const uint8_t *h, uint32_t hlen)
{
	constexpr int N = C::N;
	uint32_t qbytes = (C::QBITS + 7) / 8;
	uint32_t take = hlen < qbytes ? hlen : qbytes;
#pragma unroll
	for (int i = 0; i < N; i++) e.w[i] = 0;
	for (uint32_t i = 0; i < take; i++) {
		uint32_t pos = take - 1 - i; /* byte significance */
		uint32_t v = (uint32_t)h[i] << (8 * (pos & 3));
#pragma unroll
		for (int j = 0; j < N; j++) e.w[j] |= (j == (int)(pos >> 2)) ? v : 0u;
	}
	int sh = (int)(8 * take) - C::QBITS; /* > 0 only when bitlen(q) is not a multiple of 8 */
	if (sh > 0) {
#pragma unroll
		for (int j = 0; j < N; j++) {
			uint32_t hi = (j + 1 < N) ? e.w[j + 1] : 0u;
			e.w[j] = (e.w[j] >> sh) | (hi << (32 - sh));
		}
	}
	scalar_reduce<C>(e);
}

/*
 * The deterministic ECDSA nonce of RFC 6979 §3.2 as the reference derives it (__ecdsa_rfc6979_nonce,
 * sig/ecdsa_common.c:48-169), with HMAC over hash_type (hmac.cuh) and h the hsize-byte digest H(m):
 *   b, c. V = 0x01 .. 0x01, K = 0x00 .. 0x00 (hsize bytes each)                                          (:74-75)
 *   d.    K = HMAC_K(V || 0x00 || int2octets(x) || bits2octets(h)), bits2octets(h) = ((h >> max(0, 8*hsize -
 *         qbits)) mod q) on qlen bytes                                                                     (:81-97)
 *   e-g.  V = HMAC_K(V); K = HMAC_K(V || 0x01 || x || bits2octets(h)); V = HMAC_K(V)                     (:100-116)
 *   h.    T = the V = HMAC_K(V) blocks until T has qbits bits, k = leftmost qbits bits of T; while k >= q,
 *         K = HMAC_K(V || 0x00), V = HMAC_K(V), and again                                                (:136-165)
 * x must be in [1, q-1].  The reference takes a k of 0 (it checks k >= q only); the signer reports that k as
 * ECCB200_ERR.  V || b || x || bits2octets(h) is the two-segment source: V, then b || x || bits2octets(h) in one
 * thread-held buffer.  Returns the number of k >= q retries (the host tests count them).
 */
template <class C>
ECC_D int rfc6979_nonce(Fe<C::N> &k, int hash_type, const Fe<C::N> &x, const uint8_t *h, uint32_t hsize)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N, QL = C::QLEN, SH = 8 * C::QLEN - C::QBITS;
	uint8_t V[64], K[64], bxh[1 + 2 * QL], T[QL];
	for (uint32_t i = 0; i < hsize; i++) {
		V[i] = 0x01;
		K[i] = 0x00;
	}
	Fe<N> h1;
	digest_to_scalar<C>(h1, h, hsize); /* leftmost min(8*hsize, qbits) bits, mod q */
	bxh[0] = 0x00;
	store_be<N>(bxh + 1, x, QL);
	store_be<N>(bxh + 1 + QL, h1, QL);
	const uint64_t mlen = (uint64_t)hsize + 1 + 2 * QL;
	hmac_src(hash_type, K, hsize, Seg2{ V, hsize, bxh }, mlen, K);         /* d */
	hmac_src(hash_type, K, hsize, ByteSpan{ V }, hsize, V);                 /* e */
	bxh[0] = 0x01;
	hmac_src(hash_type, K, hsize, Seg2{ V, hsize, bxh }, mlen, K);         /* f */
	hmac_src(hash_type, K, hsize, ByteSpan{ V }, hsize, V);                 /* g */
	const uint8_t zero = 0x00;
	for (int retries = 0;; retries++) {
		for (int t = 0; t < QL; t += (int)hsize) {                      /* h.2 */
			hmac_src(hash_type, K, hsize, ByteSpan{ V }, hsize, V);
			for (int i = 0; i < (int)hsize && t + i < QL; i++) T[t + i] = V[i];
		}
		load_be<N>(k, T, QL);                                          /* h.3: bits2int(T) */
		if (SH > 0) {
#pragma unroll
			for (int j = 0; j < N; j++) {
				const uint32_t hi = (j + 1 < N) ? k.w[j + 1] : 0u;
				k.w[j] = (k.w[j] >> SH) | (hi << ((32 - SH) & 31));
			}
		}
		if (!Fq::geq_mod(k)) return retries;
		hmac_src(hash_type, K, hsize, Seg2{ V, hsize, &zero }, (uint64_t)hsize + 1, K);
		hmac_src(hash_type, K, hsize, ByteSpan{ V }, hsize, V);
	}
}

/* u = e * s^-1 mod q, v = r * s^-1 mod q (plain form): the mod-q scalar preparation of __ecdsa_verify_finalize
 * (sig/ecdsa_common.c:781-791: nn_modinv, nn_mod_mul), with s^-1 by Field::inv in the Montgomery domain of q. */
template <class C>
ECC_HD void ecdsa_uv(Fe<C::N> &u, Fe<C::N> &v, const Fe<C::N> &r, const Fe<C::N> &s, const Fe<C::N> &e)
{
	typedef Field<typename C::Fq> Fq;
	Fe<C::N> sm, wm;
	Fq::to_mont(sm, s);
	Fq::inv(wm, sm);   /* s^-1 * R mod q */
	Fq::mul(u, e, wm); /* (:786) */
	Fq::mul(v, r, wm); /* (:791) */
}

/*
 * ECDSA verification of one signature (r, s) on the reduced digest e under the public key Y (affine, validated,
 * Montgomery form).  Returns 0 = valid; 1 = r/s out of range, 2 = W' at infinity, 3 = r' != r (all map to -1).  Follows __ecdsa_verify_init's range checks (sig/ecdsa_common.c:653-658) and
 * __ecdsa_verify_finalize steps 5-10 (:781-810); differences that do not change the verdict:
 *   - s^-1 mod q by Field::inv (safegcd) in the Montgomery domain of q instead of nn_modinv's xgcd (:781);
 *   - W' = uG + vY stays Jacobian and "x(W') mod q == r" is tested without an inversion as X == c * Z^2 for the
 *     candidates c in {r, r+q} that are < p (:803-810);
 *   - uG through the comb table (K1), vY through the signed window (K2) instead of two ladders (:788,793).
 */
/* Steps 7-10 of __ecdsa_verify_finalize (sig/ecdsa_common.c:796-810) given u and v: W' = uG + vY, reject infinity,
 * accept iff x(W') mod q == r.  Returns 0 valid, 2 infinity, 3 mismatch. */
template <class C, class Inv>
ECC_HD int ecdsa_verify_tail(const Fe<C::N> &r, const Fe<C::N> &u, const Fe<C::N> &v_in, const Aff<C> &Y_in,
			     const uint32_t *__restrict__ table, int w, bool y_inf, const Inv &invert)
{
	typedef Field<typename C::Fp> F;
	constexpr int N = C::N;
	Jac<C> uG, W;
	comb_mul<C>(uG, u, table, w);
	/* A public key imported as the point at infinity (possible through the projective key formats,
	 * sig/ec_key.c:139): v*Y = infinity, exactly what the reference's complete formulas compute, so W' = uG.  The
	 * thread still walks the same code (v = 0 on a dummy base) because the inverter may be a CTA-wide one. */
	Fe<N> v = v_in;
	Aff<C> Y = Y_in;
	if (y_inf) {
#pragma unroll
		for (int i = 0; i < N; i++) {
			v.w[i] = 0;
			Y.x.w[i] = C::GX_MONT(i);
			Y.y.w[i] = C::GY_MONT(i);
		}
	}
	window_mul<C>(W, v, Y, &uG, invert); /* W' = vY + uG (:796) */
	if (EC<C>::is_inf(W)) return 2; /* (:799-800) */

	Fe<N> z2, c, t;
	F::sqr(z2, W.Z);
	bool match = false;
	if (!F::geq_mod(r)) { /* candidate x = r */
		F::to_mont(c, r);
		F::mul(t, c, z2);
		match = F::eq(t, W.X);
	}
	{ /* candidate x = r + q, when it is still a field element */
		Fe<N> rq;
		uint64_t cy = 0;
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint64_t sum = (uint64_t)r.w[i] + C::Fq::P(i) + cy;
			rq.w[i] = (uint32_t)sum;
			cy = sum >> 32;
		}
		if (cy == 0 && !F::geq_mod(rq)) {
			F::to_mont(c, rq);
			F::mul(t, c, z2);
			match = match || F::eq(t, W.X);
		}
	}
	return match ? 0 : 3;
}

template <class C>
ECC_HD int ecdsa_verify_tail(const Fe<C::N> &r, const Fe<C::N> &u, const Fe<C::N> &v, const Aff<C> &Y,
			     const uint32_t *__restrict__ table, int w, bool y_inf = false)
{
	return ecdsa_verify_tail<C>(r, u, v, Y, table, w, y_inf, ThreadInverter<C>());
}

/* ------------------------------------------------------------------------------------------ ECFSDSA (§8f.4) */

/*
 * h = OS2I(digest) mod q with the WHOLE digest (sig/ecfsdsa.c:590-592: nn_init_from_buf + nn_mod — no truncation to
 * bitlen(q), unlike ECDSA), any hlen.  Horner over chunks of 4N bytes, most significant first:
 * h <- h * 2^(32N) + chunk (mod q).  A chunk (any integer < R) is reduced by a round trip through the Montgomery
 * domain (x -> xR -> x mod q), and h * 2^(32N) mod q = h * R mod q is exactly to_mont(h).
 */
template <class C> ECC_HD void digest_full_mod_q(Fe<C::N> &e, const uint8_t *h, uint32_t hlen)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N;
	const uint32_t nchunks = (hlen + 4u * N - 1u) / (4u * N);
#pragma unroll
	for (int i = 0; i < N; i++) e.w[i] = 0;
	for (uint32_t c = nchunks; c-- > 0;) {
		Fe<N> ch, t;
#pragma unroll
		for (int i = 0; i < N; i++) ch.w[i] = 0;
		const uint32_t lo = c * 4u * N, hi = (lo + 4u * N < hlen) ? lo + 4u * N : hlen; /* byte significances */
		for (uint32_t pos = lo; pos < hi; pos++) {
			uint32_t v = (uint32_t)h[hlen - 1 - pos] << (8 * (pos & 3));
			int wi = (int)((pos - lo) >> 2);
#pragma unroll
			for (int j = 0; j < N; j++) ch.w[j] |= (j == wi) ? v : 0u;
		}
		if (c + 1 < nchunks) {
			Fq::to_mont(t, e);
			e = t;
		}
		Fq::to_mont(t, ch);
		Fq::from_mont(ch, t);
		Fq::add(e, e, ch);
	}
}

/* Steps 5-7 of _ecfsdsa_verify_finalize (sig/ecfsdsa.c:597-610): W' = sG + eY with e = -h mod q, reject infinity
 * (prj_pt_unique fails on it), accept iff W' == r.  R is the signature's point (validated, Montgomery form); the
 * comparison is done projectively (X == r_x Z^2, Y == r_y Z^3) instead of normalising W'.  0 valid, 2 infinity,
 * 3 mismatch. */
template <class C, class Inv>
ECC_HD int ecfsdsa_verify_tail(const Aff<C> &R, const Fe<C::N> &s, const Fe<C::N> &e_neg, const Aff<C> &Y,
			       const uint32_t *__restrict__ table, int w, const Inv &invert)
{
	typedef Field<typename C::Fp> F;
	Jac<C> sG, W;
	comb_mul<C>(sG, s, table, w);
	window_mul<C>(W, e_neg, Y, &sG, invert);
	if (EC<C>::is_inf(W)) return 2;
	Fe<C::N> z2, z3, t;
	F::sqr(z2, W.Z);
	F::mul(z3, z2, W.Z);
	F::mul(t, R.x, z2);
	bool ok = F::eq(t, W.X);
	F::mul(t, R.y, z3);
	ok = ok && F::eq(t, W.Y);
	return ok ? 0 : 3;
}

/* ------------------------------------------------------------------------------------------ BIP0340 (§8f.4) */

/*
 * _bip0340_verify_finalize (sig/bip0340.c:497-577) after the init checks: W' = sG + (-e)Y' with Y' the public key
 * lifted to an even y (:540-545; the caller passes Y already lifted, Montgomery form), reject infinity (:555-556),
 * reject an odd y(W') (:559-560), accept iff x(W') == r (:563-564).  Unlike ECDSA / ECFSDSA the comparison needs the
 * affine representative (the parity of y), so W' is normalised with one more inversion — `invert`, a CTA-wide one in
 * the kernel, which every thread must call: rejected items walk the same code on dummy values.
 * r: plain integer < p.  0 valid, 2 infinity, 3 mismatch / odd y.
 */
template <class C, class Inv>
ECC_HD int bip0340_verify_tail(const Fe<C::N> &r, const Fe<C::N> &s, const Fe<C::N> &e_neg, const Aff<C> &Y,
			       const uint32_t *__restrict__ table, int w, const Inv &invert)
{
	typedef Field<typename C::Fp> F;
	Jac<C> sG, W;
	comb_mul<C>(sG, s, table, w);                   /* s may be 0: the comb then returns infinity (:537) */
	window_mul<C>(W, e_neg, Y, &sG, invert);
	const bool inf = EC<C>::is_inf(W);
	Fe<C::N> z, zi, zi2, zi3, x, y, t;
	z = W.Z;
	if (inf) F::set_one(z);
	invert(zi, z);
	F::sqr(zi2, zi);
	F::mul(zi3, zi2, zi);
	F::mul(t, W.X, zi2);
	F::from_mont(x, t);
	F::mul(t, W.Y, zi3);
	F::from_mont(y, t);
	if (inf) return 2;
	if (y.w[0] & 1u) return 3;
	return F::eq(x, r) ? 0 : 3;
}

/* ------------------------------------------------------------------ Schnorr-family signing (ECSDSA .. BIP0340) */

/* ec_alg_type values of the reference (lib_ecc_types.h) for the four schemes whose hash covers W = k*G */
enum { SIG_ECSDSA = 3, SIG_ECOSDSA = 4, SIG_ECFSDSA = 5, SIG_BIP0340 = 20 };
/* the longest hash prefix: H(tag) || H(tag) || (R_x or t) || P_x with 64-byte digests on the 521-bit curve */
constexpr int kSchnorrMaxPrefix = 2 * 64 + 2 * 66;

/* r || s: hsize + qlen (ECSDSA / ECOSDSA), 2*plen + qlen (ECFSDSA), plen + qlen (BIP0340) */
template <class C> ECC_HD int schnorr_sig_len(int sig_type, int digest_size)
{
	return sig_type == SIG_ECFSDSA ? 2 * C::PLEN + C::QLEN :
	       sig_type == SIG_BIP0340 ? C::PLEN + C::QLEN : digest_size + C::QLEN;
}

/* H(tag) of the three BIP0340 tags (sig/bip0340.c:41-43): 0 aux, 1 nonce, 2 challenge */
ECC_D void bip0340_tag_hash(int hash_type, int tag, uint8_t *out)
{
	const char *s = tag == 0 ? "BIP0340/aux" : (tag == 1 ? "BIP0340/nonce" : "BIP0340/challenge");
	const uint32_t len = tag == 0 ? 11u : (tag == 1 ? 13u : 17u);
	hash_src(hash_type, ByteSpan{ (const uint8_t *)s }, len, out);
}

/*
 * The BIP0340 nonce (_bip0340_sign, sig/bip0340.c:243-297): d = x, or q - x when y(P) is odd (:237, :74-101);
 * t = d XOR H_aux(a) and k = H_nonce(t || P_x || m) mod q, with the reference's two branches (:267-280): when
 * qlen > digest size the first digest-size bytes of d are XORed and qlen bytes hashed, otherwise the first qlen bytes
 * of H_aux(a) are XORed and digest-size bytes hashed.  H_tag(z) = H(H(tag) || H(tag) || z); tag_aux / tag_nonce are
 * the H(tag) digests.  x must be in [1, q-1]; P is the affine wire key, a the qlen-byte auxiliary randomness.
 */
template <class C>
ECC_D void bip0340_nonce(Fe<C::N> &k, int hash_type, const Fe<C::N> &x, const uint8_t *P, const uint8_t *aux,
			 const uint8_t *msg, uint64_t mlen, const uint8_t *tag_aux, const uint8_t *tag_nonce)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int PL = C::PLEN, QL = C::QLEN;
	const int ds = sha2_digest_size(hash_type);
	uint8_t pre[kSchnorrMaxPrefix], h[64], db[QL];
	Fe<C::N> d = x;
	if (P[2 * PL - 1] & 1u) Fq::neg(d, d);
	store_be<C::N>(db, d, QL);
	for (int i = 0; i < ds; i++) pre[i] = pre[ds + i] = tag_aux[i];
	for (int i = 0; i < QL; i++) pre[2 * ds + i] = aux[i];
	hash_segments(hash_type, pre, (uint32_t)(2 * ds + QL), nullptr, 0, h); /* H_aux(a) */
	for (int i = 0; i < ds; i++) pre[i] = pre[ds + i] = tag_nonce[i];
	int np = 2 * ds;
	if (QL > ds) {
		for (int i = 0; i < QL; i++) pre[np + i] = db[i] ^ (i < ds ? h[i] : 0u);
		np += QL;
	} else {
		for (int i = 0; i < ds; i++) pre[np + i] = h[i] ^ (i < QL ? db[i] : 0u);
		np += ds;
	}
	for (int i = 0; i < PL; i++) pre[np + i] = P[i];
	np += PL;
	hash_segments(hash_type, pre, (uint32_t)np, msg, mlen, h);
	digest_full_mod_q<C>(k, h, (uint32_t)ds);
}

/*
 * One Schnorr-family signature from W = k*G (affine wire bytes, as K4 writes them), the private scalar x and the
 * nonce k (plain integers) and the message (in memory, read where it lies):
 *   ECSDSA  r = H(W_x || W_y || m), e = OS2I(r) mod q   (__ecsdsa_sign_init / _finalize, sig/ecsdsa_common.c:141-399)
 *   ECOSDSA r = H(W_x || m), e = OS2I(r) mod q
 *   ECFSDSA r = W_x || W_y, e = H(r || m) mod q          (sig/ecfsdsa.c:120-356)
 *   BIP0340 r = R_x, e = H_challenge(R_x || P_x || m) mod q, x and k negated when y(P) resp. y(R) is odd
 *           (sig/bip0340.c:161-371); tag_challenge = H("BIP0340/challenge"), P the affine wire key (key_ok: on the curve)
 * and s = k + e*x mod q.  e is the WHOLE digest reduced mod q (nn_init_from_buf + nn_mod), not the ECDSA truncation.
 * Returns 0 (sig written), -1 (x or k outside [1, q-1], or a BIP0340 key off the curve) or 2 (the reference fails or
 * restarts and fresh randomness would succeed: e == 0 or s == 0 for ECSDSA / ECOSDSA, s == 0 for ECFSDSA, a derived
 * k == 0 for BIP0340); sig (schnorr_sig_len bytes) is zero unless 0 is returned.
 */
template <class C>
ECC_D int schnorr_sign_core(uint8_t *sig, int sig_type, int hash_type, const uint8_t *W, const Fe<C::N> &x,
			    const Fe<C::N> &k, const uint8_t *msg, uint64_t mlen, const uint8_t *P, bool key_ok,
			    const uint8_t *tag_challenge)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N, PL = C::PLEN, QL = C::QLEN;
	const int ds = sha2_digest_size(hash_type);
	const int siglen = schnorr_sig_len<C>(sig_type, ds);
	const bool bip = sig_type == SIG_BIP0340;
	int st = 0;
	if (!key_ok || Fq::is_zero(x) || Fq::geq_mod(x)) st = -1;
	else if (Fq::is_zero(k) || Fq::geq_mod(k)) st = bip ? 2 : -1; /* BIP0340: k is derived, reduced mod q */
	if (st != 0) {
		for (int i = 0; i < siglen; i++) sig[i] = 0;
		return st;
	}
	uint8_t pre[kSchnorrMaxPrefix], h[64];
	int np = 0;
	if (bip)
		for (int i = 0; i < ds; i++) pre[i] = pre[ds + i] = tag_challenge[i];
	np = bip ? 2 * ds : 0;
	for (int i = 0; i < PL; i++) pre[np + i] = W[i];
	np += PL;
	if (sig_type == SIG_ECSDSA || sig_type == SIG_ECFSDSA) {
		for (int i = 0; i < PL; i++) pre[np + i] = W[PL + i];
		np += PL;
	} else if (bip) {
		for (int i = 0; i < PL; i++) pre[np + i] = P[i];
		np += PL;
	}
	hash_segments(hash_type, pre, (uint32_t)np, msg, mlen, h);
	Fe<N> e, xx = x, kk = k, xm, t, s;
	digest_full_mod_q<C>(e, h, (uint32_t)ds);
	if (bip) {
		if (P[2 * PL - 1] & 1u) Fq::neg(xx, xx);
		if (W[2 * PL - 1] & 1u) Fq::neg(kk, kk);
	}
	Fq::to_mont(xm, xx);
	Fq::mul(t, e, xm); /* e*x mod q (plain: one factor in the Montgomery domain) */
	Fq::add(s, kk, t);
	bool retry = (!bip && Fq::is_zero(s)) || ((sig_type == SIG_ECSDSA || sig_type == SIG_ECOSDSA) && Fq::is_zero(e));
	if (retry) {
		for (int i = 0; i < siglen; i++) sig[i] = 0;
		return 2;
	}
	const int rlen = siglen - QL;
	if (sig_type == SIG_ECSDSA || sig_type == SIG_ECOSDSA)
		for (int i = 0; i < rlen; i++) sig[i] = h[i];
	else
		for (int i = 0; i < rlen; i++) sig[i] = W[i];
	store_be<N>(sig + rlen, s, QL);
	return 0;
}

/* ------------------------------------------------------------------ message signers (ECKCDSA, ECGDSA, ECRDSA, SM2) */

/* ec_alg_type values of the reference (lib_ecc_types.h) for the randomized signers that hash the raw message */
enum { SIG_ECKCDSA = 2, SIG_ECGDSA = 6, SIG_ECRDSA = 7, SIG_SM2 = 8 };
constexpr uint32_t kSm2MaxIdLen = 8191; /* SM2_MAX_ID_LEN: ENTL = 8 * len(ID) fits 16 bits (sig/sm2.c:154) */
constexpr int kMsgsMaxPrefix = 144;    /* ECKCDSA's z: the largest block size (SHA3-224) */

#if defined(__CUDACC__)
#define ECC_D_NOINLINE __device__ __noinline__
#else
#define ECC_D_NOINLINE __attribute__((noinline))
#endif

/* r || s: r_len + qlen with r_len = min(hsize, qlen) for ECKCDSA (ECKCDSA_SIGLEN), 2*qlen for the other three */
template <class C> ECC_HD int msgs_sig_len(int sig_type, int digest_size)
{
	return sig_type == SIG_ECKCDSA ? (digest_size < C::QLEN ? digest_size : C::QLEN) + C::QLEN : 2 * C::QLEN;
}

/* One out-of-line copy of the eight hashes per kernel: the signers hash at up to three places per item. */
static ECC_D_NOINLINE void msg_hash_seg3(int hash_type, const Seg3 &src, uint64_t len, uint8_t *digest)
{
	msg_hash_src(hash_type, src, len, digest);
}

/* x in [1, q-2] (SM2 keys, sm2_init_pub_key, sig/sm2.c:72-75) or [1, q-1] (the other three) */
template <class C> ECC_HD bool msgs_key_in_range(int sig_type, const Fe<C::N> &x)
{
	typedef Field<typename C::Fq> Fq;
	if (Fq::is_zero(x) || Fq::geq_mod(x)) return false;
	if (sig_type != SIG_SM2) return true;
	Fe<C::N> one, t;
	Fq::set_zero(one);
	one.w[0] = 1;
	Fq::add(t, x, one);
	return !Fq::is_zero(t);
}

/* (1 + x) in the Montgomery domain of q: the factor SM2 inverts (step 8, sig/sm2.c:437-441) */
template <class C> ECC_HD void sm2_one_plus_x(Fe<C::N> &r, const Fe<C::N> &x)
{
	typedef Field<typename C::Fq> Fq;
	Fe<C::N> one, t;
	Fq::set_zero(one);
	one.w[0] = 1;
	Fq::add(t, x, one);
	Fq::to_mont(r, t);
}

/* SM2's Z = H(ENTL || ID || a || b || G_x || G_y || Y_x || Y_y) (sm2_compute_Z, sig/sm2.c:136-215): ENTL is held by
 * the thread, the ID is read where it lies, a || b || G || Y is assembled by the thread; Y is the affine wire key. */
template <class C> ECC_D void sm2_z(int hash_type, const uint8_t *id, uint32_t idlen, const uint8_t *Y, uint8_t *Z)
{
	typedef Field<typename C::Fp> Fp;
	constexpr int N = C::N, PL = C::PLEN;
	const uint32_t entl = (idlen * 8u) & 0xffffu;
	const uint8_t ent[2] = { (uint8_t)(entl >> 8), (uint8_t)entl };
	uint8_t tail[6 * PL];
	Fe<N> v, m;
#pragma unroll
	for (int i = 0; i < N; i++) m.w[i] = C::A_MONT(i);
	Fp::from_mont(v, m);
	store_be<N>(tail, v, PL);
#pragma unroll
	for (int i = 0; i < N; i++) m.w[i] = C::B_MONT(i);
	Fp::from_mont(v, m);
	store_be<N>(tail + PL, v, PL);
#pragma unroll
	for (int i = 0; i < N; i++) v.w[i] = C::GX(i);
	store_be<N>(tail + 2 * PL, v, PL);
#pragma unroll
	for (int i = 0; i < N; i++) v.w[i] = C::GY(i);
	store_be<N>(tail + 3 * PL, v, PL);
	for (int i = 0; i < 2 * PL; i++) tail[4 * PL + i] = Y[i];
	msg_hash_seg3(hash_type, Seg3{ ent, 2, id, idlen, tail }, 2 + (uint64_t)idlen + 6 * PL, Z);
}

/* SM2's e = OS2I(H(Z || m)) mod q (_sm2_sign_finalize step 5, _sm2_verify_finalize steps 2 and 5, sig/sm2.c:392,
 * :649-666), Z from sm2_z.  Z and h are the caller's 64-byte buffers (the signer reuses its own: a separate frame
 * here costs it registers). */
template <class C>
ECC_D void sm2_digest_scalar(Fe<C::N> &e, int hash_type, const uint8_t *id, uint32_t idlen, const uint8_t *Y,
			     const uint8_t *msg, uint64_t mlen, uint8_t *Z, uint8_t *h)
{
	const int ds = msg_hash_digest_size(hash_type);
	sm2_z<C>(hash_type, id, idlen, Y, Z);
	msg_hash_seg3(hash_type, Seg3{ Z, (uint32_t)ds, msg, mlen, nullptr }, (uint64_t)ds + mlen, h);
	digest_full_mod_q<C>(e, h, (uint32_t)ds);
}

/* ECKCDSA's H(z || m), z the first block-size bytes of Y_x || Y_y || 0... (z_len = block_size, sig/eckcdsa.c:223 sign,
 * :578-625 verify); Y is the affine wire key, z the caller's kMsgsMaxPrefix-byte buffer, h receives the whole digest */
template <class C>
ECC_D void eckcdsa_hash_zm(int hash_type, const uint8_t *Y, const uint8_t *msg, uint64_t mlen, uint8_t *z, uint8_t *h)
{
	const int bs = msg_hash_block_size(hash_type);
	for (int i = 0; i < bs; i++) z[i] = i < 2 * C::PLEN ? Y[i] : 0u;
	msg_hash_seg3(hash_type, Seg3{ z, (uint32_t)bs, msg, mlen, nullptr }, (uint64_t)bs + mlen, h);
}

/* ECRDSA's scalar of the digest h = H(m): OS2I(byte-reversed h) mod q, 0 replaced by 1 (sig/ecrdsa.c:297-313 sign,
 * :546-555 verify); rev is the caller's 64-byte buffer */
template <class C> ECC_HD void ecrdsa_digest_scalar(Fe<C::N> &e, const uint8_t *h, int ds, uint8_t *rev)
{
	for (int i = 0; i < ds; i++) rev[i] = h[ds - 1 - i];
	digest_full_mod_q<C>(e, rev, (uint32_t)ds);
	if (Field<typename C::Fq>::is_zero(e)) e.w[0] = 1;
}

/*
 * One ECKCDSA / ECGDSA / ECRDSA / SM2 signature from W = k*G (affine wire bytes, as K4 writes them), the private scalar
 * x and the nonce k (plain integers) and the message (in memory, read where it lies).  Every scheme follows the
 * reference's default build (sig/eckcdsa.c:202-471, ecgdsa.c:181-347, ecrdsa.c:196-346, sm2.c:136-455):
 *   ECGDSA  e = -(leftmost bitlen(q) bits of H(m)) mod q, r = W_x mod q, s = x*(k*r + e) mod q
 *   ECRDSA  e = OS2I(byte-reversed H(m)) mod q (0 -> 1), r = W_x mod q, s = r*x + k*e mod q
 *   ECKCDSA r = the rightmost r_len = min(hsize, qlen) bytes of H(W_x), h those of H(z || m) with z the first
 *           block-size bytes of Y_x || Y_y || 0...; e = OS2I(r XOR h) mod q, s = x*(k - e) mod q
 *   SM2     e = OS2I(H(Z || m)) (sm2_z), r = (e + W_x) mod q, s = (1 + x)^-1 * (k - r*x) mod q with inv1x = (1 + x)^-1
 *           in the Montgomery domain of q (the caller inverts, CTA-wide on the device).  Like the reference (step 7,
 *           sig/sm2.c:406-411 compares r + q with q) there is no restart on r + k == q.
 * Y is the affine wire key (ECKCDSA and SM2; key_ok: on the curve), id / idlen SM2's ID.
 * Returns 0 (sig written), -1 (x outside [1, q-1] (SM2: [1, q-2]), k outside [1, q-1], a key off the curve or an ID
 * longer than 8191 bytes) or 2 (a reference restart: r == 0 for ECGDSA / ECRDSA / SM2, s == 0 for all four); sig
 * (msgs_sig_len bytes) is zero unless 0 is returned.
 */
template <class C>
ECC_D int msgs_sign_core(uint8_t *sig, int sig_type, int hash_type, const uint8_t *W, const Fe<C::N> &x,
			 const Fe<C::N> &k, const uint8_t *msg, uint64_t mlen, const uint8_t *Y, bool key_ok,
			 const uint8_t *id, uint32_t idlen, const Fe<C::N> &inv1x)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N, PL = C::PLEN, QL = C::QLEN;
	const int ds = msg_hash_digest_size(hash_type);
	const int siglen = msgs_sig_len<C>(sig_type, ds);
	const bool sm2 = sig_type == SIG_SM2;
	if (!key_ok || !msgs_key_in_range<C>(sig_type, x) || Fq::is_zero(k) || Fq::geq_mod(k) || (sm2 && idlen > kSm2MaxIdLen)) {
		for (int i = 0; i < siglen; i++) sig[i] = 0;
		return -1;
	}
	uint8_t pre[kMsgsMaxPrefix], h[64];
	Fe<N> e, r, s, t, xm, km;
	Fq::to_mont(xm, x);
	Fq::to_mont(km, k);
	load_be<N>(r, W, PL);
	scalar_reduce<C>(r); /* W_x mod q */
	bool retry = false;
	int rlen = QL, shift = 0;
	if (sig_type == SIG_ECKCDSA) {
		uint8_t hr[64];
		eckcdsa_hash_zm<C>(hash_type, Y, msg, mlen, pre, h);                                       /* H(z || m) */
		msg_hash_seg3(hash_type, Seg3{ W, (uint32_t)PL, nullptr, 0, nullptr }, (uint64_t)PL, hr); /* H(W_x)    */
		rlen = ds < QL ? ds : QL;
		shift = ds - rlen;
		for (int i = 0; i < rlen; i++) {
			h[i] = h[shift + i] ^ hr[shift + i];
			pre[i] = hr[shift + i];
		}
		digest_full_mod_q<C>(e, h, (uint32_t)rlen);
		Fq::sub(t, k, e);
		Fq::mul(s, t, xm); /* x*(k - e) */
	} else if (sm2) {
		sm2_digest_scalar<C>(e, hash_type, id, idlen, Y, msg, mlen, pre, h);
		Fq::add(r, e, r);  /* (OS2I(H) + W_x) mod q */
		retry = Fq::is_zero(r);
		Fq::mul(t, r, xm); /* r*x */
		Fq::sub(t, k, t);
		Fq::mul(s, t, inv1x);
	} else {
		msg_hash_seg3(hash_type, Seg3{ nullptr, 0, msg, mlen, nullptr }, mlen, h);
		retry = Fq::is_zero(r);
		if (sig_type == SIG_ECGDSA) {
			digest_to_scalar<C>(e, h, (uint32_t)ds);
			Fq::neg(e, e);
			Fq::mul(t, r, km); /* k*r */
			Fq::add(t, t, e);
			Fq::mul(s, t, xm);
		} else {
			ecrdsa_digest_scalar<C>(e, h, ds, pre);
			Fq::mul(t, r, xm); /* r*x */
			Fq::mul(s, e, km); /* k*e */
			Fq::add(s, s, t);
		}
	}
	if (retry || Fq::is_zero(s)) {
		for (int i = 0; i < siglen; i++) sig[i] = 0;
		return 2;
	}
	if (sig_type == SIG_ECKCDSA)
		for (int i = 0; i < rlen; i++) sig[i] = pre[i];
	else
		store_be<N>(sig, r, QL);
	store_be<N>(sig + rlen, s, QL);
	return 0;
}

/* r, s in [1, q-1]?  (__ecdsa_verify_init, sig/ecdsa_common.c:653-658) */
template <class C> ECC_HD bool ecdsa_rs_in_range(const Fe<C::N> &r, const Fe<C::N> &s)
{
	typedef Field<typename C::Fq> Fq;
	return !(Fq::is_zero(r) || Fq::is_zero(s) || Fq::geq_mod(r) || Fq::geq_mod(s));
}

/* Whole verification of one signature with a per-item inversion of s (host build of the tests and reference for the
 * kernel, which replaces the inversion by a CTA-wide simultaneous one). */
template <class C>
ECC_HD int ecdsa_verify_core(const Fe<C::N> &r, const Fe<C::N> &s, const Fe<C::N> &e, const Aff<C> &Y,
			     const uint32_t *__restrict__ table, int w)
{
	if (!ecdsa_rs_in_range<C>(r, s)) return 1;
	Fe<C::N> u, v;
	ecdsa_uv<C>(u, v, r, s, e);
	return ecdsa_verify_tail<C>(r, u, v, Y, table, w);
}

/* ------------------------------------------------------------------------------------- ECDSA public-key recovery */

/*
 * __ecdsa_public_key_from_sig (sig/ecdsa_common.c:867-1011) in pieces shared by the kernel (k_ecdsa_recover) and the
 * host build of the tests.  Only x = r is ever tried: the reference's restart with r + k*q (:914-931, :960-971) can
 * not succeed on a curve of cofactor 1 (r + 2q >= p exits, or fp_set_nn refuses it), so it always ends in -1.
 */

/* r, s in [1, q-1] (:900-912) and r < p, which fp_set_nn requires (:958; only FRP256V1 has q > p) */
template <class C> ECC_HD bool ecdsa_recover_rs_ok(const Fe<C::N> &r, const Fe<C::N> &s)
{
	return ecdsa_rs_in_range<C>(r, s) && !Field<typename C::Fp>::geq_mod(r);
}

/* R1 = (r, sqrt1) with sqrt1 the first root of fp_sqrt (aff_pt_y_from_x, curves/aff_pt.c); false when
 * r^3 + ar + b is not a square.  r < p. */
template <class C> ECC_HD bool ecdsa_recover_point(Aff<C> &R, const Fe<C::N> &r, int *loops = nullptr)
{
	typedef Field<typename C::Fp> F;
	Fe<C::N> alpha;
	F::to_mont(R.x, r);
	EC<C>::curve_rhs(alpha, R.x);
	return F::sqrt(R.y, alpha, loops);
}

/* u = -e * r^-1 mod q, v = s * r^-1 mod q (plain form) from ri = r^-1 in the Montgomery domain of q (:981-990) */
template <class C>
ECC_HD void ecdsa_recover_uv(Fe<C::N> &u, Fe<C::N> &v, const Fe<C::N> &e, const Fe<C::N> &s, const Fe<C::N> &ri)
{
	typedef Field<typename C::Fq> Fq;
	Fq::mul(u, e, ri);
	Fq::neg(u, u); /* nn_mod_neg: 0 stays 0 */
	Fq::mul(v, s, ri);
}

/* Y1 = v*R1 + uG and Y2 = v*R2 + uG = uG - v*R1 (:992-999) from uG and V = v*R1: one scalar multiplication for both
 * keys.  add_full resolves uG = +-V and the points at infinity; either key may be the point at infinity. */
template <class C> ECC_HD void ecdsa_recover_keys(Jac<C> &Y1, Jac<C> &Y2, const Jac<C> &uG, const Jac<C> &V)
{
	Jac<C> Vn;
	EC<C>::neg(Vn, V);
	EC<C>::add_full(Y1, uG, V);
	EC<C>::add_full(Y2, uG, Vn);
}

/* The whole recovery of one item with a per-item inversion of r (host build of the tests; the kernel shares the
 * inversions across its CTA).  Returns false where the reference returns -1. */
template <class C>
ECC_HD bool ecdsa_recover_core(Jac<C> &Y1, Jac<C> &Y2, const Fe<C::N> &r, const Fe<C::N> &s, const Fe<C::N> &e,
			       const uint32_t *__restrict__ table, int w)
{
	typedef Field<typename C::Fq> Fq;
	Aff<C> R;
	if (!ecdsa_recover_rs_ok<C>(r, s) || !ecdsa_recover_point<C>(R, r)) return false;
	Fe<C::N> rm, ri, u, v;
	Fq::to_mont(rm, r);
	Fq::inv(ri, rm);
	ecdsa_recover_uv<C>(u, v, e, s, ri);
	Jac<C> uG, V;
	comb_mul<C>(uG, u, table, w);
	window_mul<C>(V, v, R, nullptr, ThreadInverter<C>());
	ecdsa_recover_keys<C>(Y1, Y2, uG, V);
	return true;
}

/* ---------------------------------------- message verifiers (ECKCDSA, ECSDSA, ECOSDSA, ECGDSA, ECRDSA, SM2) */

/* r || s: hsize + qlen (ECSDSA / ECOSDSA), min(hsize, qlen) + qlen (ECKCDSA), 2*qlen (ECGDSA, ECRDSA, SM2) */
template <class C> ECC_HD int msgs_verify_sig_len(int sig_type, int digest_size)
{
	return sig_type == SIG_ECSDSA || sig_type == SIG_ECOSDSA ? digest_size + C::QLEN :
								   msgs_sig_len<C>(sig_type, digest_size);
}

/* ECGDSA (r^-1) and ECRDSA (h^-1) need one inversion mod q per item to form their scalars */
ECC_HD bool msgs_verify_inverts(int sig_type) { return sig_type == SIG_ECGDSA || sig_type == SIG_ECRDSA; }

/*
 * First half of one verification, before W' = a*G + b*Y: the signature checks, the hash of the message and the mod-q
 * scalars (plain integers < q), each scheme as the reference's default build (the drop-in's DsScheme objects restate
 * the same rules):
 *   ECSDSA / ECOSDSA  s in ]0, q[, e = -(OS2I(r) mod q) != 0; a = s, b = e     (sig/ecsdsa_common.c:475-498)
 *   ECKCDSA           s in ]0, q[, e = OS2I(r XOR rightmost r_len bytes of H(z || m)) mod q; a = e, b = s
 *                                                                              (sig/eckcdsa.c:592-773)
 *   ECGDSA            r, s in ]0, q[, e = leftmost bitlen(q) bits of H(m); a = e, b = s, den = r
 *                                                                              (sig/ecgdsa.c:451-568)
 *   ECRDSA            r, s in ]0, q[, h = ecrdsa_digest_scalar(H(m)); a = s, b = -r, den = h
 *                     (the reference never range-checks r, sig/ecrdsa.c:448-449; an r >= q fails its final comparison
 *                     with r' < q, so refusing it here gives the same verdict)  (:546-569)
 *   SM2               r, s in ]0, q[, t = r + s mod q != 0, ID at most 8191 bytes; a = s, b = t  (sig/sm2.c:553-671)
 * For ECGDSA and ECRDSA a and b are still to be multiplied by den^-1 (msgs_verify_scale); den is 0 for the other
 * schemes.  Y is the affine wire key (read by ECKCDSA only).  Returns false (a = b = den = 0) when the reference
 * rejects the item before W'; a valid item never has a = b = 0, because s != 0 is one of its scalars.
 */
template <class C>
ECC_D bool msgs_verify_prep_core(int sig_type, int hash_type, const uint8_t *sig, const uint8_t *Y, const uint8_t *msg,
				 uint64_t mlen, uint32_t idlen, Fe<C::N> &a, Fe<C::N> &b, Fe<C::N> &den)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N, QL = C::QLEN;
	const int ds = msg_hash_digest_size(hash_type);
	Fq::set_zero(a);
	Fq::set_zero(b);
	Fq::set_zero(den);
	Fe<N> r, s;
	uint8_t pre[kMsgsMaxPrefix], h[64];
	if (sig_type == SIG_ECSDSA || sig_type == SIG_ECOSDSA) {
		load_be<N>(s, sig + ds, QL);
		if (Fq::is_zero(s) || Fq::geq_mod(s)) return false;
		digest_full_mod_q<C>(r, sig, (uint32_t)ds);
		if (Fq::is_zero(r)) return false;
		a = s;
		Fq::neg(b, r);
		return true;
	}
	if (sig_type == SIG_ECKCDSA) {
		const int rlen = ds < QL ? ds : QL, shift = ds - rlen;
		load_be<N>(s, sig + rlen, QL);
		if (Fq::is_zero(s) || Fq::geq_mod(s)) return false;
		eckcdsa_hash_zm<C>(hash_type, Y, msg, mlen, pre, h);
		for (int i = 0; i < rlen; i++) h[i] = h[shift + i] ^ sig[i];
		digest_full_mod_q<C>(a, h, (uint32_t)rlen);
		b = s;
		return true;
	}
	load_be<N>(r, sig, QL);
	load_be<N>(s, sig + QL, QL);
	if (!ecdsa_rs_in_range<C>(r, s)) return false;
	if (sig_type == SIG_SM2) {
		Fe<N> t;
		Fq::add(t, r, s);
		if (idlen > kSm2MaxIdLen || Fq::is_zero(t)) return false;
		a = s;
		b = t;
		return true;
	}
	msg_hash_seg3(hash_type, Seg3{ nullptr, 0, msg, mlen, nullptr }, mlen, h);
	if (sig_type == SIG_ECGDSA) {
		digest_to_scalar<C>(a, h, (uint32_t)ds);
		b = s;
		den = r;
	} else {
		ecrdsa_digest_scalar<C>(den, h, ds, pre);
		a = s;
		Fq::neg(b, r);
	}
	return true;
}

/* ECGDSA / ECRDSA: a, b <- a * den^-1, b * den^-1 mod q, inv = den^-1 in the Montgomery domain of q */
template <class C> ECC_HD void msgs_verify_scale(Fe<C::N> &a, Fe<C::N> &b, const Fe<C::N> &inv)
{
	typedef Field<typename C::Fq> Fq;
	Fe<C::N> t;
	Fq::mul(t, a, inv);
	a = t;
	Fq::mul(t, b, inv);
	b = t;
}

/*
 * Second half, after a finite W' (affine wire bytes): the scheme's acceptance test.
 *   ECSDSA / ECOSDSA  H(W'_x || W'_y || m) resp. H(W'_x || m) == r      (sig/ecsdsa_common.c:500-520, :606)
 *   ECKCDSA           rightmost r_len bytes of H(W'_x) == r             (sig/eckcdsa.c:778-800)
 *   ECGDSA / ECRDSA   W'_x mod q == r                                   (sig/ecgdsa.c:577-585, ecrdsa.c:580-585)
 *   SM2               (OS2I(H(Z || m)) + W'_x) mod q == r               (sig/sm2.c:664-688)
 * Y is the affine wire key (SM2's Z), id / idlen SM2's ID (at most 8191 bytes: the prep refused longer ones).
 */
template <class C>
ECC_D bool msgs_verify_accept(int sig_type, int hash_type, const uint8_t *sig, const uint8_t *W, const uint8_t *Y,
			      const uint8_t *msg, uint64_t mlen, const uint8_t *id, uint32_t idlen)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N, PL = C::PLEN, QL = C::QLEN;
	const int ds = msg_hash_digest_size(hash_type);
	uint8_t h[64];
	if (sig_type == SIG_ECSDSA || sig_type == SIG_ECOSDSA) {
		const uint32_t nw = sig_type == SIG_ECSDSA ? 2 * PL : PL;
		msg_hash_seg3(hash_type, Seg3{ W, nw, msg, mlen, nullptr }, (uint64_t)nw + mlen, h);
		uint8_t diff = 0;
		for (int i = 0; i < ds; i++) diff |= h[i] ^ sig[i];
		return diff == 0;
	}
	if (sig_type == SIG_ECKCDSA) {
		const int rlen = ds < QL ? ds : QL, shift = ds - rlen;
		msg_hash_seg3(hash_type, Seg3{ W, (uint32_t)PL, nullptr, 0, nullptr }, (uint64_t)PL, h);
		uint8_t diff = 0;
		for (int i = 0; i < rlen; i++) diff |= h[shift + i] ^ sig[i];
		return diff == 0;
	}
	Fe<N> x, r;
	load_be<N>(x, W, PL);
	scalar_reduce<C>(x); /* W'_x mod q */
	load_be<N>(r, sig, QL);
	if (sig_type == SIG_SM2) {
		Fe<N> e;
		uint8_t Z[64];
		sm2_digest_scalar<C>(e, hash_type, id, idlen, Y, msg, mlen, Z, h);
		Fq::add(x, x, e);
	}
	return Fq::eq(x, r);
}

/* ----------------------------------------------------------------------- BIGN / DBIGN (STB 34.101.45) of messages */

enum { SIG_BIGN = 18, SIG_DBIGN = 19 }; /* ec_alg_type values of the reference (lib_ecc_types.h) */
constexpr uint32_t kBignMaxAdata = 0xffff; /* the reference's adata_len is a u16 */

/* Digest size of the BIGN message hashes: SHA-224 (1), SHA-256 .. SHA3-512 (2..8), SM3 (11), BELT-HASH (16) and
 * BASH224 .. BASH512 (17..20); 0 for any other type.  Only the BIGN entry points accept 16..20. */
SHA3_HD int bign_hash_digest_size(int hash_type)
{
	return hash_type == HASH_BELT ? 32 : bash_digest_size(hash_type) ? bash_digest_size(hash_type) :
									    decdsa_hash_digest_size(hash_type);
}

/* Any of them over a byte source; H is the BELT S-box (belt.cuh: shared memory on the device) */
template <class Src>
ECC_D void bign_hash_src(int hash_type, const Src &m, uint64_t len, uint8_t *digest, const uint8_t *H)
{
	if (hash_type == HASH_BELT) belt_hash_src(m, len, digest, H);
	else if (bash_digest_size(hash_type)) bash_src(m, len, digest, bash_digest_size(hash_type));
	else decdsa_hash_src(hash_type, m, len, digest);
}

/* The adata record oid_len (2 bytes, big-endian) || t_len (2 bytes, big-endian) || oid || t || any trailing bytes
 * (bign_get_oid_from_adata / bign_get_t_from_adata, sig/bign_common.c:97-147): valid iff 4 <= len <= 65535 and
 * oid_len + t_len <= len - 4.  The OID is not checked against the hash, as in the reference. */
ECC_HD bool bign_adata_parse(const uint8_t *ad, uint64_t len, uint32_t &oid_len, uint32_t &t_len)
{
	oid_len = t_len = 0;
	if (len < 4 || len > kBignMaxAdata) return false;
	oid_len = (uint32_t)ad[0] << 8 | ad[1];
	t_len = (uint32_t)ad[2] << 8 | ad[3];
	return oid_len + t_len <= len - 4;
}

/* len little-endian bytes -> N words */
template <int N> ECC_HD void load_le(Fe<N> &r, const uint8_t *buf, int len)
{
	for (int i = 0; i < N; i++) r.w[i] = 0;
	for (int j = 0; j < len && j < 4 * N; j++) r.w[j >> 2] |= (uint32_t)buf[j] << (8 * (j & 3));
}

/* a < b on N-word integers */
template <int N> ECC_HD bool fe_less(const Fe<N> &a, const Fe<N> &b)
{
	uint32_t borrow = 0;
#pragma unroll
	for (int i = 0; i < N; i++) {
		const uint64_t t = (uint64_t)a.w[i] - b.w[i] - borrow;
		borrow = (uint32_t)(t >> 32) & 1u;
	}
	return borrow != 0;
}

/*
 * s0 = the first min(l, 32) bytes of BELT-HASH(oid || the first 2l bytes of LE(W_x) || h), zero-padded to l bytes,
 * l = qlen / 2 (step 4 of __bign_sign_finalize, sig/bign_common.c:626-645; step 6 of __bign_verify_finalize,
 * :939-957).  2l <= plen on every curve, so W_y never enters.  W is the affine wire point, h the hs-byte digest H(m);
 * the concatenation is the three-segment source, never built in memory.
 */
template <class C>
ECC_D void bign_s0(uint8_t *s0, const uint8_t *oid, uint32_t oid_len, const uint8_t *W, const uint8_t *h, int hs,
		   const uint8_t *H)
{
	constexpr int L = C::QLEN / 2, PL = C::PLEN;
	static_assert(2 * L <= PL, "bign_s0: 2l bytes of W_x");
	uint8_t wle[2 * L], d[32];
	for (int i = 0; i < 2 * L; i++) wle[i] = W[PL - 1 - i];
	belt_hash_src(Seg3{ oid, oid_len, wle, (uint64_t)(2 * L), h }, (uint64_t)oid_len + 2 * L + (uint64_t)hs, d, H);
	for (int i = 0; i < L; i++) s0[i] = i < 32 ? d[i] : 0u;
}

/* h-bar = OS2I(byte-reversed h) mod q over the whole digest (:650-652 sign, :913-915 verify); rev: 64 bytes */
template <class C> ECC_HD void bign_digest_scalar(Fe<C::N> &e, const uint8_t *h, int hs, uint8_t *rev)
{
	for (int i = 0; i < hs; i++) rev[i] = h[hs - 1 - i];
	digest_full_mod_q<C>(e, rev, (uint32_t)hs);
}

/* s0-bar + 2^(8l) from the l-byte s0.  s0-bar < 2^(8l) and 2^(8l+1) < q on every curve, so the sum is already
 * reduced, never 0, and 2^(8l) mod q is the constant bit 8l (:659-663 sign, :924-928 verify). */
template <class C> ECC_HD void bign_s0_scalar(Fe<C::N> &b, const uint8_t *s0)
{
	constexpr int L = C::QLEN / 2;
	static_assert(8 * L + 1 < C::QBITS, "bign: 2^(8l+1) < q");
	load_le<C::N>(b, s0, L);
	b.w[(8 * L) / 32] |= 1u << ((8 * L) % 32);
}

/*
 * DBIGN's nonce (__bign_determinitic_nonce, sig/bign_common.c:200-342; STB 34.101.45 §6.3.3) from the key
 * theta = BELT-HASH(oid || first 2l bytes of LE(x) || t) and the hlen-byte digest h, for the group order q of qbits
 * bits (arguments, so that the host tests can run it on the STB curves):
 *   r = h zero-padded to n = max(2, hlen / 16) blocks r_1 .. r_n;  for i = 1, 2, ...:
 *     s = r_1 ^ .. ^ r_{n-1};  r <- r_2 .. r_{n-1} || belt-block(s, theta) ^ r_n ^ <i>_128 || s;
 *     k = the first qlen bytes of r read little-endian, masked to qbits bits (all 16n bytes, unmasked, when
 *     qlen >= 16n: SECP521R1 with a digest of 64 bytes or fewer);
 *   until i >= 2n and 0 < k < q.  Returns the number of rounds.
 */
template <int N>
ECC_HD uint32_t bign_det_nonce(Fe<N> &k, const uint8_t *theta, const uint8_t *h, int hlen, const Fe<N> &q, int qbits,
			       const uint8_t *H)
{
	uint32_t key[8], r[4][4];
	belt_load_block(key, theta);
	belt_load_block(key + 4, theta + 16);
	const int n = hlen / 16 > 2 ? hlen / 16 : 2, qlen = (qbits + 7) / 8;
	const bool whole = qlen >= 16 * n;
#pragma unroll
	for (int j = 0; j < 4; j++) {
		uint8_t blk[16];
		for (int z = 0; z < 16; z++) blk[z] = 16 * j + z < hlen ? h[16 * j + z] : 0u;
		belt_load_block(r[j], blk);
	}
	for (uint32_t i = 1;; i++) {
		uint32_t s[4] = { 0, 0, 0, 0 }, e[4];
#pragma unroll
		for (int j = 0; j < 3; j++)
			if (j < n - 1)
				for (int w = 0; w < 4; w++) s[w] ^= r[j][w];
		for (int w = 0; w < 4; w++) e[w] = s[w];
		belt_block(e, key, H);
		e[0] ^= i;
#pragma unroll
		for (int j = 0; j < 4; j++) {
			if (j + 1 < n)
				for (int w = 0; w < 4; w++) r[j][w] = r[j + 1][w] ^ (j + 2 == n ? e[w] : 0u);
			else if (j + 1 == n)
				for (int w = 0; w < 4; w++) r[j][w] = s[w];
		}
#pragma unroll
		for (int m = 0; m < N; m++) {
			uint32_t v = m < 16 && m < 4 * n ? r[(m >> 2) & 3][m & 3] : 0u;
			if (!whole) {
				const int lo = 32 * m;
				v = lo >= qbits ? 0u : (qbits - lo >= 32 ? v : v & ((1u << (qbits - lo)) - 1u));
			}
			k.w[m] = v;
		}
		bool zero = true;
#pragma unroll
		for (int m = 0; m < N; m++) zero = zero && k.w[m] == 0;
		if (i >= (uint32_t)(2 * n) && !zero && fe_less<N>(k, q)) return i;
	}
}

/* theta of bign_det_nonce: BELT-HASH(oid || first 2l bytes of LE(x) || t) (:233-248), x the plain private scalar */
template <class C>
ECC_D void bign_theta(uint8_t *theta, const uint8_t *oid, uint32_t oid_len, const uint8_t *t, uint32_t t_len,
		      const Fe<C::N> &x, const uint8_t *H)
{
	constexpr int L = C::QLEN / 2;
	uint8_t xle[2 * L];
	for (int i = 0; i < 2 * L; i++) xle[i] = (uint8_t)(x.w[i >> 2] >> (8 * (i & 3)));
	belt_hash_src(Seg3{ oid, oid_len, xle, (uint64_t)(2 * L), t }, (uint64_t)oid_len + 2 * L + t_len, theta, H);
}

/* The group order q of the curve as N words */
template <class C> ECC_HD void bign_order(Fe<C::N> &q)
{
#pragma unroll
	for (int i = 0; i < C::N; i++) q.w[i] = C::Fq::P(i);
}

/*
 * One BIGN signature s0 || LE(s1) (l + qlen bytes) from W = k*G (affine wire bytes), the plain scalars x and k, the
 * digest h = H(m) and the adata record (__bign_sign_finalize steps 4-5, sig/bign_common.c:626-690):
 *   s1 = (k - h-bar - (s0-bar + 2^(8l)) * x) mod q.
 * There is no restart case: s1 = 0 is a signature the verifier accepts.  Returns 0, or -1 (sig zeroed) for x or k
 * outside [1, q-1] or a malformed adata record.
 */
template <class C>
ECC_D int bign_sign_core(uint8_t *sig, const uint8_t *W, const Fe<C::N> &x, const Fe<C::N> &k, const uint8_t *h,
			 int hs, const uint8_t *ad, uint64_t adlen, const uint8_t *H)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N, QL = C::QLEN, L = C::QLEN / 2;
	uint32_t oid_len, t_len;
	if (!bign_adata_parse(ad, adlen, oid_len, t_len) || Fq::is_zero(x) || Fq::geq_mod(x) || Fq::is_zero(k) ||
	    Fq::geq_mod(k)) {
		for (int i = 0; i < L + QL; i++) sig[i] = 0;
		return -1;
	}
	bign_s0<C>(sig, ad + 4, oid_len, W, h, hs, H);
	uint8_t rev[64];
	Fe<N> hb, b, xm, t, s1;
	bign_digest_scalar<C>(hb, h, hs, rev);
	bign_s0_scalar<C>(b, sig);
	Fq::to_mont(xm, x);
	Fq::mul(t, b, xm); /* (s0-bar + 2^(8l)) * x */
	Fq::sub(s1, k, hb);
	Fq::sub(s1, s1, t);
	for (int i = 0; i < QL; i++) sig[L + i] = (uint8_t)(s1.w[i >> 2] >> (8 * (i & 3)));
	return 0;
}

/*
 * First half of a BIGN verification (__bign_verify_init / __bign_verify_finalize, sig/bign_common.c:742-936): from the
 * signature s0 || LE(s1) and the digest h, the scalars a = (s1 + h-bar) mod q and b = s0-bar + 2^(8l) of
 * W' = a*G + b*Y.  False (a = b = 0) for s1 >= q or a malformed adata record.
 */
template <class C>
ECC_HD bool bign_verify_prep_core(Fe<C::N> &a, Fe<C::N> &b, const uint8_t *sig, const uint8_t *h, int hs,
				  const uint8_t *ad, uint64_t adlen)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N, QL = C::QLEN, L = C::QLEN / 2;
	uint32_t oid_len, t_len;
	Fe<N> s1;
	load_le<N>(s1, sig + L, QL);
	Fq::set_zero(a);
	Fq::set_zero(b);
	if (!bign_adata_parse(ad, adlen, oid_len, t_len) || Fq::geq_mod(s1)) return false;
	uint8_t rev[64];
	Fe<N> hb;
	bign_digest_scalar<C>(hb, h, hs, rev);
	Fq::add(a, s1, hb);
	bign_s0_scalar<C>(b, sig);
	return true;
}

} // namespace eccb200
