/*
 * kernels.cuh — the sm_90a kernels of the engine (SURVEY.md §2 "new kernel" table: K1..K5), the kernels of the
 * "next" rows built so far (ECDSA sign, ECC-CDH), and the measurement / experiment kernels DESIGN.md cites.
 *
 * Layout in HBM (all produced / consumed by these kernels):
 *   wire buffers   : libecc big-endian byte strings, array-of-structures (scalars [n][qlen], affine points
 *                    [n][2*plen], signatures [n][2*qlen], digests [n][hlen]); a warp reads 32 consecutive items, i.e.
 *                    contiguous 1-3 KiB, each thread with 16-byte vector loads.
 *   Jacobian buffer: [n][3N] 32-bit words (X, Y, Z in Montgomery form) between the scalar-mult kernels and the
 *                    batched normalisation.
 *   comb table     : [(nwin << w)][2N] words, entry (i << w) + d = d * 2^(w*i) * G affine, Montgomery form
 *                    (64 B per entry for 256-bit curves = half a 128 B line, fetched with four 16 B loads).
 *   prefix buffer  : [n][N] words of running products for the simultaneous inversion.
 */
#pragma once
#include "ec.cuh"

/* cluster-wide inversion experiment, see cta_inverse_128 */
#ifndef ECC_CLUSTER_INV
#define ECC_CLUSTER_INV 1
#endif
#if ECC_CLUSTER_INV > 1
#include <cooperative_groups.h>
#define ECC_CLUSTER_ATTR __cluster_dims__(ECC_CLUSTER_INV, 1, 1)
#else
#define ECC_CLUSTER_ATTR
#endif

namespace eccb200 {

/* ------------------------------------------------------------------------------------------ device wire helpers */

__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }

/* A wire field is LEN big-endian bytes holding an N-word value (LEN <= 4N).  LEN == 4N with N a multiple of 4 (the
 * 256- and 384-bit curves) is read with 16-byte vector loads — item strides are then multiples of 16 bytes; any
 * other length (66 bytes for the 521-bit curve) has no alignment to rely on and is read byte by byte. */
template <int N, int LEN> __device__ __forceinline__ void load_wire(Fe<N> &r, const uint8_t *buf)
{
	if (LEN == 4 * N && N % 4 == 0) {
		const uint4 *p = reinterpret_cast<const uint4 *>(buf);
#pragma unroll
		for (int j = 0; j < N / 4; j++) {
			uint4 v = __ldg(p + j);
			/* bytes [16j, 16j+16) hold words N-1-4j .. N-4-4j (most significant first) */
			r.w[N - 1 - 4 * j] = bswap32(v.x);
			r.w[N - 2 - 4 * j] = bswap32(v.y);
			r.w[N - 3 - 4 * j] = bswap32(v.z);
			r.w[N - 4 - 4 * j] = bswap32(v.w);
		}
	} else {
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint32_t v = 0;
#pragma unroll
			for (int b = 0; b < 4; b++) {
				const int pos = LEN - 1 - (4 * i + b); /* byte of significance 4i+b */
				if (pos >= 0) v |= (uint32_t)__ldg(buf + pos) << (8 * b);
			}
			r.w[i] = v;
		}
	}
}

template <int N, int LEN> __device__ __forceinline__ void store_wire(uint8_t *buf, const Fe<N> &a)
{
	if (LEN == 4 * N && N % 4 == 0) {
		uint4 *p = reinterpret_cast<uint4 *>(buf);
#pragma unroll
		for (int j = 0; j < N / 4; j++) {
			uint4 v;
			v.x = bswap32(a.w[N - 1 - 4 * j]);
			v.y = bswap32(a.w[N - 2 - 4 * j]);
			v.z = bswap32(a.w[N - 3 - 4 * j]);
			v.w = bswap32(a.w[N - 4 - 4 * j]);
			p[j] = v;
		}
	} else {
#pragma unroll
		for (int i = 0; i < N; i++) {
#pragma unroll
			for (int b = 0; b < 4; b++) {
				const int pos = LEN - 1 - (4 * i + b);
				if (pos >= 0) buf[pos] = (uint8_t)(a.w[i] >> (8 * b));
			}
		}
	}
}

/* word buffers written by these kernels (Jacobian, prefix, table): 16-byte accesses when N is a multiple of 4,
 * 8-byte ones otherwise (N is always even: two words per reference limb) */
template <int N> __device__ __forceinline__ void load_words(Fe<N> &r, const uint32_t *src)
{
	if (N % 4 == 0) {
		const uint4 *p = reinterpret_cast<const uint4 *>(src);
#pragma unroll
		for (int j = 0; j < N / 4; j++) {
			uint4 v = p[j];
			r.w[4 * j] = v.x;
			r.w[4 * j + 1] = v.y;
			r.w[4 * j + 2] = v.z;
			r.w[4 * j + 3] = v.w;
		}
	} else {
		const uint2 *p = reinterpret_cast<const uint2 *>(src);
#pragma unroll
		for (int j = 0; j < N / 2; j++) {
			uint2 v = p[j];
			r.w[2 * j] = v.x;
			r.w[2 * j + 1] = v.y;
		}
	}
}

template <int N> __device__ __forceinline__ void store_words(uint32_t *dst, const Fe<N> &a)
{
	if (N % 4 == 0) {
		uint4 *p = reinterpret_cast<uint4 *>(dst);
#pragma unroll
		for (int j = 0; j < N / 4; j++) {
			uint4 v;
			v.x = a.w[4 * j];
			v.y = a.w[4 * j + 1];
			v.z = a.w[4 * j + 2];
			v.w = a.w[4 * j + 3];
			p[j] = v;
		}
	} else {
		uint2 *p = reinterpret_cast<uint2 *>(dst);
#pragma unroll
		for (int j = 0; j < N / 2; j++) {
			uint2 v;
			v.x = a.w[2 * j];
			v.y = a.w[2 * j + 1];
			p[j] = v;
		}
	}
}

template <class C> __device__ __forceinline__ void store_jac(uint32_t *jac, uint32_t idx, const Jac<C> &p)
{
	uint32_t *b = jac + (size_t)idx * (3 * C::N);
	store_words<C::N>(b, p.X);
	store_words<C::N>(b + C::N, p.Y);
	store_words<C::N>(b + 2 * C::N, p.Z);
}

/* Load an affine wire point, validate it the way the reference's import does (coordinates < p,
 * fp_import_from_buf; on the curve, curves/prj_pt.c:541-545) and convert it to Montgomery form. */
template <class C> __device__ __forceinline__ bool load_affine_checked(Aff<C> &P, const uint8_t *buf)
{
	typedef Field<typename C::Fp> F;
	Fe<C::N> x, y;
	load_wire<C::N, C::PLEN>(x, buf);
	load_wire<C::N, C::PLEN>(y, buf + C::PLEN);
	bool ok = !F::geq_mod(x) && !F::geq_mod(y);
	F::to_mont(P.x, x);
	F::to_mont(P.y, y);
	ok = ok && EC<C>::on_curve(P);
	return ok;
}

/* ------------------------------------------------------------------------------------------ CTA-wide inversion */

/*
 * Simultaneous inversion across the 128 threads of a CTA: every thread passes a non-zero Montgomery-form element
 * `acc` and gets acc^-1 back.  Two shared-memory scans (inclusive prefix P and suffix S, 7 doubling steps), ONE warp
 * runs the inversion (Field::inv: safegcd division steps) on the CTA product,
 * and thread t computes inv_total * P[t-1] * S[t+1].
 * Must be called by all 128 threads of the CTA (it synchronises).  Cost per thread: 16 products + 1/4 inversion.
 */
/*
 * Experimental (off by default, -DECC_CLUSTER_INV=2|4|8): K2 / K3 run as thread-block clusters and ONE inversion chain
 * serves the whole cluster — the CTA totals are exchanged through distributed shared memory, rank 0 inverts their
 * product and hands every CTA the inverse of its own total.  The chain's share per thread drops from 330/4 to
 * 330/(4*CL) product-equivalents (roofline.py: cta_inv).  Not part of the validated default build.
 */
#define ECC_CTA_INV_WORDS(N) ((4 * 128 + 2 + 8) * (N)) /* shared words one CTA-wide inversion needs */
template <class FT, int CL = 1>
__device__ __forceinline__ void cta_inverse_128(Fe<FT::N> &inv, const Fe<FT::N> &acc, uint32_t *__restrict__ sh)
{
	typedef Field<FT> F;
	constexpr int N = FT::N;
	/* sh: ECC_CTA_INV_WORDS(N) words of shared memory, owned by the kernel so that calls for different fields (mod q
	 * and mod p in K3) reuse the same 16-37 KB */
	uint32_t *sP[2] = { sh, sh + 128 * N };                 /* double-buffered prefix scan */
	uint32_t *sS[2] = { sh + 2 * 128 * N, sh + 3 * 128 * N }; /* double-buffered suffix scan */
	uint32_t *sInv = sh + 4 * 128 * N;
	const int t = threadIdx.x;
	auto st_sh = [&](uint32_t *base, int idx, const Fe<N> &v) {
#pragma unroll
		for (int j = 0; j < N; j++) base[idx * N + j] = v.w[j];
	};
	auto ld_sh = [&](Fe<N> &v, const uint32_t *base, int idx) {
#pragma unroll
		for (int j = 0; j < N; j++) v.w[j] = base[idx * N + j];
	};
	Fe<N> pv = acc, sv = acc;
	st_sh(sP[0], t, pv);
	st_sh(sS[0], t, sv);
	__syncthreads();
	int cur = 0;
#pragma unroll 1
	for (int d = 1; d < 128; d <<= 1) {
		Fe<N> o, r;
		if (t >= d) {
			ld_sh(o, sP[cur], t - d);
			F::mul(r, pv, o);
			pv = r;
		}
		if (t + d < 128) {
			ld_sh(o, sS[cur], t + d);
			F::mul(r, sv, o);
			sv = r;
		}
		st_sh(sP[cur ^ 1], t, pv);
		st_sh(sS[cur ^ 1], t, sv);
		__syncthreads();
		cur ^= 1;
	}
	/* pv = prod_{u <= t} acc_u, sv = prod_{u >= t} acc_u; CTA product = P[127] */
#if ECC_CLUSTER_INV > 1
	if (CL > 1) {
		namespace cg = cooperative_groups;
		cg::cluster_group cluster = cg::this_cluster();
		const unsigned rank = cluster.block_rank();
		uint32_t *sTot = sh + (4 * 128 + 1) * N;  /* this CTA's total, read by rank 0 */
		uint32_t *sInvs = sh + (4 * 128 + 2) * N; /* rank 0: inverse of every CTA's total, [CL][N] */
		if (t == 0) {
			Fe<N> tot;
			ld_sh(tot, sP[cur], 127);
#pragma unroll
			for (int j = 0; j < N; j++) sTot[j] = tot.w[j];
		}
		cluster.sync();
		if (rank == 0 && t < 32) {
			Fe<N> T[CL], pre[CL], suf[CL], ti, r;
#pragma unroll
			for (int c = 0; c < CL; c++) {
				const uint32_t *rt = cluster.map_shared_rank(sTot, c);
#pragma unroll
				for (int j = 0; j < N; j++) T[c].w[j] = rt[j];
			}
			pre[0] = T[0];
#pragma unroll
			for (int c = 1; c < CL; c++) F::mul(pre[c], pre[c - 1], T[c]);
			suf[CL - 1] = T[CL - 1];
#pragma unroll
			for (int c = CL - 2; c >= 0; c--) F::mul(suf[c], suf[c + 1], T[c]);
			F::inv(ti, pre[CL - 1]);
#pragma unroll
			for (int c = 0; c < CL; c++) {
				Fe<N> v = ti;
				if (c > 0) {
					F::mul(r, v, pre[c - 1]);
					v = r;
				}
				if (c < CL - 1) {
					F::mul(r, v, suf[c + 1]);
					v = r;
				}
				if (t == 0) {
#pragma unroll
					for (int j = 0; j < N; j++) sInvs[c * N + j] = v.w[j];
				}
			}
		}
		cluster.sync();
		{
			const uint32_t *r0 = cluster.map_shared_rank(sInvs, 0);
#pragma unroll
			for (int j = 0; j < N; j++) inv.w[j] = r0[rank * N + j];
		}
		cluster.sync(); /* rank 0's shared memory has been read by everyone */
	} else
#endif
	{
		if (t < 32) {
			Fe<N> tot, ti;
			ld_sh(tot, sP[cur], 127);
			F::inv(ti, tot);
			if (t == 0) {
#pragma unroll
				for (int j = 0; j < N; j++) sInv[j] = ti.w[j];
			}
		}
		__syncthreads();
#pragma unroll
		for (int j = 0; j < N; j++) inv.w[j] = sInv[j];
	}
	Fe<N> o, r;
	if (t > 0) {
		ld_sh(o, sP[cur], t - 1);
		F::mul(r, inv, o);
		inv = r;
	}
	if (t < 127) {
		ld_sh(o, sS[cur], t + 1);
		F::mul(r, inv, o);
		inv = r;
	}
	__syncthreads(); /* the buffers may be reused by a second call */
}

/* ------------------------------------------------------------------------------------------ K1: fixed base */

/* minimum resident CTAs per SM of K1 (register cap), left at 1: the kernel is bound by the integer pipes, not by
 * latency hiding, so a tighter cap with spills did not pay (chosen on the previous GPU target and not re-measured on H100). */
#ifndef ECC_MINB_FIXED
#define ECC_MINB_FIXED 1
#endif
template <class C>
__global__ void __launch_bounds__(128, ECC_MINB_FIXED) k_smul_fixed(uint32_t n, const uint8_t *__restrict__ scalars,
						    const uint32_t *__restrict__ table, int w,
						    uint32_t *__restrict__ jac, int8_t *__restrict__ status)
{
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<C::N> k;
	load_wire<C::N, C::QLEN>(k, scalars + (size_t)idx * C::QLEN);
	scalar_reduce<C>(k);
	Jac<C> acc;
	comb_mul<C>(acc, k, table, w);
	store_jac<C>(jac, idx, acc);
	status[idx] = 0;
}

/*
 * Staging experiment (DESIGN.md §3): K1 with the CTA's 128 scalars brought into shared memory by ONE bulk
 * asynchronous copy (cp.async.bulk -> SASS UBLKCP, completion on an mbarrier) instead of per-thread 16-byte loads.
 * Same results; selected with ECCB200_TMA_STAGING=1 so that both variants can be timed.  The scalar traffic is 32 B
 * per ~100 field products, so no effect is expected — and none was measured.
 */
template <class C>
__global__ void __launch_bounds__(128) k_smul_fixed_tma(uint32_t n, const uint8_t *__restrict__ scalars,
							 const uint32_t *__restrict__ table, int w,
							 uint32_t *__restrict__ jac, int8_t *__restrict__ status)
{
	constexpr int N = C::N;
	__shared__ __align__(128) uint8_t sbuf[128 * 4 * N];
	__shared__ __align__(8) uint64_t bar;
	const uint32_t base = blockIdx.x * 128u;
	const uint32_t cnt = (n - base < 128u) ? (n - base) : 128u;
	const uint32_t bytes = cnt * 4u * N; /* multiple of 16 */
	const uint32_t bar_addr = (uint32_t)__cvta_generic_to_shared(&bar);
	const uint32_t dst_addr = (uint32_t)__cvta_generic_to_shared(sbuf);
	if (threadIdx.x == 0) {
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_addr));
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_addr), "r"(bytes) : "memory");
		asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
			     ::"r"(dst_addr), "l"(scalars + (size_t)base * (4 * N)), "r"(bytes), "r"(bar_addr)
			     : "memory");
	}
	{ /* every thread waits for phase 0 of the barrier */
		uint32_t done = 0;
		while (!done) {
			asm volatile("{\n\t.reg .pred p;\n\t"
				     "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
				     "selp.u32 %0, 1, 0, p;\n\t}"
				     : "=r"(done)
				     : "r"(bar_addr)
				     : "memory");
		}
	}
	if (threadIdx.x >= cnt) return;
	const uint32_t idx = base + threadIdx.x;
	Fe<N> k;
	{
		const uint4 *p = reinterpret_cast<const uint4 *>(sbuf + (size_t)threadIdx.x * (4 * N));
#pragma unroll
		for (int j = 0; j < N / 4; j++) {
			uint4 v = p[j];
			k.w[N - 1 - 4 * j] = bswap32(v.x);
			k.w[N - 2 - 4 * j] = bswap32(v.y);
			k.w[N - 3 - 4 * j] = bswap32(v.z);
			k.w[N - 4 - 4 * j] = bswap32(v.w);
		}
	}
	scalar_reduce<C>(k);
	Jac<C> acc;
	comb_mul<C>(acc, k, table, w);
	store_jac<C>(jac, idx, acc);
	status[idx] = 0;
}

/* ------------------------------------------------------------------------------------------ K2: variable base */

/* Minimum resident CTAs per SM for K2 / K3.  With the out-of-line multiplier the extra warps hide its fixed-latency
 * dependency chains better than the few spills cost (chosen on the previous GPU target and not re-measured on H100).  The caps follow from the register file (64 K 32-bit registers
 * and at most 2048 threads per SM on sm_90): 7 CTAs of 128 threads leave 72 registers per thread. */
#ifndef ECC_MINB_VAR
#define ECC_MINB_VAR 7
#endif
#ifndef ECC_MINB_VERIFY
#define ECC_MINB_VERIFY 7
#endif
/* 12-word fields (P-384) need 1.5x the registers per element: keep their caps at 168 / 128 registers;
 * 18-word fields (P-521) get the full 255 (2 CTAs per SM) */
#ifndef ECC_MINB_VAR_WIDE
#define ECC_MINB_VAR_WIDE 3
#endif
#ifndef ECC_MINB_VERIFY_WIDE
#define ECC_MINB_VERIFY_WIDE 4
#endif
template <class C>
__global__ void ECC_CLUSTER_ATTR __launch_bounds__(128, (C::N <= 8 ? ECC_MINB_VAR : (C::N <= 12 ? ECC_MINB_VAR_WIDE : 2))) k_smul_var(uint32_t n, const uint8_t *__restrict__ scalars,
						  const uint8_t *__restrict__ points, uint32_t *__restrict__ jac,
						  int8_t *__restrict__ status)
{
	/* every thread of the CTA walks the whole kernel (the table inversion is CTA-wide); threads past n and threads
	 * whose point was rejected work on the generator and discard the result */
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = idx < n;
	const uint32_t i0 = active ? idx : 0;
	__shared__ uint32_t sh_inv[ECC_CTA_INV_WORDS(C::N)];
	Fe<C::N> k;
	load_wire<C::N, C::QLEN>(k, scalars + (size_t)i0 * C::QLEN);
	scalar_reduce<C>(k);
	Aff<C> P;
	bool ok = load_affine_checked<C>(P, points + (size_t)i0 * (2 * C::PLEN));
	if (!ok) {
#pragma unroll
		for (int j = 0; j < C::N; j++) {
			P.x.w[j] = C::GX_MONT(j);
			P.y.w[j] = C::GY_MONT(j);
		}
	}
	Jac<C> acc;
	window_mul<C>(acc, k, P, nullptr, [&](Fe<C::N> &r, const Fe<C::N> &a) {
		cta_inverse_128<typename C::Fp, ECC_CLUSTER_INV>(r, a, sh_inv);
	});
	if (!active) return;
	if (!ok) EC<C>::set_inf(acc);
	store_jac<C>(jac, idx, acc);
	status[idx] = ok ? 0 : -1;
}

/* Comb-table build (w <= 16, and the half-width base table of wider ones): entry e = (i << w) + d  ->
 * (d << (w*i)) * G, through the same window_mul as K2. */
template <class C>
__global__ void __launch_bounds__(128) k_table_points(uint32_t n_entries, int w, uint32_t *__restrict__ jac)
{
	uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= n_entries) return;
	constexpr int N = C::N;
	uint32_t d = e & ((1u << w) - 1u);
	int i = (int)(e >> w);
	int bit = i * w;
	Fe<N> k;
#pragma unroll
	for (int j = 0; j < N; j++) k.w[j] = 0;
	Jac<C> acc;
	EC<C>::set_inf(acc);
	if (d != 0 && bit < 32 * N) {
		uint64_t v = (uint64_t)d << (bit & 31);
		int wi = bit >> 5;
#pragma unroll
		for (int j = 0; j < N; j++) {
			if (j == wi) k.w[j] = (uint32_t)v;
			if (j == wi + 1) k.w[j] = (uint32_t)(v >> 32);
		}
		/* entries whose scalar would not be < q are never addressed by a reduced scalar; leave them at infinity */
		if (!Field<typename C::Fq>::geq_mod(k)) {
			Aff<C> G;
#pragma unroll
			for (int j = 0; j < N; j++) {
				G.x.w[j] = C::GX_MONT(j);
				G.y.w[j] = C::GY_MONT(j);
			}
			window_mul<C>(acc, k, G);
		}
	}
	store_jac<C>(jac, e, acc);
}

/*
 * Wide comb tables (w > 16) are built from a half-width one: entry (i, d) of the w-bit table is
 * T_h[2i][d mod 2^h] + T_h[2i+1][d >> h] with h = w/2 — one affine+affine addition per entry instead of a scalar
 * multiplication, then the batched normalisation.  An all-zero base entry stands for the point at infinity.
 * count entries starting at wide index first_entry; results (Jacobian) go to jac[0 .. count).
 */
template <class C>
__global__ void __launch_bounds__(128) k_table_merge(uint32_t count, uint64_t first_entry, int w, int nwin_half,
						     const uint32_t *__restrict__ half_table,
						     uint32_t *__restrict__ jac)
{
	typedef Field<typename C::Fp> F;
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= count) return;
	const int h = w >> 1;
	uint64_t e = first_entry + idx;
	uint32_t i = (uint32_t)(e >> w);
	uint32_t d = (uint32_t)(e & ((1ull << w) - 1ull));
	uint32_t lo = d & ((1u << h) - 1u), hi = d >> h;
	Jac<C> acc;
	EC<C>::set_inf(acc);
	bool valid = !(hi != 0 && (int)(2 * i + 1) >= nwin_half) && (int)(2 * i) < nwin_half;
	if (valid && lo != 0) {
		Aff<C> a;
		load_table_entry<C>(a, half_table, ((size_t)(2 * i) << h) + lo);
		if (F::is_zero(a.x) && F::is_zero(a.y)) valid = false;
		else EC<C>::from_affine(acc, a);
	}
	if (valid && hi != 0) {
		Aff<C> b;
		load_table_entry<C>(b, half_table, ((size_t)(2 * i + 1) << h) + hi);
		if (F::is_zero(b.x) && F::is_zero(b.y)) valid = false;
		else {
			Jac<C> r;
			EC<C>::add_mixed(r, acc, b);
			acc = r;
		}
	}
	if (!valid) EC<C>::set_inf(acc);
	store_jac<C>(jac, idx, acc);
}

/* ------------------------------------------------------------------------------------------ K4: normalisation */

/*
 * Jacobian -> affine for a whole batch with ONE field inversion per CTA (Montgomery's simultaneous inversion, two
 * levels): thread t owns items t, t+T, t+2T, ... (T = total threads, so every pass over the batch is coalesced), keeps
 * the running product of their Z in registers and stores the prefix products; the CTA's 128 thread products are then
 * combined through shared memory, one warp inverts, and each thread walks back over its items.
 * Replaces n calls of prj_pt_unique (curves/prj_pt.c:241) -> fp_inv (fp/fp_mul.c:51, ~1.5*bitlen(p) products each).
 * MODE 0: Jacobian in, writes big-endian affine bytes + status (0 -> stays 0, infinity -> 1, -1 untouched).
 * MODE 1: Jacobian in, writes Montgomery-form words (comb table entry format), infinity as all-zero.
 * MODE 2: homogeneous projective in (x = X/Z, y = Y/Z, the reference's prj_pt), output as MODE 0: the batched
 *         prj_pt_unique + prj_pt_export_to_aff_buf (curves/prj_pt.c:241, :600).
 * MODE 3: Jacobian in, writes only the big-endian x coordinate ([n][plen]); infinity is an error (-1): the shared
 *         secret of ecccdh_derive_secret (ecdh/ecccdh.c:209-224).
 */
/*
 * Result gather fused into K4 (multi-GPU, one process per GPU; DESIGN.md §5): besides its own `out` / `status` the
 * kernel stores every item's affine bytes and status byte straight into up to ECC_MAX_GATHER_DST other buffers — the
 * gathered result buffers of peer GPUs, mapped through CUDA IPC, so the stores travel over NVLink while the kernel
 * computes — and the LAST CTA to finish publishes `flag_value` to each destination's arrival flag with a
 * system-scope release store.  No separate collective kernel runs, so nothing competes with K1 for the SMs.
 */
#define ECC_MAX_GATHER_DST 8
struct GatherDst {
	int n = 0;                              /* remote destinations (0: plain K4) */
	uint8_t *out[ECC_MAX_GATHER_DST];       /* slot base of this rank's shard in destination j: [n_items][2*plen] */
	int8_t *status[ECC_MAX_GATHER_DST];     /* [n_items] */
	uint32_t *flag[ECC_MAX_GATHER_DST];     /* arrival flag of this rank at destination j */
	uint32_t flag_value = 0;
	int signal = 1;                         /* publish the flags when this launch has stored everything (the last
	                                         * launch of a batch that is normalised in several slices) */
	unsigned int *counter = nullptr;        /* local: CTAs finished (reset by the last one) */
};

__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v)
{
	asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p)
{
	uint32_t v;
	asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}

template <class C, int MODE>
__global__ void __launch_bounds__(128) k_to_affine(uint32_t n, const uint32_t *__restrict__ jac,
						   uint32_t *__restrict__ prefix, uint8_t *__restrict__ out,
						   int8_t *__restrict__ status, uint32_t *__restrict__ table_out,
						   const GatherDst gd)
{
	typedef Field<typename C::Fp> F;
	constexpr int N = C::N;
	constexpr int PL = C::PLEN;
	constexpr bool TABLE = (MODE == 1);
	const uint32_t T = gridDim.x * blockDim.x;
	const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = tid < n; /* idle threads still take part in the block-wide inversion below */
	Fe<N> acc;
	F::set_one(acc);
	uint32_t last = tid;
	if (active) {
		for (uint32_t e = tid; e < n; e += T) {
			Fe<N> z;
			load_words<N>(z, jac + (size_t)e * (3 * N) + 2 * N);
			store_words<N>(prefix + (size_t)e * N, acc);
			if (!F::is_zero(z)) {
				Fe<N> t;
				F::mul(t, acc, z);
				acc = t;
			}
			last = e;
			if (n - e <= T) break; /* avoid uint32 overflow of e += T */
		}
	}
	Fe<N> inv;
	__shared__ __align__(16) uint32_t sh_inv[ECC_CTA_INV_WORDS(N)]; /* reused by the gather stores below */
	cta_inverse_128<typename C::Fp>(inv, acc, sh_inv); /* one inversion per CTA instead of one per thread */
	if (active)
	for (uint32_t e = last;; e -= T) {
		Fe<N> z, pre, X, Y, gx, gy; /* gx, gy, gst: what the gather stores for this item (MODE 0) */
		int8_t gst = 0;
		const uint32_t *b = jac + (size_t)e * (3 * N);
		load_words<N>(z, b + 2 * N);
		bool inf = F::is_zero(z);
		bool err = (!TABLE) && (status[e] < 0);
		if (!inf) {
			Fe<N> zi, zi2, zi3, t;
			load_words<N>(pre, prefix + (size_t)e * N);
			load_words<N>(X, b);
			load_words<N>(Y, b + N);
			F::mul(zi, inv, pre);  /* 1/z_e */
			F::mul(t, inv, z);
			inv = t;               /* drop z_e from the running inverse */
			if (TABLE) { /* Montgomery-form output: 1/z^2, 1/z^3 stay in the Montgomery domain */
				F::sqr(zi2, zi);
				F::mul(zi3, zi2, zi);
			} else {
				/* byte output: take 1/z OUT of the Montgomery domain once (zp = z^-1 as a plain integer); products of
				 * a plain factor and a Montgomery-form factor are plain, so X * zp^2 and Y * zp^3 come out as the
				 * plain coordinates directly — one product less than normalising in the domain and leaving it twice */
				Fe<N> zp;
				F::from_mont(zp, zi);
				if (MODE == 2) {
					zi2 = zp;
					zi3 = zp;
				} else {
					F::mul(zi2, zp, zi);
					F::mul(zi3, zi2, zi);
				}
			}
			F::mul(t, X, zi2);
			X = t;
			F::mul(t, Y, zi3);
			Y = t;
			if (TABLE) {
				store_words<N>(table_out + (size_t)e * (2 * N), X);
				store_words<N>(table_out + (size_t)e * (2 * N) + N, Y);
			} else if (MODE == 3) {
				t = X;
				store_wire<N, PL>(out + (size_t)e * PL, t);
			} else {
				t = X;
				zi = Y;
				store_wire<N, PL>(out + (size_t)e * (2 * PL), t);
				store_wire<N, PL>(out + (size_t)e * (2 * PL) + PL, zi);
				if (MODE == 0) {
					gx = t;
					gy = zi;
					gst = err ? (int8_t)-1 : (int8_t)0;
				}
			}
		} else {
			Fe<N> zero;
			F::set_zero(zero);
			if (TABLE) {
				store_words<N>(table_out + (size_t)e * (2 * N), zero);
				store_words<N>(table_out + (size_t)e * (2 * N) + N, zero);
			} else if (MODE == 3) {
				store_wire<N, PL>(out + (size_t)e * PL, zero);
				status[e] = -1;
			} else {
				store_wire<N, PL>(out + (size_t)e * (2 * PL), zero);
				store_wire<N, PL>(out + (size_t)e * (2 * PL) + PL, zero);
				if (!err) status[e] = 1;
				if (MODE == 0) {
					gx = zero;
					gy = zero;
					gst = err ? (int8_t)-1 : (int8_t)1;
				}
			}
		}
		if (MODE == 0 && gd.n > 0) {
			/* the gather stores.  A fully active warp holds 32 consecutive items = 32 * 2*PL contiguous bytes per
			 * destination: they are transposed through shared memory so that every store instruction writes 512
			 * contiguous bytes (whole 128-byte lines on the NVLink) instead of 32 separate 16-byte pieces. */
			const unsigned act = __activemask();
			const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
			bool coop = (N % 4 == 0) && (PL == 4 * N) && act == 0xffffffffu;
			if (coop) { /* all 32 lanes are here together: are they also on the same pass over the batch? */
				const uint32_t first = e - (uint32_t)lane;
				coop = __all_sync(0xffffffffu, first == __shfl_sync(0xffffffffu, first, 0));
			}
			if (coop) {
				constexpr int W4 = 2 * N / 4;               /* uint4 per item */
				uint4 *row = reinterpret_cast<uint4 *>(sh_inv) + warp * (32 * W4 + 2);
#pragma unroll
				for (int k = 0; k < N / 4; k++) {
					uint4 vx, vy;
					vx.x = bswap32(gx.w[N - 1 - 4 * k]);
					vx.y = bswap32(gx.w[N - 2 - 4 * k]);
					vx.z = bswap32(gx.w[N - 3 - 4 * k]);
					vx.w = bswap32(gx.w[N - 4 - 4 * k]);
					vy.x = bswap32(gy.w[N - 1 - 4 * k]);
					vy.y = bswap32(gy.w[N - 2 - 4 * k]);
					vy.z = bswap32(gy.w[N - 3 - 4 * k]);
					vy.w = bswap32(gy.w[N - 4 - 4 * k]);
					row[lane * W4 + k] = vx;
					row[lane * W4 + N / 4 + k] = vy;
				}
				reinterpret_cast<int8_t *>(row + 32 * W4)[lane] = gst;
				__syncwarp();
				const size_t e0 = (size_t)(e - (uint32_t)lane); /* item of lane 0 (consecutive lanes, consecutive items) */
				for (int j = 0; j < gd.n; j++) {
					uint4 *dst = reinterpret_cast<uint4 *>(gd.out[j] + e0 * (2 * PL));
#pragma unroll
					for (int k = 0; k < W4; k++) dst[k * 32 + lane] = row[k * 32 + lane];
					if (lane < 2) reinterpret_cast<uint4 *>(gd.status[j] + e0)[lane] = row[32 * W4 + lane];
				}
				__syncwarp();
			} else {
				for (int j = 0; j < gd.n; j++) {
					store_wire<N, PL>(gd.out[j] + (size_t)e * (2 * PL), gx);
					store_wire<N, PL>(gd.out[j] + (size_t)e * (2 * PL) + PL, gy);
					gd.status[j][e] = gst;
				}
			}
		}
		if (e < T || e - T < tid) break;
	}
	if (MODE == 0 && gd.n > 0 && gd.signal) {
		/* every thread's remote stores are ordered before the counter increment; the last CTA publishes the flags */
		__threadfence_system();
		__syncthreads();
		if (threadIdx.x == 0) {
			const unsigned int done = atomicAdd(gd.counter, 1u);
			if (done == gridDim.x - 1) {
				*gd.counter = 0;
				__threadfence_system();
				for (int j = 0; j < gd.n; j++) st_release_sys(gd.flag[j], gd.flag_value);
			}
		}
	}
}

/* Loads homogeneous projective wire points (X||Y||Z big-endian, prj_pt_export_to_buf curves/prj_pt.c:562), checks
 * them like prj_pt_import_from_buf (:462-500: coordinates < p, Y^2 Z == X^3 + a X Z^2 + b Z^3) and writes
 * Montgomery-form words for k_to_affine<MODE 2>.  status: 0 ok, -1 rejected (then Z is written as 0). */
template <class C>
__global__ void __launch_bounds__(128) k_prj_load(uint32_t n, const uint8_t *__restrict__ prj,
						  uint32_t *__restrict__ jac, int8_t *__restrict__ status)
{
	typedef Field<typename C::Fp> F;
	constexpr int N = C::N;
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<N> x, y, z;
	const uint8_t *b = prj + (size_t)idx * (3 * C::PLEN);
	load_wire<N, C::PLEN>(x, b);
	load_wire<N, C::PLEN>(y, b + C::PLEN);
	load_wire<N, C::PLEN>(z, b + 2 * C::PLEN);
	bool ok = !F::geq_mod(x) && !F::geq_mod(y) && !F::geq_mod(z);
	Jac<C> P;
	F::to_mont(P.X, x);
	F::to_mont(P.Y, y);
	F::to_mont(P.Z, z);
	{ /* Y^2 Z == X^3 + a X Z^2 + b Z^3 */
		Fe<N> l, r, t, z2, bm;
		F::sqr(t, P.Y);
		F::mul(l, t, P.Z);
		F::sqr(t, P.X);
		F::mul(r, t, P.X);
		F::sqr(z2, P.Z);
		F::mul(t, P.X, z2);
		if (C::A_KIND == 0) {
			F::sub(r, r, t);
			F::sub(r, r, t);
			F::sub(r, r, t);
		} else if (C::A_KIND == 2) {
			Fe<N> am, at;
			EC<C>::load_a(am);
			F::mul(at, am, t);
			F::add(r, r, at);
		}
#pragma unroll
		for (int i = 0; i < N; i++) bm.w[i] = C::B_MONT(i);
		F::mul(t, z2, P.Z);
		F::mul(z2, t, bm);
		F::add(r, r, z2);
		ok = ok && F::eq(l, r);
	}
	if (!ok) F::set_zero(P.Z);
	store_jac<C>(jac, idx, P);
	status[idx] = ok ? 0 : -1;
}

/* ------------------------------------------------------------------------------------------ K3: ECDSA verify */

/*
 * One signature per thread.  Follows __ecdsa_verify_init (sig/ecdsa_common.c:645-658) and
 * __ecdsa_verify_finalize (:760-810) step by step; differences that do not change the verdict:
 *   - s^-1 mod q by Field::inv (safegcd) in the Montgomery domain of q instead of nn_modinv's xgcd (:781);
 *   - W' = uG + vY is kept Jacobian and "x(W') mod q == r" is tested without an inversion as
 *     X == c * Z^2 for the candidates c in {r, r+q} that are < p (:803-810);
 *   - uG via the comb table (K1), vY via the signed window (K2) instead of two ladders (:788,793).
 * digests: hlen bytes each; e = leftmost min(8*hlen, bitlen(q)) bits (:760-775), reduced mod q (:777).
 */
template <class C, int SCHEME = 0>
__global__ void ECC_CLUSTER_ATTR __launch_bounds__(128, (C::N <= 8 ? ECC_MINB_VERIFY : (C::N <= 12 ? ECC_MINB_VERIFY_WIDE : 2))) k_ecdsa_verify(uint32_t n, const uint8_t *__restrict__ sigs,
						      const uint8_t *__restrict__ pubkeys,
						      const uint8_t *__restrict__ digests, uint32_t hlen,
						      const uint32_t *__restrict__ table, int w,
						      int8_t *__restrict__ verdict,
						      const int8_t *__restrict__ key_state,
						      uint8_t *__restrict__ aux_out)
{
	/* key_state (optional, from the structured-key import): 0 = pubkeys[i] is a validated affine point, 1 = the key
	 * is the point at infinity (pubkeys[i] ignored), -1 = the key or signature record was rejected */
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N;
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = idx < n;
	const uint32_t i0 = active ? idx : 0; /* idle threads of the last CTA still join the CTA-wide inversion */

	if (SCHEME == 1) {
		/* ECFSDSA (sig/ecfsdsa.c:416-610, SURVEY.md §8f.4): signature r || s with r = W_x || W_y a curve point and s in
		 * ]0, q[; digests[i] = H(r || m); W' = sG + (-h mod q) Y must equal r.  Same double-scalar core as ECDSA — comb
		 * for the generator, signed window for the key — without the mod-q inversion. */
		__shared__ uint32_t sh_inv1[ECC_CTA_INV_WORDS(N)];
		const uint8_t *sg = sigs + (size_t)i0 * (2 * C::PLEN + C::QLEN);
		Aff<C> Rp, Y;
		Fe<N> s, h;
		const bool r_ok = load_affine_checked<C>(Rp, sg);                 /* (:453-460) */
		load_wire<N, C::QLEN>(s, sg + 2 * C::PLEN);
		const bool s_ok = !Fq::is_zero(s) && !Fq::geq_mod(s);            /* (:465-470) */
		const bool key_ok = load_affine_checked<C>(Y, pubkeys + (size_t)i0 * (2 * C::PLEN));
		digest_full_mod_q<C>(h, digests + (size_t)i0 * hlen, hlen);      /* (:590-592) */
		Fq::neg(h, h);                                                    /* e = -h mod q (:594) */
		const bool run = r_ok && s_ok && key_ok;
		if (!run) {
			Fq::set_zero(s);
			Fq::set_zero(h);
#pragma unroll
			for (int j = 0; j < N; j++) {
				Y.x.w[j] = C::GX_MONT(j);
				Y.y.w[j] = C::GY_MONT(j);
			}
		}
		int code = ecfsdsa_verify_tail<C>(Rp, s, h, Y, table, w, [&](Fe<N> &o, const Fe<N> &a) {
			cta_inverse_128<typename C::Fp, ECC_CLUSTER_INV>(o, a, sh_inv1);
		});
		if (!active) return;
		if (!run) code = 1;
		verdict[idx] = code ? -1 : 0;
		return;
	}

	if (SCHEME == 3) {
		/*
		 * Generic double-scalar multiplication W = a*G + b*Y with an affine result: the EC core of every remaining
		 * Schnorr-type verification of the reference (ECSDSA / ECOSDSA sig/ecsdsa_common.c:493-497: W' = sG + eY;
		 * ECKCDSA: W' = sY + eG; ...), i.e. the sequence prj_pt_mul, prj_pt_mul, prj_pt_add, prj_pt_unique.  Those
		 * schemes hash the recomputed point, which stays on the host (src/hash); this kernel hands it W'.
		 * sigs[i] = a || b (QLEN bytes each, any value: reduced mod q like the ladder does); verdict: 0 finite,
		 * 1 infinity (prj_pt_unique fails on it), -1 key rejected; aux_out [n][2*PLEN] affine bytes (zero if not finite).
		 */
		typedef Field<typename C::Fp> F;
		__shared__ uint32_t sh_inv3[ECC_CTA_INV_WORDS(N)];
		const uint8_t *sg = sigs + (size_t)i0 * (2 * C::QLEN);
		Fe<N> a, b;
		Aff<C> Y;
		load_wire<N, C::QLEN>(a, sg);
		load_wire<N, C::QLEN>(b, sg + C::QLEN);
		scalar_reduce<C>(a);
		scalar_reduce<C>(b);
		const bool key_ok = load_affine_checked<C>(Y, pubkeys + (size_t)i0 * (2 * C::PLEN));
		if (!key_ok) {
			Fq::set_zero(a);
			Fq::set_zero(b);
#pragma unroll
			for (int j = 0; j < N; j++) {
				Y.x.w[j] = C::GX_MONT(j);
				Y.y.w[j] = C::GY_MONT(j);
			}
		}
		Jac<C> aG, W;
		comb_mul<C>(aG, a, table, w);
		window_mul<C>(W, b, Y, &aG, [&](Fe<N> &o, const Fe<N> &v) {
			cta_inverse_128<typename C::Fp, ECC_CLUSTER_INV>(o, v, sh_inv3);
		});
		const bool inf = EC<C>::is_inf(W);
		Fe<N> z = W.Z, zi, zp, zi2, zi3, x, y;
		if (inf) F::set_one(z);
		cta_inverse_128<typename C::Fp, ECC_CLUSTER_INV>(zi, z, sh_inv3);
		F::from_mont(zp, zi);        /* 1/z out of the Montgomery domain once: X * zp^2, Y * zp^3 are plain */
		F::mul(zi2, zp, zi);
		F::mul(zi3, zi2, zi);
		F::mul(x, W.X, zi2);
		F::mul(y, W.Y, zi3);
		if (!active) return;
		const bool fin = key_ok && !inf;
		if (!fin) {
			F::set_zero(x);
			F::set_zero(y);
		}
		store_wire<N, C::PLEN>(aux_out + (size_t)idx * (2 * C::PLEN), x);
		store_wire<N, C::PLEN>(aux_out + (size_t)idx * (2 * C::PLEN) + C::PLEN, y);
		verdict[idx] = !key_ok ? (int8_t)-1 : (inf ? (int8_t)1 : (int8_t)0);
		return;
	}

	if (SCHEME == 2) {
		/* BIP0340 (sig/bip0340.c:383-577, SURVEY.md §8f.4): signature r || s with r a field element (the x coordinate
		 * of the nonce point) and s < q; digests[i] = the tagged hash H(H(tag) || H(tag) || r || Y_x || m) computed by the
		 * host; W' = sG - eY' with the key lifted to an even y; accept iff W' is finite, y(W') even and x(W') == r. */
		typedef Field<typename C::Fp> F;
		__shared__ uint32_t sh_inv2[ECC_CTA_INV_WORDS(N)];
		const uint8_t *sg = sigs + (size_t)i0 * (C::PLEN + C::QLEN);
		const uint8_t *pkb = pubkeys + (size_t)i0 * (2 * C::PLEN);
		Fe<N> r, s, h, yraw;
		Aff<C> Y;
		load_wire<N, C::PLEN>(r, sg);
		load_wire<N, C::QLEN>(s, sg + C::PLEN);
		const bool r_ok = !F::geq_mod(r);                                 /* fp_import_from_buf (:431) */
		const bool s_ok = !Fq::geq_mod(s);                                /* s < q (:433-434); s = 0 is not excluded */
		load_wire<N, C::PLEN>(yraw, pkb + C::PLEN);
		const bool key_ok = load_affine_checked<C>(Y, pkb);
		if (yraw.w[0] & 1u) F::neg(Y.y, Y.y);                             /* lift to the even y (:540-545) */
		digest_full_mod_q<C>(h, digests + (size_t)i0 * hlen, hlen);      /* e = OS2I(hash) mod q (:530-531) */
		Fq::neg(h, h);                                                    /* -e mod q (:538) */
		const bool run = r_ok && s_ok && key_ok;
		if (!run) {
			Fq::set_zero(s);
			Fq::set_zero(h);
#pragma unroll
			for (int j = 0; j < N; j++) {
				Y.x.w[j] = C::GX_MONT(j);
				Y.y.w[j] = C::GY_MONT(j);
			}
		}
		int code = bip0340_verify_tail<C>(r, s, h, Y, table, w, [&](Fe<N> &o, const Fe<N> &a) {
			cta_inverse_128<typename C::Fp, ECC_CLUSTER_INV>(o, a, sh_inv2);
		});
		if (!active) return;
		if (!run) code = 1;
		verdict[idx] = code ? -1 : 0;
		return;
	}

	Fe<N> r, s, e;
	load_wire<N, C::QLEN>(r, sigs + (size_t)i0 * (2 * C::QLEN));
	load_wire<N, C::QLEN>(s, sigs + (size_t)i0 * (2 * C::QLEN) + C::QLEN);
	const bool rs_ok = ecdsa_rs_in_range<C>(r, s);
	/* s^-1 mod q for the whole CTA at once (sig/ecdsa_common.c:781 does one nn_modinv per signature) */
	__shared__ uint32_t sh_inv[ECC_CTA_INV_WORDS(N)];
	Fe<N> sm, wm;
	Fq::set_one(sm);
	if (rs_ok) Fq::to_mont(sm, s);
	cta_inverse_128<typename C::Fq, ECC_CLUSTER_INV>(wm, sm, sh_inv);
	Aff<C> Y;
	const int ks = key_state ? (int)key_state[i0] : 0;
	bool key_ok = load_affine_checked<C>(Y, pubkeys + (size_t)i0 * (2 * C::PLEN));
	key_ok = (key_ok && ks == 0) || ks == 1;
	digest_to_scalar<C>(e, digests + (size_t)i0 * hlen, hlen);
	/* Every thread of the CTA runs the tail (its window table is normalised by a CTA-wide inversion); a rejected
	 * item runs it on u = v = 0 and the generator — the cheapest walk — and its result is ignored. */
	const bool run = key_ok && rs_ok;
	Fe<N> u, v;
	Fq::mul(u, e, wm); /* u = e * s^-1 mod q  (:786) */
	Fq::mul(v, r, wm); /* v = r * s^-1 mod q  (:791) */
	if (!run) {
		Fq::set_zero(u);
		Fq::set_zero(v);
	}
	if (!run || ks == 1) {
#pragma unroll
		for (int j = 0; j < N; j++) {
			Y.x.w[j] = C::GX_MONT(j);
			Y.y.w[j] = C::GY_MONT(j);
		}
	}
	int code = ecdsa_verify_tail<C>(r, u, v, Y, table, w, ks == 1, [&](Fe<N> &o, const Fe<N> &a) {
		cta_inverse_128<typename C::Fp, ECC_CLUSTER_INV>(o, a, sh_inv);
	});
	if (!active) return;
	if (!key_ok) code = 4;
	else if (!rs_ok) code = 1;
#if defined(ECC_VERDICT_DEBUG)
	verdict[idx] = (int8_t)(-code);
#else
	verdict[idx] = code ? -1 : 0;
#endif
}

/* ------------------------------------------------------------------------------------------ ECDSA key recovery */

/*
 * Batched ECDSA public-key recovery, __ecdsa_public_key_from_sig (sig/ecdsa_common.c:867-1011), one item per thread:
 * sigs[i] = r || s (2*QLEN bytes), digests[i] hlen bytes -> keys[i] = Y1 || Y2 (affine, 2*PLEN bytes each) and
 * status[i] = { s1, s2 }: 0 finite, 1 the point at infinity, -1 both where the reference returns -1.
 *   - range checks and r < p (ecdsa_recover_rs_ok), e as for verification (digest_to_scalar, :942-950);
 *   - r^-1 mod q for the whole CTA at once (one nn_modinv per item in the reference, :984); rejected items give 1;
 *   - R1 = (r, sqrt1) with the reference's root (Field::sqrt), x = r only (ec.cuh);
 *   - u*G through the comb, V = v*R1 through the signed window, then Y1 = uG + V and Y2 = uG - V: the EC work of ONE
 *     verification plus one addition, where the reference runs three ladders;
 *   - both keys normalised by one CTA-wide inversion of Z1*Z2 (Z taken as 1 at infinity).
 * A rejected item walks the same code on u = v = 0 and the generator: every CTA-wide inversion stays collective.
 */
template <class C>
__global__ void ECC_CLUSTER_ATTR __launch_bounds__(128, (C::N <= 8 ? ECC_MINB_VERIFY : (C::N <= 12 ? ECC_MINB_VERIFY_WIDE : 2))) k_ecdsa_recover(uint32_t n, const uint8_t *__restrict__ sigs,
								const uint8_t *__restrict__ digests, uint32_t hlen,
								const uint32_t *__restrict__ table, int w,
								uint8_t *__restrict__ keys, int8_t *__restrict__ status)
{
	typedef Field<typename C::Fq> Fq;
	typedef Field<typename C::Fp> F;
	constexpr int N = C::N;
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = idx < n;
	const uint32_t i0 = active ? idx : 0; /* idle threads of the last CTA still join the CTA-wide inversions */
	__shared__ uint32_t sh_inv[ECC_CTA_INV_WORDS(N)];
	Fe<N> r, s, e;
	load_wire<N, C::QLEN>(r, sigs + (size_t)i0 * (2 * C::QLEN));
	load_wire<N, C::QLEN>(s, sigs + (size_t)i0 * (2 * C::QLEN) + C::QLEN);
	const bool rs_ok = ecdsa_recover_rs_ok<C>(r, s);
	Fe<N> rm, ri;
	Fq::set_one(rm);
	if (rs_ok) Fq::to_mont(rm, r);
	cta_inverse_128<typename C::Fq, ECC_CLUSTER_INV>(ri, rm, sh_inv);
	digest_to_scalar<C>(e, digests + (size_t)i0 * hlen, hlen);
	Aff<C> R;
	const bool ok = rs_ok && ecdsa_recover_point<C>(R, r);
	Fe<N> u, v;
	ecdsa_recover_uv<C>(u, v, e, s, ri);
	if (!ok) {
		Fq::set_zero(u);
		Fq::set_zero(v);
#pragma unroll
		for (int j = 0; j < N; j++) {
			R.x.w[j] = C::GX_MONT(j);
			R.y.w[j] = C::GY_MONT(j);
		}
	}
	Jac<C> uG, V, Y1, Y2;
	comb_mul<C>(uG, u, table, w);
	window_mul<C>(V, v, R, nullptr, [&](Fe<N> &o, const Fe<N> &a) {
		cta_inverse_128<typename C::Fp, ECC_CLUSTER_INV>(o, a, sh_inv);
	});
	ecdsa_recover_keys<C>(Y1, Y2, uG, V);
	const bool inf1 = EC<C>::is_inf(Y1), inf2 = EC<C>::is_inf(Y2);
	Fe<N> z1 = Y1.Z, z2 = Y2.Z, z12, zi;
	if (inf1) F::set_one(z1);
	if (inf2) F::set_one(z2);
	F::mul(z12, z1, z2);
	cta_inverse_128<typename C::Fp, ECC_CLUSTER_INV>(zi, z12, sh_inv);
	if (!active) return;
	uint8_t *out = keys + (size_t)idx * (4 * C::PLEN);
	/* 1/Z1 = zi * Z2, 1/Z2 = zi * Z1; 1/Z out of the Montgomery domain once, so X * zp^2 and Y * zp^3 come out plain */
	auto put = [&](uint8_t *o, const Jac<C> &P, const Fe<N> &zo, bool fin) {
		Fe<N> zk, zp, zk2, zk3, x, y;
		F::mul(zk, zi, zo);
		F::from_mont(zp, zk);
		F::mul(zk2, zp, zk);
		F::mul(zk3, zk2, zk);
		F::mul(x, P.X, zk2);
		F::mul(y, P.Y, zk3);
		if (!fin) {
			F::set_zero(x);
			F::set_zero(y);
		}
		store_wire<N, C::PLEN>(o, x);
		store_wire<N, C::PLEN>(o + C::PLEN, y);
	};
	put(out, Y1, z2, ok && !inf1);
	put(out + 2 * C::PLEN, Y2, z1, ok && !inf2);
	status[2 * (size_t)idx] = !ok ? (int8_t)-1 : (inf1 ? (int8_t)1 : (int8_t)0);
	status[2 * (size_t)idx + 1] = !ok ? (int8_t)-1 : (inf2 ? (int8_t)1 : (int8_t)0);
}

/* ------------------------------------------------------------------------------------------ ECDSA sign (next row f.1) */

/*
 * Second half of a batched ECDSA signature (__ecdsa_sign_finalize steps 6-11, sig/ecdsa_common.c:479-560), after K1
 * computed k*G and K4 normalised it:  r = x(kG) mod q,  s = k^-1 (e + r*d) mod q.
 * k^-1 mod q uses the same two-level simultaneous inversion as K4 (one inversion mod q per CTA; the reference does
 * one nn_modinv_fermat per signature, :537).  status: 0 ok; 2 = the reference's "restart with a new nonce" cases
 * (r == 0 :487, e == r*d :513, s == 0 :545); -1 = d or k outside [1, q-1].
 */
template <class C>
__global__ void __launch_bounds__(128) k_ecdsa_sign_finish(uint32_t n, const uint8_t *__restrict__ privkeys,
							    const uint8_t *__restrict__ nonces,
							    const uint8_t *__restrict__ digests, uint32_t hlen,
							    const uint8_t *__restrict__ kG_aff,
							    uint32_t *__restrict__ prefix, uint8_t *__restrict__ sigs,
							    int8_t *__restrict__ status)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N;
	const uint32_t T = gridDim.x * blockDim.x;
	const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = tid < n;
	Fe<N> acc;
	Fq::set_one(acc);
	uint32_t last = tid;
	if (active) {
		for (uint32_t e = tid; e < n; e += T) {
			Fe<N> kk, km;
			load_wire<N, C::QLEN>(kk, nonces + (size_t)e * C::QLEN);
			store_words<N>(prefix + (size_t)e * N, acc);
			if (!Fq::is_zero(kk) && !Fq::geq_mod(kk)) {
				Fe<N> t;
				Fq::to_mont(km, kk);
				Fq::mul(t, acc, km);
				acc = t;
			}
			last = e;
			if (n - e <= T) break;
		}
	}
	Fe<N> inv;
	__shared__ uint32_t sh_inv[ECC_CTA_INV_WORDS(N)];
	cta_inverse_128<typename C::Fq>(inv, acc, sh_inv);
	if (!active) return;
	for (uint32_t e = last;; e -= T) {
		Fe<N> kk, d, x, r, ev, s, zero;
		Fq::set_zero(zero);
		load_wire<N, C::QLEN>(kk, nonces + (size_t)e * C::QLEN);
		load_wire<N, C::QLEN>(d, privkeys + (size_t)e * C::QLEN);
		bool k_ok = !Fq::is_zero(kk) && !Fq::geq_mod(kk);
		bool d_ok = !Fq::is_zero(d) && !Fq::geq_mod(d);
		int st = 0;
		r = zero;
		s = zero;
		if (k_ok) {
			Fe<N> km, pre, kinv, t, dm;
			load_words<N>(pre, prefix + (size_t)e * N);
			Fq::to_mont(km, kk);
			Fq::mul(kinv, inv, pre);  /* k^-1 in Montgomery form */
			Fq::mul(t, inv, km);
			inv = t;
			load_wire<N, C::PLEN>(x, kG_aff + (size_t)e * (2 * C::PLEN));
			r = x;
			scalar_reduce<C>(r);                        /* r = W_x mod q          (:483) */
			digest_to_scalar<C>(ev, digests + (size_t)e * hlen, hlen);
			Fq::to_mont(dm, d);
			Fq::mul(t, r, dm);                          /* x*r mod q              (:510) */
			bool restart = Fq::is_zero(r) || Fq::eq(t, ev);
			Fq::add(t, t, ev);                          /* e + x*r                (:521) */
			Fq::mul(s, t, kinv);                        /* s = k^-1 (e + x*r)     (:540) */
			restart = restart || Fq::is_zero(s);
			st = d_ok ? (restart ? 2 : 0) : -1;
		} else {
			st = -1;
		}
		if (st != 0) {
			r = zero;
			s = zero;
		}
		store_wire<N, C::QLEN>(sigs + (size_t)e * (2 * C::QLEN), r);
		store_wire<N, C::QLEN>(sigs + (size_t)e * (2 * C::QLEN) + C::QLEN, s);
		status[e] = (int8_t)st;
		if (e < T) break;
	}
}

/*
 * Before K1 of the deterministic and raw-message forms of the ECDSA signer, one item per thread.  With dig_out: the
 * digest H(m) into dig_out ([n][digest size]; message i is msgs[off[i] .. off[i+1]), as k_sha2_batch).  With k_out: the
 * RFC 6979 nonce of x and that digest (or of digests[i] without dig_out) into k_out (rfc6979_nonce), or 0 without any
 * HMAC work where x is outside [1, q-1] (k_ecdsa_sign_finish then reports ECCB200_ERR).  hash_type: 1..8 or 11.
 */
template <class C>
__global__ void __launch_bounds__(128) k_ecdsa_nonce(uint32_t n, int hash_type, const uint8_t *__restrict__ privkeys,
						     const uint8_t *__restrict__ digests, const uint8_t *__restrict__ msgs,
						     const uint64_t *__restrict__ off, uint8_t *__restrict__ dig_out,
						     uint8_t *__restrict__ k_out)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N;
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	const uint32_t ds = (uint32_t)decdsa_hash_digest_size(hash_type);
	uint8_t hm[64];
	const uint8_t *h = dig_out ? hm : digests + (size_t)idx * ds;
	if (dig_out) {
		decdsa_hash_src(hash_type, ByteSpan{ msgs + off[idx] }, off[idx + 1] - off[idx], hm);
		for (uint32_t i = 0; i < ds; i++) dig_out[(size_t)idx * ds + i] = hm[i];
	}
	if (!k_out) return;
	Fe<N> x, k;
	load_wire<N, C::QLEN>(x, privkeys + (size_t)idx * C::QLEN);
	Fq::set_zero(k);
	if (!Fq::is_zero(x) && !Fq::geq_mod(x)) rfc6979_nonce<C>(k, hash_type, x, h, ds);
	store_wire<N, C::QLEN>(k_out + (size_t)idx * C::QLEN, k);
}

/* ------------------------------------------------------------------------- ECKCDSA / ECGDSA / ECRDSA / SM2 sign */

/*
 * After K1 (k*G) and K4 (affine W): the hashes over the message (and SM2's Z, ECKCDSA's z and H(W_x)), then r and s
 * (msgs_sign_core).  Each thread owns items tid, tid + T, ... (T = the grid's threads), like k_ecdsa_sign_finish.  For
 * SM2, (1 + x)^-1 mod q comes from the same two-level simultaneous inversion: a serial prefix product over the
 * thread's items (prefix scratch), one CTA-wide inversion, then the items in reverse order.  Items whose x is outside
 * [1, q-2] stay out of the product.  The other schemes invert nothing and run one item per thread.
 * Messages / IDs as k_sha2_batch: item i's are msgs[off[i] .. off[i+1]) and ids[id_off[i] .. id_off[i+1]).
 * sigs: [n][msgs_sig_len], status: 0 / -1 / 2 (ECCB200_OK / _ERR / _RETRY).
 */
template <class C>
__global__ void __launch_bounds__(128) k_msgs_sign_finish(uint32_t n, int sig_type, int hash_type,
							  const uint8_t *__restrict__ privkeys,
							  const uint8_t *__restrict__ pubkeys,
							  const uint8_t *__restrict__ nonces,
							  const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off,
							  const uint8_t *__restrict__ ids,
							  const uint64_t *__restrict__ id_off,
							  const uint8_t *__restrict__ W_aff, uint32_t *__restrict__ prefix,
							  uint8_t *__restrict__ sigs, int8_t *__restrict__ status)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N;
	const bool sm2 = sig_type == SIG_SM2;
	const uint32_t T = gridDim.x * blockDim.x;
	const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = tid < n;
	Fe<N> inv;
	Fq::set_one(inv);
	uint32_t last = tid;
	if (active) last = tid + (n - 1 - tid) / T * T;
	if (sm2) {
		Fe<N> acc;
		Fq::set_one(acc);
		if (active) {
			for (uint32_t e = tid; e < n; e += T) {
				Fe<N> x;
				load_wire<N, C::QLEN>(x, privkeys + (size_t)e * C::QLEN);
				store_words<N>(prefix + (size_t)e * N, acc);
				if (msgs_key_in_range<C>(SIG_SM2, x)) {
					Fe<N> t, u;
					sm2_one_plus_x<C>(u, x);
					Fq::mul(t, acc, u);
					acc = t;
				}
				if (n - e <= T) break;
			}
		}
		__shared__ uint32_t sh_inv[ECC_CTA_INV_WORDS(N)];
		cta_inverse_128<typename C::Fq>(inv, acc, sh_inv);
	}
	if (!active) return;
	const int siglen = msgs_sig_len<C>(sig_type, msg_hash_digest_size(hash_type));
	const bool with_key = sm2 || sig_type == SIG_ECKCDSA;
	for (uint32_t e = last;; e -= T) {
		Fe<N> x, k, ix;
		load_wire<N, C::QLEN>(x, privkeys + (size_t)e * C::QLEN);
		load_wire<N, C::QLEN>(k, nonces + (size_t)e * C::QLEN);
		Fq::set_zero(ix);
		if (sm2 && msgs_key_in_range<C>(SIG_SM2, x)) {
			Fe<N> pre, u, t;
			load_words<N>(pre, prefix + (size_t)e * N);
			Fq::mul(ix, inv, pre); /* (1 + x)^-1 in Montgomery form */
			sm2_one_plus_x<C>(u, x);
			Fq::mul(t, inv, u);
			inv = t;
		}
		const uint8_t *pk = with_key ? pubkeys + (size_t)e * (2 * C::PLEN) : nullptr;
		bool key_ok = true;
		if (with_key) {
			Aff<C> P;
			key_ok = load_affine_checked<C>(P, pk);
		}
		const uint8_t *id = sm2 ? ids + id_off[e] : nullptr;
		const uint64_t idlen = sm2 ? id_off[e + 1] - id_off[e] : 0;
		status[e] = (int8_t)msgs_sign_core<C>(sigs + (size_t)e * siglen, sig_type, hash_type,
						      W_aff + (size_t)e * (2 * C::PLEN), x, k, msgs + off[e],
						      off[e + 1] - off[e], pk, key_ok, id,
						      idlen > kSm2MaxIdLen ? kSm2MaxIdLen + 1 : (uint32_t)idlen, ix);
		if (e < T) break;
	}
}

/* ------------------------------------------------- ECKCDSA / ECSDSA / ECOSDSA / ECGDSA / ECRDSA / SM2 verify */

/*
 * First of the three launches of a message verification: per item the signature checks, the hash of the message and
 * the scalars a || b of W' = a*G + b*Y (msgs_verify_prep_core), written to ab ([n][2*qlen], the double-scalar kernel's
 * input).  A rejected item gets a = b = 0: W' is then infinity and the double-scalar kernel reports status 1 for it.
 * ECGDSA and ECRDSA multiply by den^-1 (r^-1, h^-1) from the two-level simultaneous inversion of k_msgs_sign_finish: a
 * serial prefix product over the thread's items (prefix scratch; den in the Montgomery domain in den_buf, 0 for a
 * rejected item, which stays out of the product), one CTA-wide inversion, then the items in reverse order.  The other
 * schemes invert nothing and run one item per thread.  Messages as k_sha2_batch; id_off: SM2's ID lengths only.
 */
template <class C>
__global__ void __launch_bounds__(128) k_msgs_verify_prep(uint32_t n, int sig_type, int hash_type,
							  const uint8_t *__restrict__ sigs,
							  const uint8_t *__restrict__ pubkeys,
							  const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off,
							  const uint64_t *__restrict__ id_off, uint32_t *__restrict__ prefix,
							  uint32_t *__restrict__ den_buf, uint8_t *__restrict__ ab)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N, QL = C::QLEN;
	const bool inverting = msgs_verify_inverts(sig_type);
	const uint32_t T = gridDim.x * blockDim.x;
	const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = tid < n;
	const int siglen = msgs_verify_sig_len<C>(sig_type, msg_hash_digest_size(hash_type));
	Fe<N> acc;
	Fq::set_one(acc);
	uint32_t last = tid;
	if (active) {
		for (uint32_t e = tid; e < n; e += T) {
			Fe<N> a, b, den;
			const uint64_t idlen = id_off ? id_off[e + 1] - id_off[e] : 0;
			const bool ok = msgs_verify_prep_core<C>(sig_type, hash_type, sigs + (size_t)e * siglen,
								 pubkeys + (size_t)e * (2 * C::PLEN), msgs + off[e],
								 off[e + 1] - off[e],
								 idlen > kSm2MaxIdLen ? kSm2MaxIdLen + 1 : (uint32_t)idlen,
								 a, b, den);
			store_wire<N, QL>(ab + (size_t)e * (2 * QL), a);
			store_wire<N, QL>(ab + (size_t)e * (2 * QL) + QL, b);
			if (inverting) {
				Fe<N> dm, t;
				store_words<N>(prefix + (size_t)e * N, acc);
				Fq::set_zero(dm);
				if (ok) {
					Fq::to_mont(dm, den);
					Fq::mul(t, acc, dm);
					acc = t;
				}
				store_words<N>(den_buf + (size_t)e * N, dm);
			}
			last = e;
			if (n - e <= T) break;
		}
	}
	if (!inverting) return; /* uniform: sig_type is the same for the whole grid */
	Fe<N> inv;
	__shared__ uint32_t sh_inv[ECC_CTA_INV_WORDS(N)];
	cta_inverse_128<typename C::Fq>(inv, acc, sh_inv);
	if (!active) return;
	for (uint32_t e = last;; e -= T) {
		Fe<N> dm;
		load_words<N>(dm, den_buf + (size_t)e * N);
		if (!Fq::is_zero(dm)) {
			Fe<N> pre, di, t, a, b;
			load_words<N>(pre, prefix + (size_t)e * N);
			Fq::mul(di, inv, pre); /* den^-1 in Montgomery form */
			Fq::mul(t, inv, dm);
			inv = t;
			load_wire<N, QL>(a, ab + (size_t)e * (2 * QL));
			load_wire<N, QL>(b, ab + (size_t)e * (2 * QL) + QL);
			msgs_verify_scale<C>(a, b, di);
			store_wire<N, QL>(ab + (size_t)e * (2 * QL), a);
			store_wire<N, QL>(ab + (size_t)e * (2 * QL) + QL, b);
		}
		if (e < T) break;
	}
}

/*
 * Last launch, one item per thread: verdict holds the double-scalar kernel's status (0 W' finite, 1 infinity, -1 key
 * off the curve) and W_aff its affine W'.  Status 0 and the scheme's acceptance test (msgs_verify_accept: the hash of
 * W' || m for ECSDSA / ECOSDSA, of W'_x for ECKCDSA, SM2's Z and H(Z || m)) give 0; anything else gives -1.
 */
template <class C>
__global__ void __launch_bounds__(128) k_msgs_verify_finish(uint32_t n, int sig_type, int hash_type,
							    const uint8_t *__restrict__ sigs,
							    const uint8_t *__restrict__ pubkeys,
							    const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off,
							    const uint8_t *__restrict__ ids,
							    const uint64_t *__restrict__ id_off,
							    const uint8_t *__restrict__ W_aff, int8_t *__restrict__ verdict)
{
	const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= n) return;
	bool ok = verdict[e] == 0;
	if (ok) {
		const int siglen = msgs_verify_sig_len<C>(sig_type, msg_hash_digest_size(hash_type));
		const uint64_t idlen = ids ? id_off[e + 1] - id_off[e] : 0;
		ok = msgs_verify_accept<C>(sig_type, hash_type, sigs + (size_t)e * siglen, W_aff + (size_t)e * (2 * C::PLEN),
					   pubkeys + (size_t)e * (2 * C::PLEN), msgs + off[e], off[e + 1] - off[e],
					   ids ? ids + id_off[e] : nullptr,
					   idlen > kSm2MaxIdLen ? kSm2MaxIdLen : (uint32_t)idlen);
	}
	verdict[e] = ok ? 0 : -1;
}

/* ------------------------------------------------------------------------------------- BIGN / DBIGN sign and verify */

/*
 * Before K1 of the BIGN signers, one item per thread: H(m) into dig_out ([n][digest size]; message i is
 * msgs[off[i] .. off[i+1]), as k_sha2_batch).  With k_out (DBIGN): the nonce of bign_det_nonce, keyed by the
 * BELT-HASH of the OID, x and t of item i's adata record (ad[ad_off[i] .. ad_off[i+1])), into k_out; 0 without any
 * BELT work where x is outside [1, q-1] or the record is malformed (k_bign_sign_finish then reports ECCB200_ERR).
 */
template <class C>
__global__ void __launch_bounds__(128) k_bign_nonce(uint32_t n, int hash_type, const uint8_t *__restrict__ privkeys,
						    const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off,
						    const uint8_t *__restrict__ ad, const uint64_t *__restrict__ ad_off,
						    uint8_t *__restrict__ dig_out, uint8_t *__restrict__ k_out)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N;
	__shared__ uint8_t sbox[256];
	belt_sbox_to_shared(sbox);
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	const int ds = bign_hash_digest_size(hash_type);
	uint8_t h[64];
	bign_hash_src(hash_type, ByteSpan{ msgs + off[idx] }, off[idx + 1] - off[idx], h, sbox);
	for (int i = 0; i < ds; i++) dig_out[(size_t)idx * ds + i] = h[i];
	if (!k_out) return;
	Fe<N> x, k;
	load_wire<N, C::QLEN>(x, privkeys + (size_t)idx * C::QLEN);
	Fq::set_zero(k);
	const uint8_t *rec = ad + ad_off[idx];
	uint32_t oid_len, t_len;
	if (!Fq::is_zero(x) && !Fq::geq_mod(x) && bign_adata_parse(rec, ad_off[idx + 1] - ad_off[idx], oid_len, t_len)) {
		uint8_t theta[32];
		Fe<N> q;
		bign_theta<C>(theta, rec + 4, oid_len, rec + 4 + oid_len, t_len, x, sbox);
		bign_order<C>(q);
		bign_det_nonce<N>(k, theta, h, ds, q, C::QBITS, sbox);
	}
	store_wire<N, C::QLEN>(k_out + (size_t)idx * C::QLEN, k);
}

/* After K1 (k*G) and K4 (affine W), one item per thread: s0 || LE(s1) (bign_sign_core) from the digest column.
 * sigs: [n][l + qlen], status: 0 / -1 (ECCB200_OK / _ERR). */
template <class C>
__global__ void __launch_bounds__(128) k_bign_sign_finish(uint32_t n, int hash_type,
							  const uint8_t *__restrict__ privkeys,
							  const uint8_t *__restrict__ nonces,
							  const uint8_t *__restrict__ digests, const uint8_t *__restrict__ ad,
							  const uint64_t *__restrict__ ad_off, const uint8_t *__restrict__ W_aff,
							  uint8_t *__restrict__ sigs, int8_t *__restrict__ status)
{
	constexpr int N = C::N, SL = C::QLEN / 2 + C::QLEN;
	__shared__ uint8_t sbox[256];
	belt_sbox_to_shared(sbox);
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	const int ds = bign_hash_digest_size(hash_type);
	Fe<N> x, k;
	load_wire<N, C::QLEN>(x, privkeys + (size_t)idx * C::QLEN);
	load_wire<N, C::QLEN>(k, nonces + (size_t)idx * C::QLEN);
	status[idx] = (int8_t)bign_sign_core<C>(sigs + (size_t)idx * SL, W_aff + (size_t)idx * (2 * C::PLEN), x, k,
						digests + (size_t)idx * ds, ds, ad + ad_off[idx],
						ad_off[idx + 1] - ad_off[idx], sbox);
}

/* First launch of a BIGN verification, one item per thread: H(m) into dig_out, and a || b of W' = a*G + b*Y
 * (bign_verify_prep_core) into ab ([n][2*qlen]); a rejected item gets a = b = 0, which the double-scalar kernel turns
 * into infinity (status 1).  b is never 0 otherwise, so a valid item never reaches infinity. */
template <class C>
__global__ void __launch_bounds__(128) k_bign_verify_prep(uint32_t n, int hash_type, const uint8_t *__restrict__ sigs,
							  const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off,
							  const uint8_t *__restrict__ ad, const uint64_t *__restrict__ ad_off,
							  uint8_t *__restrict__ dig_out, uint8_t *__restrict__ ab)
{
	constexpr int N = C::N, QL = C::QLEN, SL = C::QLEN / 2 + C::QLEN;
	__shared__ uint8_t sbox[256];
	belt_sbox_to_shared(sbox);
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	const int ds = bign_hash_digest_size(hash_type);
	uint8_t h[64];
	bign_hash_src(hash_type, ByteSpan{ msgs + off[idx] }, off[idx + 1] - off[idx], h, sbox);
	for (int i = 0; i < ds; i++) dig_out[(size_t)idx * ds + i] = h[i];
	Fe<N> a, b;
	bign_verify_prep_core<C>(a, b, sigs + (size_t)idx * SL, h, ds, ad + ad_off[idx], ad_off[idx + 1] - ad_off[idx]);
	store_wire<N, QL>(ab + (size_t)idx * (2 * QL), a);
	store_wire<N, QL>(ab + (size_t)idx * (2 * QL) + QL, b);
}

/* Last launch, one item per thread: verdict holds the double-scalar kernel's status (0 W' finite, 1 infinity, -1 key
 * off the curve), W_aff the affine W'.  Status 0, a well-formed adata record and s0 == the first l bytes of
 * BELT-HASH(oid || LE(W'_x) || h) (bign_s0) give 0; anything else gives -1. */
template <class C>
__global__ void __launch_bounds__(128) k_bign_verify_finish(uint32_t n, const uint8_t *__restrict__ sigs,
							    const uint8_t *__restrict__ ad, const uint64_t *__restrict__ ad_off,
							    const uint8_t *__restrict__ digests, int ds,
							    const uint8_t *__restrict__ W_aff, int8_t *__restrict__ verdict)
{
	constexpr int L = C::QLEN / 2, SL = C::QLEN / 2 + C::QLEN;
	__shared__ uint8_t sbox[256];
	belt_sbox_to_shared(sbox);
	const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= n) return;
	const uint8_t *rec = ad + ad_off[e];
	uint32_t oid_len, t_len;
	bool ok = verdict[e] == 0 && bign_adata_parse(rec, ad_off[e + 1] - ad_off[e], oid_len, t_len);
	if (ok) {
		uint8_t s0[L];
		bign_s0<C>(s0, rec + 4, oid_len, W_aff + (size_t)e * (2 * C::PLEN), digests + (size_t)e * ds, ds, sbox);
		const uint8_t *sig = sigs + (size_t)e * SL;
		uint8_t diff = 0;
		for (int i = 0; i < L; i++) diff |= s0[i] ^ sig[i];
		ok = diff == 0;
	}
	verdict[e] = ok ? 0 : -1;
}

/* ------------------------------------------------------------------------------------------ Schnorr-family sign */

/* H(tag) of BIP0340 tags tag0 .. tag0 + ntags - 1 into shared memory, one thread per tag: once per CTA, not per item */
__device__ __forceinline__ void bip0340_tags_shared(uint8_t (*tags)[64], int hash_type, int tag0, int ntags)
{
	if ((int)threadIdx.x < ntags) bip0340_tag_hash(hash_type, tag0 + (int)threadIdx.x, tags[threadIdx.x]);
	__syncthreads();
}

/* BIP0340 nonces before K1: k[i] = H_nonce(t || P_x || m) mod q (bip0340_nonce), or 0 when x is outside [1, q-1] or
 * the key is not on the curve (the finish kernel tells those apart from a derived k == 0).  Messages as
 * k_sha2_batch: message i is msgs[off[i] .. off[i+1]). */
template <class C>
__global__ void __launch_bounds__(128) k_bip0340_nonce(uint32_t n, int hash_type, const uint8_t *__restrict__ privkeys,
						       const uint8_t *__restrict__ pubkeys, const uint8_t *__restrict__ aux,
						       const uint8_t *__restrict__ msgs, const uint64_t *__restrict__ off,
						       uint8_t *__restrict__ k_out)
{
	typedef Field<typename C::Fq> Fq;
	constexpr int N = C::N;
	__shared__ uint8_t tags[2][64];
	bip0340_tags_shared(tags, hash_type, 0, 2);
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<N> x, k;
	Aff<C> P;
	load_wire<N, C::QLEN>(x, privkeys + (size_t)idx * C::QLEN);
	const uint8_t *pk = pubkeys + (size_t)idx * (2 * C::PLEN);
	Fq::set_zero(k);
	if (load_affine_checked<C>(P, pk) && !Fq::is_zero(x) && !Fq::geq_mod(x))
		bip0340_nonce<C>(k, hash_type, x, pk, aux + (size_t)idx * C::QLEN, msgs + off[idx], off[idx + 1] - off[idx],
				 tags[0], tags[1]);
	store_wire<N, C::QLEN>(k_out + (size_t)idx * C::QLEN, k);
}

/* After K1 (k*G) and K4 (affine W): the hash over W and the message, then s = k + e*x mod q (schnorr_sign_core).
 * sigs: [n][schnorr_sig_len], status: 0 / -1 / 2 (ECCB200_OK / _ERR / _RETRY). */
template <class C>
__global__ void __launch_bounds__(128) k_schnorr_sign_finish(uint32_t n, int sig_type, int hash_type,
							     const uint8_t *__restrict__ privkeys,
							     const uint8_t *__restrict__ pubkeys,
							     const uint8_t *__restrict__ nonces,
							     const uint8_t *__restrict__ msgs,
							     const uint64_t *__restrict__ off,
							     const uint8_t *__restrict__ W_aff, uint8_t *__restrict__ sigs,
							     int8_t *__restrict__ status)
{
	constexpr int N = C::N;
	const bool bip = sig_type == SIG_BIP0340;
	__shared__ uint8_t tags[1][64];
	if (bip) bip0340_tags_shared(tags, hash_type, 2, 1);
	const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<N> x, k;
	load_wire<N, C::QLEN>(x, privkeys + (size_t)idx * C::QLEN);
	load_wire<N, C::QLEN>(k, nonces + (size_t)idx * C::QLEN);
	const uint8_t *pk = bip ? pubkeys + (size_t)idx * (2 * C::PLEN) : nullptr;
	bool key_ok = true;
	if (bip) {
		Aff<C> P;
		key_ok = load_affine_checked<C>(P, pk);
	}
	const int siglen = schnorr_sig_len<C>(sig_type, sha2_digest_size(hash_type));
	status[idx] = (int8_t)schnorr_sign_core<C>(sigs + (size_t)idx * siglen, sig_type, hash_type,
						   W_aff + (size_t)idx * (2 * C::PLEN), x, k, msgs + off[idx],
						   off[idx + 1] - off[idx], pk, key_ok, tags[0]);
}

/* Private-key sanity check of __ecdsa_init_pub_key (sig/ecdsa_common.c:188): x < q, else the key is rejected (-1).
 * Run before K1, which would silently reduce x mod q.  state[i] is only ever lowered to -1. */
template <class C>
__global__ void __launch_bounds__(128) k_scalar_below_order(uint32_t n, const uint8_t *__restrict__ scalars,
							     int8_t *__restrict__ state)
{
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<C::N> k;
	load_wire<C::N, C::QLEN>(k, scalars + (size_t)idx * C::QLEN);
	if (Field<typename C::Fq>::geq_mod(k)) state[idx] = -1;
}

/* ------------------------------------------------------------------------------------------ unit-test kernels */

/* mod-q scalar preparation of ECDSA verify alone: out[i] = u || v (big-endian), for the arithmetic unit tests */
template <class C>
__global__ void __launch_bounds__(128) k_ecdsa_uv(uint32_t n, const uint8_t *__restrict__ sigs,
						  const uint8_t *__restrict__ digests, uint32_t hlen,
						  uint8_t *__restrict__ out)
{
	constexpr int N = C::N;
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<N> r, s, e, u, v;
	load_wire<N, C::QLEN>(r, sigs + (size_t)idx * (2 * C::QLEN));
	load_wire<N, C::QLEN>(s, sigs + (size_t)idx * (2 * C::QLEN) + C::QLEN);
	digest_to_scalar<C>(e, digests + (size_t)idx * hlen, hlen);
	ecdsa_uv<C>(u, v, r, s, e);
	store_wire<N, C::QLEN>(out + (size_t)idx * (2 * C::QLEN), u);
	store_wire<N, C::QLEN>(out + (size_t)idx * (2 * C::QLEN) + C::QLEN, v);
}

template <class FT>
__global__ void k_fp_mul_monty(uint32_t n, const uint8_t *__restrict__ a, const uint8_t *__restrict__ b,
			       uint8_t *__restrict__ out)
{
	constexpr int N = FT::N;
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<N> x, y, z;
	load_wire<N, FT::BYTES>(x, a + (size_t)idx * FT::BYTES);
	load_wire<N, FT::BYTES>(y, b + (size_t)idx * FT::BYTES);
	Field<FT>::mul(z, x, y);
	store_wire<N, FT::BYTES>(out + (size_t)idx * FT::BYTES, z);
}

/* fp_add_monty / fp_sub_monty / fp_sqr_monty (fp/fp_montgomery.c:26,35,53) as direct unit kernels of the PTX back
 * end: op 0 = a + b, 1 = a - b, 2 = a * a * R^-1 (b unused); operands < modulus. */
template <class FT>
__global__ void k_fp_addsub(uint32_t n, int op, const uint8_t *__restrict__ a, const uint8_t *__restrict__ b,
			    uint8_t *__restrict__ out)
{
	constexpr int N = FT::N;
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<N> x, y, z;
	load_wire<N, FT::BYTES>(x, a + (size_t)idx * FT::BYTES);
	load_wire<N, FT::BYTES>(y, b + (size_t)idx * FT::BYTES);
	if (op == 0) Field<FT>::add(z, x, y);
	else if (op == 1) Field<FT>::sub(z, x, y);
	else Field<FT>::sqr(z, x);
	store_wire<N, FT::BYTES>(out + (size_t)idx * FT::BYTES, z);
}

/*
 * Layout experiment (DESIGN.md §3): the SAME Montgomery product with the N = 8 words of an element striped across
 * 8 lanes (4 elements per warp) and every cross-word carry / broadcast done with __shfl_sync, as the north star
 * sketches — versus the production layout (one thread owns the element).  Both kernels run `iters` dependent
 * products x <- x*y per element so that only arithmetic is timed; k_fp_mul_chain is the production multiplier.
 * Striped algorithm per row i: b_i broadcast; t_j += lo(a_j b_i), t_{j+1} += hi(a_j b_i) (shfl_up); m = t_0*M0
 * broadcast; the same with p_j m; one-word right shift (shfl_down).  t_j are 64-bit with deferred carries; a final
 * ripple normalises and subtracts p.  8-word fields only.
 */
template <class FT>
__global__ void __launch_bounds__(128) k_fp_mul_chain(uint32_t n, const uint8_t *__restrict__ a,
						      const uint8_t *__restrict__ b, uint8_t *__restrict__ out, int iters)
{
	constexpr int N = FT::N;
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	Fe<N> x, y;
	load_wire<N, FT::BYTES>(x, a + (size_t)idx * FT::BYTES);
	load_wire<N, FT::BYTES>(y, b + (size_t)idx * FT::BYTES);
#pragma unroll 1
	for (int i = 0; i < iters; i++) Field<FT>::mul(x, x, y);
	store_wire<N, FT::BYTES>(out + (size_t)idx * FT::BYTES, x);
}

template <class FT>
__global__ void __launch_bounds__(128) k_fp_mul_striped_chain(uint32_t n, const uint8_t *__restrict__ a,
							      const uint8_t *__restrict__ b,
							      uint8_t *__restrict__ out, int iters)
{
	static_assert(FT::N == 8, "striped experiment is written for 8-word fields");
	constexpr int N = 8;
	const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t elem = gtid / N;
	const int j = (int)(gtid % N); /* word index = lane within the 8-lane group */
	if (elem >= n) return;         /* n is a multiple of 4 in the benchmark, so whole groups exit together */
	/* big-endian wire: word j (little-endian index) sits at byte offset 4*(N-1-j) */
	auto ldw = [&](const uint8_t *base) {
		uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(base + (size_t)elem * (4 * N) + 4 * (N - 1 - j)));
		return bswap32(v);
	};
	uint32_t x = ldw(a), y = ldw(b);
	uint32_t pj = 0;
#pragma unroll
	for (int k = 0; k < N; k++) pj = (k == j) ? FT::P(k) : pj;
	const unsigned full = 0xffffffffu;
#pragma unroll 1
	for (int it = 0; it < iters; it++) {
		uint64_t t = 0, tN = 0; /* position j, and (lane N-1 only) position N */
#pragma unroll
		for (int i = 0; i < N; i++) {
			uint32_t bi = __shfl_sync(full, y, i, N);
			uint64_t pr = (uint64_t)x * bi;
			t += (uint32_t)pr;
			uint32_t hi = (uint32_t)(pr >> 32);
			uint32_t up = __shfl_up_sync(full, hi, 1, N);
			if (j > 0) t += up;
			if (j == N - 1) tN += hi;
			uint32_t m = __shfl_sync(full, (uint32_t)t * FT::M0, 0, N);
			pr = (uint64_t)pj * m;
			t += (uint32_t)pr;
			hi = (uint32_t)(pr >> 32);
			up = __shfl_up_sync(full, hi, 1, N);
			if (j > 0) t += up;
			if (j == N - 1) tN += hi;
			/* shift right by one word; lane 0 keeps the carry of the word that drops out */
			uint64_t c0 = t >> 32;
			uint32_t dlo = __shfl_down_sync(full, (uint32_t)t, 1, N);
			uint32_t dhi = __shfl_down_sync(full, (uint32_t)(t >> 32), 1, N);
			uint64_t nt = ((uint64_t)dhi << 32) | dlo;
			if (j == N - 1) {
				nt = tN;
				tN = 0;
			}
			if (j == 0) nt += c0;
			t = nt;
		}
		/* ripple the deferred carries, word by word */
		uint32_t topc = 0;
#pragma unroll
		for (int k = 0; k < N; k++) {
			uint32_t c = (uint32_t)(t >> 32);
			uint32_t cin = __shfl_up_sync(full, c, 1, N);
			if (j == k) t &= 0xffffffffull;
			if (j == k + 1) t += cin;
			if (k == N - 1) topc = __shfl_sync(full, c, N - 1, N);
		}
		uint32_t r = (uint32_t)t;
		/* d = r - p with a rippled borrow; take d when r >= p or the carry word is set */
		uint32_t borrow = 0, dword = r;
#pragma unroll
		for (int k = 0; k < N; k++) {
			uint32_t bin = __shfl_sync(full, borrow, (k == 0) ? 0 : k - 1, N);
			if (k == 0) bin = 0;
			if (j == k) {
				uint64_t dd = (uint64_t)r - pj - bin;
				dword = (uint32_t)dd;
				borrow = (uint32_t)(dd >> 63);
			}
		}
		uint32_t last_borrow = __shfl_sync(full, borrow, N - 1, N);
		x = (topc != 0 || last_borrow == 0) ? dword : r;
	}
	uint32_t *o = reinterpret_cast<uint32_t *>(out + (size_t)elem * (4 * N) + 4 * (N - 1 - j));
	*o = bswap32(x);
}

} // namespace eccb200

/* ------------------------------------------------------------------------------------------ launchers */
/*
 * Host-side launch wrappers, one struct per kernel group so that each (group, curve) pair can live in its own
 * translation unit (tu_*.cu) and the groups compile in parallel; eccb200.cu only sees the declarations.
 */
#include <cuda_runtime.h>
namespace eccb200 {

static const int kThreads = 128;
static inline uint32_t grid_for(uint32_t n) { return (n + kThreads - 1) / kThreads; }
/* grids of the cluster kernels are whole clusters (idle CTAs take part in the inversion and write nothing) */
static inline uint32_t grid_clustered(uint32_t n)
{
	return (grid_for(n) + ECC_CLUSTER_INV - 1) / ECC_CLUSTER_INV * ECC_CLUSTER_INV;
}

/* K1 group: compiled with the multiplier INLINED (ECC_INLINE_MUL): its loop body is one mixed addition and runs
 * faster that way; K2 / K3 groups call the out-of-line multiplier, which keeps their much larger loop bodies inside
 * the instruction cache (both chosen on the previous GPU target and not re-measured on H100). */
template <class C> struct LaunchFixed {
	static void fixed(uint32_t n, const uint8_t *scalars, const uint32_t *table, int w, uint32_t *jac,
			  int8_t *status, cudaStream_t st);
	static int fixed_ctas_per_sm(); /* resident CTAs of k_smul_fixed per SM (register-limited): the wave size */
	static void fixed_tma(uint32_t n, const uint8_t *scalars, const uint32_t *table, int w, uint32_t *jac,
			      int8_t *status, cudaStream_t st);
	static void table_merge(uint32_t count, uint64_t first_entry, int w, int nwin_half, const uint32_t *half_table,
				uint32_t *jac, cudaStream_t st);
};

template <class C> struct LaunchVar {
	static void var(uint32_t n, const uint8_t *scalars, const uint8_t *points, uint32_t *jac, int8_t *status,
			cudaStream_t st);
	static void table_points(uint32_t entries, int w, uint32_t *jac, cudaStream_t st);
};

template <class C> struct LaunchMisc {
	static void to_affine(uint32_t blocks, uint32_t n, const uint32_t *jac, uint32_t *prefix, uint8_t *out,
			      int8_t *status, cudaStream_t st, const GatherDst *gd = nullptr);
	static void to_table(uint32_t blocks, uint32_t n, const uint32_t *jac, uint32_t *prefix, uint32_t *table,
			     cudaStream_t st);
	static void prj_unique(uint32_t blocks, uint32_t n, const uint8_t *prj, uint32_t *jac, uint32_t *prefix,
			       uint8_t *out, int8_t *status, cudaStream_t st);
	static void to_x_only(uint32_t blocks, uint32_t n, const uint32_t *jac, uint32_t *prefix, uint8_t *out,
			      int8_t *status, cudaStream_t st);
	static void sign_finish(uint32_t blocks, uint32_t n, const uint8_t *privkeys, const uint8_t *nonces,
				const uint8_t *digests, uint32_t hlen, const uint8_t *kG_aff, uint32_t *prefix,
				uint8_t *sigs, int8_t *status, cudaStream_t st);
	static void ecdsa_nonce(uint32_t n, int hash_type, const uint8_t *privkeys, const uint8_t *digests,
				const uint8_t *msgs, const uint64_t *off, uint8_t *dig_out, uint8_t *k_out, cudaStream_t st);
	static void bip0340_nonce(uint32_t n, int hash_type, const uint8_t *privkeys, const uint8_t *pubkeys,
				  const uint8_t *aux, const uint8_t *msgs, const uint64_t *off, uint8_t *k_out,
				  cudaStream_t st);
	static void schnorr_finish(uint32_t n, int sig_type, int hash_type, const uint8_t *privkeys,
				   const uint8_t *pubkeys, const uint8_t *nonces, const uint8_t *msgs, const uint64_t *off,
				   const uint8_t *W_aff, uint8_t *sigs, int8_t *status, cudaStream_t st);
	static void msgs_sign_finish(uint32_t blocks, uint32_t n, int sig_type, int hash_type, const uint8_t *privkeys,
				     const uint8_t *pubkeys, const uint8_t *nonces, const uint8_t *msgs, const uint64_t *off,
				     const uint8_t *ids, const uint64_t *id_off, const uint8_t *W_aff, uint32_t *prefix,
				     uint8_t *sigs, int8_t *status, cudaStream_t st);
	static void msgs_verify_prep(uint32_t blocks, uint32_t n, int sig_type, int hash_type, const uint8_t *sigs,
				     const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *off, const uint64_t *id_off,
				     uint32_t *prefix, uint32_t *den, uint8_t *ab, cudaStream_t st);
	static void msgs_verify_finish(uint32_t n, int sig_type, int hash_type, const uint8_t *sigs, const uint8_t *pubkeys,
				       const uint8_t *msgs, const uint64_t *off, const uint8_t *ids, const uint64_t *id_off,
				       const uint8_t *W_aff, int8_t *verdict, cudaStream_t st);
	static void bign_nonce(uint32_t n, int hash_type, const uint8_t *privkeys, const uint8_t *msgs, const uint64_t *off,
			       const uint8_t *ad, const uint64_t *ad_off, uint8_t *dig_out, uint8_t *k_out, cudaStream_t st);
	static void bign_sign_finish(uint32_t n, int hash_type, const uint8_t *privkeys, const uint8_t *nonces,
				     const uint8_t *digests, const uint8_t *ad, const uint64_t *ad_off, const uint8_t *W_aff,
				     uint8_t *sigs, int8_t *status, cudaStream_t st);
	static void bign_verify_prep(uint32_t n, int hash_type, const uint8_t *sigs, const uint8_t *msgs, const uint64_t *off,
				     const uint8_t *ad, const uint64_t *ad_off, uint8_t *dig_out, uint8_t *ab, cudaStream_t st);
	static void bign_verify_finish(uint32_t n, const uint8_t *sigs, const uint8_t *ad, const uint64_t *ad_off,
				       const uint8_t *digests, int ds, const uint8_t *W_aff, int8_t *verdict, cudaStream_t st);
	static void fp_mul(int which, uint32_t n, const uint8_t *a, const uint8_t *b, uint8_t *out, cudaStream_t st);
	static void fp_addsub(int which, int op, uint32_t n, const uint8_t *a, const uint8_t *b, uint8_t *out,
			      cudaStream_t st);
	static void scalar_below_order(uint32_t n, const uint8_t *scalars, int8_t *state, cudaStream_t st);
	static void fp_mul_chain(int striped, uint32_t n, const uint8_t *a, const uint8_t *b, uint8_t *out, int iters,
				 cudaStream_t st);
};

template <class C> struct LaunchVerify {
	static void verify(uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys, const uint8_t *digests,
			   uint32_t hlen, const uint32_t *table, int w, int8_t *verdict, cudaStream_t st,
			   const int8_t *key_state = nullptr);
	static void ecfsdsa(uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys, const uint8_t *digests,
			    uint32_t hlen, const uint32_t *table, int w, int8_t *verdict, cudaStream_t st);
	static void bip0340(uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys, const uint8_t *digests,
			    uint32_t hlen, const uint32_t *table, int w, int8_t *verdict, cudaStream_t st);
	static void double_smul(uint32_t n, const uint8_t *ab, const uint8_t *pubkeys, const uint32_t *table, int w,
				uint8_t *out, int8_t *status, cudaStream_t st);
	static void uv(uint32_t n, const uint8_t *sigs, const uint8_t *digests, uint32_t hlen, uint8_t *out,
		       cudaStream_t st);
	static void recover(uint32_t n, const uint8_t *sigs, const uint8_t *digests, uint32_t hlen, const uint32_t *table,
			    int w, uint8_t *keys, int8_t *status, cudaStream_t st);
};

#if defined(ECC_TU_FIXED)
template <class C>
void LaunchFixed<C>::fixed(uint32_t n, const uint8_t *scalars, const uint32_t *table, int w, uint32_t *jac,
			   int8_t *status, cudaStream_t st)
{
	k_smul_fixed<C><<<grid_for(n), kThreads, 0, st>>>(n, scalars, table, w, jac, status);
}
template <class C> int LaunchFixed<C>::fixed_ctas_per_sm()
{
	int nb = 0;
	if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_smul_fixed<C>, kThreads, 0) != cudaSuccess || nb < 1) {
		cudaGetLastError();
		nb = 4;
	}
	return nb;
}
template <class C>
void LaunchFixed<C>::fixed_tma(uint32_t n, const uint8_t *scalars, const uint32_t *table, int w, uint32_t *jac,
			       int8_t *status, cudaStream_t st)
{
	if constexpr (C::QLEN == 4 * C::N && C::N % 4 == 0) /* the bulk copy needs 16-byte multiples */
		k_smul_fixed_tma<C><<<grid_for(n), kThreads, 0, st>>>(n, scalars, table, w, jac, status);
	else
		k_smul_fixed<C><<<grid_for(n), kThreads, 0, st>>>(n, scalars, table, w, jac, status);
}
template <class C>
void LaunchFixed<C>::table_merge(uint32_t count, uint64_t first_entry, int w, int nwin_half,
				 const uint32_t *half_table, uint32_t *jac, cudaStream_t st)
{
	k_table_merge<C><<<grid_for(count), kThreads, 0, st>>>(count, first_entry, w, nwin_half, half_table, jac);
}
#endif

#if defined(ECC_TU_VAR)
template <class C>
void LaunchVar<C>::var(uint32_t n, const uint8_t *scalars, const uint8_t *points, uint32_t *jac, int8_t *status,
		       cudaStream_t st)
{
	k_smul_var<C><<<grid_clustered(n), kThreads, 0, st>>>(n, scalars, points, jac, status);
}
template <class C> void LaunchVar<C>::table_points(uint32_t entries, int w, uint32_t *jac, cudaStream_t st)
{
	k_table_points<C><<<grid_for(entries), kThreads, 0, st>>>(entries, w, jac);
}
#endif

#if defined(ECC_TU_MISC)
template <class C>
void LaunchMisc<C>::to_affine(uint32_t blocks, uint32_t n, const uint32_t *jac, uint32_t *prefix, uint8_t *out,
			      int8_t *status, cudaStream_t st, const GatherDst *gd)
{
	k_to_affine<C, 0><<<blocks, kThreads, 0, st>>>(n, jac, prefix, out, status, nullptr, gd ? *gd : GatherDst());
}
template <class C>
void LaunchMisc<C>::to_x_only(uint32_t blocks, uint32_t n, const uint32_t *jac, uint32_t *prefix, uint8_t *out,
			      int8_t *status, cudaStream_t st)
{
	k_to_affine<C, 3><<<blocks, kThreads, 0, st>>>(n, jac, prefix, out, status, nullptr, GatherDst());
}
template <class C>
void LaunchMisc<C>::sign_finish(uint32_t blocks, uint32_t n, const uint8_t *privkeys, const uint8_t *nonces,
				const uint8_t *digests, uint32_t hlen, const uint8_t *kG_aff, uint32_t *prefix,
				uint8_t *sigs, int8_t *status, cudaStream_t st)
{
	k_ecdsa_sign_finish<C><<<blocks, kThreads, 0, st>>>(n, privkeys, nonces, digests, hlen, kG_aff, prefix, sigs,
							     status);
}
template <class C>
void LaunchMisc<C>::ecdsa_nonce(uint32_t n, int hash_type, const uint8_t *privkeys, const uint8_t *digests,
				const uint8_t *msgs, const uint64_t *off, uint8_t *dig_out, uint8_t *k_out, cudaStream_t st)
{
	k_ecdsa_nonce<C><<<grid_for(n), kThreads, 0, st>>>(n, hash_type, privkeys, digests, msgs, off, dig_out, k_out);
}
template <class C>
void LaunchMisc<C>::bip0340_nonce(uint32_t n, int hash_type, const uint8_t *privkeys, const uint8_t *pubkeys,
				  const uint8_t *aux, const uint8_t *msgs, const uint64_t *off, uint8_t *k_out,
				  cudaStream_t st)
{
	k_bip0340_nonce<C><<<grid_for(n), kThreads, 0, st>>>(n, hash_type, privkeys, pubkeys, aux, msgs, off, k_out);
}
template <class C>
void LaunchMisc<C>::schnorr_finish(uint32_t n, int sig_type, int hash_type, const uint8_t *privkeys,
				   const uint8_t *pubkeys, const uint8_t *nonces, const uint8_t *msgs, const uint64_t *off,
				   const uint8_t *W_aff, uint8_t *sigs, int8_t *status, cudaStream_t st)
{
	k_schnorr_sign_finish<C><<<grid_for(n), kThreads, 0, st>>>(n, sig_type, hash_type, privkeys, pubkeys, nonces, msgs,
								    off, W_aff, sigs, status);
}
template <class C>
void LaunchMisc<C>::msgs_sign_finish(uint32_t blocks, uint32_t n, int sig_type, int hash_type, const uint8_t *privkeys,
				     const uint8_t *pubkeys, const uint8_t *nonces, const uint8_t *msgs, const uint64_t *off,
				     const uint8_t *ids, const uint64_t *id_off, const uint8_t *W_aff, uint32_t *prefix,
				     uint8_t *sigs, int8_t *status, cudaStream_t st)
{
	k_msgs_sign_finish<C><<<blocks, kThreads, 0, st>>>(n, sig_type, hash_type, privkeys, pubkeys, nonces, msgs, off, ids,
							    id_off, W_aff, prefix, sigs, status);
}
template <class C>
void LaunchMisc<C>::msgs_verify_prep(uint32_t blocks, uint32_t n, int sig_type, int hash_type, const uint8_t *sigs,
				     const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *off, const uint64_t *id_off,
				     uint32_t *prefix, uint32_t *den, uint8_t *ab, cudaStream_t st)
{
	k_msgs_verify_prep<C><<<blocks, kThreads, 0, st>>>(n, sig_type, hash_type, sigs, pubkeys, msgs, off, id_off, prefix,
							    den, ab);
}
template <class C>
void LaunchMisc<C>::msgs_verify_finish(uint32_t n, int sig_type, int hash_type, const uint8_t *sigs,
				       const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *off, const uint8_t *ids,
				       const uint64_t *id_off, const uint8_t *W_aff, int8_t *verdict, cudaStream_t st)
{
	k_msgs_verify_finish<C><<<grid_for(n), kThreads, 0, st>>>(n, sig_type, hash_type, sigs, pubkeys, msgs, off, ids,
								   id_off, W_aff, verdict);
}
template <class C>
void LaunchMisc<C>::bign_nonce(uint32_t n, int hash_type, const uint8_t *privkeys, const uint8_t *msgs, const uint64_t *off,
			       const uint8_t *ad, const uint64_t *ad_off, uint8_t *dig_out, uint8_t *k_out, cudaStream_t st)
{
	k_bign_nonce<C><<<grid_for(n), kThreads, 0, st>>>(n, hash_type, privkeys, msgs, off, ad, ad_off, dig_out, k_out);
}
template <class C>
void LaunchMisc<C>::bign_sign_finish(uint32_t n, int hash_type, const uint8_t *privkeys, const uint8_t *nonces,
				     const uint8_t *digests, const uint8_t *ad, const uint64_t *ad_off, const uint8_t *W_aff,
				     uint8_t *sigs, int8_t *status, cudaStream_t st)
{
	k_bign_sign_finish<C><<<grid_for(n), kThreads, 0, st>>>(n, hash_type, privkeys, nonces, digests, ad, ad_off, W_aff,
								 sigs, status);
}
template <class C>
void LaunchMisc<C>::bign_verify_prep(uint32_t n, int hash_type, const uint8_t *sigs, const uint8_t *msgs,
				     const uint64_t *off, const uint8_t *ad, const uint64_t *ad_off, uint8_t *dig_out,
				     uint8_t *ab, cudaStream_t st)
{
	k_bign_verify_prep<C><<<grid_for(n), kThreads, 0, st>>>(n, hash_type, sigs, msgs, off, ad, ad_off, dig_out, ab);
}
template <class C>
void LaunchMisc<C>::bign_verify_finish(uint32_t n, const uint8_t *sigs, const uint8_t *ad, const uint64_t *ad_off,
				       const uint8_t *digests, int ds, const uint8_t *W_aff, int8_t *verdict, cudaStream_t st)
{
	k_bign_verify_finish<C><<<grid_for(n), kThreads, 0, st>>>(n, sigs, ad, ad_off, digests, ds, W_aff, verdict);
}
template <class C>
void LaunchMisc<C>::prj_unique(uint32_t blocks, uint32_t n, const uint8_t *prj, uint32_t *jac, uint32_t *prefix,
			       uint8_t *out, int8_t *status, cudaStream_t st)
{
	k_prj_load<C><<<grid_for(n), kThreads, 0, st>>>(n, prj, jac, status);
	k_to_affine<C, 2><<<blocks, kThreads, 0, st>>>(n, jac, prefix, out, status, nullptr, GatherDst());
}
template <class C>
void LaunchMisc<C>::to_table(uint32_t blocks, uint32_t n, const uint32_t *jac, uint32_t *prefix, uint32_t *table,
			     cudaStream_t st)
{
	k_to_affine<C, 1><<<blocks, kThreads, 0, st>>>(n, jac, prefix, nullptr, nullptr, table, GatherDst());
}
template <class C>
void LaunchMisc<C>::scalar_below_order(uint32_t n, const uint8_t *scalars, int8_t *state, cudaStream_t st)
{
	k_scalar_below_order<C><<<grid_for(n), kThreads, 0, st>>>(n, scalars, state);
}
template <class C>
void LaunchMisc<C>::fp_mul(int which, uint32_t n, const uint8_t *a, const uint8_t *b, uint8_t *out, cudaStream_t st)
{
	if (which == 0)
		k_fp_mul_monty<typename C::Fp><<<grid_for(n), kThreads, 0, st>>>(n, a, b, out);
	else
		k_fp_mul_monty<typename C::Fq><<<grid_for(n), kThreads, 0, st>>>(n, a, b, out);
}
#endif

#if defined(ECC_TU_MISC)
template <class C>
void LaunchMisc<C>::fp_addsub(int which, int op, uint32_t n, const uint8_t *a, const uint8_t *b, uint8_t *out,
			      cudaStream_t st)
{
	if (which == 0)
		k_fp_addsub<typename C::Fp><<<grid_for(n), kThreads, 0, st>>>(n, op, a, b, out);
	else
		k_fp_addsub<typename C::Fq><<<grid_for(n), kThreads, 0, st>>>(n, op, a, b, out);
}
#endif

#if defined(ECC_TU_MISC)
template <class C, int NW> struct StripedLaunch {
	static void go(uint32_t, const uint8_t *, const uint8_t *, uint8_t *, int, cudaStream_t) {}
};
template <class C> struct StripedLaunch<C, 8> {
	static void go(uint32_t n, const uint8_t *a, const uint8_t *b, uint8_t *out, int iters, cudaStream_t st)
	{
		k_fp_mul_striped_chain<typename C::Fp><<<grid_for(n * 8), kThreads, 0, st>>>(n, a, b, out, iters);
	}
};
template <class C>
void LaunchMisc<C>::fp_mul_chain(int striped, uint32_t n, const uint8_t *a, const uint8_t *b, uint8_t *out,
				 int iters, cudaStream_t st)
{
	if (striped)
		StripedLaunch<C, C::N>::go(n, a, b, out, iters, st);
	else
		k_fp_mul_chain<typename C::Fp><<<grid_for(n), kThreads, 0, st>>>(n, a, b, out, iters);
}
#endif

#if defined(ECC_TU_VERIFY)
template <class C>
void LaunchVerify<C>::verify(uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys, const uint8_t *digests,
			     uint32_t hlen, const uint32_t *table, int w, int8_t *verdict, cudaStream_t st,
			     const int8_t *key_state)
{
	k_ecdsa_verify<C><<<grid_clustered(n), kThreads, 0, st>>>(n, sigs, pubkeys, digests, hlen, table, w, verdict,
							     key_state, nullptr);
}
template <class C>
void LaunchVerify<C>::ecfsdsa(uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys, const uint8_t *digests,
			      uint32_t hlen, const uint32_t *table, int w, int8_t *verdict, cudaStream_t st)
{
	k_ecdsa_verify<C, 1><<<grid_clustered(n), kThreads, 0, st>>>(n, sigs, pubkeys, digests, hlen, table, w, verdict, nullptr,
								nullptr);
}
template <class C>
void LaunchVerify<C>::bip0340(uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys, const uint8_t *digests,
			      uint32_t hlen, const uint32_t *table, int w, int8_t *verdict, cudaStream_t st)
{
	k_ecdsa_verify<C, 2><<<grid_clustered(n), kThreads, 0, st>>>(n, sigs, pubkeys, digests, hlen, table, w, verdict, nullptr,
								nullptr);
}
template <class C>
void LaunchVerify<C>::double_smul(uint32_t n, const uint8_t *ab, const uint8_t *pubkeys, const uint32_t *table, int w,
				  uint8_t *out, int8_t *status, cudaStream_t st)
{
	k_ecdsa_verify<C, 3><<<grid_clustered(n), kThreads, 0, st>>>(n, ab, pubkeys, nullptr, 0, table, w, status, nullptr, out);
}
template <class C>
void LaunchVerify<C>::uv(uint32_t n, const uint8_t *sigs, const uint8_t *digests, uint32_t hlen, uint8_t *out,
			 cudaStream_t st)
{
	k_ecdsa_uv<C><<<grid_for(n), kThreads, 0, st>>>(n, sigs, digests, hlen, out);
}
template <class C>
void LaunchVerify<C>::recover(uint32_t n, const uint8_t *sigs, const uint8_t *digests, uint32_t hlen,
			      const uint32_t *table, int w, uint8_t *keys, int8_t *status, cudaStream_t st)
{
	k_ecdsa_recover<C><<<grid_clustered(n), kThreads, 0, st>>>(n, sigs, digests, hlen, table, w, keys, status);
}
#endif

} // namespace eccb200
