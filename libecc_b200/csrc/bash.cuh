/*
 * bash.cuh — BASH224 / 256 / 384 / 512 (STB 34.101.77-2020; hash_alg_type 17..20) over the byte sources of sha3.cuh,
 * one thread per message: message hashes of the BIGN signers (ec.cuh: bign_*).  Reference counterparts (relative to
 * /root/reference/src): _bash_init / _bash_update / _bash_finalize, hash/bash.c, with the digest sizes of
 * hash/bash224.c .. hash/bash512.c.
 *
 * A sponge over the 192-byte state S = 24 little-endian 64-bit words: S[23] = the digest size in bytes (<l/4>_64),
 * rate r = 192 - 2*digest bytes.  Each r-byte block overwrites S[0 .. r) (it is not XORed in), then bash-f runs.  The
 * last block holds the message's tail, the byte 0x40 and zeros; it is a block of its own when the length is a multiple
 * of r (the empty message included).  The digest is the first bytes of S.  Constants come from
 * tools/gen_bash_constants.py.  Plain C++ outside nvcc, like sha2.cuh.
 */
#pragma once
#include <stdint.h>
#include "sha3.cuh"

namespace eccb200 {

#include "bash_constants.inc"

enum { HASH_BASH224 = 17, HASH_BASH512 = 20 }; /* hash_alg_type of the reference (lib_ecc_types.h) */

/* 28, 32, 48 or 64 for BASH224 .. BASH512, 0 for any other type */
SHA3_HD int bash_digest_size(int hash_type)
{
	return hash_type == 17 ? 28 : hash_type == 18 ? 32 : hash_type == 19 ? 48 : hash_type == 20 ? 64 : 0;
}

/* bash-s (§6.1): the S-box step on one column (w0, w1, w2) with rotations m1, n1, m2, n2 */
SHA3_HD void bash_s(uint64_t &w0, uint64_t &w1, uint64_t &w2, int m1, int n1, int m2, int n2)
{
	const uint64_t t0 = rotl64_(w0, m1);
	w0 ^= w1 ^ w2;
	const uint64_t t1 = w1 ^ rotl64_(w0, n1);
	w1 = t0 ^ t1;
	w2 = w2 ^ rotl64_(w2, m2) ^ rotl64_(t1, n2);
	const uint64_t u0 = ~w2 | w1, u1 = w0 | w2, u2 = w0 & w1;
	w1 ^= u1;
	w2 ^= u2;
	w0 ^= u0;
}

/* bash-f (§6.2): 24 rounds of eight column steps, the word permutation and the round constant into S[23] */
SHA3_HD void bash_f(uint64_t S[24])
{
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
	for (int round = 0; round < 24; round++) {
		uint64_t T[24];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int v = 0; v < 8; v++)
			bash_s(S[v], S[v + 8], S[v + 16], bash_rot(v, 0), bash_rot(v, 1), bash_rot(v, 2), bash_rot(v, 3));
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int i = 0; i < 24; i++) T[i] = S[bash_perm(i)];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int i = 0; i < 24; i++) S[i] = T[i];
		S[23] ^= bash_rc(round);
	}
}

/* BASH of len bytes of a byte source, digest_bytes in {28, 32, 48, 64} */
template <class Src> SHA3_HD void bash_src(const Src &m, uint64_t len, uint8_t *digest, int digest_bytes)
{
	const int rate = 192 - 2 * digest_bytes;
	uint64_t S[24];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
	for (int i = 0; i < 24; i++) S[i] = 0;
	S[23] = (uint64_t)digest_bytes;
	const uint64_t nblocks = len / (uint64_t)rate + 1;
	for (uint64_t b = 0; b < nblocks; b++) {
		const uint64_t base = b * (uint64_t)rate;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int lane = 0; lane < 17; lane++) { /* at most 136 / 8 lanes absorb */
			if (8 * lane < rate) {
				uint64_t w = 0;
				for (int k = 0; k < 8; k++) {
					const uint64_t i = base + 8 * (uint64_t)lane + (uint64_t)k;
					const uint64_t byte = i < len ? (uint64_t)m[i] : (i == len ? 0x40u : 0u);
					w |= byte << (8 * k);
				}
				S[lane] = w;
			}
		}
		bash_f(S);
	}
	for (int i = 0; i < digest_bytes; i++) digest[i] = (uint8_t)(S[i >> 3] >> (8 * (i & 7)));
}

} // namespace eccb200
