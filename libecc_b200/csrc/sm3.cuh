/*
 * sm3.cuh — SM3 (GB/T 32905-2016, the hash of the SM2 signature scheme) over the byte sources of sha3.cuh, one thread
 * per message.  Reference counterpart (relative to /root/reference/src): sm3_init/update/final hash/sm3.c.  Padding
 * and message loading are SHA-256's (64-byte blocks, 0x80, 64-bit big-endian bit length).
 *
 * Also the hash front end of the message signers of ec.cuh (ECKCDSA, ECGDSA, ECRDSA, SM2): the seven hashes of
 * sha2.cuh plus SM3 (hash_alg_type 11).  The older entry points keep sha2_digest_size, which knows no SM3.
 * Plain C++ outside nvcc, like sha2.cuh, so that the host build of the tests runs the same code.
 */
#pragma once
#include <stdint.h>
#include "sha2.cuh"

namespace eccb200 {

enum { HASH_SM3 = 11 }; /* hash_alg_type of the reference (lib_ecc_types.h) */

SHA2_D uint32_t sm3_rotl(uint32_t x, int n)
{
#if defined(__CUDA_ARCH__)
	return __funnelshift_l(x, x, n);
#else
	return (x << (n & 31)) | (x >> ((32 - n) & 31));
#endif
}

/* digest: 32 bytes, big-endian words */
template <class Src> SHA2_D void sm3_src(const Src &m, uint64_t len, uint8_t *__restrict__ digest)
{
	uint32_t h[8] = { 0x7380166fu, 0x4914b2b9u, 0x172442d7u, 0xda8a0600u,
			  0xa96f30bcu, 0x163138aau, 0xe38dee4du, 0xb0fb0e4eu };
	const uint64_t nblocks = (len + 9 + 63) / 64;
#pragma unroll 1
	for (uint64_t b = 0; b < nblocks; b++) {
		uint32_t w[16]; /* ring of W[t-12 .. t+3]: W[t + 4] is expanded at step t, into the slot of W[t - 12] */
#pragma unroll
		for (int j = 0; j < 16; j++) {
			uint64_t o = b * 64 + 4 * (uint64_t)j;
			w[j] = (padded_byte(m, len, o) << 24) | (padded_byte(m, len, o + 1) << 16) |
			       (padded_byte(m, len, o + 2) << 8) | padded_byte(m, len, o + 3);
		}
		if (b == nblocks - 1) { /* 64-bit message length in bits */
			w[14] = (uint32_t)((len << 3) >> 32);
			w[15] = (uint32_t)(len << 3);
		}
		uint32_t a = h[0], bb = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll 1
		for (int t0 = 0; t0 < 64; t0 += 16) {
#pragma unroll
			for (int j = 0; j < 16; j++) {
				const int t = t0 + j;
				if (t0 > 0 || j >= 12) { /* W[i] = P1(W[i-16] ^ W[i-9] ^ (W[i-3] <<< 15)) ^ (W[i-13] <<< 7) ^ W[i-6] */
					uint32_t v = w[(j + 4) & 15] ^ w[(j + 11) & 15] ^ sm3_rotl(w[(j + 1) & 15], 15);
					v = v ^ sm3_rotl(v, 15) ^ sm3_rotl(v, 23);
					w[(j + 4) & 15] = v ^ sm3_rotl(w[(j + 7) & 15], 7) ^ w[(j + 14) & 15];
				}
				const uint32_t wj = w[j], wp = wj ^ w[(j + 4) & 15];
				const uint32_t a12 = sm3_rotl(a, 12);
				const uint32_t ss1 = sm3_rotl(a12 + e + sm3_rotl(t0 == 0 ? 0x79cc4519u : 0x7a879d8au, t & 31), 7);
				const uint32_t ss2 = ss1 ^ a12;
				const uint32_t ff = t0 == 0 ? (a ^ bb ^ c) : ((a & bb) | (a & c) | (bb & c));
				const uint32_t gg = t0 == 0 ? (e ^ f ^ g) : ((e & f) | (~e & g));
				const uint32_t tt1 = ff + d + ss2 + wp;
				const uint32_t tt2 = gg + hh + ss1 + wj;
				d = c;
				c = sm3_rotl(bb, 9);
				bb = a;
				a = tt1;
				hh = g;
				g = sm3_rotl(f, 19);
				f = e;
				e = tt2 ^ sm3_rotl(tt2, 9) ^ sm3_rotl(tt2, 17); /* P0 */
			}
		}
		h[0] ^= a; h[1] ^= bb; h[2] ^= c; h[3] ^= d; h[4] ^= e; h[5] ^= f; h[6] ^= g; h[7] ^= hh;
	}
#pragma unroll
	for (int i = 0; i < 8; i++) {
		digest[4 * i] = (uint8_t)(h[i] >> 24);
		digest[4 * i + 1] = (uint8_t)(h[i] >> 16);
		digest[4 * i + 2] = (uint8_t)(h[i] >> 8);
		digest[4 * i + 3] = (uint8_t)h[i];
	}
}

/* digest size of the message signers' hashes: SHA256 .. SHA3_512 (2..8) and SM3 (11); 0 for any other type */
SHA3_HD int msg_hash_digest_size(int hash_type) { return hash_type == HASH_SM3 ? 32 : sha2_digest_size(hash_type); }

/* block size of those hashes (hm->block_size): the length of ECKCDSA's z */
SHA3_HD int msg_hash_block_size(int hash_type)
{
	return hash_type == 2 || hash_type == HASH_SM3 ? 64 : hash_type == 3 || hash_type == 4 ? 128 :
	       hash_type == 5 ? 144 : hash_type == 6 ? 136 : hash_type == 7 ? 104 : hash_type == 8 ? 72 : 0;
}

/* Any of the eight over a byte source of len bytes; hash_type must have a non-zero msg_hash_digest_size. */
template <class Src> SHA2_D void msg_hash_src(int hash_type, const Src &m, uint64_t len, uint8_t *digest)
{
	if (hash_type == HASH_SM3) sm3_src(m, len, digest);
	else hash_src(hash_type, m, len, digest);
}

} // namespace eccb200
