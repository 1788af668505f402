/*
 * belt.cuh — the BELT block cipher (belt-block, 256-bit key) and BELT-HASH of STB 34.101.31-2011, one thread per item:
 * the internal hash of the BIGN signature scheme (STB 34.101.45) and the cipher of deterministic BIGN's nonce
 * generator (ec.cuh: bign_*).  Reference counterparts (relative to /root/reference/src): belt_encrypt, belt_hash_init /
 * belt_hash_update / belt_hash_final, hash/belt-hash.c.
 *
 * The S-box H is looked up four times per G_r, with a different byte in every lane.  The kernels copy it into shared
 * memory once per CTA (belt_sbox_to_shared): 256 bytes over 32 banks give at most two-way conflicts, where __constant__
 * would serialise the 32 distinct addresses of a warp.  Every function takes the table as a pointer, so that the host
 * build of the tests runs the same code on kBeltH itself.  Plain C++ outside nvcc, like sha2.cuh.
 */
#pragma once
#include <stdint.h>
#include "sha3.cuh"

namespace eccb200 {

enum { HASH_BELT = 16 }; /* hash_alg_type of the reference (lib_ecc_types.h) */

/*
 * The substitution H : {0,1}^8 -> {0,1}^8 of STB 34.101.31-2011 (§6.1.2, table 1), entry u at index u, as published.
 * It is standard data, not derived here; tests/test_bign_host.py pins every entry against the reference.  Its first
 * 32 bytes are also BELT-HASH's initial value (§6.9: h = B194BAC80A08F53B366D008E584A5DE48504FA9D1BB6C7AC252E72C202FDCE0D).
 */
#if defined(__CUDACC__)
__device__
#endif
static const uint8_t kBeltH[256] = {
	0xB1, 0x94, 0xBA, 0xC8, 0x0A, 0x08, 0xF5, 0x3B, 0x36, 0x6D, 0x00, 0x8E, 0x58, 0x4A, 0x5D, 0xE4,
	0x85, 0x04, 0xFA, 0x9D, 0x1B, 0xB6, 0xC7, 0xAC, 0x25, 0x2E, 0x72, 0xC2, 0x02, 0xFD, 0xCE, 0x0D,
	0x5B, 0xE3, 0xD6, 0x12, 0x17, 0xB9, 0x61, 0x81, 0xFE, 0x67, 0x86, 0xAD, 0x71, 0x6B, 0x89, 0x0B,
	0x5C, 0xB0, 0xC0, 0xFF, 0x33, 0xC3, 0x56, 0xB8, 0x35, 0xC4, 0x05, 0xAE, 0xD8, 0xE0, 0x7F, 0x99,
	0xE1, 0x2B, 0xDC, 0x1A, 0xE2, 0x82, 0x57, 0xEC, 0x70, 0x3F, 0xCC, 0xF0, 0x95, 0xEE, 0x8D, 0xF1,
	0xC1, 0xAB, 0x76, 0x38, 0x9F, 0xE6, 0x78, 0xCA, 0xF7, 0xC6, 0xF8, 0x60, 0xD5, 0xBB, 0x9C, 0x4F,
	0xF3, 0x3C, 0x65, 0x7B, 0x63, 0x7C, 0x30, 0x6A, 0xDD, 0x4E, 0xA7, 0x79, 0x9E, 0xB2, 0x3D, 0x31,
	0x3E, 0x98, 0xB5, 0x6E, 0x27, 0xD3, 0xBC, 0xCF, 0x59, 0x1E, 0x18, 0x1F, 0x4C, 0x5A, 0xB7, 0x93,
	0xE9, 0xDE, 0xE7, 0x2C, 0x8F, 0x0C, 0x0F, 0xA6, 0x2D, 0xDB, 0x49, 0xF4, 0x6F, 0x73, 0x96, 0x47,
	0x06, 0x07, 0x53, 0x16, 0xED, 0x24, 0x7A, 0x37, 0x39, 0xCB, 0xA3, 0x83, 0x03, 0xA9, 0x8B, 0xF6,
	0x92, 0xBD, 0x9B, 0x1C, 0xE5, 0xD1, 0x41, 0x01, 0x54, 0x45, 0xFB, 0xC9, 0x5E, 0x4D, 0x0E, 0xF2,
	0x68, 0x20, 0x80, 0xAA, 0x22, 0x7D, 0x64, 0x2F, 0x26, 0x87, 0xF9, 0x34, 0x90, 0x40, 0x55, 0x11,
	0xBE, 0x32, 0x97, 0x13, 0x43, 0xFC, 0x9A, 0x48, 0xA0, 0x2A, 0x88, 0x5F, 0x19, 0x4B, 0x09, 0xA1,
	0x7E, 0xCD, 0xA4, 0xD0, 0x15, 0x44, 0xAF, 0x8C, 0xA5, 0x84, 0x50, 0xBF, 0x66, 0xD2, 0xE8, 0x8A,
	0xA2, 0xD7, 0x46, 0x52, 0x42, 0xA8, 0xDF, 0xB3, 0x69, 0x74, 0xC5, 0x51, 0xEB, 0x23, 0x29, 0x21,
	0xD4, 0xEF, 0xD9, 0xB4, 0x3A, 0x62, 0x28, 0x75, 0x91, 0x14, 0x10, 0xEA, 0x77, 0x6C, 0xDA, 0x1D,
};

#if defined(__CUDACC__)
/* H into the CTA's shared copy.  Every thread of the CTA must call it (it ends in a barrier), before any thread leaves
 * for an index past the batch. */
__device__ __forceinline__ void belt_sbox_to_shared(uint8_t *sh)
{
	for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) sh[i] = kBeltH[i];
	__syncthreads();
}
#endif

/* G_r(u) = RotHi^r(H(u_1) || H(u_2) || H(u_3) || H(u_4)) on a little-endian word (§6.1.3) */
SHA3_HD uint32_t belt_g(const uint8_t *H, uint32_t u, int r)
{
	const uint32_t v = (uint32_t)H[u & 0xff] | (uint32_t)H[(u >> 8) & 0xff] << 8 | (uint32_t)H[(u >> 16) & 0xff] << 16 |
			   (uint32_t)H[u >> 24] << 24;
	return (v << r) | (v >> (32 - r));
}

/*
 * belt-block encryption (§6.1.4) of the block x (four little-endian words) under the key k (eight little-endian words
 * θ_1 .. θ_8), in place.  Round i (1..8) uses the round keys K_{7i-6} .. K_{7i}, K_j = θ_{((j - 1) mod 8) + 1}.
 */
SHA3_HD void belt_block(uint32_t x[4], const uint32_t k[8], const uint8_t *H)
{
	uint32_t a = x[0], b = x[1], c = x[2], d = x[3];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
	for (int i = 0; i < 8; i++) {
		const int j = 7 * i; /* K_{7i+1 ..} with 0-based i */
		b ^= belt_g(H, a + k[j & 7], 5);
		c ^= belt_g(H, d + k[(j + 1) & 7], 21);
		a -= belt_g(H, b + k[(j + 2) & 7], 13);
		const uint32_t e = belt_g(H, b + c + k[(j + 3) & 7], 21) ^ (uint32_t)(i + 1);
		b += e;
		c -= e;
		d += belt_g(H, c + k[(j + 4) & 7], 13);
		b ^= belt_g(H, a + k[(j + 5) & 7], 21);
		c ^= belt_g(H, d + k[(j + 6) & 7], 5);
		const uint32_t ta = a, tc = c;
		a = b;       /* a <-> b */
		c = d;       /* c <-> d */
		d = tc;
		b = c;       /* b <-> c */
		c = ta;
	}
	x[0] = b;
	x[1] = d;
	x[2] = a;
	x[3] = c;
}

/* 16 little-endian bytes <-> four words */
SHA3_HD void belt_load_block(uint32_t w[4], const uint8_t *p)
{
	for (int i = 0; i < 4; i++)
		w[i] = (uint32_t)p[4 * i] | (uint32_t)p[4 * i + 1] << 8 | (uint32_t)p[4 * i + 2] << 16 | (uint32_t)p[4 * i + 3] << 24;
}
SHA3_HD void belt_store_block(uint8_t *p, const uint32_t w[4])
{
	for (int i = 0; i < 4; i++) {
		p[4 * i] = (uint8_t)w[i];
		p[4 * i + 1] = (uint8_t)(w[i] >> 8);
		p[4 * i + 2] = (uint8_t)(w[i] >> 16);
		p[4 * i + 3] = (uint8_t)(w[i] >> 24);
	}
}

/*
 * One BELT-HASH step on u = x || h (x the 256-bit block or key, h the 256-bit chaining value; §6.9.1):
 *   sigma1(u) = belt-block(h_1 ^ h_2, x) ^ h_1 ^ h_2                         -> s1
 *   sigma2(u) = (belt-block(x_1, sigma1(u) || h_2) ^ x_1) || (belt-block(x_2, ~sigma1(u) || h_1) ^ x_2)   -> h
 * The compression of a message block uses both, so sigma1 is computed once: three encryptions per step.
 */
SHA3_HD void belt_sigma(const uint32_t x[8], uint32_t h[8], uint32_t s1[4], const uint8_t *H)
{
	uint32_t key[8], y1[4], y2[4];
	for (int i = 0; i < 4; i++) s1[i] = h[i] ^ h[4 + i];
	const uint32_t u[4] = { s1[0], s1[1], s1[2], s1[3] };
	belt_block(s1, x, H);
	for (int i = 0; i < 4; i++) {
		s1[i] ^= u[i];
		key[i] = s1[i];
		key[4 + i] = h[4 + i];
		y1[i] = x[i];
		y2[i] = x[4 + i];
	}
	belt_block(y1, key, H);
	for (int i = 0; i < 4; i++) {
		key[i] = ~s1[i];
		key[4 + i] = h[i];
	}
	belt_block(y2, key, H);
	for (int i = 0; i < 4; i++) {
		h[i] = y1[i] ^ x[i];
		h[4 + i] = y2[i] ^ x[4 + i];
	}
}

/*
 * BELT-HASH (§6.9) of len bytes of a byte source (sha3.cuh), 32 bytes out: the message zero-padded to 32-byte blocks
 * X_1 .. X_n (n = 0 for the empty message); s = 0, h = the first 32 bytes of H; (s, h) <- (s ^ sigma1(X_i || h),
 * sigma2(X_i || h)) per block; the digest is sigma2(<8*len>_128 || s || h).
 */
template <class Src> SHA3_HD void belt_hash_src(const Src &m, uint64_t len, uint8_t *digest, const uint8_t *H)
{
	uint32_t h[8], s[4] = { 0, 0, 0, 0 }, x[8], s1[4];
	belt_load_block(h, H);
	belt_load_block(h + 4, H + 16);
	const uint64_t nblocks = (len + 31) / 32;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
	for (uint64_t b = 0; b < nblocks; b++) {
		for (int i = 0; i < 8; i++) {
			uint32_t w = 0;
			for (int j = 0; j < 4; j++) {
				const uint64_t o = 32 * b + 4 * (uint64_t)i + (uint64_t)j;
				w |= (o < len ? (uint32_t)m[o] : 0u) << (8 * j);
			}
			x[i] = w;
		}
		belt_sigma(x, h, s1, H);
		for (int i = 0; i < 4; i++) s[i] ^= s1[i];
	}
	const uint64_t bits = len << 3;
	x[0] = (uint32_t)bits;
	x[1] = (uint32_t)(bits >> 32);
	x[2] = (uint32_t)(len >> 61);
	x[3] = 0;
	for (int i = 0; i < 4; i++) x[4 + i] = s[i];
	belt_sigma(x, h, s1, H);
	belt_store_block(digest, h);
	belt_store_block(digest + 16, h + 4);
}

} // namespace eccb200
