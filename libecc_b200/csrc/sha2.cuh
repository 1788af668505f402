/*
 * sha2.cuh — SHA-256 / SHA-384 / SHA-512 of short messages on the device (SURVEY.md §8f.3: "host-side hashing on
 * device", the step before the ECDSA path), and SHA-224 for the deterministic ECDSA signer (hmac.cuh).  One thread
 * hashes one message of arbitrary length.
 *
 * Reference counterparts (relative to /root/reference/src): sha256_init/update/final hash/sha256.c:70,96,145 (scattered
 * form :201), SHA-384/512 hash/sha384.c, hash/sha512.c over hash/sha512_core.c; generic front end hash_mapping
 * hash/hash_algs.h:232-241.  The algorithm is FIPS 180-4; constants come from tools/gen_sha2_constants.py.
 *
 * The input is a byte source: one contiguous message (ByteSpan), or a short prefix held by the thread followed by a
 * message in global memory (Seg2: the Schnorr-family signers hash W || m or H(tag) || H(tag) || ... || m without
 * building the concatenation).  Plain C++ outside nvcc, so that the host build of the tests runs the same code.
 */
#pragma once
#include <stdint.h>
#include "sha3.cuh"

#if defined(__CUDACC__)
#define SHA2_D __device__ __forceinline__
#else
#define SHA2_D inline
#endif

namespace eccb200 {

/* internal linkage: every translation unit that hashes gets its own copy of the constants */
namespace {
#if defined(__CUDACC__)
#include "sha2_constants.inc"
#else
#define __device__
#define __constant__
#include "sha2_constants.inc"
#undef __device__
#undef __constant__
#endif
} // namespace

SHA2_D uint32_t rotr32(uint32_t x, int n)
{
#if defined(__CUDA_ARCH__)
	return __funnelshift_r(x, x, n);
#else
	return (x >> n) | (x << (32 - n));
#endif
}
SHA2_D uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

/* byte i of the padded message: data, then 0x80, then zeros; the caller overrides the trailing length field */
template <class Src> SHA2_D uint32_t padded_byte(const Src &m, uint64_t len, uint64_t i)
{
	return (i < len) ? m[i] : ((i == len) ? 0x80u : 0u);
}

/* SHA-224's initial value (FIPS 180-4 §5.3.2) */
SHA2_D uint32_t sha224_iv(int i)
{
	return i == 0 ? 0xc1059ed8u : i == 1 ? 0x367cd507u : i == 2 ? 0x3070dd17u : i == 3 ? 0xf70e5939u :
	       i == 4 ? 0xffc00b31u : i == 5 ? 0x68581511u : i == 6 ? 0x64f98fa7u : 0xbefa4fa4u;
}

/* digest: 32 bytes, big-endian words; sha224: SHA-224 (the same compression from its own initial value, 28 bytes out) */
template <class Src>
SHA2_D void sha256_src(const Src &m, uint64_t len, uint8_t *__restrict__ digest, bool sha224 = false)
{
	uint32_t h[8];
#pragma unroll
	for (int i = 0; i < 8; i++) h[i] = sha224 ? sha224_iv(i) : kSha256H[i];
	const uint64_t nblocks = (len + 9 + 63) / 64;
#pragma unroll 1
	for (uint64_t b = 0; b < nblocks; b++) {
		uint32_t w[16];
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
				if (t0 > 0) {
					uint32_t w15 = w[(j + 1) & 15], w2 = w[(j + 14) & 15];
					uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
					uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
					w[j] = w[j] + s0 + w[(j + 9) & 15] + s1;
				}
				uint32_t S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
				uint32_t ch = (e & f) ^ (~e & g);
				uint32_t t1 = hh + S1 + ch + kSha256K[t0 + j] + w[j];
				uint32_t S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
				uint32_t mj = (a & bb) ^ (a & c) ^ (bb & c);
				uint32_t t2 = S0 + mj;
				hh = g; g = f; f = e; e = d + t1; d = c; c = bb; bb = a; a = t1 + t2;
			}
		}
		h[0] += a; h[1] += bb; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
	}
#pragma unroll
	for (int i = 0; i < 8; i++) {
		if (sha224 && i == 7) break;
		digest[4 * i] = (uint8_t)(h[i] >> 24);
		digest[4 * i + 1] = (uint8_t)(h[i] >> 16);
		digest[4 * i + 2] = (uint8_t)(h[i] >> 8);
		digest[4 * i + 3] = (uint8_t)h[i];
	}
}

/* SHA-512 core with selectable initial value; out_bytes = 48 (SHA-384) or 64 (SHA-512) */
template <class Src>
SHA2_D void sha512_family_src(const Src &m, uint64_t len, uint8_t *__restrict__ digest, const uint64_t *__restrict__ iv,
			      int out_bytes)
{
	uint64_t h[8];
#pragma unroll
	for (int i = 0; i < 8; i++) h[i] = iv[i];
	const uint64_t nblocks = (len + 17 + 127) / 128;
#pragma unroll 1
	for (uint64_t b = 0; b < nblocks; b++) {
		uint64_t w[16];
#pragma unroll
		for (int j = 0; j < 16; j++) {
			uint64_t o = b * 128 + 8 * (uint64_t)j, v = 0;
#pragma unroll
			for (int k = 0; k < 8; k++) v = (v << 8) | padded_byte(m, len, o + k);
			w[j] = v;
		}
		if (b == nblocks - 1) { /* 128-bit message length in bits (lengths here fit 64 bits) */
			w[14] = len >> 61;
			w[15] = len << 3;
		}
		uint64_t a = h[0], bb = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll 1
		for (int t0 = 0; t0 < 80; t0 += 16) {
#pragma unroll
			for (int j = 0; j < 16; j++) {
				if (t0 > 0) {
					uint64_t w15 = w[(j + 1) & 15], w2 = w[(j + 14) & 15];
					uint64_t s0 = rotr64(w15, 1) ^ rotr64(w15, 8) ^ (w15 >> 7);
					uint64_t s1 = rotr64(w2, 19) ^ rotr64(w2, 61) ^ (w2 >> 6);
					w[j] = w[j] + s0 + w[(j + 9) & 15] + s1;
				}
				uint64_t S1 = rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41);
				uint64_t ch = (e & f) ^ (~e & g);
				uint64_t t1 = hh + S1 + ch + kSha512K[t0 + j] + w[j];
				uint64_t S0 = rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39);
				uint64_t mj = (a & bb) ^ (a & c) ^ (bb & c);
				uint64_t t2 = S0 + mj;
				hh = g; g = f; f = e; e = d + t1; d = c; c = bb; bb = a; a = t1 + t2;
			}
		}
		h[0] += a; h[1] += bb; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
	}
	for (int i = 0; i < out_bytes; i++) digest[i] = (uint8_t)(h[i >> 3] >> (8 * (7 - (i & 7))));
}

SHA2_D void sha256_device(const uint8_t *__restrict__ m, uint64_t len, uint8_t *__restrict__ digest)
{
	sha256_src(ByteSpan{ m }, len, digest);
}
SHA2_D void sha512_family_device(const uint8_t *__restrict__ m, uint64_t len, uint8_t *__restrict__ digest,
				 const uint64_t *__restrict__ iv, int out_bytes)
{
	sha512_family_src(ByteSpan{ m }, len, digest, iv, out_bytes);
}

/* hash_alg_type values of the reference (lib_ecc_types.h:82-): SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224 = 5,
 * SHA3_256 = 6, SHA3_384 = 7, SHA3_512 = 8 (sha3.cuh) */
SHA3_HD int sha2_digest_size(int hash_type)
{
	return hash_type == 2 ? 32 : hash_type == 3 ? 48 : hash_type == 4 ? 64 : hash_type == 5 ? 28 : hash_type == 6 ? 32 :
	       hash_type == 7 ? 48 : hash_type == 8 ? 64 : 0;
}

/* Any of the seven hashes over a byte source of len bytes; digest: sha2_digest_size(hash_type) bytes.  hash_type must
 * be one of 2..8. */
template <class Src> SHA2_D void hash_src(int hash_type, const Src &m, uint64_t len, uint8_t *digest)
{
	if (hash_type == 2) sha256_src(m, len, digest);
	else if (hash_type == 3) sha512_family_src(m, len, digest, kSha384H, 48);
	else if (hash_type == 4) sha512_family_src(m, len, digest, kSha512H, 64);
	else sha3_src(m, len, digest, sha2_digest_size(hash_type));
}

/* H(pre[0 .. npre) || msg[0 .. nmsg)): the prefix lives with the thread, the message in (global) memory */
SHA2_D void hash_segments(int hash_type, const uint8_t *pre, uint32_t npre, const uint8_t *msg, uint64_t nmsg,
			  uint8_t *digest)
{
	hash_src(hash_type, Seg2{ pre, npre, msg }, (uint64_t)npre + nmsg, digest);
}

#if defined(__CUDACC__)
/* messages are concatenated in `msgs`; message i is msgs[off[i] .. off[i+1]); digests are [n][digest_size] */
static __global__ void __launch_bounds__(128) k_sha2_batch(uint32_t n, int hash_type, const uint8_t *__restrict__ msgs,
							   const uint64_t *__restrict__ off, uint8_t *__restrict__ digests)
{
	uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= n) return;
	const uint8_t *m = msgs + off[idx];
	const uint64_t len = off[idx + 1] - off[idx];
	const int ds = sha2_digest_size(hash_type);
	uint8_t *out = digests + (size_t)idx * ds;
	if (hash_type == 2) sha256_device(m, len, out);
	else if (hash_type == 3) sha512_family_device(m, len, out, kSha384H, 48);
	else if (hash_type == 4) sha512_family_device(m, len, out, kSha512H, 64);
	else sha3_device(m, len, out, ds);
}
#endif

} // namespace eccb200
