/*
 * sha3.cuh — SHA3-224 / 256 / 384 / 512 of short messages, one thread per message (the remaining hash functions the
 * reference's ECDSA / ECFSDSA known-answer tests use: src/hash/sha3-256.c etc. over src/hash/sha3.c; generic front end
 * hash_mapping, src/hash/hash_algs.h:232-241).  FIPS 202: Keccak-f[1600] sponge, rate 200 - 2*digest bytes, domain
 * byte 0x06, final bit 0x80.  Constants come from tools/gen_sha3_constants.py (derived from their definition).
 * Plain C++ so that the host build of the tests (tests/hostsim) runs the same code against hashlib.
 */
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define SHA3_HD __host__ __device__ __forceinline__
#else
#define SHA3_HD inline
#endif

namespace eccb200 {

#include "sha3_constants.inc"

/* Byte sources of the hash functions (sha2.cuh as well): m[i] for i < the length the caller passes. */
struct ByteSpan { /* one contiguous message */
	const uint8_t *p;
	SHA3_HD uint32_t operator[](uint64_t i) const { return p[i]; }
};
struct Seg2 { /* pre[0 .. npre) followed by msg */
	const uint8_t *pre;
	uint32_t npre;
	const uint8_t *msg;
	SHA3_HD uint32_t operator[](uint64_t i) const { return i < npre ? pre[i] : msg[i - npre]; }
};
struct Seg3 { /* pre[0 .. npre), then mid[0 .. nmid), then post: SM2's Z = H(ENTL || ID || a || b || G || Y) */
	const uint8_t *pre;
	uint32_t npre;
	const uint8_t *mid;
	uint64_t nmid;
	const uint8_t *post;
	SHA3_HD uint32_t operator[](uint64_t i) const
	{
		return i < npre ? pre[i] : (i - npre < nmid ? mid[i - npre] : post[i - npre - nmid]);
	}
};

static SHA3_HD uint64_t rotl64_(uint64_t x, int n) { return n ? ((x << n) | (x >> (64 - n))) : x; }

/* Keccak-f[1600] on 25 lanes, lane (x, y) at index x + 5*y */
static SHA3_HD void keccak_f1600(uint64_t a[25])
{
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
	for (int round = 0; round < 24; round++) {
		uint64_t c[5], d[5], b[25];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];   /* theta */
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int x = 0; x < 5; x++) d[x] = c[(x + 4) % 5] ^ rotl64_(c[(x + 1) % 5], 1);
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int i = 0; i < 25; i++) {
			const int x = i % 5, y = i / 5;
			/* rho + pi: lane (x, y) rotated moves to (y, 2x + 3y) */
			b[y + 5 * ((2 * x + 3 * y) % 5)] = rotl64_(a[i] ^ d[x], keccak_rot(i));
		}
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int i = 0; i < 25; i++) {
			const int x = i % 5, y = i / 5;
			a[i] = b[i] ^ (~b[(x + 1) % 5 + 5 * y] & b[(x + 2) % 5 + 5 * y]);                    /* chi */
		}
		a[0] ^= keccak_rc(round);                                                                      /* iota */
	}
}

/* digest_bytes in {28, 32, 48, 64} */
template <class Src> SHA3_HD void sha3_src(const Src &m, uint64_t len, uint8_t *digest, int digest_bytes)
{
	const int rate = 200 - 2 * digest_bytes;
	const uint64_t total = ((len + 1 + (uint64_t)rate - 1) / (uint64_t)rate) * (uint64_t)rate; /* padded length */
	uint64_t st[25];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
	for (int i = 0; i < 25; i++) st[i] = 0;
	for (uint64_t base = 0; base < total; base += (uint64_t)rate) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
		for (int lane = 0; lane < 18; lane++) { /* at most 144 / 8 lanes absorb */
			if (8 * lane < rate) {
				uint64_t w = 0;
				for (int k = 0; k < 8; k++) {
					const uint64_t i = base + 8 * (uint64_t)lane + (uint64_t)k;
					uint64_t byte = (i < len) ? (uint64_t)m[i] : 0;
					if (i == len) byte ^= 0x06;
					if (i == total - 1) byte ^= 0x80;
					w |= byte << (8 * k);
				}
				st[lane] ^= w;
			}
		}
		keccak_f1600(st);
	}
	for (int i = 0; i < digest_bytes; i++) digest[i] = (uint8_t)(st[i >> 3] >> (8 * (i & 7)));
}

static SHA3_HD void sha3_device(const uint8_t *m, uint64_t len, uint8_t *digest, int digest_bytes)
{
	sha3_src(ByteSpan{ m }, len, digest, digest_bytes);
}

} // namespace eccb200
