/*
 * hmac.cuh — HMAC (RFC 2104) over the hashes of the device, one thread per item: the pseudo-random function of
 * deterministic ECDSA's nonce generation (RFC 6979 §3.2, ec.cuh: rfc6979_nonce).  Reference counterpart (relative to
 * /root/reference/src): hmac_init / hmac_update / hmac_finalize, hash/hmac.c:16-134.
 *
 * The hash set is that of the message signers (sm3.cuh: SHA-256 .. SHA3-512 and SM3) plus SHA-224 (hash_alg_type 1),
 * which only the deterministic-ECDSA entry points accept: sha2_digest_size and msg_hash_digest_size keep refusing it,
 * so the older entry points keep their behaviour.  Plain C++ outside nvcc, like sha2.cuh, so that the host build of the
 * tests runs the same code.
 */
#pragma once
#include <stdint.h>
#include "sm3.cuh"

namespace eccb200 {

enum { HASH_SHA224 = 1 }; /* hash_alg_type of the reference (lib_ecc_types.h) */

/* digest size of the deterministic-ECDSA hashes: SHA-224 (1), SHA-256 .. SHA3-512 (2..8), SM3 (11); 0 otherwise */
SHA3_HD int decdsa_hash_digest_size(int hash_type)
{
	return hash_type == HASH_SHA224 ? 28 : msg_hash_digest_size(hash_type);
}

/* their block size (hm->block_size), the length HMAC pads its key to */
SHA3_HD int decdsa_hash_block_size(int hash_type)
{
	return hash_type == HASH_SHA224 ? 64 : msg_hash_block_size(hash_type);
}

/* Any of the nine over a byte source of len bytes; hash_type must have a non-zero decdsa_hash_digest_size. */
template <class Src> SHA2_D void decdsa_hash_src(int hash_type, const Src &m, uint64_t len, uint8_t *digest)
{
	if (hash_type == HASH_SHA224) sha256_src(m, len, digest, true);
	else msg_hash_src(hash_type, m, len, digest);
}

/* (K XOR pad) zero-extended to the block size bs, then the message: the input of HMAC's inner (pad 0x36) and outer
 * (pad 0x5c) hash (hash/hmac.c:67-75).  K is klen <= bs bytes held by the thread. */
template <class Src> struct HmacPadSrc {
	const uint8_t *key;
	uint32_t klen;
	uint32_t bs;
	uint32_t pad;
	Src msg;
	SHA3_HD uint32_t operator[](uint64_t i) const
	{
		return i < bs ? ((i < klen ? (uint32_t)key[i] : 0u) ^ pad) : msg[i - bs];
	}
};

/*
 * out = HMAC_K(m) = H((K ^ opad) || H((K ^ ipad) || m)) with H = hash_type (decdsa_hash_digest_size(hash_type) bytes
 * out).  The key must not be longer than the block size: RFC 6979 keys HMAC with a digest-sized K, and the reference
 * hashes longer keys first (hash/hmac.c:45-56), a branch this never needs.  out may alias the key or the message: the
 * hashes write the digest after they have read their last block.  Two hashes of bs + |m| and bs + hsize bytes; no
 * midstate is kept across HMACs with the same key.
 */
template <class Src>
SHA2_D void hmac_src(int hash_type, const uint8_t *key, uint32_t klen, const Src &m, uint64_t mlen, uint8_t *out)
{
	const uint32_t bs = (uint32_t)decdsa_hash_block_size(hash_type), ds = (uint32_t)decdsa_hash_digest_size(hash_type);
	uint8_t inner[64];
	decdsa_hash_src(hash_type, HmacPadSrc<Src>{ key, klen, bs, 0x36u, m }, (uint64_t)bs + mlen, inner);
	decdsa_hash_src(hash_type, HmacPadSrc<ByteSpan>{ key, klen, bs, 0x5cu, ByteSpan{ inner } }, (uint64_t)bs + ds, out);
}

} // namespace eccb200
