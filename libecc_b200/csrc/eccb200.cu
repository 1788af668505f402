/*
 * eccb200.cu — C-ABI implementation (include/libecc_b200.h): context management, kernel dispatch, and the
 * chunked host<->device pipeline of the host-pointer entry points.  No arithmetic happens on the host.
 */
#include "../../include/libecc_b200.h"
#include "kernels.cuh"
#include "msm.cuh"
#include "sha2.cuh"
#include "wire.cuh"

#include <cuda_runtime.h>
#include <sys/random.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

using namespace eccb200;

static thread_local std::string g_err;
static int fail(const std::string &m)
{
	g_err = m;
	return -1;
}
#define CUDA_OK(expr)                                                                                      \
	do {                                                                                               \
		cudaError_t e_ = (expr);                                                                   \
		if (e_ != cudaSuccess)                                                                     \
			return fail(std::string(#expr) + ": " + cudaGetErrorString(e_));                   \
	} while (0)

extern "C" const char *eccb200_last_error(void) { return g_err.c_str(); }

static const int kStages = 3; /* pipeline depth of the host-pointer API */

struct eccb200_ctx {
	int curve_id = 0;
	int device = 0;
	int N = 0;           /* 32-bit words per element */
	uint32_t plen = 0, qlen = 0;
	int w = 0;           /* comb window */
	int nwin = 0;
	int sm_count = 0;
	uint32_t wave = 0;     /* items of one full wave of K1: SMs * 4 CTAs * 128 threads */
	uint32_t chunk_eq = 0; /* items per equal pipeline chunk: four waves (ECCB200_CHUNK_WAVES) */
	uint32_t chunk = 0;    /* capacity of the stage buffers: the largest chunk (eight waves) */
	uint32_t *table = nullptr;
	/* work buffers (grown on demand) */
	uint32_t cap = 0;
	uint32_t *jac = nullptr;
	uint32_t *prefix = nullptr;
	uint8_t *aff = nullptr;  /* [cap][2*plen] scratch (k*G of the signing path) */
	/* host-pointer pipeline */
	cudaStream_t streams[kStages] = {};
	cudaEvent_t kdone[kStages] = {}; /* the next chunk's kernels may start: recorded after the chunk's LAST kernel, or
	                                  * by the launcher after its throughput-bound kernel (kdone_set) so that the short
	                                  * latency-bound normalisation overlaps the next chunk's scalar multiplications */
	bool kdone_set = false;
	cudaStream_t hi[kStages] = {};    /* highest-priority streams for the short normalisation kernels of the pipeline */
	cudaEvent_t ndone[kStages] = {};  /* normalisation of the stage's chunk finished */
	uint8_t *h_in[kStages] = {};   /* pinned */
	uint8_t *h_out[kStages] = {};  /* pinned */
	uint8_t *d_in[kStages] = {};
	uint8_t *d_out[kStages] = {};
	size_t stage_in_bytes = 0, stage_out_bytes = 0;
	uint32_t *stage_jac[kStages] = {};
	uint32_t *stage_prefix[kStages] = {};
	uint8_t *stage_aff[kStages] = {};
	uint8_t *stage_state[kStages] = {}; /* [chunk] per-key states of the projective-key verification */
	uint64_t launches = 0;
	/* The device-pointer entry points share ONE scratch set (jac / prefix / aff).  Calls may come in on different
	 * streams: every call first makes its stream wait for scratch_done (recorded behind the previous call's last
	 * kernel), so calls are serialised on the device in the order they were issued — never racing on the scratch. */
	cudaEvent_t scratch_done = nullptr;
	bool scratch_used = false;
	unsigned int *gather_counter = nullptr; /* CTA counter of the fused K4 gather (kernels.cuh GatherDst) */
	/* K6 (msm.cuh): work buffers of the multi-scalar-multiplication batch verification, grown on demand */
	MsmBuffers msm = {};
	uint32_t msm_cap_n = 0, msm_cap_total = 0;
	size_t msm_cap_list = 0;
	uint8_t *msm_in = nullptr; /* device copy of the host-pointer entry point's inputs */
	size_t msm_in_bytes = 0;
	uint8_t *unique_io = nullptr; /* device buffer of eccb200_prj_pt_unique_batch (in || out || status), grown on demand:
	                               * a cudaMalloc / cudaFree pair per call cost up to a second on a busy allocator */
	size_t unique_io_bytes = 0;
	uint8_t *sign_k = nullptr; /* [sign_k_cap][qlen] scratch of the device-pointer signers, grown on demand: BIP0340, RFC 6979
	                            * and DBIGN nonces, and the digests of the ECDSA and BIGN message signers and of the BIGN
	                            * verifier after them */
	size_t sign_k_cap = 0;
	/* optional per-kernel timing of the device-pointer API (bench.py's roofline leg) */
	bool profiling = false;
	static const int kProfCalls = 64;
	cudaEvent_t ev[kProfCalls][3];  /* per timed call: before kernel 0, between, after kernel 1 */
	int ev_kernels[kProfCalls];     /* kernels timed by that call (1 or 2) */
	int ev_calls = 0;               /* timed device-pointer calls since the last eccb200_profile_read */
	bool ev_ready = false;
};

template <class Fn> static int dispatch(int curve_id, Fn &&fn)
{
	switch (curve_id) {
	case ECCB200_SECP256R1: return fn(Curve_SECP256R1());
	case ECCB200_FRP256V1: return fn(Curve_FRP256V1());
	case ECCB200_SECP384R1: return fn(Curve_SECP384R1());
	case ECCB200_BRAINPOOLP256R1: return fn(Curve_BRAINPOOLP256R1());
	case ECCB200_BRAINPOOLP384R1: return fn(Curve_BRAINPOOLP384R1());
	case ECCB200_SECP256K1: return fn(Curve_SECP256K1());
	case ECCB200_SECP521R1: return fn(Curve_SECP521R1());
	case ECCB200_SM2P256V1: return fn(Curve_SM2P256V1());
	case ECCB200_BRAINPOOLP512R1: return fn(Curve_BRAINPOOLP512R1());
	case ECCB200_SECP224R1: return fn(Curve_SECP224R1());
	case ECCB200_SECP192R1: return fn(Curve_SECP192R1());
	default: return fail("unknown curve id");
	}
}

extern "C" int eccb200_curve_sizes(int curve_id, uint32_t *plen, uint32_t *qlen)
{
	return dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		*plen = C::PLEN;
		*qlen = C::QLEN;
		return 0;
	});
}

extern "C" const char *eccb200_curve_name(int curve_id)
{
	const char *n = nullptr;
	dispatch(curve_id, [&](auto c) {
		n = decltype(c)::name();
		return 0;
	});
	return n;
}

/* threads for the batched normalisation: enough to fill the machine, few enough that every thread amortises its
 * inversion over many items */
static uint32_t affine_grid(const eccb200_ctx *ctx, uint32_t n, bool for_throughput = false)
{
	/* Two regimes.  On its own in a stream the kernel is latency-bound for small n (two passes of dependent items per
	 * thread around one inversion): as many CTAs as the machine holds, one item per thread if need be.  Running UNDER the
	 * next chunk's scalar multiplication (side stream of the host pipeline) its work is what counts: every thread then
	 * owns at least ~8 items, which share the 16 products per thread of the CTA-wide inversion. */
	uint32_t want = for_throughput ? (n + kThreads * 8 - 1) / (kThreads * 8) : grid_for(n);
	static int per_sm = 0; /* CTAs of 128 threads per SM; ECCB200_AFFINE_CTAS overrides (tuning knob) */
	if (!per_sm) {
		const char *e = getenv("ECCB200_AFFINE_CTAS");
		per_sm = (e && atoi(e) > 0) ? atoi(e) : 4;
	}
	uint32_t cap = (uint32_t)ctx->sm_count * (uint32_t)per_sm;
	return std::max(1u, std::min(want, cap));
}

static int ensure_work(eccb200_ctx *ctx, uint32_t n)
{
	if (n <= ctx->cap) return 0;
	CUDA_OK(cudaDeviceSynchronize()); /* earlier calls may still be using the scratch that is about to be replaced */
	if (ctx->jac) cudaFree(ctx->jac);
	if (ctx->prefix) cudaFree(ctx->prefix);
	if (ctx->aff) cudaFree(ctx->aff);
	ctx->jac = ctx->prefix = nullptr;
	ctx->aff = nullptr;
	ctx->cap = 0;
	CUDA_OK(cudaMalloc(&ctx->jac, (size_t)n * 3 * ctx->N * sizeof(uint32_t)));
	CUDA_OK(cudaMalloc(&ctx->prefix, (size_t)n * ctx->N * sizeof(uint32_t)));
	CUDA_OK(cudaMalloc(&ctx->aff, (size_t)n * 2 * ctx->plen));
	ctx->cap = n;
	return 0;
}

extern "C" int eccb200_ctx_create(eccb200_ctx **out, int curve_id, int device, int comb_window)
{
	if (!out) return fail("null ctx pointer");
	*out = nullptr;
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
		return fail("no CUDA device: libecc_b200 has no CPU fallback");
	if (device < 0 || device >= ndev) return fail("bad device index");
	CUDA_OK(cudaSetDevice(device));
	cudaDeviceProp prop;
	CUDA_OK(cudaGetDeviceProperties(&prop, device));
	if (prop.major != 9) return fail("libecc_b200 is built for sm_90a (H100) only");
	if (const char *ss = getenv("ECCB200_STACK")) cudaDeviceSetLimit(cudaLimitStackSize, (size_t)atoi(ss));
	/* tuning knob: L2 fetch granularity for the random 64-96 B comb-table gathers (32, 64 or 128; measured: no
	 * effect on the kernel time, which is integer-pipe bound — left at the device default unless requested) */
	if (const char *lf = getenv("ECCB200_L2_FETCH")) {
		size_t g = (size_t)atoi(lf);
		if (g == 32 || g == 64 || g == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, g);
		cudaGetLastError();
	}
	/* default: 22-bit windows (12 adds per 256-bit scalar, 3.2 GB table); 20-bit for the 521-bit curve (27 adds, 4 GB) */
	uint32_t plen_probe = 0, qlen_probe = 0;
	if (eccb200_curve_sizes(curve_id, &plen_probe, &qlen_probe)) return -1;
	int w = comb_window ? comb_window : (plen_probe > 48 ? 20 : 22);
	if (w < 4 || w > 26 || (w > 16 && (w & 1))) return fail("comb_window must be in [4,16] or even in [18,26]");

	eccb200_ctx *ctx = new eccb200_ctx();
	ctx->curve_id = curve_id;
	ctx->device = device;
	ctx->w = w;
	ctx->sm_count = prop.multiProcessorCount;
	{ /* pipeline chunk = full K1 waves (SMs x resident CTAs x 128 items; the residency is the kernel's real,
	   * register-limited one from the occupancy API — a chunk that is not a
	   * whole number of waves leaves the SMs idle at its tail); ECCB200_CHUNK_WAVES overrides the wave count */
		const char *cw = getenv("ECCB200_CHUNK_WAVES");
		uint32_t waves = (cw && atoi(cw) > 0 && atoi(cw) <= 64) ? (uint32_t)atoi(cw) : 4u;
		int occ = 4;
		dispatch(curve_id, [&](auto c) {
			occ = LaunchFixed<decltype(c)>::fixed_ctas_per_sm();
			return 0;
		});
		ctx->wave = (uint32_t)prop.multiProcessorCount * (uint32_t)occ * 128u;
		ctx->chunk_eq = waves * ctx->wave;
		ctx->chunk = std::max(8u, waves) * ctx->wave; /* stage capacity: the largest chunk the pipeline may cut */
	}
	int rc = dispatch(curve_id, [&](auto c) {
		typedef decltype(c) C;
		ctx->N = C::N;
		ctx->plen = C::PLEN;
		ctx->qlen = C::QLEN;
		ctx->nwin = (C::QBITS + w - 1) / w;
		const size_t entries = (size_t)ctx->nwin << w;
		CUDA_OK(cudaMalloc(&ctx->table, entries * 2 * C::N * sizeof(uint32_t)));
		if (w <= 16) {
			/* direct build: every entry is a scalar multiplication d * 2^(w*i) * G (K2's window_mul) */
			if (ensure_work(ctx, (uint32_t)entries)) return -1;
			LaunchVar<C>::table_points((uint32_t)entries, w, ctx->jac, 0);
			LaunchMisc<C>::to_table(affine_grid(ctx, (uint32_t)entries), (uint32_t)entries, ctx->jac, ctx->prefix,
						ctx->table, 0);
			ctx->launches += 2;
		} else {
			/* wide table from a half-width one: one addition per entry (k_table_merge), window by window */
			const int h = w / 2, nwin_half = (C::QBITS + h - 1) / h;
			const uint32_t half_entries = (uint32_t)nwin_half << h, per_win = 1u << w;
			/* merged in slices of at most 2^22 entries so that the scratch stays small next to a table of tens of GB */
			const uint32_t slice = std::min(per_win, 1u << 22);
			uint32_t *half = nullptr;
			CUDA_OK(cudaMalloc(&half, (size_t)half_entries * 2 * C::N * sizeof(uint32_t)));
			if (ensure_work(ctx, std::max(half_entries, slice))) return -1;
			LaunchVar<C>::table_points(half_entries, h, ctx->jac, 0);
			LaunchMisc<C>::to_table(affine_grid(ctx, half_entries), half_entries, ctx->jac, ctx->prefix, half, 0);
			ctx->launches += 2;
			for (int i = 0; i < ctx->nwin; i++) {
				for (uint32_t off = 0; off < per_win; off += slice) {
					const uint64_t first = ((uint64_t)i << w) + off;
					LaunchFixed<C>::table_merge(slice, first, w, nwin_half, half, ctx->jac, 0);
					LaunchMisc<C>::to_table(affine_grid(ctx, slice), slice, ctx->jac, ctx->prefix,
								ctx->table + (size_t)first * 2 * C::N, 0);
					ctx->launches += 2;
				}
			}
			CUDA_OK(cudaDeviceSynchronize());
			cudaFree(half);
		}
		CUDA_OK(cudaGetLastError());
		CUDA_OK(cudaDeviceSynchronize());
		return 0;
	});
	if (rc) {
		eccb200_ctx_destroy(ctx);
		return -1;
	}
	if (cudaEventCreateWithFlags(&ctx->scratch_done, cudaEventDisableTiming) != cudaSuccess ||
	    cudaMalloc(&ctx->gather_counter, sizeof(unsigned int)) != cudaSuccess ||
	    cudaMemset(ctx->gather_counter, 0, sizeof(unsigned int)) != cudaSuccess) {
		eccb200_ctx_destroy(ctx);
		return fail("context event / counter allocation failed");
	}
	for (int s = 0; s < kStages; s++) {
		int least = 0, greatest = 0;
		cudaDeviceGetStreamPriorityRange(&least, &greatest);
		if (cudaStreamCreateWithPriority(&ctx->streams[s], cudaStreamNonBlocking, least) != cudaSuccess ||
		    cudaStreamCreateWithPriority(&ctx->hi[s], cudaStreamNonBlocking, greatest) != cudaSuccess ||
		    cudaEventCreateWithFlags(&ctx->kdone[s], cudaEventDisableTiming) != cudaSuccess ||
		    cudaEventCreateWithFlags(&ctx->ndone[s], cudaEventDisableTiming) != cudaSuccess) {
			eccb200_ctx_destroy(ctx);
			return fail("cudaStreamCreate failed");
		}
	}
	*out = ctx;
	return 0;
}

static void msm_release(eccb200_ctx *ctx)
{
	uint32_t *bufs[] = { ctx->msm.pts, ctx->msm.scal, ctx->msm.partial, ctx->msm.count, ctx->msm.offs, ctx->msm.fill,
			     ctx->msm.list, ctx->msm.buckets, ctx->msm.parts, ctx->msm.winsum, ctx->msm.order, ctx->msm.aux };
	for (uint32_t *b : bufs)
		if (b) cudaFree(b);
	if (ctx->msm.flags) cudaFree(ctx->msm.flags);
	ctx->msm = MsmBuffers{};
	ctx->msm_cap_n = ctx->msm_cap_total = 0;
	ctx->msm_cap_list = 0;
}

extern "C" void eccb200_ctx_destroy(eccb200_ctx *ctx)
{
	if (!ctx) return;
	cudaSetDevice(ctx->device);
	cudaDeviceSynchronize();
	for (int s = 0; s < kStages; s++) {
		if (ctx->streams[s]) cudaStreamDestroy(ctx->streams[s]);
		if (ctx->kdone[s]) cudaEventDestroy(ctx->kdone[s]);
		if (ctx->hi[s]) cudaStreamDestroy(ctx->hi[s]);
		if (ctx->ndone[s]) cudaEventDestroy(ctx->ndone[s]);
		if (ctx->h_in[s]) cudaFreeHost(ctx->h_in[s]);
		if (ctx->h_out[s]) cudaFreeHost(ctx->h_out[s]);
		if (ctx->d_in[s]) cudaFree(ctx->d_in[s]);
		if (ctx->d_out[s]) cudaFree(ctx->d_out[s]);
		if (ctx->stage_jac[s]) cudaFree(ctx->stage_jac[s]);
		if (ctx->stage_prefix[s]) cudaFree(ctx->stage_prefix[s]);
		if (ctx->stage_aff[s]) cudaFree(ctx->stage_aff[s]);
		if (ctx->stage_state[s]) cudaFree(ctx->stage_state[s]);
	}
	if (ctx->ev_ready)
		for (int c = 0; c < eccb200_ctx::kProfCalls; c++)
			for (int i = 0; i < 3; i++) cudaEventDestroy(ctx->ev[c][i]);
	if (ctx->scratch_done) cudaEventDestroy(ctx->scratch_done);
	if (ctx->gather_counter) cudaFree(ctx->gather_counter);
	msm_release(ctx);
	if (ctx->msm_in) cudaFree(ctx->msm_in);
	if (ctx->unique_io) cudaFree(ctx->unique_io);
	if (ctx->sign_k) cudaFree(ctx->sign_k);
	if (ctx->table) cudaFree(ctx->table);
	if (ctx->jac) cudaFree(ctx->jac);
	if (ctx->prefix) cudaFree(ctx->prefix);
	if (ctx->aff) cudaFree(ctx->aff);
	delete ctx;
}

extern "C" int eccb200_profile_enable(eccb200_ctx *ctx, int on)
{
	if (!ctx) return fail("null ctx");
	CUDA_OK(cudaSetDevice(ctx->device));
	if (on && !ctx->ev_ready) {
		for (int c = 0; c < eccb200_ctx::kProfCalls; c++)
			for (int i = 0; i < 3; i++) CUDA_OK(cudaEventCreate(&ctx->ev[c][i]));
		ctx->ev_ready = true;
	}
	ctx->profiling = on != 0;
	ctx->ev_calls = 0;
	return 0;
}

/* Sums, per kernel position, the device time of every timed device-pointer call since the previous read. */
extern "C" int eccb200_profile_read(eccb200_ctx *ctx, float *ms, int cap)
{
	if (!ctx || !ms) return fail("null argument");
	if (!ctx->profiling || ctx->ev_calls == 0) return 0;
	int kmax = 0;
	for (int k = 0; k < cap && k < 2; k++) ms[k] = 0.f;
	for (int c = 0; c < ctx->ev_calls; c++) {
		CUDA_OK(cudaEventSynchronize(ctx->ev[c][ctx->ev_kernels[c]]));
		for (int k = 0; k < ctx->ev_kernels[c] && k < cap; k++) {
			float t = 0.f;
			CUDA_OK(cudaEventElapsedTime(&t, ctx->ev[c][k], ctx->ev[c][k + 1]));
			ms[k] += t;
		}
		if (ctx->ev_kernels[c] > kmax) kmax = ctx->ev_kernels[c];
	}
	ctx->ev_calls = 0;
	return kmax < cap ? kmax : cap;
}

extern "C" int eccb200_comb_window(const eccb200_ctx *ctx) { return ctx ? ctx->w : -1; }
extern "C" uint64_t eccb200_kernel_launches(const eccb200_ctx *ctx) { return ctx ? ctx->launches : 0; }

/* ------------------------------------------------------------------------------------------ device-pointer API */

/* ECCB200_TMA_STAGING=1 selects the K1 variant that stages the scalars with cp.async.bulk (layout experiment) */
static bool tma_staging_enabled()
{
	static int v = -1;
	if (v < 0) {
		const char *e = getenv("ECCB200_TMA_STAGING");
		v = (e && atoi(e) != 0) ? 1 : 0;
	}
	return v == 1;
}

/* see eccb200_ctx::scratch_done */
static void scratch_enter(eccb200_ctx *ctx, cudaStream_t st)
{
	if (ctx->scratch_used) cudaStreamWaitEvent(st, ctx->scratch_done, 0);
}
static void scratch_leave(eccb200_ctx *ctx, cudaStream_t st)
{
	cudaEventRecord(ctx->scratch_done, st);
	ctx->scratch_used = true;
}

/* The 256-, 384- and 512-bit curves read and write their wire fields with 16-byte vector accesses (load_wire /
 * store_wire): caller-supplied device (or zero-copy host) buffers must be 16-byte aligned there. */
static bool misaligned16(const eccb200_ctx *ctx, std::initializer_list<const void *> ptrs)
{
	if (ctx->plen % 16) return false; /* byte-granular loaders */
	for (const void *p : ptrs)
		if (p && ((uintptr_t)p & 15)) return true;
	return false;
}
static const char *kAlignMsg = "buffer not 16-byte aligned (required for the 256/384/512-bit curves' vector accesses)";

/* waits until flags[i] >= value for i < count (flags in this GPU's memory, written by peers; wrap-safe compare) */
__global__ void k_flag_wait(const uint32_t *flags, int count, uint32_t value)
{
	for (int i = threadIdx.x; i < count; i += blockDim.x)
		while ((int32_t)(ld_acquire_sys(flags + i) - value) < 0) __nanosleep(200);
}

struct FlagList {
	uint32_t *p[ECC_MAX_GATHER_DST];
};
/* publishes value to up to ECC_MAX_GATHER_DST (peer-mapped) flags; everything earlier in the stream is visible first */
__global__ void k_flag_signal(FlagList fl, int count, uint32_t value)
{
	__threadfence_system();
	if ((int)threadIdx.x < count) st_release_sys(fl.p[threadIdx.x], value);
}

static int smul_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_scalars, const uint8_t *d_points, uint8_t *d_out,
		    int8_t *d_status, uint32_t *jac, uint32_t *prefix, cudaStream_t st, cudaEvent_t after_smul = nullptr,
		    cudaStream_t st_norm = nullptr, cudaEvent_t after_norm = nullptr, const GatherDst *gd = nullptr,
		    const uint32_t *d_wait_flags = nullptr, int wait_count = 0, uint32_t wait_value = 0)
{
	/* Pipeline form (after_smul / st_norm / after_norm given): the normalisation runs on a highest-priority stream
	 * behind the scalar multiplication, so the NEXT chunk's scalar multiplication (which only waits for after_smul)
	 * overlaps its latency-bound inversion without delaying it; `st` resumes (for the D2H) after after_norm. */
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		const bool own_scratch = jac == ctx->jac;
		if (own_scratch) scratch_enter(ctx, st);
		const bool prof = ctx->profiling && own_scratch && ctx->ev_calls < eccb200_ctx::kProfCalls;
		cudaEvent_t *pe = prof ? ctx->ev[ctx->ev_calls] : nullptr;
		if (prof) cudaEventRecord(pe[0], st);
		if (d_points)
			LaunchVar<C>::var(n, d_scalars, d_points, jac, d_status, st);
		else if (tma_staging_enabled())
			LaunchFixed<C>::fixed_tma(n, d_scalars, ctx->table, ctx->w, jac, d_status, st);
		else
			LaunchFixed<C>::fixed(n, d_scalars, ctx->table, ctx->w, jac, d_status, st);
		if (prof) cudaEventRecord(pe[1], st);
		if (after_smul) cudaEventRecord(after_smul, st);
		if (st_norm && after_smul && after_norm) {
			cudaStreamWaitEvent(st_norm, after_smul, 0);
			LaunchMisc<C>::to_affine(affine_grid(ctx, n, true), n, jac, prefix, d_out, d_status, st_norm);
			cudaEventRecord(after_norm, st_norm);
			cudaStreamWaitEvent(st, after_norm, 0);
		} else {
			/* multi-GPU gather: the destination's consumer must have released the buffer (ack flag) before K4 stores
			 * into it; K1 above does not wait */
			if (d_wait_flags && wait_count > 0) {
				k_flag_wait<<<1, 32, 0, st>>>(d_wait_flags, wait_count, wait_value);
				ctx->launches += 1;
			}
			LaunchMisc<C>::to_affine(affine_grid(ctx, n), n, jac, prefix, d_out, d_status, st, gd);
		}
		if (prof) {
			cudaEventRecord(pe[2], st);
			ctx->ev_kernels[ctx->ev_calls++] = 2;
		}
		if (own_scratch) scratch_leave(ctx, st);
		ctx->launches += 2;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_prj_pt_mul_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_scalars,
					    const uint8_t *d_points, uint8_t *d_out, int8_t *d_status, void *stream)
{
	if (!ctx || (n && (!d_scalars || !d_out || !d_status))) return fail("null argument");
	if (misaligned16(ctx, { d_scalars, d_points, d_out })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	return smul_dev(ctx, n, d_scalars, d_points, d_out, d_status, ctx->jac, ctx->prefix, (cudaStream_t)stream);
}

/* ------------------------------------------------------------------------------------------ multi-GPU result gather */

extern "C" int eccb200_ipc_alloc(eccb200_ctx *ctx, size_t bytes, void **d_ptr, uint8_t handle[64])
{
	if (!ctx || !d_ptr || !handle || bytes == 0) return fail("bad argument");
	static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
	CUDA_OK(cudaSetDevice(ctx->device));
	void *p = nullptr;
	CUDA_OK(cudaMalloc(&p, bytes));
	if (cudaMemset(p, 0, bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
		cudaFree(p);
		return fail("cudaMemset of the IPC allocation failed");
	}
	cudaIpcMemHandle_t h;
	cudaError_t e = cudaIpcGetMemHandle(&h, p);
	if (e != cudaSuccess) {
		cudaFree(p);
		return fail(std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e));
	}
	memcpy(handle, &h, 64);
	*d_ptr = p;
	return 0;
}

extern "C" int eccb200_ipc_open(eccb200_ctx *ctx, const uint8_t handle[64], void **d_ptr)
{
	if (!ctx || !d_ptr || !handle) return fail("bad argument");
	CUDA_OK(cudaSetDevice(ctx->device));
	cudaIpcMemHandle_t h;
	memcpy(&h, handle, 64);
	CUDA_OK(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
	return 0;
}

extern "C" int eccb200_ipc_close(eccb200_ctx *ctx, void *d_ptr)
{
	if (!ctx || !d_ptr) return fail("bad argument");
	CUDA_OK(cudaSetDevice(ctx->device));
	CUDA_OK(cudaIpcCloseMemHandle(d_ptr));
	return 0;
}

extern "C" int eccb200_ipc_free(eccb200_ctx *ctx, void *d_ptr)
{
	if (!ctx || !d_ptr) return fail("bad argument");
	CUDA_OK(cudaSetDevice(ctx->device));
	CUDA_OK(cudaFree(d_ptr));
	return 0;
}

/*
 * Sliced form of smul_dev for the multi-GPU gather: the batch is cut into the pipeline's four-wave slices; slice c's
 * scalar multiplication runs on the caller's stream and its normalisation — the kernel whose stores travel to the
 * peers — on the context's high-priority stream behind it, so the NVLink traffic of slice c overlaps the arithmetic of
 * slice c + 1 instead of arriving at the destination in one burst at the end of the step (eight GPUs storing 68 MB
 * each into one root would otherwise queue on the root's NVLink ingress).  The arrival flags are published by the
 * last slice's normalisation; the caller's stream then waits for it.
 */
static int smul_dev_sliced(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_scalars, const uint8_t *d_points,
			   uint8_t *d_out, int8_t *d_status, cudaStream_t st, const GatherDst *gd,
			   const uint32_t *d_wait_flags, int wait_count, uint32_t wait_value, uint32_t slice)
{
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		constexpr size_t QL = C::QLEN, PL2 = 2 * (size_t)C::PLEN, JW = 3 * (size_t)C::N;
		cudaStream_t H = ctx->hi[0];
		scratch_enter(ctx, st);
		const bool prof = ctx->profiling && ctx->ev_calls < eccb200_ctx::kProfCalls;
		cudaEvent_t *pe = prof ? ctx->ev[ctx->ev_calls] : nullptr;
		if (prof) cudaEventRecord(pe[0], st);
		uint32_t idx = 0;
		for (uint32_t lo = 0; lo < n; lo += slice, idx++) {
			const uint32_t cnt = std::min(slice, n - lo);
			const bool last = lo + cnt >= n;
			uint32_t *jac = ctx->jac + (size_t)lo * JW;
			if (d_points)
				LaunchVar<C>::var(cnt, d_scalars + lo * QL, d_points + lo * PL2, jac, d_status + lo, st);
			else
				LaunchFixed<C>::fixed(cnt, d_scalars + lo * QL, ctx->table, ctx->w, jac, d_status + lo, st);
			cudaEvent_t ev = ctx->kdone[idx % kStages];
			cudaEventRecord(ev, st);
			cudaStreamWaitEvent(H, ev, 0);
			if (idx == 0 && d_wait_flags && wait_count > 0) {
				k_flag_wait<<<1, 32, 0, H>>>(d_wait_flags, wait_count, wait_value);
				ctx->launches += 1;
			}
			GatherDst g = gd ? *gd : GatherDst();
			for (int j = 0; j < g.n; j++) {
				g.out[j] += lo * PL2;
				g.status[j] += lo;
			}
			g.signal = last ? 1 : 0;
			LaunchMisc<C>::to_affine(affine_grid(ctx, cnt, true), cnt, jac, ctx->prefix + (size_t)lo * C::N, d_out + lo * PL2,
						 d_status + lo, H, &g);
			ctx->launches += 2;
		}
		if (prof) cudaEventRecord(pe[1], st); /* scalar multiplications done (the normalisations overlap them) */
		cudaEventRecord(ctx->ndone[0], H);
		cudaStreamWaitEvent(st, ctx->ndone[0], 0);
		if (prof) {
			cudaEventRecord(pe[2], st);
			ctx->ev_kernels[ctx->ev_calls++] = 2;
		}
		scratch_leave(ctx, st);
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

/* slices per gather call: ECCB200_GATHER_SLICE_WAVES waves of the fixed-base kernel each (default: the pipeline's
 * chunk, four waves); 0 = one slice (the whole batch, normalisation behind the scalar multiplication on one stream) */
static uint32_t gather_slice(const eccb200_ctx *ctx)
{
	static int waves = -1;
	if (waves < 0) {
		const char *e = getenv("ECCB200_GATHER_SLICE_WAVES");
		waves = e ? atoi(e) : 4;
		if (waves < 0 || waves > 64) waves = 4;
	}
	return waves ? (uint32_t)waves * ctx->wave : 0u;
}

extern "C" int eccb200_prj_pt_mul_batch_dev_gather(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_scalars,
						   const uint8_t *d_points, uint8_t *d_out, int8_t *d_status, int n_dst,
						   uint8_t *const *dst_out, int8_t *const *dst_status,
						   uint32_t *const *dst_flag, uint32_t flag_value,
						   const uint32_t *d_wait_flags, int wait_count, uint32_t wait_value,
						   void *stream)
{
	if (!ctx || (n && (!d_scalars || !d_out || !d_status))) return fail("null argument");
	if (n_dst < 0 || n_dst > ECC_MAX_GATHER_DST || (n_dst && (!dst_out || !dst_status || !dst_flag)))
		return fail("bad destination list");
	if (n == 0) return fail("empty batch: the gather signals arrival from the normalisation kernel");
	if (misaligned16(ctx, { d_scalars, d_points, d_out })) return fail(kAlignMsg);
	GatherDst gd;
	gd.n = n_dst;
	for (int j = 0; j < n_dst; j++) {
		if (!dst_out[j] || !dst_status[j] || !dst_flag[j]) return fail("null destination");
		if (misaligned16(ctx, { dst_out[j] })) return fail(kAlignMsg);
		gd.out[j] = dst_out[j];
		gd.status[j] = dst_status[j];
		gd.flag[j] = dst_flag[j];
	}
	gd.flag_value = flag_value;
	gd.counter = ctx->gather_counter;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	const uint32_t slice = gather_slice(ctx);
	if (slice && n > slice)
		return smul_dev_sliced(ctx, n, d_scalars, d_points, d_out, d_status, (cudaStream_t)stream,
				       n_dst ? &gd : nullptr, d_wait_flags, wait_count, wait_value, slice);
	return smul_dev(ctx, n, d_scalars, d_points, d_out, d_status, ctx->jac, ctx->prefix, (cudaStream_t)stream, nullptr,
			nullptr, nullptr, n_dst ? &gd : nullptr, d_wait_flags, wait_count, wait_value);
}

/*
 * Copy-engine form of the gather: push `bytes` of local results to up to ECC_MAX_GATHER_DST peer-mapped buffers with
 * DMA transfers (cudaMemcpyAsync on peer pointers: NVLink, no SM involved) on `stream`, then publish flag_value to the
 * destinations' arrival flags.  If wait_count > 0 the transfers first wait for the destinations' acknowledgements
 * (flags in this GPU's memory).  The caller orders `stream` behind the kernels that produce `d_src` (an event).
 */
extern "C" int eccb200_push_results(eccb200_ctx *ctx, int n_dst, void *const *dst, const void *d_src, size_t bytes,
				    uint32_t *const *dst_flag, uint32_t flag_value, const uint32_t *d_wait_flags,
				    int wait_count, uint32_t wait_value, void *stream)
{
	if (!ctx || !d_src || n_dst <= 0 || n_dst > ECC_MAX_GATHER_DST || !dst || !dst_flag) return fail("bad argument");
	CUDA_OK(cudaSetDevice(ctx->device));
	cudaStream_t st = (cudaStream_t)stream;
	if (d_wait_flags && wait_count > 0) {
		k_flag_wait<<<1, 32, 0, st>>>(d_wait_flags, wait_count, wait_value);
		ctx->launches += 1;
	}
	FlagList fl;
	for (int j = 0; j < n_dst; j++) {
		if (!dst[j] || !dst_flag[j]) return fail("null destination");
		CUDA_OK(cudaMemcpyAsync(dst[j], d_src, bytes, cudaMemcpyDeviceToDevice, st));
		fl.p[j] = dst_flag[j];
	}
	k_flag_signal<<<1, 32, 0, st>>>(fl, n_dst, flag_value);
	ctx->launches += 1;
	CUDA_OK(cudaGetLastError());
	return 0;
}

extern "C" int eccb200_flag_wait(eccb200_ctx *ctx, const uint32_t *d_flags, int count, uint32_t value, void *stream)
{
	if (!ctx || !d_flags || count <= 0 || count > 1024) return fail("bad argument");
	CUDA_OK(cudaSetDevice(ctx->device));
	k_flag_wait<<<1, 32, 0, (cudaStream_t)stream>>>(d_flags, count, value);
	ctx->launches += 1;
	CUDA_OK(cudaGetLastError());
	return 0;
}

extern "C" int eccb200_flag_signal(eccb200_ctx *ctx, uint32_t *const *d_flags, int count, uint32_t value, void *stream)
{
	if (!ctx || !d_flags || count <= 0 || count > ECC_MAX_GATHER_DST) return fail("bad argument");
	CUDA_OK(cudaSetDevice(ctx->device));
	FlagList fl;
	for (int i = 0; i < count; i++) fl.p[i] = d_flags[i];
	k_flag_signal<<<1, 32, 0, (cudaStream_t)stream>>>(fl, count, value);
	ctx->launches += 1;
	CUDA_OK(cudaGetLastError());
	return 0;
}

static int verify_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
		      const uint8_t *d_digests, uint32_t hlen, int8_t *d_verdict, cudaStream_t st,
		      const int8_t *d_key_state = nullptr)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		bool staged = false; /* calls made by the host-pointer pipeline are not timed */
		for (int s = 0; s < kStages; s++) staged = staged || d_verdict == (int8_t *)ctx->d_out[s];
		const bool prof = ctx->profiling && !staged && ctx->ev_calls < eccb200_ctx::kProfCalls;
		cudaEvent_t *pe = prof ? ctx->ev[ctx->ev_calls] : nullptr;
		if (prof) cudaEventRecord(pe[0], st);
		LaunchVerify<C>::verify(n, d_sigs, d_pubkeys, d_digests, hlen, ctx->table, ctx->w, d_verdict, st, d_key_state);
		if (prof) {
			cudaEventRecord(pe[1], st);
			ctx->ev_kernels[ctx->ev_calls++] = 1;
		}
		ctx->launches += 1;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_ecdsa_verify_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs,
					      const uint8_t *d_pubkeys, const uint8_t *d_digests, uint32_t hlen,
					      int8_t *d_verdict, void *stream)
{
	if (!ctx || (n && (!d_sigs || !d_pubkeys || !d_digests || !d_verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (misaligned16(ctx, { d_sigs, d_pubkeys })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	return verify_dev(ctx, n, d_sigs, d_pubkeys, d_digests, hlen, d_verdict, (cudaStream_t)stream);
}

static int recover_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_digests, uint32_t hlen,
		       uint8_t *d_keys, int8_t *d_status, cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		LaunchVerify<C>::recover(n, d_sigs, d_digests, hlen, ctx->table, ctx->w, d_keys, d_status, st);
		ctx->launches += 1;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_ecdsa_recover_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs,
					       const uint8_t *d_digests, uint32_t hlen, uint8_t *d_keys, int8_t *d_status,
					       void *stream)
{
	if (!ctx || (n && (!d_sigs || !d_digests || !d_keys || !d_status))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (misaligned16(ctx, { d_sigs, d_keys })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	return recover_dev(ctx, n, d_sigs, d_digests, hlen, d_keys, d_status, (cudaStream_t)stream);
}

static int ecfsdsa_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
		       const uint8_t *d_digests, uint32_t hlen, int8_t *d_verdict, cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		LaunchVerify<C>::ecfsdsa(n, d_sigs, d_pubkeys, d_digests, hlen, ctx->table, ctx->w, d_verdict, st);
		ctx->launches += 1;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_ecfsdsa_verify_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs,
						  const uint8_t *d_pubkeys, const uint8_t *d_digests, uint32_t hlen,
						  int8_t *d_verdict, void *stream)
{
	if (!ctx || (n && (!d_sigs || !d_pubkeys || !d_digests || !d_verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (misaligned16(ctx, { d_sigs, d_pubkeys })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	return ecfsdsa_dev(ctx, n, d_sigs, d_pubkeys, d_digests, hlen, d_verdict, (cudaStream_t)stream);
}

static int double_smul_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_ab, const uint8_t *d_pubkeys, uint8_t *d_out,
			   int8_t *d_status, cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		LaunchVerify<C>::double_smul(n, d_ab, d_pubkeys, ctx->table, ctx->w, d_out, d_status, st);
		ctx->launches += 1;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_double_smul_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_ab, const uint8_t *d_pubkeys,
					       uint8_t *d_out, int8_t *d_status, void *stream)
{
	if (!ctx || (n && (!d_ab || !d_pubkeys || !d_out || !d_status))) return fail("null argument");
	if (misaligned16(ctx, { d_ab, d_pubkeys, d_out })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	return double_smul_dev(ctx, n, d_ab, d_pubkeys, d_out, d_status, (cudaStream_t)stream);
}

static int bip0340_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
		       const uint8_t *d_digests, uint32_t hlen, int8_t *d_verdict, cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		LaunchVerify<C>::bip0340(n, d_sigs, d_pubkeys, d_digests, hlen, ctx->table, ctx->w, d_verdict, st);
		ctx->launches += 1;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_bip0340_verify_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs,
						  const uint8_t *d_pubkeys, const uint8_t *d_digests, uint32_t hlen,
						  int8_t *d_verdict, void *stream)
{
	if (!ctx || (n && (!d_sigs || !d_pubkeys || !d_digests || !d_verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (misaligned16(ctx, { d_sigs, d_pubkeys })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	return bip0340_dev(ctx, n, d_sigs, d_pubkeys, d_digests, hlen, d_verdict, (cudaStream_t)stream);
}

/* ------------------------------------------------------------------------------------------ host-pointer API */

static int ensure_stages(eccb200_ctx *ctx, size_t in_bytes, size_t out_bytes)
{
	if (in_bytes <= ctx->stage_in_bytes && out_bytes <= ctx->stage_out_bytes && ctx->stage_jac[0]) return 0;
	size_t ib = std::max(in_bytes, ctx->stage_in_bytes), ob = std::max(out_bytes, ctx->stage_out_bytes);
	/* nothing may still be using the buffers that are about to be replaced; and until the reallocation has fully
	 * succeeded the recorded sizes are zero, so that a later, smaller call cannot pass the size check on null pointers */
	CUDA_OK(cudaDeviceSynchronize());
	ctx->stage_in_bytes = ctx->stage_out_bytes = 0;
	for (int s = 0; s < kStages; s++) {
		if (ctx->h_in[s]) cudaFreeHost(ctx->h_in[s]);
		if (ctx->h_out[s]) cudaFreeHost(ctx->h_out[s]);
		if (ctx->d_in[s]) cudaFree(ctx->d_in[s]);
		if (ctx->d_out[s]) cudaFree(ctx->d_out[s]);
		ctx->h_in[s] = ctx->h_out[s] = ctx->d_in[s] = ctx->d_out[s] = nullptr;
		CUDA_OK(cudaMallocHost(&ctx->h_in[s], ib));
		CUDA_OK(cudaMallocHost(&ctx->h_out[s], ob));
		CUDA_OK(cudaMalloc(&ctx->d_in[s], ib));
		CUDA_OK(cudaMalloc(&ctx->d_out[s], ob));
		if (!ctx->stage_jac[s]) {
			CUDA_OK(cudaMalloc(&ctx->stage_jac[s], (size_t)ctx->chunk * 3 * ctx->N * sizeof(uint32_t)));
			CUDA_OK(cudaMalloc(&ctx->stage_prefix[s], (size_t)ctx->chunk * ctx->N * sizeof(uint32_t)));
			CUDA_OK(cudaMalloc(&ctx->stage_aff[s], (size_t)ctx->chunk * 2 * ctx->plen));
			CUDA_OK(cudaMalloc(&ctx->stage_state[s], (size_t)ctx->chunk));
		}
	}
	ctx->stage_in_bytes = ib;
	ctx->stage_out_bytes = ob;
	return 0;
}

/* One array of fixed-size records on the host side of a batch call. */
struct HostCol {
	uint8_t *host;   /* caller's buffer (inputs are only read) */
	size_t item;     /* bytes per item */
	bool pinned;     /* page-locked (cudaHostAlloc / cudaHostRegister / eccb200_host_alloc): DMA straight from/to it */
};

static bool is_pinned(const void *p)
{
	cudaPointerAttributes at;
	if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
		cudaGetLastError();
		return false;
	}
	return at.type == cudaMemoryTypeHost;
}

/*
 * Chunked, multi-stream pipeline of the host-pointer entry points.  Chunk c uses stage c % kStages:
 *   H2D of the chunk's input columns -> kernels -> D2H of its output columns, all on the stage's stream, so the
 *   copies of one chunk overlap the kernels of the others.  In the stage buffers the columns of a chunk are stored
 *   one after the other ([cnt][item0], [cnt][item1], ...), every item size except possibly the last input column's
 *   being a multiple of 16 bytes, which keeps each column 16-byte aligned for the kernels' vector loads.
 * Page-locked caller buffers are copied directly by the DMA engines; pageable ones go through the context's pinned
 * staging buffers (one extra memcpy each way).
 */
template <class Launch>
static int run_pipeline_body(eccb200_ctx *ctx, uint32_t n, std::vector<HostCol> &in, std::vector<HostCol> &out,
			     Launch launch, bool ordered);

/*
 * Chunk boundaries of the host pipeline.
 *  - unordered pipelines (the long K2 / K3 kernels): equal chunks of four waves;
 *  - ordered ones (fixed base: short kernels, the copies are what shows): the chunk sizes ramp up 1, 2, 4 (, 8) waves so
 *    that the first kernel starts after a 2.4 MB copy instead of a 9.7 MB one, run at four waves (eight for batches
 *    beyond 64 waves: fewer per-chunk gaps) and ramp down 2, 1 so that the last device->host copy is short.
 * With a Fermat inversion in K4 every extra chunk would expose that long serial chain; the safegcd inversion keeps it
 * short, so the shaping pays (DESIGN.md §7).  ECCB200_PIPE_SHAPE=0 restores equal chunks.
 */
static std::vector<uint32_t> chunk_bounds(uint32_t n, uint32_t w, uint32_t chunk_eq, uint32_t capacity, bool shaped)
{
	std::vector<uint32_t> bounds{ 0 };
	if (!shaped || n <= 2 * w) {
		for (uint32_t lo = 0; lo < n;) {
			lo += std::min(chunk_eq, n - lo);
			bounds.push_back(lo);
		}
		return bounds;
	}
	const uint32_t maxw = std::min<uint32_t>(capacity / w, (n / w >= 64) ? 8u : 4u);
	uint32_t lo = 0;
	auto push = [&](uint32_t cnt) {
		lo += cnt;
		bounds.push_back(lo);
	};
	for (uint32_t u = 1; u < maxw && (uint64_t)(n - lo) > (uint64_t)(u + 3) * w; u *= 2) push(u * w); /* ramp up */
	while ((uint64_t)(n - lo) > (uint64_t)(maxw + 3) * w) push(maxw * w);                                /* steady state */
	if (n - lo > 3 * w) push(n - lo - 3 * w);                                                             /* ramp down */
	if (n - lo > w) push(n - lo - w);
	if (n - lo > 0) push(n - lo);
	return bounds;
}

static std::vector<uint32_t> pipeline_bounds(const eccb200_ctx *ctx, uint32_t n, bool ordered)
{
	static const bool shape = !(getenv("ECCB200_PIPE_SHAPE") && atoi(getenv("ECCB200_PIPE_SHAPE")) == 0);
	return chunk_bounds(n, ctx->wave, ctx->chunk_eq, ctx->chunk, ordered && shape);
}

/* The chunking rule as a pure function (host logic, testable without a GPU): writes at most cap boundaries
 * (0 = b[0] < b[1] < ... = n) and returns how many there are. */
extern "C" int eccb200_pipeline_chunk_bounds(uint32_t n, uint32_t wave_items, uint32_t equal_chunk_items,
					     uint32_t capacity_items, int shaped, uint32_t *bounds, int cap)
{
	if (!bounds || cap < 2 || wave_items == 0 || equal_chunk_items == 0 || capacity_items < wave_items)
		return fail("bad argument");
	const std::vector<uint32_t> b = chunk_bounds(n, wave_items, equal_chunk_items, capacity_items, shaped != 0);
	for (size_t i = 0; i < b.size() && (int)i < cap; i++) bounds[i] = b[i];
	return (int)b.size();
}

template <class Launch>
static int run_pipeline(eccb200_ctx *ctx, uint32_t n, std::vector<HostCol> &in, std::vector<HostCol> &out,
			Launch launch, bool ordered = false)
{
	const int rc = run_pipeline_body(ctx, n, in, out, launch, ordered);
	if (rc) {
		/* a failed enqueue leaves copies into the caller's buffers and kernels on the stage buffers in flight: drain
		 * every stream before the caller may free its memory or the next call reshapes the stages */
		const std::string keep = g_err;
		for (int s = 0; s < kStages; s++) {
			if (ctx->streams[s]) cudaStreamSynchronize(ctx->streams[s]);
			if (ctx->hi[s]) cudaStreamSynchronize(ctx->hi[s]);
		}
		cudaGetLastError();
		g_err = keep;
	}
	return rc;
}

template <class Launch>
static int run_pipeline_body(eccb200_ctx *ctx, uint32_t n, std::vector<HostCol> &in, std::vector<HostCol> &out,
			     Launch launch, bool ordered)
{
	/* ordered: the chunks' kernels run in chunk order (event chain).  Right for the short fixed-base kernels, whose
	 * D2H must overlap the next chunk's arithmetic; wrong for the long K2 / K3 launches, where letting the next chunk's
	 * CTAs fill the tail of the previous one is worth more (chosen on the previous GPU target and not re-measured on H100). */
	CUDA_OK(cudaSetDevice(ctx->device));
	size_t in_item = 0, out_item = 0;
	for (auto &c : in) {
		in_item += c.item;
		c.pinned = is_pinned(c.host);
	}
	for (auto &c : out) {
		out_item += c.item;
		c.pinned = is_pinned(c.host);
	}
	const uint32_t kChunk = ctx->chunk;
	if (ensure_stages(ctx, (size_t)kChunk * in_item, (size_t)kChunk * out_item)) return -1;
	const std::vector<uint32_t> bounds = pipeline_bounds(ctx, n, ordered);
	const uint32_t nchunks = (uint32_t)bounds.size() - 1;
	bool all_pinned = true;
	for (auto &c : in) all_pinned = all_pinned && c.pinned;
	for (auto &c : out) all_pinned = all_pinned && c.pinned;
	if (all_pinned) {
		/* No host-side staging: enqueue every chunk without a single host synchronisation.  Stage buffers are
		 * reused by chunk c + kStages on the SAME stream, so stream order alone keeps them safe.
		 * ECCB200_PIPE_TRACE=1 records an event after each phase of each chunk and prints the timeline
		 * (diagnostic for DESIGN.md §7; the events cost a few microseconds per chunk). */
		static const bool trace = getenv("ECCB200_PIPE_TRACE") && atoi(getenv("ECCB200_PIPE_TRACE")) != 0;
		std::vector<cudaEvent_t> ev;
		if (trace) {
			ev.resize((size_t)nchunks * 4);
			for (auto &e : ev) CUDA_OK(cudaEventCreate(&e));
		}
		for (uint32_t c = 0; c < nchunks; c++) {
			int s = (int)(c % kStages);
			uint32_t lo = bounds[c], cnt = bounds[c + 1] - lo;
			size_t off = 0;
			if (trace) cudaEventRecord(ev[4 * c + 0], ctx->streams[s]);
			for (auto &col : in) {
				size_t bytes = (size_t)cnt * col.item;
				CUDA_OK(cudaMemcpyAsync(ctx->d_in[s] + off, col.host + (size_t)lo * col.item, bytes,
							cudaMemcpyHostToDevice, ctx->streams[s]));
				off += bytes;
			}
			if (trace) cudaEventRecord(ev[4 * c + 1], ctx->streams[s]);
			/* kernels run in chunk order: without this the block scheduler interleaves the CTAs of the chunks
			 * queued on the other streams, every chunk finishes late and no D2H overlaps the arithmetic */
			if (ordered && c > 0) CUDA_OK(cudaStreamWaitEvent(ctx->streams[s], ctx->kdone[(c - 1) % kStages], 0));
			ctx->kdone_set = false;
			if (launch(s, cnt)) return -1;
			if (!ctx->kdone_set) CUDA_OK(cudaEventRecord(ctx->kdone[s], ctx->streams[s]));
			if (trace) cudaEventRecord(ev[4 * c + 2], ctx->streams[s]);
			off = 0;
			for (auto &col : out) {
				size_t bytes = (size_t)cnt * col.item;
				CUDA_OK(cudaMemcpyAsync(col.host + (size_t)lo * col.item, ctx->d_out[s] + off, bytes,
							cudaMemcpyDeviceToHost, ctx->streams[s]));
				off += bytes;
			}
			if (trace) cudaEventRecord(ev[4 * c + 3], ctx->streams[s]);
		}
		for (int s = 0; s < kStages; s++) CUDA_OK(cudaStreamSynchronize(ctx->streams[s]));
		if (trace) {
			fprintf(stderr, "[eccb200 pipe] n=%u chunk=%u: per chunk, ms since the first copy was enqueued: "
					"h2d_start h2d_end kernels_end d2h_end\n", n, kChunk);
			for (uint32_t c = 0; c < nchunks; c++) {
				float t[4];
				for (int k = 0; k < 4; k++) cudaEventElapsedTime(&t[k], ev[0], ev[4 * c + k]);
				fprintf(stderr, "[eccb200 pipe]   chunk %u (stream %u): %.3f %.3f %.3f %.3f\n", c, c % kStages, t[0], t[1],
					t[2], t[3]);
			}
			for (auto &e : ev) cudaEventDestroy(e);
		}
		return 0;
	}
	std::vector<uint32_t> pending_lo(kStages, 0), pending_cnt(kStages, 0);
	for (uint32_t c = 0; c < nchunks + kStages; c++) {
		int s = (int)(c % kStages);
		if (pending_cnt[s]) { /* retire what this stage was doing */
			CUDA_OK(cudaStreamSynchronize(ctx->streams[s]));
			size_t off = 0;
			for (auto &col : out) {
				if (!col.pinned)
					memcpy(col.host + (size_t)pending_lo[s] * col.item, ctx->h_out[s] + off,
					       (size_t)pending_cnt[s] * col.item);
				off += (size_t)pending_cnt[s] * col.item;
			}
			pending_cnt[s] = 0;
		}
		if (c >= nchunks) continue;
		uint32_t lo = bounds[c], cnt = bounds[c + 1] - lo;
		size_t off = 0;
		for (auto &col : in) {
			const uint8_t *src = col.host + (size_t)lo * col.item;
			size_t bytes = (size_t)cnt * col.item;
			if (!col.pinned) {
				memcpy(ctx->h_in[s] + off, src, bytes);
				src = ctx->h_in[s] + off;
			}
			CUDA_OK(cudaMemcpyAsync(ctx->d_in[s] + off, src, bytes, cudaMemcpyHostToDevice, ctx->streams[s]));
			off += bytes;
		}
		if (ordered && c > 0) CUDA_OK(cudaStreamWaitEvent(ctx->streams[s], ctx->kdone[(c - 1) % kStages], 0));
		ctx->kdone_set = false;
		if (launch(s, cnt)) return -1;
		if (!ctx->kdone_set) CUDA_OK(cudaEventRecord(ctx->kdone[s], ctx->streams[s]));
		off = 0;
		for (auto &col : out) {
			size_t bytes = (size_t)cnt * col.item;
			uint8_t *dst = col.pinned ? col.host + (size_t)lo * col.item : ctx->h_out[s] + off;
			CUDA_OK(cudaMemcpyAsync(dst, ctx->d_out[s] + off, bytes, cudaMemcpyDeviceToHost, ctx->streams[s]));
			off += bytes;
		}
		pending_lo[s] = lo;
		pending_cnt[s] = cnt;
	}
	return 0;
}

/* Page-locked buffers are visible to the device through unified addressing: with ECCB200_ZEROCOPY=1 the kernels read
 * their operands from, and write their results to, the caller's host memory directly, so the PCIe traffic overlaps
 * the arithmetic warp by warp and no staging copy or copy-engine transfer is issued at all. */
static bool zero_copy_enabled()
{
	static int v = -1;
	if (v < 0) {
		const char *e = getenv("ECCB200_ZEROCOPY");
		v = (e && atoi(e) != 0) ? 1 : 0;
	}
	return v == 1;
}

extern "C" int eccb200_prj_pt_mul_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *scalars, const uint8_t *points,
					uint8_t *out, int8_t *status)
{
	if (!ctx || (n && (!scalars || !out || !status))) return fail("null argument");
	if (n == 0) return 0;
	if (zero_copy_enabled() && is_pinned(scalars) && is_pinned(out) && is_pinned(status) &&
	    (!points || is_pinned(points))) {
		if (misaligned16(ctx, { scalars, points, out })) return fail(kAlignMsg);
		CUDA_OK(cudaSetDevice(ctx->device));
		if (ensure_work(ctx, n)) return -1;
		if (smul_dev(ctx, n, scalars, points, out, status, ctx->jac, ctx->prefix, ctx->streams[0])) return -1;
		CUDA_OK(cudaStreamSynchronize(ctx->streams[0]));
		return 0;
	}
	const size_t sl = ctx->qlen, pl = 2 * (size_t)ctx->plen;
	std::vector<HostCol> in = { { (uint8_t *)scalars, sl, false } };
	if (points) in.push_back({ (uint8_t *)points, pl, false });
	std::vector<HostCol> outc = { { out, pl, false }, { (uint8_t *)status, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d_sc = ctx->d_in[s];
		const uint8_t *d_pt = points ? ctx->d_in[s] + (size_t)cnt * sl : nullptr;
		uint8_t *d_o = ctx->d_out[s];
		int8_t *d_st = (int8_t *)(ctx->d_out[s] + (size_t)cnt * pl);
		if (points) /* variable base: one long kernel per chunk, left unordered (see run_pipeline) */
			return smul_dev(ctx, cnt, d_sc, d_pt, d_o, d_st, ctx->stage_jac[s], ctx->stage_prefix[s],
					ctx->streams[s]);
		/* Where the normalisation of a chunk runs (DESIGN.md §7): on the chunk's own stream behind K1, the next chunk's
		 * K1 waiting for it, or on a high-priority side stream under the next chunk's K1.  The first wins while the batch
		 * is a handful of chunks, the second once the steady state dominates; the 24-wave threshold was
		 * chosen on the previous GPU target and not re-measured on H100.  ECCB200_PIPE_K4_INLINE=0/1 forces one. */
		static const int k4_force = getenv("ECCB200_PIPE_K4_INLINE") ? atoi(getenv("ECCB200_PIPE_K4_INLINE")) : -1;
		const bool k4_inline = k4_force >= 0 ? k4_force != 0 : n <= 24u * ctx->wave;
		if (k4_inline)
			return smul_dev(ctx, cnt, d_sc, d_pt, d_o, d_st, ctx->stage_jac[s], ctx->stage_prefix[s],
					ctx->streams[s]);
		ctx->kdone_set = true;
		return smul_dev(ctx, cnt, d_sc, d_pt, d_o, d_st, ctx->stage_jac[s], ctx->stage_prefix[s], ctx->streams[s],
				ctx->kdone[s], ctx->hi[s], ctx->ndone[s]);
	}, /*ordered=*/points == nullptr);
}

extern "C" int eccb200_ecdsa_verify_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
					  const uint8_t *digests, uint32_t hlen, int8_t *verdict)
{
	if (!ctx || (n && (!sigs || !pubkeys || !digests || !verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	const size_t sg = 2 * (size_t)ctx->qlen, pk = 2 * (size_t)ctx->plen;
	/* the digest column goes last: it is the only one whose item size need not be a multiple of 16 */
	std::vector<HostCol> in = { { (uint8_t *)sigs, sg, false }, { (uint8_t *)pubkeys, pk, false },
				    { (uint8_t *)digests, hlen, false } };
	std::vector<HostCol> outc = { { (uint8_t *)verdict, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		return verify_dev(ctx, cnt, d, d + (size_t)cnt * sg, d + (size_t)cnt * (sg + pk), hlen,
				  (int8_t *)ctx->d_out[s], ctx->streams[s]);
	});
}

extern "C" int eccb200_ecdsa_recover_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *digests,
					   uint32_t hlen, uint8_t *keys, int8_t *status)
{
	if (!ctx || (n && (!sigs || !digests || !keys || !status))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	const size_t sg = 2 * (size_t)ctx->qlen, kl = 4 * (size_t)ctx->plen;
	/* the digest column goes last: it is the only one whose item size need not be a multiple of 16 */
	std::vector<HostCol> in = { { (uint8_t *)sigs, sg, false }, { (uint8_t *)digests, hlen, false } };
	std::vector<HostCol> outc = { { keys, kl, false }, { (uint8_t *)status, 2, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		return recover_dev(ctx, cnt, d, d + (size_t)cnt * sg, hlen, ctx->d_out[s],
				   (int8_t *)(ctx->d_out[s] + (size_t)cnt * kl), ctx->streams[s]);
	});
}

/* With a per-key state column (0 = affine key in pubkeys[i], 1 = the key is the point at infinity, -1 = rejected): the
 * reference's ec_verify accepts an ec_pub_key whose y is the point at infinity and then computes W' = u*G
 * (prj_pt_mul on infinity gives infinity, curves/prj_pt.c:1767-1775); callers holding reference structs need it. */
extern "C" int eccb200_ecdsa_verify_keystate_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs,
						   const uint8_t *pubkeys, const int8_t *key_state,
						   const uint8_t *digests, uint32_t hlen, int8_t *verdict)
{
	if (!ctx || (n && (!sigs || !pubkeys || !key_state || !digests || !verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	const size_t sg = 2 * (size_t)ctx->qlen, pk = 2 * (size_t)ctx->plen;
	std::vector<HostCol> in = { { (uint8_t *)sigs, sg, false }, { (uint8_t *)pubkeys, pk, false },
				    { (uint8_t *)key_state, 1, false }, { (uint8_t *)digests, hlen, false } };
	std::vector<HostCol> outc = { { (uint8_t *)verdict, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		return verify_dev(ctx, cnt, d, d + (size_t)cnt * sg, d + (size_t)cnt * (sg + pk + 1), hlen,
				  (int8_t *)ctx->d_out[s], ctx->streams[s], (const int8_t *)(d + (size_t)cnt * (sg + pk)));
	});
}

/*
 * ECDSA verification with the public keys in the reference's HOMOGENEOUS PROJECTIVE form (X || Y || Z, what an
 * ec_pub_key holds: the output of a prj_pt_mul, Z != 1 in general).  Per pipeline chunk: key import + batched
 * prj_pt_unique on the device (k_prj_load + K4 mode 2, one inversion per CTA) feeding the verification kernel its
 * affine keys and key states — the keys never go back to the host.
 */
extern "C" int eccb200_ecdsa_verify_prj_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs,
					      const uint8_t *prj_pubkeys, const uint8_t *digests, uint32_t hlen,
					      int8_t *verdict)
{
	if (!ctx || (n && (!sigs || !prj_pubkeys || !digests || !verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	const size_t sg = 2 * (size_t)ctx->qlen, pk = 3 * (size_t)ctx->plen;
	std::vector<HostCol> in = { { (uint8_t *)sigs, sg, false }, { (uint8_t *)prj_pubkeys, pk, false },
				    { (uint8_t *)digests, hlen, false } };
	std::vector<HostCol> outc = { { (uint8_t *)verdict, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		cudaStream_t st = ctx->streams[s];
		/* the stage's affine scratch receives the normalised keys, its state scratch the key states (0 / 1 / -1) */
		int8_t *state = (int8_t *)ctx->stage_state[s];
		int rc = dispatch(ctx->curve_id, [&](auto c) {
			typedef decltype(c) C;
			LaunchMisc<C>::prj_unique(affine_grid(ctx, cnt), cnt, d + (size_t)cnt * sg, ctx->stage_jac[s],
						  ctx->stage_prefix[s], ctx->stage_aff[s], state, st);
			ctx->launches += 2;
			return 0;
		});
		if (rc) return rc;
		return verify_dev(ctx, cnt, d, ctx->stage_aff[s], d + (size_t)cnt * (sg + pk), hlen, (int8_t *)ctx->d_out[s], st,
				  state);
	});
}

extern "C" int eccb200_ecfsdsa_verify_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
					    const uint8_t *digests, uint32_t hlen, int8_t *verdict)
{
	if (!ctx || (n && (!sigs || !pubkeys || !digests || !verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	const size_t pk = 2 * (size_t)ctx->plen, sg = pk + (size_t)ctx->qlen;
	/* column order keeps the 16-byte-multiple items first (256/384-bit curves): keys, signatures, digests */
	std::vector<HostCol> in = { { (uint8_t *)pubkeys, pk, false }, { (uint8_t *)sigs, sg, false },
				    { (uint8_t *)digests, hlen, false } };
	std::vector<HostCol> outc = { { (uint8_t *)verdict, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		return ecfsdsa_dev(ctx, cnt, d + (size_t)cnt * pk, d, d + (size_t)cnt * (pk + sg), hlen,
				   (int8_t *)ctx->d_out[s], ctx->streams[s]);
	});
}

extern "C" int eccb200_double_smul_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *ab, const uint8_t *pubkeys,
					   uint8_t *out, int8_t *status)
{
	if (!ctx || (n && (!ab || !pubkeys || !out || !status))) return fail("null argument");
	if (n == 0) return 0;
	const size_t sc = 2 * (size_t)ctx->qlen, pk = 2 * (size_t)ctx->plen;
	std::vector<HostCol> in = { { (uint8_t *)ab, sc, false }, { (uint8_t *)pubkeys, pk, false } };
	std::vector<HostCol> outc = { { out, pk, false }, { (uint8_t *)status, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		return double_smul_dev(ctx, cnt, d, d + (size_t)cnt * sc, ctx->d_out[s],
				       (int8_t *)(ctx->d_out[s] + (size_t)cnt * pk), ctx->streams[s]);
	});
}

extern "C" int eccb200_bip0340_verify_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
					    const uint8_t *digests, uint32_t hlen, int8_t *verdict)
{
	if (!ctx || (n && (!sigs || !pubkeys || !digests || !verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	const size_t pk = 2 * (size_t)ctx->plen, sg = (size_t)ctx->plen + (size_t)ctx->qlen;
	std::vector<HostCol> in = { { (uint8_t *)pubkeys, pk, false }, { (uint8_t *)sigs, sg, false },
				    { (uint8_t *)digests, hlen, false } };
	std::vector<HostCol> outc = { { (uint8_t *)verdict, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		return bip0340_dev(ctx, cnt, d + (size_t)cnt * pk, d, d + (size_t)cnt * (pk + sg), hlen,
				   (int8_t *)ctx->d_out[s], ctx->streams[s]);
	});
}

/* ------------------------------------------------------------------------------------------ K6: batch verification as one MSM */

/* Window width of the bucket method: the c in [2, 16] that minimises (mixed additions of the accumulation) + (additions
 * and conversions of the bucket reduction), in field products; ECCB200_MSM_WINDOW overrides (tests walk small c). */
static int msm_pick_window(uint32_t n, int qbits)
{
	/* the bucket scan handles up to 2^20 buckets (1024 tiles of 1024): wide orders stop below c = 16 */
	auto fits = [&](int c) { return (uint64_t)msm_windows(qbits - 1, c) << (c - 1) <= (1u << 20); };
	if (const char *e = getenv("ECCB200_MSM_WINDOW")) {
		int c = atoi(e);
		if (c >= 2 && c <= 16) {
			while (!fits(c)) c--;
			return c;
		}
	}
	/* time ~ max(total work / threads in flight, the longest chain one thread adds up): the chain is the expected load
	 * of a bucket of the top window, which holds only t = (qbits - 1) mod c bits (msm_core.cuh) */
	int best = 2;
	double best_cost = 0;
	for (int c = 2; c <= 16 && fits(c); c++) {
		const int nw = msm_windows(qbits - 1, c), nwa = msm_windows(msm_coefficient_bits(c), c), t = (qbits - 1) % c;
		const double acc = (double)n * (nwa + nw) * 10.0;
		const double red = (double)nw * (double)(1u << (c - 1)) * (2 * 16.0 + 2.0);
		const double chain = (double)n / (double)(1u << t) * 10.0;
		const double cost = std::max((acc + red) / 65536.0, chain);
		if (c == 2 || cost < best_cost) {
			best = c;
			best_cost = cost;
		}
	}
	return best;
}

static int msm_ensure(eccb200_ctx *ctx, uint32_t n, int c)
{
	const int qbits = (int)ctx->qlen * 8; /* upper bound of bitlen(q): only sizes buffers */
	const int nwin = msm_windows(qbits - 1, c);
	const uint32_t nb = 1u << (c - 1), total = (uint32_t)nwin * nb;
	/* list: every W_i owns at most ceil(128 / c) non-zero digits, every Y_i and the generator at most nwin */
	const size_t list_need = (size_t)n * (size_t)(msm_windows(msm_coefficient_bits(c), c) + nwin) + (size_t)nwin;
	if (n <= ctx->msm_cap_n && total <= ctx->msm_cap_total && list_need <= ctx->msm_cap_list) return 0;
	const uint32_t cap_n = std::max(n, ctx->msm_cap_n), cap_total = std::max(total, ctx->msm_cap_total);
	const size_t cap_list = std::max(list_need, ctx->msm_cap_list);
	cudaDeviceSynchronize();
	msm_release(ctx);
	const size_t N = (size_t)ctx->N, npts = 2 * (size_t)cap_n + 1;
	MsmBuffers &b = ctx->msm;
	if (cudaMalloc(&b.pts, npts * 2 * N * 4) != cudaSuccess || cudaMalloc(&b.scal, npts * N * 4) != cudaSuccess ||
	    cudaMalloc(&b.partial, ((size_t)cap_n / 128 + 1) * N * 4) != cudaSuccess ||
	    cudaMalloc(&b.count, (size_t)cap_total * 4) != cudaSuccess || cudaMalloc(&b.offs, (size_t)cap_total * 4) != cudaSuccess ||
	    cudaMalloc(&b.fill, (size_t)cap_total * 4) != cudaSuccess || cudaMalloc(&b.list, cap_list * 4) != cudaSuccess ||
	    cudaMalloc(&b.buckets, (size_t)cap_total * 3 * N * 4) != cudaSuccess ||
	    cudaMalloc(&b.parts, (size_t)cap_total * 3 * N * 4) != cudaSuccess ||
	    cudaMalloc(&b.winsum, (size_t)msm_windows(qbits - 1, 2) * 3 * N * 4) != cudaSuccess ||
	    cudaMalloc(&b.order, (size_t)cap_total * 4) != cudaSuccess || cudaMalloc(&b.aux, 3072 * 4) != cudaSuccess ||
	    cudaMalloc(&b.flags, 2 * sizeof(int)) != cudaSuccess) {
		cudaGetLastError();
		msm_release(ctx);
		return fail("out of device memory for the multi-scalar-multiplication buffers");
	}
	ctx->msm_cap_n = cap_n;
	ctx->msm_cap_total = cap_total;
	ctx->msm_cap_list = cap_list;
	return 0;
}

static int msm_seed(MsmKey &key, const uint8_t *seed)
{
	uint8_t buf[32];
	if (seed) {
		memcpy(buf, seed, 32);
	} else {
		size_t got = 0;
		while (got < sizeof buf) {
			const ssize_t r = getrandom(buf + got, sizeof buf - got, 0);
			if (r <= 0) return fail("getrandom failed: no entropy for the batch coefficients");
			got += (size_t)r;
		}
	}
	for (int i = 0; i < 8; i++)
		key.k[i] = (uint32_t)buf[4 * i] | ((uint32_t)buf[4 * i + 1] << 8) | ((uint32_t)buf[4 * i + 2] << 16) |
			   ((uint32_t)buf[4 * i + 3] << 24);
	return 0;
}

static int schnorr_msm_dev(eccb200_ctx *ctx, int scheme, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
			   const uint8_t *d_digests, uint32_t hlen, const uint8_t *seed, int *all_valid, cudaStream_t st)
{
	*all_valid = 0;
	if (n == 0) return 0; /* the reference's implementations reject an empty batch (sig/ecfsdsa.c:740) */
	if (n > (1u << 26)) return fail("batch too large for one multi-scalar multiplication (2^26 signatures): split it");
	MsmKey key;
	if (msm_seed(key, seed)) return -1;
	int flags[2] = { 0, 0 };
	int rc = dispatch(ctx->curve_id, [&](auto cv) {
		typedef decltype(cv) C;
		const int c = msm_pick_window(n, C::QBITS);
		if (msm_ensure(ctx, n, c)) return -1;
		scratch_enter(ctx, st);
		const int launched = LaunchMsm<C>::verify(scheme, n, d_sigs, d_pubkeys, d_digests, hlen, key, c, ctx->msm, st);
		if (launched < 0) return fail("BIP0340 batch verification by multi-scalar multiplication needs p = 3 mod 4 (not this curve)");
		ctx->launches += (uint64_t)launched;
		CUDA_OK(cudaGetLastError());
		CUDA_OK(cudaMemcpyAsync(flags, ctx->msm.flags, sizeof flags, cudaMemcpyDeviceToHost, st));
		scratch_leave(ctx, st);
		CUDA_OK(cudaStreamSynchronize(st));
		return 0;
	});
	if (rc) return rc;
	*all_valid = flags[1] == 1 ? 1 : 0;
	return 0;
}

static int schnorr_msm_dev_checked(eccb200_ctx *ctx, int scheme, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pubkeys,
				   const uint8_t *d_digests, uint32_t hlen, const uint8_t *seed, int *all_valid, void *stream)
{
	if (!ctx || !all_valid || (n && (!d_sigs || !d_pubkeys || !d_digests))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (misaligned16(ctx, { d_sigs, d_pubkeys })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	return schnorr_msm_dev(ctx, scheme, n, d_sigs, d_pubkeys, d_digests, hlen, seed, all_valid, (cudaStream_t)stream);
}

extern "C" int eccb200_ecfsdsa_verify_msm_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs,
						      const uint8_t *d_pubkeys, const uint8_t *d_digests, uint32_t hlen,
						      const uint8_t *seed, int *all_valid, void *stream)
{
	return schnorr_msm_dev_checked(ctx, 1, n, d_sigs, d_pubkeys, d_digests, hlen, seed, all_valid, stream);
}

extern "C" int eccb200_bip0340_verify_msm_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_sigs,
						      const uint8_t *d_pubkeys, const uint8_t *d_digests, uint32_t hlen,
						      const uint8_t *seed, int *all_valid, void *stream)
{
	return schnorr_msm_dev_checked(ctx, 2, n, d_sigs, d_pubkeys, d_digests, hlen, seed, all_valid, stream);
}

static inline size_t msm_align16(size_t v) { return (v + 15) & ~(size_t)15; }

static int schnorr_msm_host(eccb200_ctx *ctx, int scheme, uint32_t n, const uint8_t *sigs, const uint8_t *pubkeys,
			    const uint8_t *digests, uint32_t hlen, const uint8_t *seed, int *all_valid)
{
	if (!ctx || !all_valid || (n && (!sigs || !pubkeys || !digests))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	*all_valid = 0;
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	const size_t pk = 2 * (size_t)ctx->plen, sg = (scheme == 2 ? (size_t)ctx->plen : pk) + (size_t)ctx->qlen;
	const size_t b_sg = msm_align16((size_t)n * sg), b_pk = msm_align16((size_t)n * pk), b_dg = msm_align16((size_t)n * hlen);
	if (ctx->msm_in_bytes < b_sg + b_pk + b_dg) {
		if (ctx->msm_in) cudaFree(ctx->msm_in);
		ctx->msm_in = nullptr;
		ctx->msm_in_bytes = 0;
		CUDA_OK(cudaMalloc(&ctx->msm_in, b_sg + b_pk + b_dg));
		ctx->msm_in_bytes = b_sg + b_pk + b_dg;
	}
	cudaStream_t st = ctx->streams[0];
	uint8_t *d = ctx->msm_in;
	CUDA_OK(cudaMemcpyAsync(d, sigs, (size_t)n * sg, cudaMemcpyHostToDevice, st));
	CUDA_OK(cudaMemcpyAsync(d + b_sg, pubkeys, (size_t)n * pk, cudaMemcpyHostToDevice, st));
	CUDA_OK(cudaMemcpyAsync(d + b_sg + b_pk, digests, (size_t)n * hlen, cudaMemcpyHostToDevice, st));
	return schnorr_msm_dev(ctx, scheme, n, d, d + b_sg, d + b_sg + b_pk, hlen, seed, all_valid, st);
}

extern "C" int eccb200_ecfsdsa_verify_msm_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs,
						  const uint8_t *pubkeys, const uint8_t *digests, uint32_t hlen,
						  const uint8_t *seed, int *all_valid)
{
	return schnorr_msm_host(ctx, 1, n, sigs, pubkeys, digests, hlen, seed, all_valid);
}

extern "C" int eccb200_bip0340_verify_msm_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs,
						  const uint8_t *pubkeys, const uint8_t *digests, uint32_t hlen,
						  const uint8_t *seed, int *all_valid)
{
	return schnorr_msm_host(ctx, 2, n, sigs, pubkeys, digests, hlen, seed, all_valid);
}

/* ------------------------------------------------------------------------------------------ sign / ECC-CDH (§8f) */

static int sign_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_priv, const uint8_t *d_nonce, const uint8_t *d_dig,
		    uint32_t hlen, uint8_t *d_sigs, int8_t *d_status, uint32_t *jac, uint32_t *prefix, uint8_t *aff,
		    cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		if (jac == ctx->jac) scratch_enter(ctx, st);
		LaunchFixed<C>::fixed(n, d_nonce, ctx->table, ctx->w, jac, d_status, st);       /* k*G          */
		LaunchMisc<C>::to_affine(affine_grid(ctx, n), n, jac, prefix, aff, d_status, st); /* affine (x, y) */
		LaunchMisc<C>::sign_finish(affine_grid(ctx, n), n, d_priv, d_nonce, d_dig, hlen, aff, prefix, d_sigs,
					   d_status, st);                                        /* r, s          */
		if (jac == ctx->jac) scratch_leave(ctx, st);
		ctx->launches += 3;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_ecdsa_sign_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_privkeys,
					    const uint8_t *d_nonces, const uint8_t *d_digests, uint32_t hlen,
					    uint8_t *d_sigs, int8_t *d_status, void *stream)
{
	if (!ctx || (n && (!d_privkeys || !d_nonces || !d_digests || !d_sigs || !d_status))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (misaligned16(ctx, { d_privkeys, d_nonces, d_sigs })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	return sign_dev(ctx, n, d_privkeys, d_nonces, d_digests, hlen, d_sigs, d_status, ctx->jac, ctx->prefix, ctx->aff,
			(cudaStream_t)stream);
}

extern "C" int eccb200_ecdsa_sign_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *privkeys, const uint8_t *nonces,
					const uint8_t *digests, uint32_t hlen, uint8_t *sigs, int8_t *status)
{
	if (!ctx || (n && (!privkeys || !nonces || !digests || !sigs || !status))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	const size_t ql = ctx->qlen;
	std::vector<HostCol> in = { { (uint8_t *)privkeys, ql, false }, { (uint8_t *)nonces, ql, false },
				    { (uint8_t *)digests, hlen, false } };
	std::vector<HostCol> outc = { { sigs, 2 * ql, false }, { (uint8_t *)status, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		return sign_dev(ctx, cnt, d, d + (size_t)cnt * ql, d + (size_t)cnt * 2 * ql, hlen, ctx->d_out[s],
				(int8_t *)(ctx->d_out[s] + (size_t)cnt * 2 * ql), ctx->stage_jac[s], ctx->stage_prefix[s],
				ctx->stage_aff[s], ctx->streams[s]);
	}, /*ordered=*/true);
}

static int ecdh_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_priv, const uint8_t *d_peers, uint8_t *d_shared,
		    int8_t *d_status, uint32_t *jac, uint32_t *prefix, cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		if (jac == ctx->jac) scratch_enter(ctx, st);
		LaunchVar<C>::var(n, d_priv, d_peers, jac, d_status, st);
		LaunchMisc<C>::to_x_only(affine_grid(ctx, n), n, jac, prefix, d_shared, d_status, st);
		if (jac == ctx->jac) scratch_leave(ctx, st);
		ctx->launches += 2;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_ecccdh_derive_batch_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_privkeys,
					       const uint8_t *d_peer_pubkeys, uint8_t *d_shared, int8_t *d_status,
					       void *stream)
{
	if (!ctx || (n && (!d_privkeys || !d_peer_pubkeys || !d_shared || !d_status))) return fail("null argument");
	if (misaligned16(ctx, { d_privkeys, d_peer_pubkeys, d_shared })) return fail(kAlignMsg);
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	return ecdh_dev(ctx, n, d_privkeys, d_peer_pubkeys, d_shared, d_status, ctx->jac, ctx->prefix,
			(cudaStream_t)stream);
}

extern "C" int eccb200_ecccdh_derive_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *privkeys,
					   const uint8_t *peer_pubkeys, uint8_t *shared, int8_t *status)
{
	if (!ctx || (n && (!privkeys || !peer_pubkeys || !shared || !status))) return fail("null argument");
	if (n == 0) return 0;
	const size_t ql = ctx->qlen, pl = ctx->plen;
	std::vector<HostCol> in = { { (uint8_t *)privkeys, ql, false }, { (uint8_t *)peer_pubkeys, 2 * pl, false } };
	std::vector<HostCol> outc = { { shared, pl, false }, { (uint8_t *)status, 1, false } };
	return run_pipeline(ctx, n, in, outc, [&](int s, uint32_t cnt) {
		const uint8_t *d = ctx->d_in[s];
		return ecdh_dev(ctx, cnt, d, d + (size_t)cnt * ql, ctx->d_out[s],
				(int8_t *)(ctx->d_out[s] + (size_t)cnt * pl), ctx->stage_jac[s], ctx->stage_prefix[s],
				ctx->streams[s]);
	});
}

/* ------------------------------------------------------------------------------------------ hashing on device (§8f.3) */

static int hash_dev(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *d_msgs, const uint64_t *d_off,
		    uint8_t *d_digests, cudaStream_t st)
{
	if (n == 0) return 0;
	if (!sha2_digest_size(hash_type)) return fail("unsupported hash (SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = 5..8)");
	k_sha2_batch<<<grid_for(n), kThreads, 0, st>>>(n, hash_type, d_msgs, d_off, d_digests);
	ctx->launches += 1;
	CUDA_OK(cudaGetLastError());
	return 0;
}

static inline size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

/* offsets[0] == 0 and non-decreasing: message i is msgs[offsets[i], offsets[i+1]) inside the offsets[n] bytes copied */
static bool offsets_ok(const uint64_t *offsets, uint32_t n)
{
	if (offsets[0] != 0) return false;
	for (uint32_t i = 0; i < n; i++)
		if (offsets[i + 1] < offsets[i]) return false;
	return true;
}

extern "C" int eccb200_hash_batch(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *msgs,
				  const uint64_t *offsets, uint8_t *digests)
{
	if (!ctx || (n && (!offsets || !digests))) return fail("null argument");
	const int ds = sha2_digest_size(hash_type);
	if (!ds) return fail("unsupported hash (SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = 5..8)");
	if (n == 0) return 0;
	if (!offsets_ok(offsets, n)) return fail("offsets must start at 0 and be non-decreasing");
	CUDA_OK(cudaSetDevice(ctx->device));
	const uint64_t total = offsets[n];
	if (total && !msgs) return fail("null argument");
	uint8_t *d = nullptr;
	const size_t off_b = ((size_t)total + 15) & ~(size_t)15, offs_bytes = (size_t)(n + 1) * sizeof(uint64_t);
	CUDA_OK(cudaMalloc(&d, off_b + offs_bytes + (size_t)n * ds + 16));
	int rc = 0;
	if ((total && cudaMemcpy(d, msgs, total, cudaMemcpyHostToDevice) != cudaSuccess) ||
	    cudaMemcpy(d + off_b, offsets, offs_bytes, cudaMemcpyHostToDevice) != cudaSuccess)
		rc = fail("H2D copy failed");
	if (!rc) rc = hash_dev(ctx, hash_type, n, d, (const uint64_t *)(d + off_b), d + off_b + offs_bytes, 0);
	if (!rc && cudaMemcpy(digests, d + off_b + offs_bytes, (size_t)n * ds, cudaMemcpyDeviceToHost) != cudaSuccess)
		rc = fail("D2H copy failed");
	cudaFree(d);
	return rc;
}

/* ECDSA verification of raw messages: hashing on the device, then K3 — per chunk of four waves, on two streams, so
 * that the copies of one chunk overlap the kernels of the other (variable-length messages: a chunk's slice of `msgs`
 * is msgs[offsets[lo], offsets[hi]); the hash kernel keeps addressing it with the caller's absolute offsets). */
extern "C" int eccb200_ecdsa_verify_msgs_batch(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *sigs,
					       const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *offsets,
					       int8_t *verdict)
{
	if (!ctx || (n && (!sigs || !pubkeys || !offsets || !verdict))) return fail("null argument");
	const int ds = sha2_digest_size(hash_type);
	if (!ds) return fail("unsupported hash (SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = 5..8)");
	if (n == 0) return 0;
	if (!offsets_ok(offsets, n)) return fail("offsets must start at 0 and be non-decreasing");
	CUDA_OK(cudaSetDevice(ctx->device));
	if (offsets[n] && !msgs) return fail("null argument");
	const uint32_t step = ctx->chunk_eq;
	const size_t sgi = 2 * (size_t)ctx->qlen, pki = 2 * (size_t)ctx->plen;
	size_t max_msg = 0;
	for (uint32_t lo = 0; lo < n; lo += step) {
		const uint32_t hi = (uint32_t)std::min<uint64_t>((uint64_t)lo + step, n);
		max_msg = std::max<size_t>(max_msg, (size_t)(offsets[hi] - offsets[lo]));
	}
	const uint32_t cap = std::min(step, n);
	const size_t b_sig = align16(cap * sgi), b_pk = align16(cap * pki), b_dg = align16((size_t)cap * ds),
		     b_msg = align16(max_msg + 16), b_off = align16(((size_t)cap + 1) * sizeof(uint64_t)), b_v = align16(cap);
	const size_t stage = b_sig + b_pk + b_dg + b_msg + b_off + b_v;
	uint8_t *d = nullptr;
	CUDA_OK(cudaMalloc(&d, 2 * stage));
	int rc = 0;
	uint32_t c = 0;
	for (uint32_t lo = 0; lo < n && !rc; lo += step, c++) {
		const uint32_t hi = (uint32_t)std::min<uint64_t>((uint64_t)lo + step, n), cnt = hi - lo;
		cudaStream_t st = ctx->streams[c & 1];
		uint8_t *base = d + (size_t)(c & 1) * stage;
		uint8_t *d_sig = base, *d_pk = d_sig + b_sig, *d_dg = d_pk + b_pk, *d_msg = d_dg + b_dg, *d_off = d_msg + b_msg,
			*d_v = d_off + b_off;
		const size_t mbytes = (size_t)(offsets[hi] - offsets[lo]);
		if (cudaMemcpyAsync(d_sig, sigs + lo * sgi, cnt * sgi, cudaMemcpyHostToDevice, st) != cudaSuccess ||
		    cudaMemcpyAsync(d_pk, pubkeys + lo * pki, cnt * pki, cudaMemcpyHostToDevice, st) != cudaSuccess ||
		    (mbytes && cudaMemcpyAsync(d_msg, msgs + offsets[lo], mbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) ||
		    cudaMemcpyAsync(d_off, offsets + lo, ((size_t)cnt + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st) !=
			    cudaSuccess) {
			rc = fail("H2D copy failed");
			break;
		}
		/* the kernel adds the caller's absolute offsets to this base: the chunk's bytes start at offsets[lo] */
		rc = hash_dev(ctx, hash_type, cnt, d_msg - offsets[lo], (const uint64_t *)d_off, d_dg, st);
		if (!rc) rc = verify_dev(ctx, cnt, d_sig, d_pk, d_dg, (uint32_t)ds, (int8_t *)d_v, st);
		if (!rc && cudaMemcpyAsync(verdict + lo, d_v, cnt, cudaMemcpyDeviceToHost, st) != cudaSuccess)
			rc = fail("D2H copy failed");
	}
	const std::string keep = g_err;
	for (int s2 = 0; s2 < 2; s2++)
		if (cudaStreamSynchronize(ctx->streams[s2]) != cudaSuccess && !rc) rc = fail("stream synchronisation failed");
	if (rc && !keep.empty()) g_err = keep;
	cudaFree(d);
	return rc;
}

/* Device-resident form: messages, offsets (n + 1 entries, offsets[0] == 0, non-decreasing — NOT re-checked here) and a
 * [n][digest_size] scratch for the digests all live on the device; hash kernel + K3 on `stream`, asynchronous. */
extern "C" int eccb200_ecdsa_verify_msgs_batch_dev(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *d_sigs,
						   const uint8_t *d_pubkeys, const uint8_t *d_msgs,
						   const uint64_t *d_offsets, uint8_t *d_digests, int8_t *d_verdict,
						   void *stream)
{
	if (!ctx || (n && (!d_sigs || !d_pubkeys || !d_offsets || !d_digests || !d_verdict))) return fail("null argument");
	const int ds = sha2_digest_size(hash_type);
	if (!ds) return fail("unsupported hash (SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = 5..8)");
	if (misaligned16(ctx, { d_sigs, d_pubkeys })) return fail(kAlignMsg);
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (hash_dev(ctx, hash_type, n, d_msgs, d_offsets, d_digests, (cudaStream_t)stream)) return -1;
	return verify_dev(ctx, n, d_sigs, d_pubkeys, d_digests, (uint32_t)ds, d_verdict, (cudaStream_t)stream);
}

/* ------------------------------------------------------------------------------------------ Schnorr-family sign */

static const char *kSchnorrAlgMsg = "unsupported sig_type (ECSDSA = 3, ECOSDSA = 4, ECFSDSA = 5, BIP0340 = 20)";
static bool schnorr_alg_ok(int sig_type)
{
	return sig_type == SIG_ECSDSA || sig_type == SIG_ECOSDSA || sig_type == SIG_ECFSDSA || sig_type == SIG_BIP0340;
}

/* BIP0340 nonce kernel (k into k_buf), K1 on k (or on the caller's nonces), K4, finish kernel — all on `st` */
static int schnorr_sign_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *d_priv,
			    const uint8_t *d_pub, const uint8_t *d_rand, const uint8_t *d_msgs, const uint64_t *d_off,
			    uint8_t *d_sigs, int8_t *d_status, uint32_t *jac, uint32_t *prefix, uint8_t *aff, uint8_t *k_buf,
			    cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		if (jac == ctx->jac) scratch_enter(ctx, st);
		const uint8_t *d_k = d_rand;
		if (sig_type == SIG_BIP0340) {
			LaunchMisc<C>::bip0340_nonce(n, hash_type, d_priv, d_pub, d_rand, d_msgs, d_off, k_buf, st);
			d_k = k_buf;
			ctx->launches += 1;
		}
		LaunchFixed<C>::fixed(n, d_k, ctx->table, ctx->w, jac, d_status, st);         /* W = k*G   */
		LaunchMisc<C>::to_affine(affine_grid(ctx, n), n, jac, prefix, aff, d_status, st); /* affine W  */
		LaunchMisc<C>::schnorr_finish(n, sig_type, hash_type, d_priv, d_pub, d_k, d_msgs, d_off, aff, d_sigs,
					      d_status, st);                                   /* hash, s   */
		if (jac == ctx->jac) scratch_leave(ctx, st);
		ctx->launches += 3;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

/* ctx->sign_k holds at least `slots` qlen-byte entries */
static int ensure_sign_k(eccb200_ctx *ctx, size_t slots)
{
	if (ctx->sign_k_cap >= slots) return 0;
	CUDA_OK(cudaDeviceSynchronize()); /* an earlier call may still read the buffer that is about to be replaced */
	if (ctx->sign_k) cudaFree(ctx->sign_k);
	ctx->sign_k = nullptr;
	ctx->sign_k_cap = 0;
	CUDA_OK(cudaMalloc(&ctx->sign_k, slots * ctx->qlen));
	ctx->sign_k_cap = slots;
	return 0;
}

extern "C" int eccb200_schnorr_sign_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
						   const uint8_t *d_privkeys, const uint8_t *d_pubkeys,
						   const uint8_t *d_randomness, const uint8_t *d_msgs,
						   const uint64_t *d_offsets, uint8_t *d_sigs, int8_t *d_status, void *stream)
{
	if (!ctx) return fail("null argument");
	if (!schnorr_alg_ok(sig_type)) return fail(kSchnorrAlgMsg);
	if (!sha2_digest_size(hash_type)) return fail("unsupported hash (SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = 5..8)");
	if (n && (!d_privkeys || !d_randomness || !d_offsets || !d_sigs || !d_status ||
		  (sig_type == SIG_BIP0340 && !d_pubkeys)))
		return fail("null argument");
	if (misaligned16(ctx, { d_privkeys, d_pubkeys, d_randomness, d_sigs })) return fail(kAlignMsg);
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	if (sig_type == SIG_BIP0340 && ensure_sign_k(ctx, n)) return -1;
	return schnorr_sign_dev(ctx, sig_type, hash_type, n, d_privkeys, d_pubkeys, d_randomness, d_msgs, d_offsets, d_sigs,
				d_status, ctx->jac, ctx->prefix, ctx->aff, ctx->sign_k, (cudaStream_t)stream);
}

/* A per-item input of the host-pointer message signers: `width` bytes per item (host == nullptr: not used) */
struct SignCol {
	const uint8_t *host;
	size_t width;
};
/* A ragged input: item i's bytes are data[off[i] .. off[i+1]) (off == nullptr: not used) */
struct SignRagged {
	const uint8_t *data;
	const uint64_t *off;
};
/* One chunk's device buffers, in the order of the inputs (nullptr where an input is not used).  rag_base[j] is shifted
 * so that the caller's absolute offsets address it: the chunk's bytes start at off[lo]. */
struct SignChunk {
	const uint8_t *col[3];
	uint8_t *scratch; /* scratch_width bytes per item */
	const uint8_t *rag_base[2];
	const uint64_t *rag_off[2];
	uint8_t *sigs;
	int8_t *status;
};

/* Host-pointer form of the message signers (Schnorr family and the others) and of the message verifier: chunks of four
 * waves on two streams like eccb200_ecdsa_verify_msgs_batch (a chunk's copies overlap the other chunk's kernels), K1 /
 * K4 scratch from the per-stream stage buffers.  launch(s, cnt, chunk) queues one chunk's kernels on ctx->streams[s].
 * siglen == 0 (the verifier): the status column is the only output.  The caller has checked the offsets. */
template <class Launch>
static int sign_msgs_pipeline(eccb200_ctx *ctx, uint32_t n, const SignCol (&cols)[3], size_t scratch_width,
			      const SignRagged (&rag)[2], size_t siglen, uint8_t *sigs, int8_t *status, Launch launch)
{
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_stages(ctx, 1, 1)) return -1; /* the stage_jac / stage_prefix / stage_aff scratch */
	const uint32_t step = std::min(ctx->chunk_eq, ctx->chunk);
	size_t max_rag[2] = { 0, 0 };
	for (uint32_t lo = 0; lo < n; lo += step) {
		const uint32_t hi = (uint32_t)std::min<uint64_t>((uint64_t)lo + step, n);
		for (int j = 0; j < 2; j++)
			if (rag[j].off) max_rag[j] = std::max<size_t>(max_rag[j], (size_t)(rag[j].off[hi] - rag[j].off[lo]));
	}
	const uint32_t cap = std::min(step, n);
	size_t b_col[3], b_rag[2], b_roff[2];
	size_t stage = 0;
	for (int j = 0; j < 3; j++) stage += b_col[j] = cols[j].host ? align16(cap * cols[j].width) : 0;
	const size_t b_k = align16(cap * scratch_width);
	for (int j = 0; j < 2; j++) {
		stage += b_rag[j] = rag[j].off ? align16(max_rag[j] + 16) : 0;
		stage += b_roff[j] = rag[j].off ? align16(((size_t)cap + 1) * sizeof(uint64_t)) : 0;
	}
	const size_t b_sig = align16(cap * siglen), b_st = align16(cap);
	stage += b_k + b_sig + b_st;
	uint8_t *d = nullptr;
	CUDA_OK(cudaMalloc(&d, 2 * stage));
	int rc = 0;
	uint32_t c = 0;
	for (uint32_t lo = 0; lo < n && !rc; lo += step, c++) {
		const uint32_t hi = (uint32_t)std::min<uint64_t>((uint64_t)lo + step, n), cnt = hi - lo;
		const int s = (int)(c & 1);
		cudaStream_t st = ctx->streams[s];
		uint8_t *p = d + (size_t)s * stage;
		SignChunk ch = {};
		bool ok = true;
		for (int j = 0; j < 3; j++) {
			if (cols[j].host) {
				ok = ok && cudaMemcpyAsync(p, cols[j].host + lo * cols[j].width, cnt * cols[j].width,
							   cudaMemcpyHostToDevice, st) == cudaSuccess;
				ch.col[j] = p;
			}
			p += b_col[j];
		}
		ch.scratch = scratch_width ? p : nullptr;
		p += b_k;
		for (int j = 0; j < 2; j++) {
			if (rag[j].off) {
				const uint64_t *off = rag[j].off;
				const size_t bytes = (size_t)(off[hi] - off[lo]);
				ok = ok && (!bytes || cudaMemcpyAsync(p, rag[j].data + off[lo], bytes, cudaMemcpyHostToDevice, st) ==
							      cudaSuccess);
				ok = ok && cudaMemcpyAsync(p + b_rag[j], off + lo, ((size_t)cnt + 1) * sizeof(uint64_t),
							   cudaMemcpyHostToDevice, st) == cudaSuccess;
				ch.rag_base[j] = p - off[lo]; /* the kernels add the caller's absolute offsets to this base */
				ch.rag_off[j] = (const uint64_t *)(p + b_rag[j]);
			}
			p += b_rag[j] + b_roff[j];
		}
		ch.sigs = p;
		ch.status = (int8_t *)(p + b_sig);
		if (!ok) {
			rc = fail("H2D copy failed");
			break;
		}
		rc = launch(s, cnt, ch);
		if (!rc && ((siglen && cudaMemcpyAsync(sigs + lo * siglen, ch.sigs, cnt * siglen, cudaMemcpyDeviceToHost, st) !=
						cudaSuccess) ||
			    cudaMemcpyAsync(status + lo, ch.status, cnt, cudaMemcpyDeviceToHost, st) != cudaSuccess))
			rc = fail("D2H copy failed");
	}
	const std::string keep = g_err;
	for (int s2 = 0; s2 < 2; s2++)
		if (cudaStreamSynchronize(ctx->streams[s2]) != cudaSuccess && !rc) rc = fail("stream synchronisation failed");
	if (rc && !keep.empty()) g_err = keep;
	cudaFree(d);
	return rc;
}

/* Host-pointer form through sign_msgs_pipeline; the BIP0340 nonces go to the chunk's scratch column. */
extern "C" int eccb200_schnorr_sign_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
					       const uint8_t *privkeys, const uint8_t *pubkeys, const uint8_t *randomness,
					       const uint8_t *msgs, const uint64_t *offsets, uint8_t *sigs, int8_t *status)
{
	if (!ctx) return fail("null argument");
	if (!schnorr_alg_ok(sig_type)) return fail(kSchnorrAlgMsg);
	const int ds = sha2_digest_size(hash_type);
	if (!ds) return fail("unsupported hash (SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = 5..8)");
	const bool bip = sig_type == SIG_BIP0340;
	if (n && (!privkeys || !randomness || !offsets || !sigs || !status || (bip && !pubkeys))) return fail("null argument");
	if (n == 0) return 0;
	if (!offsets_ok(offsets, n)) return fail("offsets must start at 0 and be non-decreasing");
	if (offsets[n] && !msgs) return fail("null argument");
	const size_t ql = ctx->qlen;
	size_t siglen = 0;
	dispatch(ctx->curve_id, [&](auto c) {
		siglen = (size_t)schnorr_sig_len<decltype(c)>(sig_type, ds);
		return 0;
	});
	const SignCol cols[3] = { { privkeys, ql }, { bip ? pubkeys : nullptr, 2 * (size_t)ctx->plen }, { randomness, ql } };
	const SignRagged rag[2] = { { msgs, offsets }, { nullptr, nullptr } };
	return sign_msgs_pipeline(ctx, n, cols, bip ? ql : 0, rag, siglen, sigs, status,
				  [&](int s, uint32_t cnt, const SignChunk &ch) {
					  return schnorr_sign_dev(ctx, sig_type, hash_type, cnt, ch.col[0], ch.col[1],
								  ch.col[2], ch.rag_base[0], ch.rag_off[0], ch.sigs,
								  ch.status, ctx->stage_jac[s], ctx->stage_prefix[s],
								  ctx->stage_aff[s], ch.scratch, ctx->streams[s]);
				  });
}

/* ------------------------------------------------------------------------- ECKCDSA / ECGDSA / ECRDSA / SM2 sign */

static const char *kMsgsAlgMsg = "unsupported sig_type (ECKCDSA = 2, ECGDSA = 6, ECRDSA = 7, SM2 = 8)";
static const char *kMsgsHashMsg = "unsupported hash (SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = 5..8, SM3 = 11)";
static bool msgs_alg_ok(int sig_type)
{
	return sig_type == SIG_ECKCDSA || sig_type == SIG_ECGDSA || sig_type == SIG_ECRDSA || sig_type == SIG_SM2;
}

/* the checks both forms share; 0, or -1 with the reason in eccb200_last_error */
static int msgs_sign_args(const eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const void *privkeys,
			  const void *pubkeys, const void *nonces, const void *offsets, const void *ids,
			  const void *id_offsets, const void *sigs, const void *status)
{
	if (!ctx) return fail("null argument");
	if (!msgs_alg_ok(sig_type)) return fail(kMsgsAlgMsg);
	if (!msg_hash_digest_size(hash_type)) return fail(kMsgsHashMsg);
	const bool sm2 = sig_type == SIG_SM2;
	if (n && (!privkeys || !nonces || !offsets || !sigs || !status || ((sm2 || sig_type == SIG_ECKCDSA) && !pubkeys) ||
		  (sm2 && (!ids || !id_offsets))))
		return fail("null argument");
	return 0;
}

static size_t msgs_siglen(const eccb200_ctx *ctx, int sig_type, int hash_type)
{
	size_t siglen = 0;
	dispatch(ctx->curve_id, [&](auto c) {
		siglen = (size_t)msgs_sig_len<decltype(c)>(sig_type, msg_hash_digest_size(hash_type));
		return 0;
	});
	return siglen;
}

extern "C" int eccb200_sign_sig_len(eccb200_ctx *ctx, int sig_type, int hash_type)
{
	if (!ctx) return fail("null argument");
	if (!msgs_alg_ok(sig_type)) return fail(kMsgsAlgMsg);
	if (!msg_hash_digest_size(hash_type)) return fail(kMsgsHashMsg);
	return (int)msgs_siglen(ctx, sig_type, hash_type);
}

/* K1 on the nonces, K4, finish kernel — all on `st`.  SM2's finish runs on the normalisation's grid (several items per
 * thread share the CTA-wide inversion of 1 + x); the other schemes invert nothing and run one item per thread. */
static int msgs_sign_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *d_priv,
			 const uint8_t *d_pub, const uint8_t *d_nonce, const uint8_t *d_msgs, const uint64_t *d_off,
			 const uint8_t *d_ids, const uint64_t *d_id_off, uint8_t *d_sigs, int8_t *d_status, uint32_t *jac,
			 uint32_t *prefix, uint8_t *aff, cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		if (jac == ctx->jac) scratch_enter(ctx, st);
		LaunchFixed<C>::fixed(n, d_nonce, ctx->table, ctx->w, jac, d_status, st);       /* W = k*G  */
		LaunchMisc<C>::to_affine(affine_grid(ctx, n), n, jac, prefix, aff, d_status, st); /* affine W */
		LaunchMisc<C>::msgs_sign_finish(sig_type == SIG_SM2 ? affine_grid(ctx, n) : grid_for(n), n, sig_type,
						hash_type, d_priv, d_pub, d_nonce, d_msgs, d_off, d_ids, d_id_off, aff,
						prefix, d_sigs, d_status, st);                 /* hash, r, s */
		if (jac == ctx->jac) scratch_leave(ctx, st);
		ctx->launches += 3;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_sign_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
					   const uint8_t *d_privkeys, const uint8_t *d_pubkeys, const uint8_t *d_nonces,
					   const uint8_t *d_msgs, const uint64_t *d_offsets, const uint8_t *d_ids,
					   const uint64_t *d_id_offsets, uint8_t *d_sigs, int8_t *d_status, void *stream)
{
	if (msgs_sign_args(ctx, sig_type, hash_type, n, d_privkeys, d_pubkeys, d_nonces, d_offsets, d_ids, d_id_offsets,
			   d_sigs, d_status))
		return -1;
	if (misaligned16(ctx, { d_privkeys, d_pubkeys, d_nonces, d_sigs })) return fail(kAlignMsg);
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	const bool sm2 = sig_type == SIG_SM2, with_key = sm2 || sig_type == SIG_ECKCDSA;
	return msgs_sign_dev(ctx, sig_type, hash_type, n, d_privkeys, with_key ? d_pubkeys : nullptr, d_nonces, d_msgs,
			     d_offsets, sm2 ? d_ids : nullptr, sm2 ? d_id_offsets : nullptr, d_sigs, d_status, ctx->jac,
			     ctx->prefix, ctx->aff, (cudaStream_t)stream);
}

extern "C" int eccb200_sign_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
				       const uint8_t *privkeys, const uint8_t *pubkeys, const uint8_t *nonces,
				       const uint8_t *msgs, const uint64_t *offsets, const uint8_t *ids,
				       const uint64_t *id_offsets, uint8_t *sigs, int8_t *status)
{
	if (msgs_sign_args(ctx, sig_type, hash_type, n, privkeys, pubkeys, nonces, offsets, ids, id_offsets, sigs, status))
		return -1;
	if (n == 0) return 0;
	const bool sm2 = sig_type == SIG_SM2, with_key = sm2 || sig_type == SIG_ECKCDSA;
	if (!offsets_ok(offsets, n)) return fail("offsets must start at 0 and be non-decreasing");
	if (offsets[n] && !msgs) return fail("null argument");
	if (sm2) {
		if (!offsets_ok(id_offsets, n)) return fail("id_offsets must start at 0 and be non-decreasing");
		for (uint32_t i = 0; i < n; i++)
			if (id_offsets[i + 1] - id_offsets[i] > kSm2MaxIdLen) return fail("SM2 ID longer than 8191 bytes");
	}
	const size_t ql = ctx->qlen;
	const SignCol cols[3] = { { privkeys, ql }, { with_key ? pubkeys : nullptr, 2 * (size_t)ctx->plen }, { nonces, ql } };
	const SignRagged rag[2] = { { msgs, offsets }, { sm2 ? ids : nullptr, sm2 ? id_offsets : nullptr } };
	return sign_msgs_pipeline(ctx, n, cols, 0, rag, msgs_siglen(ctx, sig_type, hash_type), sigs, status,
				  [&](int s, uint32_t cnt, const SignChunk &ch) {
					  return msgs_sign_dev(ctx, sig_type, hash_type, cnt, ch.col[0], ch.col[1], ch.col[2],
							       ch.rag_base[0], ch.rag_off[0], ch.rag_base[1], ch.rag_off[1],
							       ch.sigs, ch.status, ctx->stage_jac[s], ctx->stage_prefix[s],
							       ctx->stage_aff[s], ctx->streams[s]);
				  });
}

/* ------------------------------------------------------- deterministic ECDSA (RFC 6979) and ECDSA of raw messages */

enum { SIG_ECDSA = 1, SIG_DECDSA = 14 }; /* ec_alg_type values of the reference (lib_ecc_types.h) */
static const char *kDecdsaHashMsg =
	"unsupported hash (SHA224 = 1, SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = 5..8, SM3 = 11)";

/* The nonce kernel (H(m) into dig_buf when msgs are given, the RFC 6979 k into k_buf when det), K1 on k (k_buf, or
 * the caller's d_nonce), K4, k_ecdsa_sign_finish on the digests (dig_buf, or the caller's d_dig) — all on `st`. */
static int ecdsa_det_sign_dev(eccb200_ctx *ctx, bool det, int hash_type, uint32_t n, const uint8_t *d_priv,
			      const uint8_t *d_nonce, const uint8_t *d_dig, bool with_msgs, const uint8_t *d_msgs,
			      const uint64_t *d_off, uint8_t *k_buf, uint8_t *dig_buf, uint8_t *d_sigs, int8_t *d_status,
			      uint32_t *jac, uint32_t *prefix, uint8_t *aff, cudaStream_t st)
{
	if (n == 0) return 0;
	const uint32_t ds = (uint32_t)decdsa_hash_digest_size(hash_type);
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		if (jac == ctx->jac) scratch_enter(ctx, st);
		const uint8_t *k = det ? k_buf : d_nonce, *dig = with_msgs ? dig_buf : d_dig;
		LaunchMisc<C>::ecdsa_nonce(n, hash_type, d_priv, d_dig, d_msgs, d_off, with_msgs ? dig_buf : nullptr,
					   det ? k_buf : nullptr, st);                       /* H(m), k      */
		LaunchFixed<C>::fixed(n, k, ctx->table, ctx->w, jac, d_status, st);             /* k*G          */
		LaunchMisc<C>::to_affine(affine_grid(ctx, n), n, jac, prefix, aff, d_status, st); /* affine (x, y) */
		LaunchMisc<C>::sign_finish(affine_grid(ctx, n), n, d_priv, k, dig, ds, aff, prefix, d_sigs, d_status,
					   st);                                                   /* r, s         */
		if (jac == ctx->jac) scratch_leave(ctx, st);
		ctx->launches += 4;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_decdsa_sign_batch_dev(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *d_privkeys,
					     const uint8_t *d_digests, uint8_t *d_sigs, int8_t *d_status, void *stream)
{
	if (!ctx) return fail("null argument");
	if (!decdsa_hash_digest_size(hash_type)) return fail(kDecdsaHashMsg);
	if (n && (!d_privkeys || !d_digests || !d_sigs || !d_status)) return fail("null argument");
	if (misaligned16(ctx, { d_privkeys, d_sigs })) return fail(kAlignMsg);
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n) || ensure_sign_k(ctx, n)) return -1;
	return ecdsa_det_sign_dev(ctx, true, hash_type, n, d_privkeys, nullptr, d_digests, false, nullptr, nullptr,
				  ctx->sign_k, nullptr, d_sigs, d_status, ctx->jac, ctx->prefix, ctx->aff,
				  (cudaStream_t)stream);
}

/* Host-pointer form through sign_msgs_pipeline: private keys and digests as columns, k in the scratch column. */
extern "C" int eccb200_decdsa_sign_batch(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *privkeys,
					 const uint8_t *digests, uint8_t *sigs, int8_t *status)
{
	if (!ctx) return fail("null argument");
	const int ds = decdsa_hash_digest_size(hash_type);
	if (!ds) return fail(kDecdsaHashMsg);
	if (n && (!privkeys || !digests || !sigs || !status)) return fail("null argument");
	if (n == 0) return 0;
	const size_t ql = ctx->qlen;
	const SignCol cols[3] = { { privkeys, ql }, { digests, (size_t)ds }, { nullptr, 0 } };
	const SignRagged rag[2] = { { nullptr, nullptr }, { nullptr, nullptr } };
	return sign_msgs_pipeline(ctx, n, cols, ql, rag, 2 * ql, sigs, status,
				  [&](int s, uint32_t cnt, const SignChunk &ch) {
					  return ecdsa_det_sign_dev(ctx, true, hash_type, cnt, ch.col[0], nullptr, ch.col[1],
								    false, nullptr, nullptr, ch.scratch, nullptr, ch.sigs,
								    ch.status, ctx->stage_jac[s], ctx->stage_prefix[s],
								    ctx->stage_aff[s], ctx->streams[s]);
				  });
}

/* the checks both message forms share; 0, or -1 with the reason in eccb200_last_error */
static int ecdsa_msgs_args(const eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const void *privkeys,
			   const void *nonces, const void *offsets, const void *sigs, const void *status)
{
	if (!ctx) return fail("null argument");
	if (sig_type != SIG_ECDSA && sig_type != SIG_DECDSA) return fail("unsupported sig_type (ECDSA = 1, DECDSA = 14)");
	if (!decdsa_hash_digest_size(hash_type)) return fail(kDecdsaHashMsg);
	if (sig_type == SIG_ECDSA && !nonces) return fail("ECDSA needs the caller's nonces");
	if (n && (!privkeys || !offsets || !sigs || !status)) return fail("null argument");
	return 0;
}

/* Scratch of the message forms, per chunk of cnt items: the RFC 6979 nonces (DECDSA, cnt * qlen bytes), then the
 * digests (cnt * digest size bytes).  cnt * qlen keeps the digests 16-byte aligned wherever alignment matters. */
extern "C" int eccb200_ecdsa_sign_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
						 const uint8_t *d_privkeys, const uint8_t *d_nonces, const uint8_t *d_msgs,
						 const uint64_t *d_offsets, uint8_t *d_sigs, int8_t *d_status, void *stream)
{
	if (ecdsa_msgs_args(ctx, sig_type, hash_type, n, d_privkeys, d_nonces, d_offsets, d_sigs, d_status)) return -1;
	const bool det = sig_type == SIG_DECDSA;
	if (misaligned16(ctx, { d_privkeys, det ? nullptr : d_nonces, d_sigs })) return fail(kAlignMsg);
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	const size_t ql = ctx->qlen, ds = (size_t)decdsa_hash_digest_size(hash_type);
	const size_t k_bytes = det ? (size_t)n * ql : 0;
	if (ensure_work(ctx, n) || ensure_sign_k(ctx, (k_bytes + (size_t)n * ds + ql - 1) / ql)) return -1;
	return ecdsa_det_sign_dev(ctx, det, hash_type, n, d_privkeys, det ? nullptr : d_nonces, nullptr, true, d_msgs,
				  d_offsets, det ? ctx->sign_k : nullptr, ctx->sign_k + k_bytes, d_sigs, d_status, ctx->jac,
				  ctx->prefix, ctx->aff, (cudaStream_t)stream);
}

extern "C" int eccb200_ecdsa_sign_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
					     const uint8_t *privkeys, const uint8_t *nonces, const uint8_t *msgs,
					     const uint64_t *offsets, uint8_t *sigs, int8_t *status)
{
	if (ecdsa_msgs_args(ctx, sig_type, hash_type, n, privkeys, nonces, offsets, sigs, status)) return -1;
	if (n == 0) return 0;
	if (!offsets_ok(offsets, n)) return fail("offsets must start at 0 and be non-decreasing");
	if (offsets[n] && !msgs) return fail("null argument");
	const bool det = sig_type == SIG_DECDSA;
	const size_t ql = ctx->qlen, ds = (size_t)decdsa_hash_digest_size(hash_type);
	const SignCol cols[3] = { { privkeys, ql }, { det ? nullptr : nonces, ql }, { nullptr, 0 } };
	const SignRagged rag[2] = { { msgs, offsets }, { nullptr, nullptr } };
	return sign_msgs_pipeline(ctx, n, cols, (det ? ql : 0) + ds, rag, 2 * ql, sigs, status,
				  [&](int s, uint32_t cnt, const SignChunk &ch) {
					  const size_t k_bytes = det ? (size_t)cnt * ql : 0;
					  return ecdsa_det_sign_dev(ctx, det, hash_type, cnt, ch.col[0], ch.col[1], nullptr,
								    true, ch.rag_base[0], ch.rag_off[0],
								    det ? ch.scratch : nullptr, ch.scratch + k_bytes,
								    ch.sigs, ch.status, ctx->stage_jac[s],
								    ctx->stage_prefix[s], ctx->stage_aff[s], ctx->streams[s]);
				  });
}

/* ------------------------------------------------------------------------------- BIGN / DBIGN of raw messages */

static const char *kBignHashMsg = "unsupported hash (SHA224 = 1, SHA256 = 2, SHA384 = 3, SHA512 = 4, SHA3_224..512 = "
				  "5..8, SM3 = 11, BELT_HASH = 16, BASH224..512 = 17..20)";

/* k_bign_nonce (H(m) into dig_buf; the DBIGN k into k_buf when det), K1 on k (k_buf, or the caller's d_nonce), K4,
 * k_bign_sign_finish — all on `st` */
static int bign_sign_dev(eccb200_ctx *ctx, bool det, int hash_type, uint32_t n, const uint8_t *d_priv,
			 const uint8_t *d_nonce, const uint8_t *d_msgs, const uint64_t *d_off, const uint8_t *d_ad,
			 const uint64_t *d_ad_off, uint8_t *k_buf, uint8_t *dig_buf, uint8_t *d_sigs, int8_t *d_status,
			 uint32_t *jac, uint32_t *prefix, uint8_t *aff, cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		if (jac == ctx->jac) scratch_enter(ctx, st);
		const uint8_t *k = det ? k_buf : d_nonce;
		LaunchMisc<C>::bign_nonce(n, hash_type, d_priv, d_msgs, d_off, d_ad, d_ad_off, dig_buf, det ? k_buf : nullptr,
					  st);                                                    /* H(m), k  */
		LaunchFixed<C>::fixed(n, k, ctx->table, ctx->w, jac, d_status, st);             /* W = k*G  */
		LaunchMisc<C>::to_affine(affine_grid(ctx, n), n, jac, prefix, aff, d_status, st); /* affine W */
		LaunchMisc<C>::bign_sign_finish(n, hash_type, d_priv, k, dig_buf, d_ad, d_ad_off, aff, d_sigs, d_status,
						st);                                              /* s0, s1   */
		if (jac == ctx->jac) scratch_leave(ctx, st);
		ctx->launches += 4;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

/* the checks both signing forms share; 0, or -1 with the reason in eccb200_last_error */
static int bign_sign_args(const eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const void *privkeys,
			  const void *nonces, const void *offsets, const void *adata, const void *adata_offsets,
			  const void *sigs, const void *status)
{
	if (!ctx) return fail("null argument");
	if (sig_type != SIG_BIGN && sig_type != SIG_DBIGN) return fail("unsupported sig_type (BIGN = 18, DBIGN = 19)");
	if (!bign_hash_digest_size(hash_type)) return fail(kBignHashMsg);
	if (sig_type == SIG_BIGN && !nonces) return fail("BIGN needs the caller's nonces");
	if (n && (!privkeys || !offsets || !adata || !adata_offsets || !sigs || !status)) return fail("null argument");
	return 0;
}

/* Scratch of the signers, per chunk of cnt items: the DBIGN nonces (cnt * qlen bytes), then the digests (cnt * digest
 * size bytes). */
extern "C" int eccb200_bign_sign_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
						const uint8_t *d_privkeys, const uint8_t *d_nonces, const uint8_t *d_msgs,
						const uint64_t *d_offsets, const uint8_t *d_adata,
						const uint64_t *d_adata_offsets, uint8_t *d_sigs, int8_t *d_status, void *stream)
{
	if (bign_sign_args(ctx, sig_type, hash_type, n, d_privkeys, d_nonces, d_offsets, d_adata, d_adata_offsets, d_sigs,
			   d_status))
		return -1;
	const bool det = sig_type == SIG_DBIGN;
	if (misaligned16(ctx, { d_privkeys, det ? nullptr : d_nonces, d_sigs })) return fail(kAlignMsg);
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	const size_t ql = ctx->qlen, ds = (size_t)bign_hash_digest_size(hash_type);
	const size_t k_bytes = det ? (size_t)n * ql : 0;
	if (ensure_work(ctx, n) || ensure_sign_k(ctx, (k_bytes + (size_t)n * ds + ql - 1) / ql)) return -1;
	return bign_sign_dev(ctx, det, hash_type, n, d_privkeys, det ? nullptr : d_nonces, d_msgs, d_offsets, d_adata,
			     d_adata_offsets, det ? ctx->sign_k : nullptr, ctx->sign_k + k_bytes, d_sigs, d_status, ctx->jac,
			     ctx->prefix, ctx->aff, (cudaStream_t)stream);
}

extern "C" int eccb200_bign_sign_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
					    const uint8_t *privkeys, const uint8_t *nonces, const uint8_t *msgs,
					    const uint64_t *offsets, const uint8_t *adata, const uint64_t *adata_offsets,
					    uint8_t *sigs, int8_t *status)
{
	if (bign_sign_args(ctx, sig_type, hash_type, n, privkeys, nonces, offsets, adata, adata_offsets, sigs, status))
		return -1;
	if (n == 0) return 0;
	if (!offsets_ok(offsets, n)) return fail("offsets must start at 0 and be non-decreasing");
	if (offsets[n] && !msgs) return fail("null argument");
	if (!offsets_ok(adata_offsets, n)) return fail("adata_offsets must start at 0 and be non-decreasing");
	const bool det = sig_type == SIG_DBIGN;
	const size_t ql = ctx->qlen, ds = (size_t)bign_hash_digest_size(hash_type);
	const SignCol cols[3] = { { privkeys, ql }, { det ? nullptr : nonces, ql }, { nullptr, 0 } };
	const SignRagged rag[2] = { { msgs, offsets }, { adata, adata_offsets } };
	return sign_msgs_pipeline(ctx, n, cols, (det ? ql : 0) + ds, rag, ql / 2 + ql, sigs, status,
				  [&](int s, uint32_t cnt, const SignChunk &ch) {
					  const size_t k_bytes = det ? (size_t)cnt * ql : 0;
					  return bign_sign_dev(ctx, det, hash_type, cnt, ch.col[0], ch.col[1], ch.rag_base[0],
							       ch.rag_off[0], ch.rag_base[1], ch.rag_off[1],
							       det ? ch.scratch : nullptr, ch.scratch + k_bytes, ch.sigs,
							       ch.status, ctx->stage_jac[s], ctx->stage_prefix[s],
							       ctx->stage_aff[s], ctx->streams[s]);
				  });
}

/* k_bign_verify_prep (checks, H(m) into dig_buf, a || b into jac), the double-scalar kernel (W' into aff, its status
 * into d_verdict), k_bign_verify_finish (s0 test) — all on `st` */
static int bign_verify_dev(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *d_sigs, const uint8_t *d_pub,
			   const uint8_t *d_msgs, const uint64_t *d_off, const uint8_t *d_ad, const uint64_t *d_ad_off,
			   uint8_t *dig_buf, int8_t *d_verdict, uint32_t *jac, uint8_t *aff, cudaStream_t st)
{
	if (n == 0) return 0;
	const int ds = bign_hash_digest_size(hash_type);
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		static_assert(2 * C::QLEN <= 12 * C::N, "verify scratch layout"); /* [n][2*qlen] bytes in [n][3N] words */
		uint8_t *ab = reinterpret_cast<uint8_t *>(jac);
		if (jac == ctx->jac) scratch_enter(ctx, st);
		LaunchMisc<C>::bign_verify_prep(n, hash_type, d_sigs, d_msgs, d_off, d_ad, d_ad_off, dig_buf, ab, st);
		LaunchVerify<C>::double_smul(n, ab, d_pub, ctx->table, ctx->w, aff, d_verdict, st); /* W' = aG + bY */
		LaunchMisc<C>::bign_verify_finish(n, d_sigs, d_ad, d_ad_off, dig_buf, ds, aff, d_verdict, st);
		if (jac == ctx->jac) scratch_leave(ctx, st);
		ctx->launches += 3;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

static int bign_verify_args(const eccb200_ctx *ctx, int hash_type, uint32_t n, const void *sigs, const void *pubkeys,
			    const void *offsets, const void *adata, const void *adata_offsets, const void *verdict)
{
	if (!ctx) return fail("null argument");
	if (!bign_hash_digest_size(hash_type)) return fail(kBignHashMsg);
	if (n && (!sigs || !pubkeys || !offsets || !adata || !adata_offsets || !verdict)) return fail("null argument");
	return 0;
}

extern "C" int eccb200_bign_verify_msgs_batch_dev(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *d_sigs,
						  const uint8_t *d_pubkeys, const uint8_t *d_msgs, const uint64_t *d_offsets,
						  const uint8_t *d_adata, const uint64_t *d_adata_offsets, int8_t *d_verdict,
						  void *stream)
{
	if (bign_verify_args(ctx, hash_type, n, d_sigs, d_pubkeys, d_offsets, d_adata, d_adata_offsets, d_verdict))
		return -1;
	if (misaligned16(ctx, { d_sigs, d_pubkeys })) return fail(kAlignMsg);
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	const size_t ql = ctx->qlen, ds = (size_t)bign_hash_digest_size(hash_type);
	if (ensure_work(ctx, n) || ensure_sign_k(ctx, ((size_t)n * ds + ql - 1) / ql)) return -1;
	return bign_verify_dev(ctx, hash_type, n, d_sigs, d_pubkeys, d_msgs, d_offsets, d_adata, d_adata_offsets,
			       ctx->sign_k, d_verdict, ctx->jac, ctx->aff, (cudaStream_t)stream);
}

/* Host-pointer form through sign_msgs_pipeline: signatures and keys are its columns, messages and adata its ragged
 * inputs, the digests its scratch column, the verdicts its status column. */
extern "C" int eccb200_bign_verify_msgs_batch(eccb200_ctx *ctx, int hash_type, uint32_t n, const uint8_t *sigs,
					      const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *offsets,
					      const uint8_t *adata, const uint64_t *adata_offsets, int8_t *verdict)
{
	if (bign_verify_args(ctx, hash_type, n, sigs, pubkeys, offsets, adata, adata_offsets, verdict)) return -1;
	if (n == 0) return 0;
	if (!offsets_ok(offsets, n)) return fail("offsets must start at 0 and be non-decreasing");
	if (offsets[n] && !msgs) return fail("null argument");
	if (!offsets_ok(adata_offsets, n)) return fail("adata_offsets must start at 0 and be non-decreasing");
	const size_t ql = ctx->qlen, ds = (size_t)bign_hash_digest_size(hash_type);
	const SignCol cols[3] = { { sigs, ql / 2 + ql }, { pubkeys, 2 * (size_t)ctx->plen }, { nullptr, 0 } };
	const SignRagged rag[2] = { { msgs, offsets }, { adata, adata_offsets } };
	return sign_msgs_pipeline(ctx, n, cols, ds, rag, 0, nullptr, verdict, [&](int s, uint32_t cnt, const SignChunk &ch) {
		return bign_verify_dev(ctx, hash_type, cnt, ch.col[0], ch.col[1], ch.rag_base[0], ch.rag_off[0],
				       ch.rag_base[1], ch.rag_off[1], ch.scratch, ch.status, ctx->stage_jac[s],
				       ctx->stage_aff[s], ctx->streams[s]);
	});
}

/* -------------------------------------------- ECKCDSA / ECSDSA / ECOSDSA / ECGDSA / ECRDSA / SM2 verification */

static const char *kVerifyAlgMsg =
	"unsupported sig_type (ECKCDSA = 2, ECSDSA = 3, ECOSDSA = 4, ECGDSA = 6, ECRDSA = 7, SM2 = 8)";
static bool verify_msgs_alg_ok(int sig_type)
{
	return msgs_alg_ok(sig_type) || sig_type == SIG_ECSDSA || sig_type == SIG_ECOSDSA;
}

/* the checks both forms share; 0, or -1 with the reason in eccb200_last_error */
static int msgs_verify_args(const eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const void *sigs,
			    const void *pubkeys, const void *offsets, const void *ids, const void *id_offsets,
			    const void *verdict)
{
	if (!ctx) return fail("null argument");
	if (!verify_msgs_alg_ok(sig_type)) return fail(kVerifyAlgMsg);
	if (!msg_hash_digest_size(hash_type)) return fail(kMsgsHashMsg);
	if (n && (!sigs || !pubkeys || !offsets || !verdict || (sig_type == SIG_SM2 && (!ids || !id_offsets))))
		return fail("null argument");
	return 0;
}

/* prep kernel (checks, hash, a || b into jac), the double-scalar kernel (W' into aff, its status into d_verdict), finish
 * kernel (acceptance test) — all on `st`.  The prep of ECGDSA / ECRDSA runs on the normalisation's grid (several items
 * per thread share the CTA-wide inversion; den goes to aff, which W' overwrites later); the other schemes invert nothing
 * and run one item per thread. */
static int msgs_verify_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *d_sigs,
			   const uint8_t *d_pub, const uint8_t *d_msgs, const uint64_t *d_off, const uint8_t *d_ids,
			   const uint64_t *d_id_off, int8_t *d_verdict, uint32_t *jac, uint32_t *prefix, uint8_t *aff,
			   cudaStream_t st)
{
	if (n == 0) return 0;
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		/* [n][2*qlen] bytes fit the [n][3N] words of the Jacobian scratch, [n][N] words the [n][2*plen] bytes of aff */
		static_assert(2 * C::QLEN <= 12 * C::N && 4 * C::N <= 2 * C::PLEN, "verify scratch layout");
		uint8_t *ab = reinterpret_cast<uint8_t *>(jac);
		if (jac == ctx->jac) scratch_enter(ctx, st);
		LaunchMisc<C>::msgs_verify_prep(msgs_verify_inverts(sig_type) ? affine_grid(ctx, n) : grid_for(n), n, sig_type,
						hash_type, d_sigs, d_pub, d_msgs, d_off, d_id_off, prefix,
						reinterpret_cast<uint32_t *>(aff), ab, st);           /* checks, a || b */
		LaunchVerify<C>::double_smul(n, ab, d_pub, ctx->table, ctx->w, aff, d_verdict, st); /* W' = aG + bY */
		LaunchMisc<C>::msgs_verify_finish(n, sig_type, hash_type, d_sigs, d_pub, d_msgs, d_off, d_ids, d_id_off, aff,
						  d_verdict, st);                                       /* accept */
		if (jac == ctx->jac) scratch_leave(ctx, st);
		ctx->launches += 3;
		CUDA_OK(cudaGetLastError());
		return 0;
	});
}

extern "C" int eccb200_verify_msgs_batch_dev(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n,
					     const uint8_t *d_sigs, const uint8_t *d_pubkeys, const uint8_t *d_msgs,
					     const uint64_t *d_offsets, const uint8_t *d_ids, const uint64_t *d_id_offsets,
					     int8_t *d_verdict, void *stream)
{
	if (msgs_verify_args(ctx, sig_type, hash_type, n, d_sigs, d_pubkeys, d_offsets, d_ids, d_id_offsets, d_verdict))
		return -1;
	if (misaligned16(ctx, { d_sigs, d_pubkeys })) return fail(kAlignMsg);
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	const bool sm2 = sig_type == SIG_SM2;
	return msgs_verify_dev(ctx, sig_type, hash_type, n, d_sigs, d_pubkeys, d_msgs, d_offsets, sm2 ? d_ids : nullptr,
			       sm2 ? d_id_offsets : nullptr, d_verdict, ctx->jac, ctx->prefix, ctx->aff,
			       (cudaStream_t)stream);
}

/* Host-pointer form through sign_msgs_pipeline: signatures and keys are its columns, messages and IDs its ragged
 * inputs, the verdicts its status column. */
extern "C" int eccb200_verify_msgs_batch(eccb200_ctx *ctx, int sig_type, int hash_type, uint32_t n, const uint8_t *sigs,
					 const uint8_t *pubkeys, const uint8_t *msgs, const uint64_t *offsets,
					 const uint8_t *ids, const uint64_t *id_offsets, int8_t *verdict)
{
	if (msgs_verify_args(ctx, sig_type, hash_type, n, sigs, pubkeys, offsets, ids, id_offsets, verdict)) return -1;
	if (n == 0) return 0;
	const bool sm2 = sig_type == SIG_SM2;
	if (!offsets_ok(offsets, n)) return fail("offsets must start at 0 and be non-decreasing");
	if (offsets[n] && !msgs) return fail("null argument");
	if (sm2 && !offsets_ok(id_offsets, n)) return fail("id_offsets must start at 0 and be non-decreasing");
	size_t siglen = 0;
	dispatch(ctx->curve_id, [&](auto c) {
		siglen = (size_t)msgs_verify_sig_len<decltype(c)>(sig_type, msg_hash_digest_size(hash_type));
		return 0;
	});
	const SignCol cols[3] = { { sigs, siglen }, { pubkeys, 2 * (size_t)ctx->plen }, { nullptr, 0 } };
	const SignRagged rag[2] = { { msgs, offsets }, { sm2 ? ids : nullptr, sm2 ? id_offsets : nullptr } };
	return sign_msgs_pipeline(ctx, n, cols, 0, rag, 0, nullptr, verdict, [&](int s, uint32_t cnt, const SignChunk &ch) {
		return msgs_verify_dev(ctx, sig_type, hash_type, cnt, ch.col[0], ch.col[1], ch.rag_base[0], ch.rag_off[0],
				       ch.rag_base[1], ch.rag_off[1], ch.status, ctx->stage_jac[s], ctx->stage_prefix[s],
				       ctx->stage_aff[s], ctx->streams[s]);
	});
}

/* cudaMemcpy device -> host for callers that do not link the CUDA runtime (bench.py reads peer-written buffers). */
extern "C" int eccb200_copy_to_host(eccb200_ctx *ctx, void *host_dst, const void *d_src, size_t bytes)
{
	if (!ctx || !host_dst || !d_src) return fail("null argument");
	CUDA_OK(cudaSetDevice(ctx->device));
	CUDA_OK(cudaMemcpy(host_dst, d_src, bytes, cudaMemcpyDeviceToHost));
	return 0;
}

/* ------------------------------------------------------------------------------------------ structured wire formats (§8f.2) */

static inline uint32_t grid_bytes(uint64_t total) { return (uint32_t)((total + 255) / 256); }

/* device scratch of the structured-record entry points: one allocation, carved into 16-byte aligned pieces */
struct DevArena {
	uint8_t *base = nullptr;
	size_t used = 0, cap = 0;
	std::vector<size_t> want;
	size_t reserve(size_t bytes)
	{
		want.push_back(align16(bytes));
		return want.size() - 1;
	}
	int commit()
	{
		for (size_t b : want) cap += b;
		return cudaMalloc(&base, cap ? cap : 16) == cudaSuccess ? 0 : -1;
	}
	uint8_t *get(size_t idx)
	{
		size_t off = 0;
		for (size_t i = 0; i < idx; i++) off += want[i];
		return base + off;
	}
	~DevArena()
	{
		if (base) cudaFree(base);
	}
};

/* records (device) -> validated affine keys + state (0 ok, 1 infinity, -1 rejected); d_prj: [n][3*plen] scratch */
static int structured_pub_import_dev(eccb200_ctx *ctx, uint32_t n, const uint8_t *d_rec, int alg, uint8_t *d_prj,
				     uint8_t *d_aff, int8_t *d_state, cudaStream_t st)
{
	const uint32_t pl = ctx->plen, stride = 3 + 3 * pl;
	k_struct_unpack<<<grid_bytes((uint64_t)n * 3 * pl), 256, 0, st>>>(n, d_rec, stride, 3 * pl, d_prj, 3 * pl);
	int rc = dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		scratch_enter(ctx, st);
		LaunchMisc<C>::prj_unique(affine_grid(ctx, n), n, d_prj, ctx->jac, ctx->prefix, d_aff, d_state, st);
		scratch_leave(ctx, st);
		return 0;
	});
	if (rc) return rc;
	k_struct_check<<<grid_for(n), kThreads, 0, st>>>(n, d_rec, stride, 0 /* EC_PUBKEY */, (uint8_t)alg,
							 (uint8_t)ctx->curve_id, 0, d_state);
	ctx->launches += 4;
	CUDA_OK(cudaGetLastError());
	return 0;
}

/* ec_structured_pub_key_import_from_buf (sig/ec_key.c:410-449) for n records of 3 + 3*plen bytes: header check,
 * coordinates < p, point on the curve, normalisation to affine.  status: 0 ok, 1 the key is the point at infinity
 * (the reference imports it), -1 rejected.  Rejected / infinity slots of `pubkeys` are zero. */
extern "C" int eccb200_structured_pub_key_import_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *records, int alg,
							 uint8_t *pubkeys, int8_t *status)
{
	if (!ctx || (n && (!records || !pubkeys || !status))) return fail("null argument");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	const size_t pl = ctx->plen, rec_b = (size_t)n * (3 + 3 * pl);
	DevArena a;
	const size_t i_rec = a.reserve(rec_b), i_prj = a.reserve((size_t)n * 3 * pl), i_aff = a.reserve((size_t)n * 2 * pl),
		     i_st = a.reserve(n);
	if (a.commit()) return fail("cudaMalloc failed");
	CUDA_OK(cudaMemcpy(a.get(i_rec), records, rec_b, cudaMemcpyHostToDevice));
	if (structured_pub_import_dev(ctx, n, a.get(i_rec), alg, a.get(i_prj), a.get(i_aff), (int8_t *)a.get(i_st), 0))
		return -1;
	CUDA_OK(cudaMemcpy(pubkeys, a.get(i_aff), (size_t)n * 2 * pl, cudaMemcpyDeviceToHost));
	CUDA_OK(cudaMemcpy(status, a.get(i_st), n, cudaMemcpyDeviceToHost));
	for (uint32_t i = 0; i < n; i++)
		if (status[i] < 0) memset(pubkeys + (size_t)i * 2 * pl, 0, 2 * pl);
	return 0;
}

/* ec_structured_pub_key_export_to_buf (sig/ec_key.c:451-497) for n affine keys: records of 3 + 3*plen bytes with
 * Z = 1 (a representation the reference's import accepts; its own export carries whatever Z the key holds). */
extern "C" int eccb200_structured_pub_key_export_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *pubkeys, int alg,
							 uint8_t *records)
{
	if (!ctx || (n && (!pubkeys || !records))) return fail("null argument");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	const size_t pl = ctx->plen, rec_b = (size_t)n * (3 + 3 * pl);
	DevArena a;
	const size_t i_aff = a.reserve((size_t)n * 2 * pl), i_st = a.reserve(n), i_rec = a.reserve(rec_b);
	if (a.commit()) return fail("cudaMalloc failed");
	CUDA_OK(cudaMemcpy(a.get(i_aff), pubkeys, (size_t)n * 2 * pl, cudaMemcpyHostToDevice));
	CUDA_OK(cudaMemset(a.get(i_st), 0, n));
	k_struct_pack_pub<<<grid_bytes(rec_b), 256>>>(n, a.get(i_aff), (uint32_t)pl, (const int8_t *)a.get(i_st), 0,
						     (uint8_t)alg, (uint8_t)ctx->curve_id, a.get(i_rec));
	ctx->launches += 1;
	CUDA_OK(cudaGetLastError());
	CUDA_OK(cudaMemcpy(records, a.get(i_rec), rec_b, cudaMemcpyDeviceToHost));
	return 0;
}

/* ec_structured_key_pair_import_from_priv_key_buf (sig/ec_key.c:499-545) + ec_structured_pub_key_export_to_buf for
 * n private-key records of 3 + priv_len bytes: header check, x < q (sig/ecdsa_common.c:188), Y = x*G on the
 * fixed-base path (K1 + K4), structured public-key records out.  status: 0 ok, 1 x = 0 (Y at infinity), -1 rejected. */
extern "C" int eccb200_structured_key_pair_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *priv_records,
						   uint32_t priv_len, int alg, uint8_t *pub_records, int8_t *status)
{
	if (!ctx || (n && (!priv_records || !pub_records || !status))) return fail("null argument");
	if (priv_len < ctx->qlen || priv_len > 252) return fail("priv_len must be in [qlen, 252]");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	const size_t pl = ctx->plen, ql = ctx->qlen, in_b = (size_t)n * (3 + priv_len), out_b = (size_t)n * (3 + 3 * pl);
	DevArena a;
	const size_t i_in = a.reserve(in_b), i_sc = a.reserve((size_t)n * ql), i_aff = a.reserve((size_t)n * 2 * pl),
		     i_st = a.reserve(n), i_out = a.reserve(out_b);
	if (a.commit()) return fail("cudaMalloc failed");
	CUDA_OK(cudaMemcpy(a.get(i_in), priv_records, in_b, cudaMemcpyHostToDevice));
	int8_t *d_st = (int8_t *)a.get(i_st);
	k_struct_unpack<<<grid_bytes((uint64_t)n * ql), 256>>>(n, a.get(i_in), 3 + priv_len, priv_len, a.get(i_sc),
							      (uint32_t)ql);
	if (smul_dev(ctx, n, a.get(i_sc), nullptr, a.get(i_aff), d_st, ctx->jac, ctx->prefix, 0)) return -1;
	int rc = dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		LaunchMisc<C>::scalar_below_order(n, a.get(i_sc), d_st, 0);
		return 0;
	});
	if (rc) return rc;
	k_struct_check<<<grid_for(n), kThreads>>>(n, a.get(i_in), 3 + priv_len, 1 /* EC_PRIVKEY */, (uint8_t)alg,
						  (uint8_t)ctx->curve_id, priv_len - (uint32_t)ql, d_st);
	k_struct_pack_pub<<<grid_bytes(out_b), 256>>>(n, a.get(i_aff), (uint32_t)pl, d_st, 0, (uint8_t)alg,
						     (uint8_t)ctx->curve_id, a.get(i_out));
	ctx->launches += 4;
	CUDA_OK(cudaGetLastError());
	CUDA_OK(cudaMemcpy(pub_records, a.get(i_out), out_b, cudaMemcpyDeviceToHost));
	CUDA_OK(cudaMemcpy(status, d_st, n, cudaMemcpyDeviceToHost));
	return 0;
}

/* ECDSA verification on the reference's record formats: structured signatures (3 + 2*qlen bytes,
 * ec_structured_sig_import_from_buf sig/sig_algs.c:702) and structured public keys (3 + 3*plen bytes), digests as in
 * eccb200_ecdsa_verify_batch.  A record whose header does not name (alg, hash_type, this curve) / (EC_PUBKEY, alg, this
 * curve) fails like the reference's callers fail it (tests/ec_utils.c verify path); a key imported as the point at
 * infinity is verified the way the reference's complete formulas do (W' = u*G). */
extern "C" int eccb200_ecdsa_verify_structured_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sig_records,
						       const uint8_t *pub_records, int alg, int hash_type,
						       const uint8_t *digests, uint32_t hlen, int8_t *verdict)
{
	if (!ctx || (n && (!sig_records || !pub_records || !digests || !verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	const size_t pl = ctx->plen, ql = ctx->qlen, sr_b = (size_t)n * (3 + 2 * ql), pr_b = (size_t)n * (3 + 3 * pl);
	DevArena a;
	const size_t i_sr = a.reserve(sr_b), i_pr = a.reserve(pr_b), i_dg = a.reserve((size_t)n * hlen),
		     i_sig = a.reserve((size_t)n * 2 * ql), i_prj = a.reserve((size_t)n * 3 * pl),
		     i_aff = a.reserve((size_t)n * 2 * pl), i_st = a.reserve(n), i_v = a.reserve(n);
	if (a.commit()) return fail("cudaMalloc failed");
	CUDA_OK(cudaMemcpy(a.get(i_sr), sig_records, sr_b, cudaMemcpyHostToDevice));
	CUDA_OK(cudaMemcpy(a.get(i_pr), pub_records, pr_b, cudaMemcpyHostToDevice));
	CUDA_OK(cudaMemcpy(a.get(i_dg), digests, (size_t)n * hlen, cudaMemcpyHostToDevice));
	int8_t *d_st = (int8_t *)a.get(i_st);
	if (structured_pub_import_dev(ctx, n, a.get(i_pr), alg, a.get(i_prj), a.get(i_aff), d_st, 0)) return -1;
	k_struct_unpack<<<grid_bytes((uint64_t)n * 2 * ql), 256>>>(n, a.get(i_sr), (uint32_t)(3 + 2 * ql),
								  (uint32_t)(2 * ql), a.get(i_sig), (uint32_t)(2 * ql));
	k_struct_check<<<grid_for(n), kThreads>>>(n, a.get(i_sr), (uint32_t)(3 + 2 * ql), (uint8_t)alg, (uint8_t)hash_type,
						  (uint8_t)ctx->curve_id, 0, d_st);
	int rc = dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		LaunchVerify<C>::verify(n, a.get(i_sig), a.get(i_aff), a.get(i_dg), hlen, ctx->table, ctx->w,
					(int8_t *)a.get(i_v), 0, d_st);
		return 0;
	});
	if (rc) return rc;
	ctx->launches += 3;
	CUDA_OK(cudaGetLastError());
	CUDA_OK(cudaMemcpy(verdict, a.get(i_v), n, cudaMemcpyDeviceToHost));
	return 0;
}

/* ECDSA signing on the record formats: structured private keys in, structured signatures (3 + 2*qlen bytes) out;
 * nonces and digests as in eccb200_ecdsa_sign_batch.  status as there (0 / 2 retry / -1), -1 also for a bad record. */
extern "C" int eccb200_ecdsa_sign_structured_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *priv_records,
						     uint32_t priv_len, int alg, int hash_type, const uint8_t *nonces,
						     const uint8_t *digests, uint32_t hlen, uint8_t *sig_records,
						     int8_t *status)
{
	if (!ctx || (n && (!priv_records || !nonces || !digests || !sig_records || !status))) return fail("null argument");
	if (priv_len < ctx->qlen || priv_len > 252) return fail("priv_len must be in [qlen, 252]");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	const size_t ql = ctx->qlen, in_b = (size_t)n * (3 + priv_len), out_b = (size_t)n * (3 + 2 * ql);
	DevArena a;
	const size_t i_in = a.reserve(in_b), i_d = a.reserve((size_t)n * ql), i_k = a.reserve((size_t)n * ql),
		     i_dg = a.reserve((size_t)n * hlen), i_sig = a.reserve((size_t)n * 2 * ql), i_st = a.reserve(n),
		     i_out = a.reserve(out_b);
	if (a.commit()) return fail("cudaMalloc failed");
	CUDA_OK(cudaMemcpy(a.get(i_in), priv_records, in_b, cudaMemcpyHostToDevice));
	CUDA_OK(cudaMemcpy(a.get(i_k), nonces, (size_t)n * ql, cudaMemcpyHostToDevice));
	CUDA_OK(cudaMemcpy(a.get(i_dg), digests, (size_t)n * hlen, cudaMemcpyHostToDevice));
	int8_t *d_st = (int8_t *)a.get(i_st);
	k_struct_unpack<<<grid_bytes((uint64_t)n * ql), 256>>>(n, a.get(i_in), 3 + priv_len, priv_len, a.get(i_d),
							      (uint32_t)ql);
	if (sign_dev(ctx, n, a.get(i_d), a.get(i_k), a.get(i_dg), hlen, a.get(i_sig), d_st, ctx->jac, ctx->prefix, ctx->aff,
		     0))
		return -1;
	k_struct_check<<<grid_for(n), kThreads>>>(n, a.get(i_in), 3 + priv_len, 1 /* EC_PRIVKEY */, (uint8_t)alg,
						  (uint8_t)ctx->curve_id, priv_len - (uint32_t)ql, d_st);
	k_struct_pack<<<grid_bytes(out_b), 256>>>(n, a.get(i_sig), (uint32_t)(2 * ql), d_st, (uint8_t)alg,
						 (uint8_t)hash_type, (uint8_t)ctx->curve_id, a.get(i_out));
	ctx->launches += 3;
	CUDA_OK(cudaGetLastError());
	CUDA_OK(cudaMemcpy(sig_records, a.get(i_out), out_b, cudaMemcpyDeviceToHost));
	CUDA_OK(cudaMemcpy(status, d_st, n, cudaMemcpyDeviceToHost));
	return 0;
}

/* Page-locked host memory for callers that do not link CUDA themselves (cudaHostAlloc / cudaFreeHost). */
extern "C" void *eccb200_host_alloc(size_t bytes)
{
	void *p = nullptr;
	if (cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) {
		cudaGetLastError();
		g_err = "cudaHostAlloc failed";
		return nullptr;
	}
	return p;
}

/* Write-combined page-locked memory: for INPUT buffers the host only writes (reads of it by the CPU are slow);
 * host->device DMA out of write-combined memory skips the CPU cache snoops. */
extern "C" void *eccb200_host_alloc_input(size_t bytes)
{
	void *p = nullptr;
	if (cudaHostAlloc(&p, bytes, cudaHostAllocWriteCombined | cudaHostAllocPortable) != cudaSuccess) {
		cudaGetLastError();
		g_err = "cudaHostAlloc(write-combined) failed";
		return nullptr;
	}
	return p;
}

extern "C" void eccb200_host_free(void *p)
{
	if (p) cudaFreeHost(p);
}

/* batched prj_pt_unique on homogeneous projective wire points; small host-pointer helper (not pipelined) */
extern "C" int eccb200_prj_pt_unique_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *prj, uint8_t *out,
					   int8_t *status)
{
	if (!ctx || (n && (!prj || !out || !status))) return fail("null argument");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	if (ensure_work(ctx, n)) return -1;
	const size_t in_b = (size_t)n * 3 * ctx->plen, out_b = (size_t)n * 2 * ctx->plen;
	if (ctx->unique_io_bytes < in_b + out_b + n) {
		cudaDeviceSynchronize();
		if (ctx->unique_io) cudaFree(ctx->unique_io);
		ctx->unique_io = nullptr;
		ctx->unique_io_bytes = 0;
		CUDA_OK(cudaMalloc(&ctx->unique_io, in_b + out_b + n));
		ctx->unique_io_bytes = in_b + out_b + n;
	}
	uint8_t *d = ctx->unique_io;
	if (cudaMemcpy(d, prj, in_b, cudaMemcpyHostToDevice) != cudaSuccess) return fail("H2D copy failed");
	return dispatch(ctx->curve_id, [&](auto c) {
		typedef decltype(c) C;
		scratch_enter(ctx, 0);
		LaunchMisc<C>::prj_unique(affine_grid(ctx, n), n, d, ctx->jac, ctx->prefix, d + in_b,
					  (int8_t *)(d + in_b + out_b), 0);
		scratch_leave(ctx, 0);
		ctx->launches += 2;
		CUDA_OK(cudaGetLastError());
		CUDA_OK(cudaMemcpy(out, d + in_b, out_b, cudaMemcpyDeviceToHost));
		CUDA_OK(cudaMemcpy(status, d + in_b + out_b, n, cudaMemcpyDeviceToHost));
		return 0;
	});
}

extern "C" int eccb200_fp_mul_monty_batch(eccb200_ctx *ctx, int which, uint32_t n, const uint8_t *a, const uint8_t *b,
					  uint8_t *out)
{
	if (!ctx || (n && (!a || !b || !out))) return fail("null argument");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	size_t bytes = (size_t)n * ctx->plen;
	uint8_t *d = nullptr;
	CUDA_OK(cudaMalloc(&d, 3 * bytes));
	int rc = 0;
	do {
		if (cudaMemcpy(d, a, bytes, cudaMemcpyHostToDevice) != cudaSuccess ||
		    cudaMemcpy(d + bytes, b, bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
			rc = fail("H2D copy failed");
			break;
		}
		rc = dispatch(ctx->curve_id, [&](auto c) {
			typedef decltype(c) C;
			LaunchMisc<C>::fp_mul(which, n, d, d + bytes, d + 2 * bytes, 0);
			ctx->launches += 1;
			CUDA_OK(cudaGetLastError());
			CUDA_OK(cudaMemcpy(out, d + 2 * bytes, bytes, cudaMemcpyDeviceToHost));
			return 0;
		});
	} while (0);
	cudaFree(d);
	return rc;
}

/* fp_add_monty / fp_sub_monty / fp_sqr_monty unit entry point (op 0 / 1 / 2), mod p (which = 0) or mod q (1) */
extern "C" int eccb200_fp_addsub_batch(eccb200_ctx *ctx, int which, int op, uint32_t n, const uint8_t *a,
				       const uint8_t *b, uint8_t *out)
{
	if (!ctx || (n && (!a || !b || !out))) return fail("null argument");
	if (op < 0 || op > 2) return fail("op must be 0 (add), 1 (sub) or 2 (sqr)");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	size_t bytes = (size_t)n * ctx->plen;
	uint8_t *d = nullptr;
	CUDA_OK(cudaMalloc(&d, 3 * bytes));
	int rc = 0;
	if (cudaMemcpy(d, a, bytes, cudaMemcpyHostToDevice) != cudaSuccess ||
	    cudaMemcpy(d + bytes, b, bytes, cudaMemcpyHostToDevice) != cudaSuccess)
		rc = fail("H2D copy failed");
	if (!rc)
		rc = dispatch(ctx->curve_id, [&](auto c) {
			typedef decltype(c) C;
			LaunchMisc<C>::fp_addsub(which, op, n, d, d + bytes, d + 2 * bytes, 0);
			ctx->launches += 1;
			CUDA_OK(cudaGetLastError());
			CUDA_OK(cudaMemcpy(out, d + 2 * bytes, bytes, cudaMemcpyDeviceToHost));
			return 0;
		});
	cudaFree(d);
	return rc;
}

extern "C" int eccb200_ecdsa_uv_batch(eccb200_ctx *ctx, uint32_t n, const uint8_t *sigs, const uint8_t *digests,
				      uint32_t hlen, uint8_t *out)
{
	if (!ctx || (n && (!sigs || !digests || !out))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	if (n == 0) return 0;
	CUDA_OK(cudaSetDevice(ctx->device));
	size_t sg = (size_t)n * 2 * ctx->qlen, dg = (size_t)n * hlen;
	uint8_t *d = nullptr;
	CUDA_OK(cudaMalloc(&d, 2 * sg + dg));
	int rc = 0;
	if (cudaMemcpy(d, sigs, sg, cudaMemcpyHostToDevice) != cudaSuccess ||
	    cudaMemcpy(d + 2 * sg, digests, dg, cudaMemcpyHostToDevice) != cudaSuccess)
		rc = fail("H2D copy failed");
	if (!rc)
		rc = dispatch(ctx->curve_id, [&](auto c) {
			typedef decltype(c) C;
			LaunchVerify<C>::uv(n, d, d + 2 * sg, hlen, d + sg, 0);
			ctx->launches += 1;
			CUDA_OK(cudaGetLastError());
			CUDA_OK(cudaMemcpy(out, d + sg, sg, cudaMemcpyDeviceToHost));
			return 0;
		});
	cudaFree(d);
	return rc;
}

/* Layout experiment entry point (DESIGN.md §3): out[i] = a[i] * b[i]^iters in the Montgomery sense, computed by the
 * production thread-per-element multiplier (striped = 0) or by the 8-lanes-per-element shuffle variant (striped = 1,
 * 256-bit curves only); *ms receives the kernel's device time. */
extern "C" int eccb200_fp_mul_chain_bench(eccb200_ctx *ctx, int striped, uint32_t n, const uint8_t *a,
					  const uint8_t *b, uint8_t *out, int iters, float *ms)
{
	if (!ctx || !a || !b || !out || !ms || n == 0 || (n & 3)) return fail("bad argument (n must be a multiple of 4)");
	if (striped && ctx->N != 8) return fail("striped variant exists for 8-word fields only");
	CUDA_OK(cudaSetDevice(ctx->device));
	size_t bytes = (size_t)n * ctx->plen;
	uint8_t *d = nullptr;
	CUDA_OK(cudaMalloc(&d, 3 * bytes));
	cudaEvent_t e0, e1;
	CUDA_OK(cudaEventCreate(&e0));
	CUDA_OK(cudaEventCreate(&e1));
	int rc = 0;
	if (cudaMemcpy(d, a, bytes, cudaMemcpyHostToDevice) != cudaSuccess ||
	    cudaMemcpy(d + bytes, b, bytes, cudaMemcpyHostToDevice) != cudaSuccess)
		rc = fail("H2D copy failed");
	if (!rc)
		rc = dispatch(ctx->curve_id, [&](auto c) {
			typedef decltype(c) C;
			for (int r = 0; r < 3; r++) { /* two warm-ups, keep the last timing */
				cudaEventRecord(e0, 0);
				LaunchMisc<C>::fp_mul_chain(striped, n, d, d + bytes, d + 2 * bytes, iters, 0);
				cudaEventRecord(e1, 0);
				CUDA_OK(cudaEventSynchronize(e1));
				ctx->launches += 1;
			}
			CUDA_OK(cudaGetLastError());
			CUDA_OK(cudaEventElapsedTime(ms, e0, e1));
			CUDA_OK(cudaMemcpy(out, d + 2 * bytes, bytes, cudaMemcpyDeviceToHost));
			return 0;
		});
	cudaEventDestroy(e0);
	cudaEventDestroy(e1);
	cudaFree(d);
	return rc;
}

/* ------------------------------------------------------------------------------------------ imad_peak */
/*
 * Integer multiply-add peak of the device: the denominator of the roofline (SURVEY.md §8d).  Every thread runs 8 independent 32x32+64 multiply-add chains (IMAD.WIDE.U32), enough
 * warps per SM to saturate the pipe.  Result: IMAD32 per second, best of 5 runs, and IMAD per clock per SM at the
 * SM clock the driver reports as current maximum.
 */
__global__ void __launch_bounds__(256) k_imad_peak(uint32_t *out, int iters, uint32_t seed)
{
	uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	uint32_t b = (seed ^ 0x9e3779b9u) + t;
	uint32_t l0 = t, l1 = t + 1, l2 = t + 2, l3 = t + 3, l4 = t + 4, l5 = t + 5, l6 = t + 6, l7 = t + 7;
	uint32_t h0 = seed, h1 = seed, h2 = seed, h3 = seed, h4 = seed, h5 = seed, h6 = seed, h7 = seed;
#pragma unroll 1
	for (int i = 0; i < iters; i++) {
#pragma unroll
		for (int u = 0; u < 4; u++) {
			/* chain j: (h_j:l_j) += l_{j+1} * b — the multiplicand changes every iteration, so nothing can be
			 * hoisted; the lo/hi pair is the same PTX idiom the field multiplier uses (fuses to IMAD.WIDE.U32) */
			asm volatile("mad.lo.cc.u32 %0, %1, %16, %0;\n\tmadc.hi.u32 %8, %1, %16, %8;\n\t"
				     "mad.lo.cc.u32 %1, %2, %16, %1;\n\tmadc.hi.u32 %9, %2, %16, %9;\n\t"
				     "mad.lo.cc.u32 %2, %3, %16, %2;\n\tmadc.hi.u32 %10, %3, %16, %10;\n\t"
				     "mad.lo.cc.u32 %3, %4, %16, %3;\n\tmadc.hi.u32 %11, %4, %16, %11;\n\t"
				     "mad.lo.cc.u32 %4, %5, %16, %4;\n\tmadc.hi.u32 %12, %5, %16, %12;\n\t"
				     "mad.lo.cc.u32 %5, %6, %16, %5;\n\tmadc.hi.u32 %13, %6, %16, %13;\n\t"
				     "mad.lo.cc.u32 %6, %7, %16, %6;\n\tmadc.hi.u32 %14, %7, %16, %14;\n\t"
				     "mad.lo.cc.u32 %7, %0, %16, %7;\n\tmadc.hi.u32 %15, %0, %16, %15;"
				     : "+r"(l0), "+r"(l1), "+r"(l2), "+r"(l3), "+r"(l4), "+r"(l5), "+r"(l6), "+r"(l7),
				       "+r"(h0), "+r"(h1), "+r"(h2), "+r"(h3), "+r"(h4), "+r"(h5), "+r"(h6), "+r"(h7)
				     : "r"(b));
		}
	}
	out[t] = l0 ^ l1 ^ l2 ^ l3 ^ l4 ^ l5 ^ l6 ^ l7 ^ h0 ^ h1 ^ h2 ^ h3 ^ h4 ^ h5 ^ h6 ^ h7;
}

extern "C" int eccb200_imad_peak(int device, double *imad32_per_s, double *imad_per_clk_per_sm)
{
	if (!imad32_per_s || !imad_per_clk_per_sm) return fail("null argument");
	CUDA_OK(cudaSetDevice(device));
	cudaDeviceProp prop;
	CUDA_OK(cudaGetDeviceProperties(&prop, device));
	const int blocks = prop.multiProcessorCount * 8, threads = 256, iters = 4096;
	uint32_t *d = nullptr;
	CUDA_OK(cudaMalloc(&d, (size_t)blocks * threads * sizeof(uint32_t)));
	cudaEvent_t e0, e1;
	CUDA_OK(cudaEventCreate(&e0));
	CUDA_OK(cudaEventCreate(&e1));
	double best = 0;
	for (int r = 0; r < 7; r++) {
		CUDA_OK(cudaEventRecord(e0));
		k_imad_peak<<<blocks, threads>>>(d, iters, 12345u + r);
		CUDA_OK(cudaEventRecord(e1));
		CUDA_OK(cudaEventSynchronize(e1));
		float ms = 0;
		CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
		double rate = (double)blocks * threads * iters * 32.0 / (ms * 1e-3);
		if (r >= 2 && rate > best) best = rate; /* first two runs are warm-up */
	}
	cudaEventDestroy(e0);
	cudaEventDestroy(e1);
	cudaFree(d);
	int clk_khz = 0;
	cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, device);
	*imad32_per_s = best;
	*imad_per_clk_per_sm = clk_khz ? best / ((double)clk_khz * 1e3) / prop.multiProcessorCount : 0;
	return 0;
}

/* ------------------------------------------------------------------------------------------ NUMA placement */
/*
 * Binds the CALLING host thread to the CPUs that are local to `device` (/sys/bus/pci/devices/<bdf>/local_cpulist,
 * intersected with the thread's current affinity).  Page-locked memory the thread allocates afterwards, and the
 * staging copies it performs, then sit on the GPU's NUMA node, so that eight GPUs of a two-socket box do not all DMA
 * through one socket's memory controllers (measured: bench.py e2e at N = 8).  Returns the number of CPUs bound to, 0 if
 * nothing was changed, -1 on error.
 */
#include <sched.h>
extern "C" int eccb200_bind_thread_near_device(int device)
{
	char bdf[64] = { 0 };
	if (cudaDeviceGetPCIBusId(bdf, (int)sizeof(bdf) - 1, device) != cudaSuccess) {
		cudaGetLastError();
		return fail("cudaDeviceGetPCIBusId failed");
	}
	for (char *p = bdf; *p; p++)
		if (*p >= 'A' && *p <= 'F') *p = (char)(*p - 'A' + 'a');
	std::string path = std::string("/sys/bus/pci/devices/") + bdf + "/local_cpulist";
	FILE *f = fopen(path.c_str(), "r");
	if (!f) return 0;
	char line[4096] = { 0 };
	const bool got = fgets(line, sizeof(line) - 1, f) != nullptr;
	fclose(f);
	if (!got) return 0;
	cpu_set_t cur, want;
	CPU_ZERO(&want);
	if (sched_getaffinity(0, sizeof(cur), &cur)) return 0;
	int count = 0;
	for (char *tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
		int a = 0, b = 0;
		if (sscanf(tok, "%d-%d", &a, &b) == 2) {
		} else if (sscanf(tok, "%d", &a) == 1) {
			b = a;
		} else {
			continue;
		}
		for (int c = a; c <= b && c < CPU_SETSIZE; c++)
			if (CPU_ISSET(c, &cur)) {
				CPU_SET(c, &want);
				count++;
			}
	}
	if (count == 0) return 0;
	if (sched_setaffinity(0, sizeof(want), &want)) return 0;
	return count;
}

/* ------------------------------------------------------------------------------------------ multi-device (one process) */
/*
 * SURVEY.md §8(b) "multi-GPU fan-out is internal", §8(e): a C host hands ONE batch to the library and the library
 * shards it.  Items are independent, so device g takes the contiguous range [g*n/G, (g+1)*n/G) and runs the ordinary
 * host-pointer pipeline of its own context on it (own streams, own comb table, own PCIe link), one host thread per
 * device; every device DMAs its results straight into the caller's output arrays at the shard's offset, so there is
 * no gather step at all.  Page-locked buffers must be visible to every device (eccb200_host_alloc allocates them
 * portable).
 */
struct eccb200_multi {
	std::vector<eccb200_ctx *> ctx;
};

extern "C" void eccb200_multi_destroy(eccb200_multi *m)
{
	if (!m) return;
	for (auto *c : m->ctx) eccb200_ctx_destroy(c);
	delete m;
}

extern "C" int eccb200_multi_create(eccb200_multi **out, int curve_id, const int *devices, int n_devices,
				    int comb_window)
{
	if (!out) return fail("null argument");
	*out = nullptr;
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
		return fail("no CUDA device: libecc_b200 has no CPU fallback");
	std::vector<int> devs;
	if (devices && n_devices > 0) devs.assign(devices, devices + n_devices);
	else
		for (int d = 0; d < ndev; d++) devs.push_back(d);
	if (devs.size() > 64) return fail("too many devices");
	eccb200_multi *m = new eccb200_multi();
	m->ctx.assign(devs.size(), nullptr);
	std::vector<int> rc(devs.size(), 0);
	std::vector<std::string> msg(devs.size());
	std::vector<std::thread> th;
	for (size_t g = 0; g < devs.size(); g++) /* the comb tables are built concurrently, one host thread per device */
		th.emplace_back([&, g] {
			eccb200_bind_thread_near_device(devs[g]); /* the context's pinned staging lands on the GPU's NUMA node */
			rc[g] = eccb200_ctx_create(&m->ctx[g], curve_id, devs[g], comb_window);
			if (rc[g]) msg[g] = eccb200_last_error();
		});
	for (auto &t : th) t.join();
	for (size_t g = 0; g < devs.size(); g++)
		if (rc[g]) {
			std::string e = "device " + std::to_string(devs[g]) + ": " + msg[g];
			eccb200_multi_destroy(m);
			return fail(e);
		}
	*out = m;
	return 0;
}

extern "C" int eccb200_multi_device_count(const eccb200_multi *m) { return m ? (int)m->ctx.size() : -1; }
extern "C" eccb200_ctx *eccb200_multi_ctx(eccb200_multi *m, int index)
{
	return (m && index >= 0 && index < (int)m->ctx.size()) ? m->ctx[index] : nullptr;
}

template <class Fn> static int multi_run(eccb200_multi *m, uint64_t n, Fn &&fn)
{
	if (!m) return fail("null argument");
	const size_t G = m->ctx.size();
	if (n / G >= 0xffffffffull) return fail("shard too large (2^32 - 1 items per device)");
	std::vector<int> rc(G, 0);
	std::vector<std::string> msg(G);
	std::vector<std::thread> th;
	for (size_t g = 0; g < G; g++) {
		const uint64_t lo = n * g / G, hi = n * (g + 1) / G;
		if (hi == lo) continue;
		th.emplace_back([&, g, lo, hi] {
			eccb200_bind_thread_near_device(m->ctx[g]->device);
			rc[g] = fn(m->ctx[g], lo, (uint32_t)(hi - lo));
			if (rc[g]) msg[g] = eccb200_last_error();
		});
	}
	for (auto &t : th) t.join();
	for (size_t g = 0; g < G; g++)
		if (rc[g]) return fail("device shard " + std::to_string(g) + ": " + msg[g]);
	return 0;
}

extern "C" int eccb200_multi_prj_pt_mul_batch(eccb200_multi *m, uint64_t n, const uint8_t *scalars,
					      const uint8_t *points, uint8_t *out, int8_t *status)
{
	if (!m || (n && (!scalars || !out || !status))) return fail("null argument");
	const size_t ql = m->ctx[0]->qlen, pl = 2 * (size_t)m->ctx[0]->plen;
	return multi_run(m, n, [&](eccb200_ctx *c, uint64_t lo, uint32_t cnt) {
		return eccb200_prj_pt_mul_batch(c, cnt, scalars + lo * ql, points ? points + lo * pl : nullptr,
						out + lo * pl, status + lo);
	});
}

extern "C" int eccb200_multi_ecdsa_verify_batch(eccb200_multi *m, uint64_t n, const uint8_t *sigs,
						const uint8_t *pubkeys, const uint8_t *digests, uint32_t hlen,
						int8_t *verdict)
{
	if (!m || (n && (!sigs || !pubkeys || !digests || !verdict))) return fail("null argument");
	if (hlen == 0 || hlen > 128) return fail("bad digest length");
	const size_t sg = 2 * (size_t)m->ctx[0]->qlen, pk = 2 * (size_t)m->ctx[0]->plen;
	return multi_run(m, n, [&](eccb200_ctx *c, uint64_t lo, uint32_t cnt) {
		return eccb200_ecdsa_verify_batch(c, cnt, sigs + lo * sg, pubkeys + lo * pk, digests + lo * (size_t)hlen, hlen,
						  verdict + lo);
	});
}
