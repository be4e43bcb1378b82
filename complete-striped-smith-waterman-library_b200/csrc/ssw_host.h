/* ssw_host.h -- small host-side helpers shared by the engine sources. */
#ifndef SSW_HOST_H
#define SSW_HOST_H

#include <string.h>
#include <algorithm>
#include <atomic>
#include <map>
#include <mutex>
#include <thread>
#include <utility>
#include <vector>
#include "ssw_common.cuh"

/* counts device allocations and frees made through SswDevBuf: the engine re-reads the free device memory only when
 * this changed (cudaMemGetInfo costs milliseconds while a monitoring tool polls the driver) */
inline std::atomic<unsigned long long>& ssw_alloc_epoch() { static std::atomic<unsigned long long> n{1}; return n; }

/* engines currently inside an align call: every planner may claim 1 / (engines + 1) of the free device memory for its
 * scratch, so that several engines working on one device at the same time (helper engines of a sliced batch, concurrent
 * ssw_align callers, user-made engines in several threads) cannot claim the same half twice; idle engines do not count */
inline std::atomic<int>& ssw_live_engines(int device) { static std::atomic<int> n[64]; return n[device & 63]; }      /* per device: engines of a device group do not share memory */
struct SswBusyGuard { int dev; explicit SswBusyGuard(int device) : dev(device) { ++ssw_live_engines(dev); } ~SswBusyGuard() { --ssw_live_engines(dev); } };
inline size_t ssw_budget_share(size_t bytes)
{
	int dev = 0;
	cudaGetDevice(&dev);          /* the engine made its device current on entry */
	const int n = ssw_live_engines(dev).load();
	return bytes / (size_t)((n < 1 ? 1 : n) + 1);
}

/* 64-bit content hash (four interleaved multiply-xor lanes over 8-byte words): the resident-reference cache of ssw_align */
inline uint64_t ssw_hash_bytes(const void* data, size_t len)
{
	const unsigned char* p = (const unsigned char*)data;
	uint64_t h[4] = {0x9E3779B97F4A7C15ull, 0xC2B2AE3D27D4EB4Full, 0x165667B19E3779F9ull, 0x27D4EB2F165667C5ull};
	size_t i = 0;
	for (; i + 32 <= len; i += 32) {
		uint64_t w[4];
		memcpy(w, p + i, 32);
		for (int k = 0; k < 4; ++k) { h[k] = (h[k] ^ w[k]) * 0x100000001B3ull; h[k] ^= h[k] >> 29; }
	}
	uint64_t tail[4] = {0, 0, 0, 0};
	memcpy(tail, p + i, len - i);
	for (int k = 0; k < 4; ++k) { h[k] = (h[k] ^ tail[k]) * 0x100000001B3ull; h[k] ^= h[k] >> 29; }
	uint64_t r = (uint64_t)len;
	for (int k = 0; k < 4; ++k) { r = (r ^ h[k]) * 0x9E3779B97F4A7C15ull; r ^= r >> 32; }
	return r;
}

/* grow-only device buffer */
struct SswDevBuf {
	void* p = nullptr;
	size_t cap = 0;
	bool borrowed = false;          /* a view of another engine's buffer: never freed or grown here */
	void borrow(const SswDevBuf& o) { if (!borrowed && p) { ++ssw_alloc_epoch(); cudaFree(p); } p = o.p; cap = o.cap; borrowed = true; }
	int ensure(size_t bytes)
	{
		if (bytes <= cap) return 0;
		if (borrowed) { fprintf(stderr, "[libssw-b200] internal: a borrowed buffer cannot grow\n"); return -1; }
		++ssw_alloc_epoch();
		if (p) cudaFree(p);
		p = nullptr; cap = 0;
		size_t want = bytes + bytes / 8 + 256;
		if (cudaMalloc(&p, want) != cudaSuccess) {
			fprintf(stderr, "[libssw-b200] device allocation of %zu bytes failed\n", want);
			return -1;
		}
		cap = want;
		return 0;
	}
	void release() { if (!borrowed) { ++ssw_alloc_epoch(); if (p) cudaFree(p); } p = nullptr; cap = 0; borrowed = false; }
	template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

/* opt a kernel into more than 48 KB of dynamic shared memory, once per (device, kernel, size): the attribute call costs
 * microseconds that a one-pair ssw_align would otherwise pay on every launch */
inline int ssw_ensure_dyn_smem(const void* fn, size_t smem)
{
	if (smem <= 48 * 1024) return 0;
	static std::mutex mu;
	static std::map<std::pair<int, const void*>, size_t> granted;
	int dev = 0;
	cudaGetDevice(&dev);
	std::lock_guard<std::mutex> lock(mu);
	size_t& have = granted[std::make_pair(dev, fn)];
	if (have >= smem) return 0;
	if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
	have = smem;
	return 0;
}

/* Ask for the largest shared-memory carve-out for a kernel, once per (device, kernel).  An SM's L1 / shared-memory split can
 * only change while the SM is idle, so launches whose carve-outs differ do not share an SM: the traceback launches of one
 * round (same kernel, row rings of 16 / 32 / 64 KB per CTA) can start far apart although all their CTAs would fit at once.  With one carve-out for every kernel of the long-read phases (traceback,
 * strip fills) their CTAs go wherever registers and shared memory are free. */
inline int ssw_prefer_max_smem(const void* fn)
{
#ifndef SSW_CPU_EMU
	static std::mutex mu;
	static std::map<std::pair<int, const void*>, bool> done;
	int dev = 0;
	cudaGetDevice(&dev);
	std::lock_guard<std::mutex> lock(mu);
	bool& d = done[std::make_pair(dev, fn)];
	if (d) return 0;
	if (cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared) != cudaSuccess) return -1;
	d = true;
#else
	(void)fn;
#endif
	return 0;
}

/* free memory of the current device, re-read only after one of our buffers was (re)allocated */
inline size_t ssw_free_device_bytes()
{
	static std::mutex mu;
	static size_t cache[64];
	static unsigned long long epoch[64];
	int dev = 0;
	cudaGetDevice(&dev);
	dev &= 63;
	std::lock_guard<std::mutex> lock(mu);
	const unsigned long long now = ssw_alloc_epoch().load();
	if (epoch[dev] != now) {
		size_t free_b = 0, total_b = 0;
		cudaMemGetInfo(&free_b, &total_b);
		cache[dev] = free_b;
		epoch[dev] = now;
	}
	return cache[dev];
}

/* Large device -> pageable-host copies: a plain cudaMemcpy into pageable memory runs at a few GB/s (the driver stages
 * it through one small pinned buffer).  This stages through two pinned 8 MB buffers: the copy of chunk k+1 runs while the
 * host moves chunk k to its destination. */
#ifndef SSW_D2H_CHUNK
#define SSW_D2H_CHUNK ((size_t)8 << 20)      /* the emulator build uses a tiny value so that CPU tests cross chunk borders */
#endif
struct SswStagedD2H {
	void* pin[2] = {nullptr, nullptr};
	cudaEvent_t ev[2] = {nullptr, nullptr};
	static constexpr size_t CHUNK = SSW_D2H_CHUNK;
	int copy(void* dst, const void* src_dev, size_t bytes, cudaStream_t st)
	{
		if (bytes < 2 * CHUNK) {
			if (cudaMemcpyAsync(dst, src_dev, bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return -1;
			return cudaStreamSynchronize(st) == cudaSuccess ? 0 : -1;
		}
		for (int i = 0; i < 2; ++i)
			if (!pin[i]) {
				if (cudaMallocHost(&pin[i], CHUNK) != cudaSuccess || cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming) != cudaSuccess) return -1;
			}
		const size_t n = (bytes + CHUNK - 1) / CHUNK;
		for (size_t k = 0; k <= n; ++k) {
			if (k < n) {
				const size_t len = k + 1 < n ? CHUNK : bytes - k * CHUNK;
				if (cudaMemcpyAsync(pin[k & 1], (const char*)src_dev + k * CHUNK, len, cudaMemcpyDeviceToHost, st) != cudaSuccess) return -1;
				cudaEventRecord(ev[k & 1], st);
			}
			if (k > 0) {
				const size_t j = k - 1, len = j + 1 < n ? CHUNK : bytes - j * CHUNK;
				if (cudaEventSynchronize(ev[j & 1]) != cudaSuccess) return -1;
				/* the destination is often freshly allocated memory: four threads share the copy (and its page faults) */
				char* d = (char*)dst + j * CHUNK;
				const char* sp = (const char*)pin[j & 1];
				const size_t q = (len / 4 + 4095) & ~(size_t)4095;
				std::thread th[3];
				int nt = 0;
				for (int t = 1; t < 4 && (size_t)t * q < len; ++t, ++nt) {
					const size_t o = (size_t)t * q, l = std::min(q, len - o);
					th[nt] = std::thread([=]() { memcpy(d + o, sp + o, l); });
				}
				memcpy(d, sp, std::min(q, len));
				for (int t = 0; t < nt; ++t) th[t].join();
			}
		}
		return 0;
	}
	void release()
	{
		for (int i = 0; i < 2; ++i) { if (pin[i]) cudaFreeHost(pin[i]); if (ev[i]) cudaEventDestroy(ev[i]); pin[i] = nullptr; ev[i] = nullptr; }
	}
};

/* internal entry points shared by ssw_engine.cu and ssw_capi.cu (not part of the public headers) */
struct ssw_engine;
extern "C" int ssw_engine_set_pair(ssw_engine* e, const int8_t* read, int32_t readLen, const int8_t* ref, int32_t refLen);
int ssw_default_engines_option(const char* name, int64_t value);     /* ssw_engine_set_option(NULL, ...): the engines behind ssw_align */
bool ssw_engine_has_option(const char* name);                        /* is `name` an option of ssw_engine_set_option */

/* Phase times without synchronising: start/stop only record events on the stream; the elapsed times are read and added
 * to their accumulators by collect(), once, after the call's final synchronisation.  (A stopwatch that waits for its stop
 * event costs one host<->device round trip per kernel: three per phase of a one-pair ssw_align.) */
struct SswLaps {
	struct Lap { cudaEvent_t a, b; float* acc; };
	std::vector<cudaEvent_t> pool;
	std::vector<Lap> laps;
	size_t used = 0;
	cudaEvent_t cur = nullptr;
	cudaEvent_t get() { if (used == pool.size()) { cudaEvent_t ev = nullptr; cudaEventCreate(&ev); pool.push_back(ev); } return pool[used++]; }
	void start(cudaStream_t s) { cur = get(); cudaEventRecord(cur, s); }
	void stop(cudaStream_t s, float* acc) { cudaEvent_t b = get(); cudaEventRecord(b, s); laps.push_back(Lap{cur, b, acc}); }
	/* all recorded events must have completed (the caller has synchronised the stream) */
	void collect()
	{
		for (const Lap& l : laps) { float ms = 0; if (cudaEventElapsedTime(&ms, l.a, l.b) == cudaSuccess) *l.acc += ms; }
		laps.clear(); used = 0;
	}
	~SswLaps() { for (cudaEvent_t ev : pool) if (ev) cudaEventDestroy(ev); }
};

/* CUDA-event stopwatch on one stream */
struct SswTimer {
	cudaEvent_t a = nullptr, b = nullptr;
	void start(cudaStream_t s) { if (!a) { cudaEventCreate(&a); cudaEventCreate(&b); } cudaEventRecord(a, s); }
	float stop(cudaStream_t s) { cudaEventRecord(b, s); cudaEventSynchronize(b); float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms; }
	~SswTimer() { if (a) { cudaEventDestroy(a); cudaEventDestroy(b); } }
};

#endif
