// Ingest (SURVEY.md 8f rank 4): n_streams recorded IQ files feeding one engine -- the batch form of the reference's
// Device::RAWFile (Source/Device/FileRAW.cpp:36-165): each file is read in fixed blocks, the last block of a file is
// zero-padded (FileRAW.cpp:91-94), and the stream of blocks ends when the longest file has been consumed (shorter files
// keep delivering zeros, which is what a silent receiver looks like to the models).
//
// Two pinned host buffers: reader threads fill buffer c+1 from the files while the copy and the kernels of block c are in
// flight (aisgpu_submit_async), and the frames of block c-1 are handed to the callback.  Everything goes through the
// public C ABI; the only CUDA calls are the pinned allocations.

#include "../../include/aisgpu.h"
#include "host_internal.h"

#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <string>
#include <thread>
#include <vector>

namespace {

struct Source {
	FILE *f = nullptr;
	bool eof = false;
};

// reads one block of every stream in [s0, s1) into dst (stream-major); returns through `live` whether any file still had data
void read_block(std::vector<Source> &src, int s0, int s1, unsigned char *dst, size_t block_bytes, std::atomic<int> &live) {
	for (int s = s0; s < s1; s++) {
		unsigned char *p = dst + (size_t)s * block_bytes;
		size_t got = 0;
		if (!src[s].eof) {
			got = fread(p, 1, block_bytes, src[s].f);
			if (got < block_bytes) src[s].eof = true;
			if (got > 0) live.fetch_add(1, std::memory_order_relaxed);
		}
		if (got < block_bytes) memset(p + got, 0, block_bytes - got);
	}
}

} // namespace

extern "C" int aisgpu_feed_files(aisgpu_handle *h, const char *const *paths, int n_samples, aisgpu_msg_fn fn, void *user, uint64_t *n_blocks) {
	if (!h) return AISGPU_EINVAL;
	if (aisgpu_internal_grouped(h)) {
		aisgpu_internal_set_error(h, "aisgpu_feed_files: not available for an engine group (aisgpu_attach)");
		return AISGPU_EINVAL;
	}
	const aisgpu_config *cfg = aisgpu_internal_config(h);
	if (!paths || n_samples <= 0 || n_samples > cfg->max_chunk_samples) {
		aisgpu_internal_set_error(h, "aisgpu_feed_files: bad argument");
		return AISGPU_EINVAL;
	}
	const int B = cfg->n_streams;
	const size_t bps = cfg->format == AISGPU_FMT_CF32 ? 8 : (cfg->format == AISGPU_FMT_CS16 ? 4 : 2);
	const size_t block_bytes = (size_t)n_samples * bps;
	std::vector<Source> src((size_t)B);
	auto close_all = [&]() {
		for (auto &s : src)
			if (s.f) fclose(s.f);
	};
	for (int s = 0; s < B; s++) {
		src[s].f = paths[s] ? fopen(paths[s], "rb") : nullptr;
		if (!src[s].f) { // the reference: "FILE: cannot open input file" thrown from RAWFile::Open (FileRAW.cpp:189-193)
			aisgpu_internal_set_error(h, (std::string("aisgpu_feed_files: cannot open input file \"") + (paths[s] ? paths[s] : "(null)") + "\"").c_str());
			close_all();
			return AISGPU_EINVAL;
		}
	}
	unsigned char *pin[2] = { nullptr, nullptr };
	for (int i = 0; i < 2; i++)
		if (cudaMallocHost((void **)&pin[i], block_bytes * (size_t)B) != cudaSuccess) {
			cudaGetLastError();
			if (pin[0]) cudaFreeHost(pin[0]);
			close_all();
			aisgpu_internal_set_error(h, "aisgpu_feed_files: pinned host allocation failed");
			return AISGPU_ENOMEM;
		}
	const int T = (int)std::max(1u, std::min(std::min(std::thread::hardware_concurrency(), 16u), (unsigned)B));
	auto fill = [&](unsigned char *dst) { // one block of every stream, files shared out over T threads; false once all files are drained
		std::atomic<int> live(0);
		std::vector<std::thread> th;
		for (int t = 1; t < T; t++) th.emplace_back(read_block, std::ref(src), (int)((long long)B * t / T), (int)((long long)B * (t + 1) / T), dst, block_bytes, std::ref(live));
		read_block(src, 0, (int)((long long)B / T), dst, block_bytes, live);
		for (auto &x : th) x.join();
		return live.load() > 0;
	};
	std::vector<aisgpu_msg> msgs(256);
	auto drain = [&](int64_t ticket) {
		int rc_keep = 0;
		for (;;) {
			int n = 0;
			const int rc = aisgpu_poll_upto(h, ticket, msgs.data(), (int)msgs.size(), &n);
			if (rc != 0 && rc != AISGPU_EOVERFLOW) return rc;
			if (rc == AISGPU_EOVERFLOW) rc_keep = rc; // survivors are still delivered
			if (n > 0 && fn) fn(msgs.data(), n, user);
			if (n < (int)msgs.size()) return rc_keep;
		}
	};
	int rc = 0, overflow = 0;
	uint64_t blocks = 0;
	int64_t prev = -1;
	bool more = fill(pin[0]);
	for (int cur = 0; more && rc == 0; cur ^= 1) {
		int64_t ticket = -1;
		rc = aisgpu_submit_async(h, pin[cur], n_samples, &ticket);
		if (rc) break;
		blocks++;
		// pin[cur ^ 1] was the source of block `prev`: its copy must have completed before the readers overwrite it
		if (prev >= 0) {
			rc = drain(prev);
			if (rc == AISGPU_EOVERFLOW) { overflow = 1; rc = 0; }
			if (rc) break;
		}
		more = fill(pin[cur ^ 1]);
		prev = ticket;
	}
	if (rc == 0) {
		rc = drain(-1);
		if (rc == AISGPU_EOVERFLOW) { overflow = 1; rc = 0; }
	}
	else aisgpu_sync(h);
	cudaFreeHost(pin[0]);
	cudaFreeHost(pin[1]);
	close_all();
	if (n_blocks) *n_blocks = blocks;
	return rc ? rc : (overflow ? AISGPU_EOVERFLOW : 0);
}
