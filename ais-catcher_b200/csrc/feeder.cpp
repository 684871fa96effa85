// Ingest (SURVEY.md 8f rank 4): one recorded IQ file per input row feeding one engine (n_streams of them, or n_streams / per_input
// behind a fan of tunings, aisgpu_set_tunings) -- the batch form of the reference's
// Device::RAWFile (Source/Device/FileRAW.cpp:36-165): each file is read in fixed blocks, the last block of a file is
// zero-padded (FileRAW.cpp:91-94), and the stream of blocks ends when the longest file has been consumed (shorter files
// keep delivering zeros, which is what a silent receiver looks like to the models).  WAV recordings are read the same way
// from the start of their data chunk, whose position the header walk of the reference's Device::WAVFile gives
// (Source/Device/FileWAV.cpp:49-120).
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

// reads one block of every input in [s0, s1) into dst (input-major); returns through `live` whether any file still had data
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

int check_args(aisgpu_handle *h, const char *who, const char *const *paths, int n_samples) {
	if (!h) return AISGPU_EINVAL;
	if (aisgpu_internal_grouped(h)) {
		aisgpu_internal_set_error(h, (std::string(who) + ": not available for an engine group (aisgpu_attach)").c_str());
		return AISGPU_EINVAL;
	}
	if (!paths || n_samples <= 0 || n_samples > aisgpu_internal_config(h)->max_chunk_samples) {
		aisgpu_internal_set_error(h, (std::string(who) + ": bad argument").c_str());
		return AISGPU_EINVAL;
	}
	return 0;
}

// The blocks of every input row, row s read from byte offsets[s] of paths[s] (offsets == NULL: from the start) to its end.
int feed(aisgpu_handle *h, const char *who, const char *const *paths, const int64_t *offsets, int n_samples, aisgpu_msg_fn fn, void *user,
		 uint64_t *n_blocks) {
	if (int rc = check_args(h, who, paths, n_samples)) return rc;
	const aisgpu_config *cfg = aisgpu_internal_config(h);
	const int B = aisgpu_internal_inputs(h);
	const size_t bps = cfg->format == AISGPU_FMT_CF32 ? 8 : (cfg->format == AISGPU_FMT_DC16H ? 12 : ((cfg->format == AISGPU_FMT_CS16 || cfg->format == AISGPU_FMT_F32_FS4) ? 4 : 2));
	const size_t block_bytes = (size_t)n_samples * bps;
	std::vector<Source> src((size_t)B);
	auto close_all = [&]() {
		for (auto &s : src)
			if (s.f) fclose(s.f);
	};
	for (int s = 0; s < B; s++) {
		src[s].f = paths[s] ? fopen(paths[s], "rb") : nullptr;
		if (src[s].f && offsets && fseeko(src[s].f, (off_t)offsets[s], SEEK_SET) != 0) {
			fclose(src[s].f);
			src[s].f = nullptr;
		}
		if (!src[s].f) { // the reference: "FILE: cannot open input file" thrown from RAWFile::Open (FileRAW.cpp:189-193)
			aisgpu_internal_set_error(h, (std::string(who) + ": cannot open input file \"" + (paths[s] ? paths[s] : "(null)") + "\"").c_str());
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
			aisgpu_internal_set_error(h, (std::string(who) + ": pinned host allocation failed").c_str());
			return AISGPU_ENOMEM;
		}
	const int T = (int)std::max(1u, std::min(std::min(std::thread::hardware_concurrency(), 16u), (unsigned)B));
	auto fill = [&](unsigned char *dst) { // one block of every input, files shared out over T threads; false once all files are drained
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

// WAVFile::Open's header walk (FileWAV.cpp:49-98) on an open file: "" and the file left at the first byte of the data chunk, or
// the reference's error text.  Partial reads store what they got, as std::istream::read does, and a skip past the end leaves
// nothing more to read, as std::istream::ignore does.
std::string wav_header(FILE *f, const char *path, int32_t *format, uint32_t *sample_rate) {
	uint32_t riff[3];
	if (fread(riff, 1, sizeof(riff), f) != sizeof(riff)) return std::string("cannot read header from WAV file: \"") + path + "\"";
	if (riff[0] != 0x46464952 || riff[2] != 0x45564157) return "not a supported WAV-file."; // "RIFF" ... "WAVE"
	struct {
		uint16_t wFormatTag, wChannels;
		uint32_t dwSamplesPerSec, dwAvgBytesPerSec;
		uint16_t wBlockAlign, wBitsPerSample;
	} fmt = { 0, 0, 0, 0, 0, 0 };
	static_assert(sizeof(fmt) == 16, "the fmt chunk's first 16 bytes");
	uint32_t chunk[2] = { 0, 0 }; // ID, size
	bool fmt_seen = false;
	while (fread(chunk, 1, sizeof(chunk), f) == sizeof(chunk)) {
		if (chunk[0] == 0x20746d66) { // "fmt "
			if (chunk[1] < sizeof(fmt)) return "invalid fmt chunk in WAV-file.";
			if (fread(&fmt, 1, sizeof(fmt), f) != sizeof(fmt)) return "cannot read fmt chunk from WAV-file.";
			fseeko(f, (off_t)(chunk[1] - sizeof(fmt) + (chunk[1] & 1)), SEEK_CUR);
			fmt_seen = true;
		}
		else if (chunk[0] == 0x61746164) // "data"
			break;
		else
			fseeko(f, (off_t)chunk[1] + (chunk[1] & 1), SEEK_CUR); // chunks are word-aligned
	}
	if (chunk[0] != 0x61746164 || !fmt_seen) return "no data in WAV-file.";
	if (fmt.wChannels != 2) return "WAV-file must have 2 channels (I/Q).";
	if (fmt.wFormatTag == 3 && fmt.wBitsPerSample == 32) *format = AISGPU_FMT_CF32;
	else if (fmt.wFormatTag == 1 && fmt.wBitsPerSample == 8) *format = AISGPU_FMT_CU8;
	else if (fmt.wFormatTag == 1 && fmt.wBitsPerSample == 16) *format = AISGPU_FMT_CS16;
	else return "format not supported";
	*sample_rate = fmt.dwSamplesPerSec;
	return "";
}

// "" and the header's fields, or the reference's error text
std::string wav_probe(const char *path, int32_t *format, uint32_t *sample_rate, int64_t *data_offset) {
	FILE *f = fopen(path, "rb");
	if (!f) return std::string("cannot open WAV file: \"") + path + "\"";
	std::string err = wav_header(f, path, format, sample_rate);
	// after a data chunk header cut short at the end of the file this is the file's size: the reference reads no sample
	*data_offset = (int64_t)ftello(f);
	fclose(f);
	return err;
}

const char *format_name(int32_t f) {
	switch (f) {
	case AISGPU_FMT_CF32: return "CF32";
	case AISGPU_FMT_CU8: return "CU8";
	case AISGPU_FMT_CS8: return "CS8";
	case AISGPU_FMT_CS16: return "CS16";
	case AISGPU_FMT_F32_FS4: return "F32_FS4";
	case AISGPU_FMT_DC16H: return "DC16H";
	default: return "?";
	}
}

} // namespace

extern "C" int aisgpu_feed_files(aisgpu_handle *h, const char *const *paths, int n_samples, aisgpu_msg_fn fn, void *user, uint64_t *n_blocks) {
	return feed(h, "aisgpu_feed_files", paths, nullptr, n_samples, fn, user, n_blocks);
}

extern "C" int aisgpu_wav_probe(const char *path, int32_t *format, uint32_t *sample_rate, int64_t *data_offset) {
	if (!path || !format || !sample_rate || !data_offset) {
		aisgpu_internal_set_error(nullptr, "aisgpu_wav_probe: null argument");
		return AISGPU_EINVAL;
	}
	int32_t fmt = 0;
	uint32_t rate = 0;
	int64_t off = 0;
	const std::string err = wav_probe(path, &fmt, &rate, &off);
	if (!err.empty()) {
		aisgpu_internal_set_error(nullptr, err.c_str());
		return AISGPU_EINVAL;
	}
	*format = fmt;
	*sample_rate = rate;
	*data_offset = off;
	return 0;
}

extern "C" int aisgpu_feed_wav_files(aisgpu_handle *h, const char *const *paths, int n_samples, aisgpu_msg_fn fn, void *user, uint64_t *n_blocks) {
	const char *who = "aisgpu_feed_wav_files";
	if (int rc = check_args(h, who, paths, n_samples)) return rc;
	const aisgpu_config *cfg = aisgpu_internal_config(h);
	const int B = aisgpu_internal_inputs(h);
	std::vector<int64_t> offsets((size_t)B);
	for (int s = 0; s < B; s++) {
		const std::string name = std::string(who) + ": \"" + (paths[s] ? paths[s] : "(null)") + "\": ";
		int32_t fmt = 0;
		uint32_t rate = 0;
		const std::string err = paths[s] ? wav_probe(paths[s], &fmt, &rate, &offsets[s]) : std::string("cannot open WAV file");
		std::string bad;
		if (!err.empty()) bad = err;
		else if (fmt != cfg->format)
			bad = std::string("format ") + format_name(fmt) + " differs from the engine's " + format_name(cfg->format);
		else if ((int64_t)rate != (int64_t)cfg->sample_rate)
			bad = "sample rate " + std::to_string(rate) + " differs from the engine's " + std::to_string(cfg->sample_rate);
		if (!bad.empty()) {
			aisgpu_internal_set_error(h, (name + bad).c_str());
			return AISGPU_EINVAL;
		}
	}
	return feed(h, who, paths, offsets.data(), n_samples, fn, user, n_blocks);
}
