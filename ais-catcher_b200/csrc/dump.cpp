// The 48 kHz channel dump (-go DUMP <prefix>): the FilterCIC5 outputs C_a / C_b of every dumped stream as two stereo float WAV files,
// byte for byte what the reference's Util::ConvertToRAW >> Util::WriteWAV pair writes (Utilities/StreamHelpers.h:94-161,
// StreamHelpers.cpp:135-229):
//   - the 44-byte header is written when the first block arrives, with both sizes 0; audio_format 3 (IEEE float), 2 channels,
//     32 bits, 48000 S/s, byte_rate 384000, alignment 8;
//   - every block is appended raw (CF32, I then Q);
//   - at close, wav_size = data_size + 36 goes to offset 4 and data_size to offset 40, both truncated to uint32_t as the reference
//     does (they wrap past 4 GiB of data, about 3.1 h at 48 kHz);
//   - the first failed create or write stops the dump, with the reference's wording.  A file whose write failed is closed at once
//     and keeps its header as it was, as WriteWAV::Receive does.
// The engine (aisgpu.cu) hands this unit each submit's rows from a pinned slot, on the caller's thread.
#include "dump.h"

#include <stdint.h>
#include <string.h>
#include <sys/types.h>

namespace aisgpu {

namespace {

void put_u16(unsigned char *p, uint16_t v) {
	p[0] = (unsigned char)v;
	p[1] = (unsigned char)(v >> 8);
}
void put_u32(unsigned char *p, uint32_t v) {
	for (int i = 0; i < 4; i++) p[i] = (unsigned char)(v >> (8 * i));
}

// WriteWAV::WAVHeader after Open() for Format::CF32 at 48000 S/s (StreamHelpers.h:123-144, StreamHelpers.cpp:144-171)
void wav_header(unsigned char h[44]) {
	memcpy(h, "RIFF", 4);
	put_u32(h + 4, 0);
	memcpy(h + 8, "WAVE", 4);
	memcpy(h + 12, "fmt ", 4);
	put_u32(h + 16, 16);
	put_u16(h + 20, 3);
	put_u16(h + 22, 2);
	put_u32(h + 24, 48000);
	put_u32(h + 28, 48000 * 2 * 4);
	put_u16(h + 32, 2 * 4);
	put_u16(h + 34, 32);
	memcpy(h + 36, "data", 4);
	put_u32(h + 40, 0);
}

} // namespace

ChannelDump::ChannelDump(const char *const *prefixes, int n_streams) : files_((size_t)2 * n_streams) {
	for (int s = 0; s < n_streams; s++)
		if (prefixes[s]) {
			files_[2 * s].name = std::string(prefixes[s]) + "_A.wav"; // Model.cpp:390-396: literally A and B, in CD mode too
			files_[2 * s + 1].name = std::string(prefixes[s]) + "_B.wav";
		}
}

ChannelDump::~ChannelDump() { close(); }

bool ChannelDump::write(const float *rows, long long n) {
	if (failed()) return false;
	for (size_t r = 0; r < files_.size(); r++) {
		File &f = files_[r];
		if (f.name.empty()) continue;
		if (!f.fp) { // WriteWAV::Open at the first Receive
			f.fp = fopen(f.name.c_str(), "wb");
			if (!f.fp) {
				err_ = "WAV out: Cannot open WAV file for writing: \"" + f.name + "\"";
				return false;
			}
			unsigned char h[44];
			wav_header(h);
			if (fwrite(h, 1, sizeof(h), f.fp) != sizeof(h)) {
				err_ = "WAV out: Write error on WAV file \"" + f.name + "\"";
				return false;
			}
		}
		const size_t bytes = (size_t)n * 8;
		if (fwrite(rows + (size_t)r * 2 * n, 1, bytes, f.fp) != bytes) {
			err_ = "WAV out: write failed (disk full?) on \"" + f.name + "\"";
			fclose(f.fp);
			f.fp = nullptr;
			return false;
		}
	}
	return true;
}

bool ChannelDump::close() {
	for (File &f : files_) {
		if (!f.fp) continue;
		// WriteWAV::~WriteWAV: sizes from the write position, as uint32_t
		const long long data = (long long)ftello(f.fp) - 44;
		unsigned char v[4];
		put_u32(v, (uint32_t)(data + 36));
		fseeko(f.fp, 4, SEEK_SET);
		fwrite(v, 1, 4, f.fp);
		put_u32(v, (uint32_t)data);
		fseeko(f.fp, 40, SEEK_SET);
		fwrite(v, 1, 4, f.fp);
		fclose(f.fp);
		f.fp = nullptr;
	}
	return !failed();
}

} // namespace aisgpu
