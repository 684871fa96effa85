// dump.h -- the WAV writer behind aisgpu_dump_open (dump.cpp, host-only).
#pragma once
#include <stdio.h>

#include <string>
#include <vector>

namespace aisgpu {

// The 48 kHz channel streams of a batch as the reference's -go DUMP writes them for one receiver (Model.cpp:348-353, 390-396):
// C_a of stream s to "<prefixes[s]>_A.wav", C_b to "<prefixes[s]>_B.wav", through Util::WriteWAV (StreamHelpers.cpp:135-229).
class ChannelDump {
public:
	ChannelDump(const char *const *prefixes, int n_streams); // prefixes[s] == NULL: stream s is not written
	~ChannelDump();                                          // close()
	// Appends n CF32 samples of every row: rows[r * 2 n] holds row r = 2 s + channel.  Opens a file at its first write.  After the
	// first failure nothing more is written and this returns false.
	bool write(const float *rows, long long n);
	// Patches the sizes of every open file and closes it; false if a create or write ever failed.
	bool close();
	bool failed() const { return !err_.empty(); }
	const std::string &error() const { return err_; }

private:
	struct File {
		std::string name;
		FILE *fp = nullptr;
	};
	std::vector<File> files_; // one per row
	std::string err_;
};

} // namespace aisgpu
