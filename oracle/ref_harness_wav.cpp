// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// The UNMODIFIED reference's Device::WAVFile (Source/Device/FileWAV.cpp), driven as the application drives it:
//   aisrefw_open : SetKey(FILE, path), Open(0); the format (as an AISGPU_FMT_* value: CF32 0, CU8 1, CS16 3), the sample rate and
//                  the read position after Open (-1 when the stream has failed), or the text of the exception Open threw.
//   aisrefw_read : the same, then Play() and isStreaming() until it returns false: every byte the device Sends as RAW samples.
// Built into oracle/_ref/libaisref_wav.so by oracle/wav.mk.

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "Device.h"
#include "FileWAV.h"

void StopRequest() {} // Source/Library/Common.h:72 -- the application normally defines it

namespace {

struct Bytes : public StreamIn<RAW> {
	std::vector<char> v;
	void Receive(const RAW *r, int len, TAG &) {
		for (int i = 0; i < len; i++) v.insert(v.end(), (const char *)r[i].data, (const char *)r[i].data + r[i].size);
	}
};

int fmt_id(Format f) {
	switch (f) {
	case Format::CF32: return 0;
	case Format::CU8: return 1;
	case Format::CS16: return 3;
	default: return -1;
	}
}

void copy_text(const std::string &s, char *err, long cap) {
	if (err && cap > 0) {
		strncpy(err, s.c_str(), (size_t)cap - 1);
		err[cap - 1] = 0;
	}
}

} // namespace

// 0 and *format / *rate / *pos, or -1 and the exception's text in err
extern "C" int aisrefw_open(const char *path, int *format, unsigned *rate, long long *pos, char *err, long cap) {
	Device::WAVFile d;
	try {
		d.SetKey(AIS::KEY_SETTING_FILE, path);
		d.Open(0);
	}
	catch (const std::exception &e) {
		copy_text(e.what(), err, cap);
		return -1;
	}
	*format = fmt_id(d.getFormat());
	*rate = d.getSampleRate();
	*pos = (long long)d.file.tellg();
	d.Close();
	return 0;
}

// the number of sample bytes the device delivers (copied to dst up to cap), or -1 and the exception's text in err
extern "C" long aisrefw_read(const char *path, void *dst, long cap, char *err, long errcap) {
	Device::WAVFile d;
	Bytes b;
	try {
		d.SetKey(AIS::KEY_SETTING_FILE, path);
		d.Open(0);
	}
	catch (const std::exception &e) {
		copy_text(e.what(), err, errcap);
		return -1;
	}
	d.out.Connect(&b);
	d.Play();
	while (d.isStreaming()) {
	}
	d.Stop();
	d.Close();
	if (dst) memcpy(dst, b.v.data(), std::min((size_t)cap, b.v.size()));
	return (long)b.v.size();
}
