// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// The UNMODIFIED reference's full AIS JSON (AIS::JSONAIS::ProcessMsg serialised by JSON::Serializer with JSON_DICT_FULL, the
// output of -o 5 / MSGFORMAT JSON_FULL) for one message built from raw fields:
//   aisrefj_line : payload bytes (at most MAX_AIS_BYTES are taken, the rest of the message is zero as after Message::clear), length,
//                  channel, the sentences to report under "nmea" (given, not rebuilt, so that the caller can hand the product the very
//                  same ones), station, rx time, toa, and the TAG fields the line prints.  Returns the line's length (no newline),
//                  or -1 if it does not fit in max.
// Built into oracle/_ref/libaisref_json.so by oracle/json.mk; checker for the product's aisgpu_msg_json_full and aisgpu_poll_json.

#include <cstdint>
#include <cstring>
#include <string>

#include "AIS.h"
#include "JSON/JSON.h"
#include "JSON/JSONAIS.h"
#include "JSON/Writer.h"

void StopRequest() {} // Source/Library/Common.h:72 -- the application normally defines it

extern "C" long aisrefj_line(const unsigned char *data, int nbytes, int nbits, int channel, int n_sent, const char *const *sent,
							 const int *sent_len, float level, float ppm, int version, int driver, const char *hardware, int mode,
							 long long rxtime_us, long long toa_us, int station, char *out, long max) {
	AIS::Message m;
	m.clear();
	m.setBytes(data, nbytes);
	m.setOrigin((char)channel, station, -1);
	m.setLength(nbits);
	m.setRxTimeMicros(rxtime_us);
	m.setTOA(toa_us);
	m.beginNMEA();
	for (int i = 0; i < n_sent; i++) m.pushNMEA(sent[i], (size_t)sent_len[i]);
	TAG tag;
	tag.mode = (unsigned)mode;
	tag.level = level;
	tag.ppm = ppm;
	tag.version = version;
	tag.driver = (Type)driver;
	tag.hardware = hardware ? hardware : "";
	AIS::JSONAIS j;
	j.json.clear();
	j.ProcessMsg(m, tag);
	JSON::Serializer s(JSON_DICT_FULL);
	std::string o;
	s.stringify(j.json, o);
	long n = (long)o.size();
	if (n > max) return -1;
	memcpy(out, o.data(), (size_t)n);
	return n;
}
