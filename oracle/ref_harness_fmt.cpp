// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// The UNMODIFIED reference's output records: what IO::OutputMessage appends for one message in each MessageFormat
// (Source/Library/Common.h:144-156), for a message built from raw fields as ref_harness_json.cpp builds it.
//   aisreff_record     : NMEA, NMEA_TAG, COMMUNITY_HUB, BINARY_NMEA, FULL and JSON_NMEA through OutputMessage::formatInto
//                        (IO/MsgOut.h:58-122) of one output that lives as long as the library; JSON_SPARSE, JSON_FULL and
//                        JSON_ANNOTATED through JSONAIS::ProcessMsg and JSON::Serializer (setMap(JSON_DICT_SPARSE) /
//                        setStringifyEnhanced(true)), followed by the output's suffix, as OutputMessage::Receive(JSON) writes them.
//                        Returns the record's length, or -1 if it does not fit in max.
//   aisreff_hub        : that output's hub line count (COMMUNITY_HUB), set to v when v >= 0; returns the count before.
//   aisreff_group_seed : advances the process-wide group id of Message::getNMEATagBlock until the last group it handed out is g
//                        (g = 0 and g = 9999 both make the next group 1); returns the calls it took.
//   aisreff_key_count / aisreff_key: one member (key index, an int value) serialised under JSON_DICT_FULL, JSON_DICT_SPARSE or
//                        enhanced -- the key names, units, descriptions and lookup texts as the reference prints them, for
//                        tools/gen_fmt_text.py.
// Built into oracle/_ref/libaisref_fmt.so by oracle/fmt.mk; checker for the product's aisgpu_msg_format and aisgpu_poll_lines.

#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>

#include "AIS.h"
#include "JSON/JSON.h"
#include "JSON/JSONAIS.h"
#include "JSON/Writer.h"
#include "MsgOut.h"

void StopRequest() {} // Source/Library/Common.h:72 -- the application normally defines it

namespace {

IO::OutputMessage &output() {
	static IO::OutputMessage o;
	return o;
}

void build(AIS::Message &m, const unsigned char *data, int nbytes, int nbits, int channel, int n_sent, const char *const *sent,
		   const int *sent_len, long long rxtime_us, long long toa_us, int station, int start_idx, int end_idx) {
	m.clear();
	m.setBytes(data, nbytes);
	m.setOrigin((char)channel, station, -1);
	m.setLength(nbits);
	m.setRxTimeMicros(rxtime_us);
	m.setTOA(toa_us);
	m.setStartIdx(start_idx);
	m.setEndIdx(end_idx);
	m.beginNMEA();
	for (int i = 0; i < n_sent; i++) m.pushNMEA(sent[i], (size_t)sent_len[i]);
}

} // namespace

extern "C" long aisreff_record(int fmt, const unsigned char *data, int nbytes, int nbits, int channel, int n_sent,
							   const char *const *sent, const int *sent_len, float level, float ppm, int version, int driver,
							   const char *hardware, int mode, long long rxtime_us, long long toa_us, int station, int include_ssl,
							   int start_idx, int end_idx, const char *uuid, int status, unsigned ipv4, const char *suffix, char *out,
							   long max) {
	AIS::Message m;
	build(m, data, nbytes, nbits, channel, n_sent, sent, sent_len, rxtime_us, toa_us, station, start_idx, end_idx);
	TAG tag;
	tag.mode = (unsigned)mode;
	tag.level = level;
	tag.ppm = ppm;
	tag.version = version;
	tag.driver = (Type)driver;
	tag.hardware = hardware ? hardware : "";
	tag.status = status;
	tag.ipv4 = ipv4;
	IO::OutputMessage &o = output();
	o.fmt = (MessageFormat)fmt;
	o.include_sample_start = include_ssl != 0;
	o.uuid = uuid ? uuid : "";
	o.line_suffix = suffix ? suffix : "\r\n";
	std::string r;
	if (fmt == (int)MessageFormat::JSON_SPARSE || fmt == (int)MessageFormat::JSON_FULL || fmt == (int)MessageFormat::JSON_ANNOTATED) {
		AIS::JSONAIS j;
		j.json.clear();
		j.ProcessMsg(m, tag);
		JSON::Serializer s(fmt == (int)MessageFormat::JSON_SPARSE ? JSON_DICT_SPARSE : JSON_DICT_FULL);
		s.setStringifyEnhanced(fmt == (int)MessageFormat::JSON_ANNOTATED);
		s.stringify(j.json, r, o.line_suffix);
	}
	else {
		o.formatInto(m, tag);
		r = o.json;
	}
	long n = (long)r.size();
	if (n > max) return -1;
	memcpy(out, r.data(), (size_t)n);
	return n;
}

extern "C" long long aisreff_hub(long long v) {
	const long long before = (long long)output().hub_lines;
	if (v >= 0) output().hub_lines = (uint64_t)v;
	return before;
}

extern "C" int aisreff_group_seed(int g) {
	const int want = (g % 9999 == 0) ? 9999 : g;
	AIS::Message m;
	const unsigned char d[21] = { 0 };
	const char *sent[2] = { "!AIVDM,2,1,,A,0,0*00", "!AIVDM,2,2,,A,0,0*00" };
	const int len[2] = { 20, 20 };
	build(m, d, 21, 168, 'A', 2, sent, len, 0, 0, 0, 0, 0);
	for (int calls = 1; calls <= 10000; calls++) {
		std::string s;
		m.getNMEATagBlock(s);
		const size_t at = s.find(",g:1-2-");
		if (at != std::string::npos && atoi(s.c_str() + at + 7) == want) return calls;
	}
	return -1;
}

extern "C" int aisreff_key_count() { return AIS::KEY_COUNT; }

// key k with the int value v under dict (0: full, 2: sparse) or, with enhanced, annotated; the object's text, -1 if too long
extern "C" long aisreff_key(int k, int dict, int enhanced, int v, char *out, long max) {
	JSON::JSON j;
	j.Add(k, v);
	JSON::Serializer s(dict);
	s.setStringifyEnhanced(enhanced != 0);
	std::string r;
	s.stringify(j, r);
	long n = (long)r.size();
	if (n > max) return -1;
	memcpy(out, r.data(), (size_t)n);
	return n;
}
