// Egress formats for decoded frames (SURVEY.md 8f rank 4): what the reference's outputs make of an AIS::Message after the
// demodulation path has produced it.  Host-only entry points over the host build of the record formatter in be_json.cu, the
// code the engine runs on the device for aisgpu_poll_lines:
//
//   aisgpu_msg_json   == AIS::Message::getNMEAJSON   (Source/Marine/Message.cpp:93-191; number and string formatting of
//                        JSON::Writer, Source/JSON/Writer.h:124-218, 269-345, 427-442)
//   aisgpu_msg_binary == AIS::Message::getBinaryNMEA (Source/Marine/Message.cpp:277-396; CRC of Util::Helper::CRC16,
//                        Source/Utilities/Helper.cpp:42-57)
//
// Both return the number of bytes written, or AISGPU_EINVAL (bad argument) / AISGPU_EOVERFLOW (cap too small; nothing useful
// in out).  The reference appends to a std::string; here the caller provides the buffer.

#include "../../include/aisgpu.h"
#include "be_json.h"

#include <stdint.h>

extern "C" int aisgpu_msg_json(const aisgpu_msg *m, const aisgpu_tag *tag, char *out, int cap) {
	if (!m || !tag || !out || cap <= 0 || m->n_sentences < 0 || m->n_sentences > 4) return AISGPU_EINVAL;
	const AjPrefix no_prefix; // not printed by this format
	const FmtCtx c = fmt_ctx(tag, AISGPU_MSGFORMAT_JSON_NMEA, tag->suffix, no_prefix);
	return fmt_record_host(m, &c, 0, 0, out, cap);
}

extern "C" int aisgpu_msg_binary(const aisgpu_msg *m, const aisgpu_tag *tag, int crc, uint8_t *out, int cap) {
	if (!m || !tag || !out || cap <= 0) return AISGPU_EINVAL;
	const AjPrefix no_prefix; // not printed by this format
	FmtCtx c = fmt_ctx(tag, AISGPU_MSGFORMAT_BINARY_NMEA, nullptr, no_prefix);
	c.crc = crc != 0;
	return fmt_record_host(m, &c, 0, 0, (char *)out, cap);
}
