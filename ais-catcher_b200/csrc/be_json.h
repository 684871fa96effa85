// The records of frames in every message format and the full AIS JSON of published frames (be_json.cu): the host-side view
// aisgpu.cu and egress.cpp need.
#pragma once
#include "../../include/aisgpu.h"

#include <cuda_runtime.h>
#include <string>

// What a record is printed with: the format and the tag's fields, its strings never NULL, and the full-JSON prefix of the tag
// (aj_prefix) with the place of the time members in it.  rxtime_us: the time of every record of an engine without a clock (the
// records of one with a clock take each frame's stamp instead).  suffix: the output's line suffix; crc: BINARY_NMEA's CRC flag (0
// in the outputs' records).  The engine keeps a copy of this and of its strings in device memory.
struct FmtCtx {
	int fmt, version, driver, mode, station, status, include_ssl, crc;
	unsigned ipv4;
	long long rxtime_us, toa_us;
	const char *hardware, *uuid, *suffix, *prefix;
	int prefix_len, prefix_time;
};

// The part of every full-JSON line that depends only on the tag (class .. hardware, then toa and "scaled"), ending in "scaled":true
// -- built once per engine and copied in front of every line.  The time members (rxtime / rxuxtime, where mode bit 1 is set) are
// the frame's and are written between the two parts, at time_at.
struct AjPrefix {
	std::string text;
	int time_at = 0;
};
AjPrefix aj_prefix(const aisgpu_tag *tag);

// The longest time members a full-JSON line can hold: ,"rxtime":"YYYYMMDDHHMMSS","rxuxtime":<s> with <s> of any int64 time
// (at most 21 characters)
const int kAjTimeMax = 64;

// The context of *tag for format fmt; NULL hardware / uuid as "", suffix as given (NULL: none); prefix = aj_prefix(tag).
FmtCtx fmt_ctx(const aisgpu_tag *tag, int fmt, const char *suffix, const AjPrefix &prefix);

// The record of m into out (cap bytes): its length, or AISGPU_EOVERFLOW when it does not fit.  ordinal: the frames the engine
// published before m (COMMUNITY_HUB); groups: the multi-sentence frames among them (NMEA_TAG).
int fmt_record_host(const aisgpu_msg *m, const FmtCtx *c, long long ordinal, long long groups, char *out, int cap);

// The device side of one batch of n published frames (already in d_msgs), four launches on st:
//   - d_groups[i] = groups + the multi-sentence frames of the batch before frame i, d_total[3] = those of the whole batch;
//   - record i (frame ordinal + i), printed with d_ctx[0] or, with per_stream, d_ctx[stream of frame i], and the time d_stamps[i]
//     (NULL: the context's rxtime_us), into the first cap bytes of the slot d_slots + i * slot (the rest is its scratch), its length
//     into d_len[i] (-2: longer than cap);
//   - the placement: record i is kept when the records of its submit up to and including it fit in budget bytes (d_seg[i] = index
//     of the first frame of frame i's submit; carry = the bytes the batch's first submit used in earlier batches); d_keep[i] = its
//     bytes (-1: dropped), d_off[i] = where, d_total[0] = all of them, d_total[1] the records kept and d_total[2] the bytes of the
//     batch's last submit so far (d_psum: scratch, n);
//   - the kept records packed into d_text.
// Returns the launch error, if any.
cudaError_t fmt_launch(const aisgpu_msg *d_msgs, const long long *d_stamps, int n, const FmtCtx *d_ctx, int per_stream, long long ordinal, long long groups, long long *d_groups,
					   char *d_slots, int slot, int cap, int *d_len, const int *d_seg, long long budget, long long carry,
					   long long *d_psum, long long *d_off, int *d_keep, long long *d_total, char *d_text, cudaStream_t st);
