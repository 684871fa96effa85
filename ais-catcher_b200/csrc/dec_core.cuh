// dec_core.cuh -- AIS::Decoder (Marine/AIS.h:91-181, AIS.cpp:33-142) as device functions shared by the decoder kernels
// (be_sym.cu) and the V2 engine (be_v2.cu): the bit-serial state machine, CRC-16, cannotBeValid and frame emission.
#pragma once
#include "exact.cuh"
#include "params.h"

namespace aisgpu {

struct DecCtx {
	uint32_t *frame; // shared memory, word w of this thread at frame[w * stride]
	int mode_level;  // the row's frames carry the signal level (row_level)
	int stride;      // threads sharing the frame array (32 in the decoder kernels)
};

__device__ __forceinline__ uint32_t frame_word(const DecCtx &c, int w) { return c.frame[w * c.stride]; }
__device__ __forceinline__ int dec_type(const DecCtx &c) { return (frame_word(c, 0) & 0xff) >> 2; }
__device__ __forceinline__ unsigned dec_mmsi(const DecCtx &c) {
	const uint32_t w0 = frame_word(c, 0), w1 = frame_word(c, 1);
	const unsigned d1 = (w0 >> 8) & 0xff, d2 = (w0 >> 16) & 0xff, d3 = (w0 >> 24) & 0xff, d4 = w1 & 0xff;
	return (d1 << 22) | (d2 << 14) | (d3 << 6) | (d4 >> 2);
}
__device__ __forceinline__ bool dec_cannot_be_valid(const DecCtx &c, int len) { // AIS.cpp:111-142
	if (len < 30) return false;
	const int t = dec_type(c);
	switch (len) {
	case 30: return t > 28 || t == 0;
	case 62: return dec_mmsi(c) > 999999999u;
	case 96: return t == 10;
	case 168: return t == 16;
	case 184: return t == 15 || t == 20 || t == 23;
	case 192: return t == 1 || t == 2 || t == 3 || t == 4 || t == 7 || t == 9 || t == 11 || t == 18 || t == 22 || t == 24 || t == 25 || t == 27 || t == 28;
	case 336: return t == 19;
	case 385: return t == 21;
	case 448: return t == 5;
	}
	return false;
}
// Same CRC (AIS.cpp:55-64: reflected 0x8408, init 0xFFFF, good residue 0xF0B8), eight bits per step: the frame words
// hold the bits LSB first, which is the order the reflected CRC consumes them.
__device__ __forceinline__ bool dec_crc16_bytes(const DecCtx &c, int len) {
	unsigned crc = 0xFFFF;
	const int nbytes = len >> 3;
	uint32_t w = 0;
	for (int k = 0; k < nbytes; k++) {
		if ((k & 3) == 0) w = frame_word(c, k >> 2);
		unsigned dta = ((w >> ((k & 3) * 8)) ^ crc) & 0xffu;
		dta ^= (dta << 4) & 0xffu;
		crc = (((dta << 8) | (crc >> 8)) ^ (dta >> 4) ^ (dta << 3)) & 0xffffu;
	}
	for (int i = nbytes * 8; i < len; i++) {
		const unsigned bit = (frame_word(c, i >> 5) >> (i & 31)) & 1u;
		crc = ((bit ^ crc) & 1u) ? ((crc >> 1) ^ 0x8408u) : (crc >> 1);
	}
	return crc == 0xF0B8u;
}
__device__ __forceinline__ bool dec_crc16(const DecCtx &c, int len) { // AIS.cpp:55-64
	unsigned crc = 0xFFFF;
	for (int i = 0; i < len; i++) {
		const unsigned bit = (frame_word(c, i >> 5) >> (i & 31)) & 1u;
		crc = ((bit ^ crc) & 1u) ? ((crc >> 1) ^ 0x8408u) : (crc >> 1);
	}
	return crc == 0xF0B8u;
}

// One Decoder::Run (AIS.h:91-181).  Returns true when a frame with a good CRC just completed (processData true);
// in that case fr_len = payload bits + 16 and the caller emits and performs the FOUNDMESSAGE/Reset protocol.
__device__ __forceinline__ bool dec_step(DecState &d, const DecCtx &c, float sample, float sample_lvl, long long sample_idx, int &fr_len,
										 float &fr_level, int &lastBit_before) {
	const int dd = sample > 0.0f;
	const int Bit = !(dd ^ d.prev);
	d.prev = dd;
	lastBit_before = d.lastBit;
	bool found = false;
	switch (d.state) {
	case ST_TRAINING:
		if (Bit != d.lastBit) d.position++;
		else {
			if (d.position > 4) {
				d.start_idx = sample_idx;
				d.state = ST_STARTFLAG;
				d.position = Bit ? 3 : 1;
				d.one_seq = 0;
			}
			else { d.state = ST_TRAINING; d.position = 0; d.one_seq = 0; }
		}
		break;
	case ST_STARTFLAG:
		if (d.position == 7) {
			if (Bit == 0) {
				d.state = ST_DATAFCS; d.position = 0; d.one_seq = 0;
				d.level = 0.0f;
				for (int w = 0; w < DEC_WORDS; w++) c.frame[w * c.stride] = 0u; // msg.clear()
			}
			else { d.state = ST_TRAINING; d.position = 0; d.one_seq = 0; }
		}
		else {
			if (Bit == 1) d.position++;
			else { d.state = ST_TRAINING; d.position = 0; d.one_seq = 0; }
		}
		break;
	case ST_DATAFCS: {
		const int pos = d.position++;
		if (pos < MAX_FRAME_BITS) { // Message::setBit (Message.h:264-273)
			uint32_t *wp = &c.frame[(pos >> 5) * c.stride];
			const uint32_t m = 1u << (pos & 31);
			*wp = Bit ? (*wp | m) : (*wp & ~m);
		}
		if (c.mode_level) d.level = __fadd_rn(d.level, sample_lvl);
		if (Bit == 1) {
			if (d.one_seq == 5) {
				fr_level = c.mode_level ? __fdiv_rn(d.level, (float)d.position) : 0.0f;
				const int len = d.position - 7;
				if (len >= 16 && dec_crc16(c, len)) {
					found = true;
					fr_len = len;
				}
				d.state = ST_TRAINING; d.position = 0; d.one_seq = 0;
			}
			else d.one_seq++;
		}
		else {
			if (d.one_seq == 5) d.position--;
			d.one_seq = 0;
		}
		if (d.position == MAX_FRAME_BITS || dec_cannot_be_valid(c, d.position)) { d.state = ST_TRAINING; d.position = 0; d.one_seq = 0; }
		break;
	}
	default: break;
	}
	d.lastBit = Bit;
	return found;
}

// The frame ring is circular: `head` only grows (one ticket per frame); a frame whose ticket is `ring_cap` or more ahead of
// what the host had drained when the kernel was launched (ticket >= limit) is dropped -- the host sees the gap in the
// ticket range and reports AISGPU_EOVERFLOW.
__device__ __forceinline__ FrameRec *ring_claim(FrameRec *__restrict__ ring, unsigned long long *__restrict__ head, unsigned long long limit, int ring_cap) {
	const unsigned long long t = atomicAdd(head, 1ull);
	return t < limit ? &ring[t % (unsigned long long)ring_cap] : nullptr;
}
__device__ __forceinline__ void emit_frame(FrameRec *__restrict__ ring, unsigned long long *__restrict__ head, unsigned long long limit, int ring_cap, int chunk,
										   int blk, const DecCtx &c, int row, int phase, int len, float level, float ppm, long long start_idx, long long end_idx) {
	FrameRec *rp = ring_claim(ring, head, limit, ring_cap);
	if (!rp) return;
	FrameRec &r = *rp;
	r.row = row;
	r.phase = phase;
	r.nbits = len - 16;
	r.level = level;
	r.ppm = ppm;
	r.chunk = chunk;
	r.blk = blk;
	r.start_idx = start_idx;
	r.end_idx = end_idx;
	for (int w = 0; w < DEC_WORDS; w++) r.data[w] = frame_word(c, w);
}

} // namespace aisgpu
