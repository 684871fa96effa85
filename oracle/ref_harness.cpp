// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// In-memory harness around the UNMODIFIED reference implementation
// (/root/reference/Source, compiled where it lies by oracle/Makefile into
// oracle/_ref/libaisref*.so).  It instantiates the reference's own
// AIS::ModelDefault / ModelStandard / ModelBase (Source/DSP/Model.h:180-228),
// feeds them RAW blocks of a caller-chosen chunk length through a
// Device::Device subclass (Source/Device/Device.h:58) exactly as a device thread
// would (Source/Device/FileRAW.cpp:121-137), and records
//   * every AIS::Message the model publishes (Source/DSP/Model.h:87,96), for ModelChallenger with the
//     decoder that published it (aisref_publishers), and
//   * optional float taps on the internal Connection<>s of the chain
// so that the CPU restatement in oracle/ais_oracle.c and the CUDA path can be
// compared against the real thing.  Built with -fno-access-control so private
// block members (CGF_a, FC_a, CD_EMA_a[], ...) can be tapped without touching
// the reference sources.  Nothing here is copied from the reference: it only
// *uses* its public block interface (Source/Library/Stream.h:36-167).
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may load the resulting library.

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "Model.h"
#include "Device.h"

void StopRequest() {} // Source/Library/Common.h:72 -- the application normally defines it

namespace {

struct MemDevice : public Device::Device {
	void push(void *p, int bytes, Format f) {
		RAW r{f, p, bytes};
		Send(&r, 1, tag);
	}
};

struct RecC : public StreamIn<CFLOAT32> {
	std::vector<float> v, ppm;
	void Receive(const CFLOAT32 *d, int len, TAG &tag) {
		const float *f = (const float *)d;
		v.insert(v.end(), f, f + 2 * (size_t)len);
		ppm.push_back(tag.ppm);
	}
};

struct RecF : public StreamIn<FLOAT32> {
	std::vector<float> v;
	void Receive(const FLOAT32 *d, int len, TAG &) { v.insert(v.end(), d, d + len); }
};

struct MsgSink : public StreamIn<AIS::Message> {
	std::string text;
	long count = 0;
	// The multi-sentence sequence id is a PROCESS-global atomic in the reference (Source/Marine/Message.cpp:28-39), so the digit
	// a message gets depends on what every other model instance of the process has published -- and on thread timing when
	// several instances run in parallel threads (tests, bench.py).  The harness therefore renumbers: every handle counts its
	// own multi-sentence messages exactly as Message::nextSeqId does (0..9, wrapping), writes that digit into the sentences
	// and recomputes their checksums.  Nothing else of the sentence changes.
	int seq = 0;
	static std::string renumber(const std::string &s, char digit) {
		std::string r = s; // "!AIVDM,n,k,<seq>,C,payload,fill*HH": the id is the 4th field
		size_t p = 0;
		for (int commas = 0; p < r.size() && commas < 3; p++)
			if (r[p] == ',') commas++;
		if (p >= r.size() || r[p] < '0' || r[p] > '9') return r;
		r[p] = digit;
		size_t star = r.rfind('*');
		if (star == std::string::npos || star + 2 >= r.size()) return r;
		unsigned c = 0;
		for (size_t k = 1; k < star; k++) c ^= (unsigned char)r[k];
		static const char hex[] = "0123456789ABCDEF";
		r[star + 1] = hex[(c >> 4) & 15];
		r[star + 2] = hex[c & 15];
		return r;
	}
	void Receive(const AIS::Message *m, int len, TAG &tag) {
		for (int i = 0; i < len; i++) {
			char buf[128];
			const AIS::Message &x = m[i];
			int nbytes = (x.getLength() + 7) / 8;
			snprintf(buf, sizeof(buf), "%c|%d|%lld|%lld|%.9g|%.9g|", x.getChannel(), x.getLength(),
					 (long long)x.start_idx, (long long)x.end_idx, (double)tag.level, (double)tag.ppm);
			text += buf;
			for (int b = 0; b < nbytes; b++) {
				snprintf(buf, sizeof(buf), "%02X", x.data[b]);
				text += buf;
			}
			text += "|";
			bool first = true;
			const bool multi = x.sentences().size() > 1;
			for (const auto &s : x.sentences()) {
				if (!first) text += " ";
				text += multi ? renumber(std::string(s.data(), s.size()), (char)('0' + seq)) : std::string(s.data(), s.size());
				first = false;
			}
			if (multi) seq = (seq + 1) % 10;
			text += "\n";
			count++;
		}
	}
};

// Which decoder published: one more sink on each decoder's own output, behind the model's output (so it hears each message
// right after MsgSink has recorded it).  code numbers the decoder as ais_oracle.c's Decoder.idx does.
struct PubSink : public StreamIn<AIS::Message> {
	std::vector<int> *dst = nullptr;
	int code = 0;
	void Receive(const AIS::Message *, int len, TAG &) {
		for (int i = 0; i < len; i++) dst->push_back(code);
	}
};

enum { MODEL_STANDARD = 0, MODEL_BASE = 1, MODEL_DEFAULT = 2, MODEL_CHALLENGER = 4, MODEL_V2 = 11 };
enum { FLAG_PS_EMA = 1, FLAG_AFC_WIDE = 2, FLAG_DROOP = 4, FLAG_TAPS = 8, FLAG_FP_DS = 16, FLAG_DSK = 32 };
static const int NTAPS_C = 11; // 0: ROT in, 1/2: ROT up/down, 3/4: C_a/C_b, 5/6: CGF or (unused), 7/8: FC, 9: US out, 10: DSK out
static const int NTAPS_F = 14; // 0..4 / 5..9: per-phase decoder inputs ch A / B; 10/11: FM out; 12/13: FR out

struct Handle {
	MemDevice dev;
	AIS::ModelDefault *md = nullptr;
	AIS::ModelStandard *ms = nullptr;
	AIS::ModelBase *mb = nullptr;
	AIS::ModelEngineV2 *mv = nullptr;
	AIS::ModelChallenger *mc = nullptr;
	bool taps = false;
	AIS::ModelFrontend *fe = nullptr;
	MsgSink sink;
	PubSink pub[2][10];
	std::vector<int> pubs;
	RecC tc[NTAPS_C];
	RecF tf[NTAPS_F];
	Format fmt = Format::CF32;
	~Handle() {
		delete md;
		delete ms;
		delete mb;
		delete mv;
		delete mc;
	}
};

// ModelChallenger: the publisher sinks on DEC_a / DEC_af (codes 0..4 / 5..9) and DEC_b / DEC_bf, and in A/B mode its taps
// (complex 5/6: CGF, 7/8: FC; float 0..4 / 5..9: CD_EMA per phase, 10/11: FM, 12/13: FR).  In single-channel mode its taps stay
// the front end's, as tests/golden/mode_x.json records them.
static void attach_challenger(Handle *h, bool two_channels) {
	AIS::ModelChallenger *m = h->mc;
	for (int c = 0; c < (two_channels ? 2 : 1); c++)
		for (int i = 0; i < 5; i++) {
			for (int k = 0; k < 2; k++) {
				PubSink &ps = h->pub[c][5 * k + i];
				ps.dst = &h->pubs;
				ps.code = 5 * k + i;
				AIS::Decoder &d = c ? (k ? m->DEC_bf[i] : m->DEC_b[i]) : (k ? m->DEC_af[i] : m->DEC_a[i]);
				d.out.Connect(&ps);
			}
		}
	if (!h->taps || !two_channels) return;
	m->CGF_a.out.Connect(&h->tc[5]);
	m->FC_a.out.Connect(&h->tc[7]);
	m->FM_af.out.Connect(&h->tf[10]);
	m->FR_af.out.Connect(&h->tf[12]);
	for (int i = 0; i < 5; i++) m->CD_EMA_a[i].out.Connect(&h->tf[i]);
	m->CGF_b.out.Connect(&h->tc[6]);
	m->FC_b.out.Connect(&h->tc[8]);
	m->FM_bf.out.Connect(&h->tf[11]);
	m->FR_bf.out.Connect(&h->tf[13]);
	for (int i = 0; i < 5; i++) m->CD_EMA_b[i].out.Connect(&h->tf[5 + i]);
}

template <typename T>
bool feeds(Connection<T> &c, StreamIn<T> *s) {
	for (auto p : c.connections)
		if (p == s) return true;
	return false;
}

} // namespace

extern "C" {

void *aisref_create(int model, int sample_rate, int format, unsigned flags, int own_mmsi) {
	Handle *h = new Handle();
	try {
		switch (format) {
		case 0: h->fmt = Format::CF32; break;
		case 1: h->fmt = Format::CU8; break;
		case 2: h->fmt = Format::CS8; break;
		case 3: h->fmt = Format::CS16; break;
		default: delete h; return nullptr;
		}
		const char *droop = (flags & FLAG_DROOP) ? "on" : "off";
		if (model == MODEL_DEFAULT) {
			h->md = new AIS::ModelDefault();
			h->fe = h->md;
			h->md->SetKey(AIS::KEY_SETTING_PS_EMA, (flags & FLAG_PS_EMA) ? "on" : "off");
			h->md->SetKey(AIS::KEY_SETTING_AFC_WIDE, (flags & FLAG_AFC_WIDE) ? "on" : "off");
		}
		else if (model == MODEL_STANDARD) {
			h->ms = new AIS::ModelStandard();
			h->fe = h->ms;
		}
		else if (model == MODEL_BASE) {
			h->mb = new AIS::ModelBase();
			h->fe = h->mb;
		}
		else if (model == MODEL_CHALLENGER) { // model 4 "v1_high" (Source/DSP/Model.cpp:601-678)
			h->mc = new AIS::ModelChallenger();
			h->fe = h->mc;
			h->mc->SetKey(AIS::KEY_SETTING_AFC_WIDE, (flags & FLAG_AFC_WIDE) ? "on" : "off");
		}
		else if (model == MODEL_V2) { // model 11 "v2_base" (Source/DSP/Model.cpp:440-460)
			h->mv = new AIS::ModelEngineV2();
			h->fe = h->mv;
		}
		else {
			delete h;
			return nullptr;
		}
		h->fe->SetKey(AIS::KEY_SETTING_DROOP, droop);
		if (flags & FLAG_FP_DS) h->fe->SetKey(AIS::KEY_SETTING_FP_DS, "on"); // -go FP_DS on (Source/DSP/Model.cpp:362-365)
		if (flags & FLAG_DSK) h->fe->SetKey(AIS::KEY_SETTING_DSK, "on");     // -go DSK on   (Source/DSP/Model.cpp:377-379)
		h->fe->setOwnMMSI(own_mmsi);
		h->dev.setFormat(h->fmt);
		h->dev.setSampleRate(sample_rate);
		h->fe->buildModel('A', 'B', sample_rate, false, &h->dev);
		h->fe->Output() >> h->sink;

		h->taps = (flags & FLAG_TAPS) != 0;
		if (flags & FLAG_TAPS) {
			AIS::ModelFrontend *fe = h->fe;
			// whichever Connection feeds ROT (depends on the rate, Source/DSP/Model.cpp:157-338)
			Connection<CFLOAT32> *cands[] = {&fe->FDC.out, &fe->DS2_1.out, &fe->DSK.out, &fe->US.out, &fe->DS16_CU8.out, &fe->convert.out};
			for (auto c : cands)
				if (feeds<CFLOAT32>(*c, &fe->ROT)) {
					c->Connect(&h->tc[0]);
					break;
				}
			fe->US.out.Connect(&h->tc[9]);   // DSP::Upsample / DownsampleKFilter outputs (only fed at resampled rates)
			fe->DSK.out.Connect(&h->tc[10]);
			fe->ROT.up.Connect(&h->tc[1]);
			fe->ROT.down.Connect(&h->tc[2]);
			fe->C_a->Connect(&h->tc[3]);
			fe->C_b->Connect(&h->tc[4]);
			if (h->md) {
				h->md->CGF_a.out.Connect(&h->tc[5]);
				h->md->CGF_b.out.Connect(&h->tc[6]);
				h->md->FC_a.out.Connect(&h->tc[7]);
				h->md->FC_b.out.Connect(&h->tc[8]);
				for (int i = 0; i < 5; i++) {
					if (flags & FLAG_PS_EMA) {
						h->md->CD_EMA_a[i].out.Connect(&h->tf[i]);
						h->md->CD_EMA_b[i].out.Connect(&h->tf[5 + i]);
					}
					else {
						h->md->CD_a[i].out.Connect(&h->tf[i]);
						h->md->CD_b[i].out.Connect(&h->tf[5 + i]);
					}
				}
			}
			if (h->ms) {
				h->ms->FM_a.out.Connect(&h->tf[10]);
				h->ms->FM_b.out.Connect(&h->tf[11]);
				h->ms->FR_a.out.Connect(&h->tf[12]);
				h->ms->FR_b.out.Connect(&h->tf[13]);
				for (int i = 0; i < 5; i++) {
					h->ms->S_a.out[i].Connect(&h->tf[i]);
					h->ms->S_b.out[i].Connect(&h->tf[5 + i]);
				}
			}
			if (h->mb) {
				h->mb->FM_a.out.Connect(&h->tf[10]);
				h->mb->FM_b.out.Connect(&h->tf[11]);
				h->mb->FR_a.out.Connect(&h->tf[12]);
				h->mb->FR_b.out.Connect(&h->tf[13]);
				h->mb->sampler_a.out.Connect(&h->tf[0]);
				h->mb->sampler_b.out.Connect(&h->tf[5]);
			}
		}
		if (h->mc) attach_challenger(h, true);
	}
	catch (const std::exception &e) {
		fprintf(stderr, "aisref_create: %s\n", e.what());
		delete h;
		return nullptr;
	}
	return h;
}

// one RAW block == one Device callback (chunk length is part of the parity contract, SURVEY.md 3.2)
int aisref_push(void *hv, const void *data, long nbytes) {
	Handle *h = (Handle *)hv;
	long long before[2] = {0, 0};
	if (h->mv && h->taps) {
		before[0] = h->mv->V2_a.sample_idx;
		before[1] = h->mv->V2_b.sample_idx;
	}
	h->dev.push((void *)data, (int)nbytes, h->fmt);
	if (h->mv && h->taps) { // the arrays of the LAST block each engine decoded in this push (taps 5/6 CGF out, 7/8 FIR17 out, 12/13 FIR37 out)
		V2::Engine *e[2] = {&h->mv->V2_a, &h->mv->V2_b};
		for (int c = 0; c < 2; c++) {
			if (e[c]->sample_idx == before[c]) continue;
			const float *fc = (const float *)e[c]->freq_corrected, *co = (const float *)e[c]->coh_filtered;
			h->tc[5 + c].v.insert(h->tc[5 + c].v.end(), fc, fc + 2 * V2::BLOCK_SIZE);
			h->tc[5 + c].ppm.push_back(e[c]->ppm);
			h->tc[7 + c].v.insert(h->tc[7 + c].v.end(), co, co + 2 * V2::BLOCK_SIZE);
			h->tf[12 + c].v.insert(h->tf[12 + c].v.end(), e[c]->fm_filtered, e[c]->fm_filtered + V2::BLOCK_SIZE);
		}
	}
	return 0;
}

// complex taps (interleaved re,im floats): returns float count; copies up to max and clears when dst != NULL
long aisref_tap_c(void *hv, int tap, float *dst, long max) {
	Handle *h = (Handle *)hv;
	if (tap < 0 || tap >= NTAPS_C) return -1;
	std::vector<float> &v = h->tc[tap].v;
	long n = (long)v.size();
	if (dst) {
		long k = n < max ? n : max;
		memcpy(dst, v.data(), k * sizeof(float));
		v.clear();
	}
	return n;
}

// tag.ppm seen at each Receive of a complex tap (one value per CGF block for taps 5..8)
long aisref_tap_ppm(void *hv, int tap, float *dst, long max) {
	Handle *h = (Handle *)hv;
	if (tap < 0 || tap >= NTAPS_C) return -1;
	std::vector<float> &v = h->tc[tap].ppm;
	long n = (long)v.size();
	if (dst) {
		long k = n < max ? n : max;
		memcpy(dst, v.data(), k * sizeof(float));
		v.clear();
	}
	return n;
}

long aisref_tap_f(void *hv, int tap, float *dst, long max) {
	Handle *h = (Handle *)hv;
	if (tap < 0 || tap >= NTAPS_F) return -1;
	std::vector<float> &v = h->tf[tap].v;
	long n = (long)v.size();
	if (dst) {
		long k = n < max ? n : max;
		memcpy(dst, v.data(), k * sizeof(float));
		v.clear();
	}
	return n;
}

long aisref_msg_count(void *hv) { return ((Handle *)hv)->sink.count; }

// ModelChallenger: the decoder that published each message aisref_messages has not yet returned, in the same order (0..4 the
// coherent phases, 5..9 the FM phases).  Copies up to max and clears when dst != NULL; returns the count.
long aisref_publishers(void *hv, int *dst, long max) {
	std::vector<int> &v = ((Handle *)hv)->pubs;
	long n = (long)v.size();
	if (dst) {
		long k = n < max ? n : max;
		memcpy(dst, v.data(), k * sizeof(int));
		v.clear();
	}
	return n;
}

// newline-separated records "ch|nbits|start_idx|end_idx|level|ppm|HEXPAYLOAD|nmea1 nmea2"
long aisref_messages(void *hv, char *dst, long max) {
	Handle *h = (Handle *)hv;
	long n = (long)h->sink.text.size();
	if (dst) {
		long k = n < max ? n : max;
		memcpy(dst, h->sink.text.data(), k);
		h->sink.text.clear();
	}
	return n;
}

// The reference's own output formatters on a message built from raw fields (no model involved): checker for the product's
// aisgpu_msg_json / aisgpu_msg_binary.  kind 0: Message::getNMEAJSON, 1: getBinaryNMEA(crc = false), 2: getBinaryNMEA(crc = true).
// The message's sentences (built by Message::buildNMEA, hence with the process-global sequence id) are returned newline-terminated
// in nmea_out so that the caller can hand the very same sentences to the product.
long aisref_format(int kind, const unsigned char *data, int nbits, int channel, int station, int own_mmsi, long long start_idx,
				   long long end_idx, long long rxtime_us, long long toa_us, float level, float ppm, int version, int driver,
				   const char *hardware, int mode, int status, unsigned ipv4, const char *uuid, int include_ssl, const char *suffix,
				   char *out, long max, char *nmea_out, long nmea_max) {
	AIS::Message m;
	m.clear();
	m.setBytes(data, (nbits + 7) / 8);
	m.setOrigin((char)channel, station, own_mmsi);
	m.setLength(nbits);
	m.setStartIdx(start_idx);
	m.setEndIdx(end_idx);
	m.setRxTimeMicros(rxtime_us);
	m.setTOA(toa_us);
	TAG tag;
	tag.mode = (unsigned)mode;
	tag.level = level;
	tag.ppm = ppm;
	tag.version = version;
	tag.driver = (Type)driver;
	tag.hardware = hardware ? hardware : "";
	tag.status = status;
	tag.ipv4 = ipv4;
	m.buildNMEA(tag);
	std::string o;
	if (kind == 0) m.getNMEAJSON(o, tag, include_ssl != 0, uuid ? std::string(uuid) : std::string(), suffix);
	else m.getBinaryNMEA(o, tag, kind == 2);
	if (nmea_out) {
		std::string all;
		for (const auto &sv : m.sentences()) {
			all.append(sv.data(), sv.size());
			all.push_back('\n');
		}
		if ((long)all.size() > nmea_max) return -1;
		memcpy(nmea_out, all.data(), all.size());
	}
	long n = (long)o.size();
	if (n > max) return -1;
	memcpy(out, o.data(), (size_t)n);
	return n;
}

void aisref_destroy(void *hv) { delete (Handle *)hv; }

} // extern "C"
