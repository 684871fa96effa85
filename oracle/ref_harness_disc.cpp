// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// The reference harness (ref_harness.cpp, included unchanged: push / taps / messages are its aisref_* functions) with one more
// constructor, aisrefd_create, for the FM-discriminator input model (-m 3, Source/DSP/Model.h:281-300, Model.cpp:702-754): the
// UNMODIFIED AIS::ModelDiscriminator, built with the caller's two channel letters.  ModelDiscriminator is a Model, not a
// ModelFrontend, so Handle has no slot for it: DiscHandle owns it, and aisrefd_destroy (never aisref_destroy, Handle's destructor is
// not virtual) frees it.  Taps keep the harness's numbering where a slot means the same thing:
//   complex 9: US out (rates below 48 kHz)
//   float   0..4 / 5..9: S_a / S_b outputs (decoder inputs), 10 / 11: RP / IP out (what feeds FR_a / FR_b), 12 / 13: FR_a / FR_b out
// Built into oracle/_ref/libaisrefd.so by oracle/disc.mk.
#include "ref_harness.cpp"

namespace {
struct DiscHandle : Handle {
	AIS::ModelDiscriminator *disc = nullptr;
	~DiscHandle() { delete disc; }
};
} // namespace

extern "C" void *aisrefd_create(int sample_rate, int format, unsigned flags, int own_mmsi, const char *letters) {
	DiscHandle *h = new DiscHandle();
	try {
		switch (format) {
		case 0: h->fmt = Format::CF32; break;
		case 1: h->fmt = Format::CU8; break;
		case 2: h->fmt = Format::CS8; break;
		case 3: h->fmt = Format::CS16; break;
		default: delete h; return nullptr;
		}
		h->disc = new AIS::ModelDiscriminator();
		h->disc->setOwnMMSI(own_mmsi);
		h->dev.setFormat(h->fmt);
		h->dev.setSampleRate(sample_rate);
		h->disc->buildModel(letters && letters[0] ? letters[0] : 'A', letters && letters[0] && letters[1] ? letters[1] : 'B', sample_rate, false, &h->dev);
		h->disc->Output() >> h->sink;
		h->taps = (flags & FLAG_TAPS) != 0;
		if (h->taps) {
			AIS::ModelDiscriminator *m = h->disc;
			m->US.out.Connect(&h->tc[9]);
			m->RP.out.Connect(&h->tf[10]);
			m->IP.out.Connect(&h->tf[11]);
			m->FR_a.out.Connect(&h->tf[12]);
			m->FR_b.out.Connect(&h->tf[13]);
			for (int i = 0; i < 5; i++) {
				m->S_a.out[i].Connect(&h->tf[i]);
				m->S_b.out[i].Connect(&h->tf[5 + i]);
			}
		}
	}
	catch (const std::exception &e) {
		fprintf(stderr, "aisrefd_create: %s\n", e.what());
		delete h;
		return nullptr;
	}
	return static_cast<Handle *>(h);
}

extern "C" void aisrefd_destroy(void *hv) { delete static_cast<DiscHandle *>(static_cast<Handle *>(hv)); }
