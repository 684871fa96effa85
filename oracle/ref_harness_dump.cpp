// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// The reference harness (ref_harness.cpp, included unchanged: push / taps / messages / destroy are its aisref_* functions) with
// one more constructor, aisref_create_dump: the same ModelFrontend models with SetKey(KEY_SETTING_DUMP, prefix) before buildModel,
// so that the reference's own Util::ConvertToRAW >> Util::WriteWAV pair writes <prefix>_A.wav / <prefix>_B.wav
// (Source/DSP/Model.cpp:348-353, 390-396).  The files are complete once aisref_destroy has run (WriteWAV::~WriteWAV patches the
// sizes).  channel_mode 3 builds single-channel mode (setMode(X), buildModel('X', 'X')), where the reference wires no dump.
// The complex taps 3 / 4 are C_a / C_b (C_a only in X).  Built into oracle/_ref/libaisref_dump.so by oracle/dump.mk.
#include "ref_harness.cpp"

extern "C" void *aisref_create_dump(int model, int sample_rate, int format, unsigned flags, int own_mmsi, int channel_mode, char ch1, char ch2,
									 const char *prefix) {
	Handle *h = new Handle();
	try {
		switch (format) {
		case 0: h->fmt = Format::CF32; break;
		case 1: h->fmt = Format::CU8; break;
		case 2: h->fmt = Format::CS8; break;
		case 3: h->fmt = Format::CS16; break;
		default: delete h; return nullptr;
		}
		if (model == MODEL_DEFAULT) {
			h->fe = h->md = new AIS::ModelDefault();
			h->md->SetKey(AIS::KEY_SETTING_PS_EMA, (flags & FLAG_PS_EMA) ? "on" : "off");
			h->md->SetKey(AIS::KEY_SETTING_AFC_WIDE, (flags & FLAG_AFC_WIDE) ? "on" : "off");
		}
		else if (model == MODEL_STANDARD) h->fe = h->ms = new AIS::ModelStandard();
		else if (model == MODEL_BASE) h->fe = h->mb = new AIS::ModelBase();
		else if (model == MODEL_CHALLENGER) {
			h->fe = h->mc = new AIS::ModelChallenger();
			h->mc->SetKey(AIS::KEY_SETTING_AFC_WIDE, (flags & FLAG_AFC_WIDE) ? "on" : "off");
		}
		else if (model == MODEL_V2) h->fe = h->mv = new AIS::ModelEngineV2();
		else {
			delete h;
			return nullptr;
		}
		h->fe->SetKey(AIS::KEY_SETTING_DROOP, (flags & FLAG_DROOP) ? "on" : "off");
		if (flags & FLAG_FP_DS) h->fe->SetKey(AIS::KEY_SETTING_FP_DS, "on");
		if (flags & FLAG_DSK) h->fe->SetKey(AIS::KEY_SETTING_DSK, "on");
		if (prefix) h->fe->SetKey(AIS::KEY_SETTING_DUMP, prefix); // -go DUMP <prefix>
		h->fe->setOwnMMSI(own_mmsi);
		const bool x = channel_mode == 3;
		if (x) h->fe->setMode(AIS::Mode::X);
		h->dev.setFormat(h->fmt);
		h->dev.setSampleRate(sample_rate);
		h->fe->buildModel(x ? 'X' : ch1, x ? 'X' : ch2, sample_rate, false, &h->dev);
		h->fe->Output() >> h->sink;
		if (flags & FLAG_TAPS) {
			h->taps = true;
			h->fe->C_a->Connect(&h->tc[3]);
			if (!x) h->fe->C_b->Connect(&h->tc[4]);
		}
	}
	catch (const std::exception &e) {
		fprintf(stderr, "aisref_create_dump: %s\n", e.what());
		delete h;
		return nullptr;
	}
	return h;
}
