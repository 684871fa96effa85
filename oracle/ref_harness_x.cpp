// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// The reference harness (ref_harness.cpp, included unchanged: push / taps / messages / destroy are its aisref_* functions) with
// one more constructor, aisrefx_create: the same models in single-channel mode (-c X, Source/DSP/Model.cpp:35-107) --
// setMode(AIS::Mode::X) before buildModel('X', 'X', ...), the Receiver's default letters for X (Receiver.cpp:87-98).
// Only channel A's chain exists in X; its taps keep the harness's numbering:
//   complex 0: whatever Connection feeds FCIC5_a (FDC / DS2_1 / US / convert), 3: C_a, 5: CGF_a, 7: FC_a, 9: US out
//   float   0..4: decoder inputs, 10: FM_a, 12: FR_a
// Built into oracle/_ref/libaisrefx.so by oracle/mode_x.mk.
#include "ref_harness.cpp"

extern "C" void *aisrefx_create(int model, int sample_rate, int format, unsigned flags, int own_mmsi) {
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
			h->md = new AIS::ModelDefault();
			h->fe = h->md;
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
		h->fe->setOwnMMSI(own_mmsi);
		h->fe->setMode(AIS::Mode::X);
		h->dev.setFormat(h->fmt);
		h->dev.setSampleRate(sample_rate);
		h->fe->buildModel('X', 'X', sample_rate, false, &h->dev);
		h->fe->Output() >> h->sink;
		h->taps = (flags & FLAG_TAPS) != 0;
		if (h->taps) {
			AIS::ModelFrontend *fe = h->fe;
			Connection<CFLOAT32> *cands[] = {&fe->FDC.out, &fe->DS2_1.out, &fe->US.out, &fe->convert.out};
			for (auto c : cands)
				if (feeds<CFLOAT32>(*c, &fe->FCIC5_a)) {
					c->Connect(&h->tc[0]);
					break;
				}
			fe->US.out.Connect(&h->tc[9]);
			fe->C_a->Connect(&h->tc[3]);
			if (h->md) {
				h->md->CGF_a.out.Connect(&h->tc[5]);
				h->md->FC_a.out.Connect(&h->tc[7]);
				for (int i = 0; i < 5; i++) {
					if (flags & FLAG_PS_EMA) h->md->CD_EMA_a[i].out.Connect(&h->tf[i]);
					else h->md->CD_a[i].out.Connect(&h->tf[i]);
				}
			}
			if (h->ms) {
				h->ms->FM_a.out.Connect(&h->tf[10]);
				h->ms->FR_a.out.Connect(&h->tf[12]);
				for (int i = 0; i < 5; i++) h->ms->S_a.out[i].Connect(&h->tf[i]);
			}
			if (h->mb) {
				h->mb->FM_a.out.Connect(&h->tf[10]);
				h->mb->FR_a.out.Connect(&h->tf[12]);
				h->mb->sampler_a.out.Connect(&h->tf[0]);
			}
		}
	}
	catch (const std::exception &e) {
		fprintf(stderr, "aisrefx_create: %s\n", e.what());
		delete h;
		return nullptr;
	}
	return h;
}
