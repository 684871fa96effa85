// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// One of the reference harnesses (AFC_BASE: ref_harness.cpp or ref_harness_x.cpp, included unchanged) with two more entry points
// for the tests of frequency correction over its whole range (tests/test_afc.py):
//   aisref_v2_state    the state a V2::Engine of ModelEngineV2 holds after the last push: the slot predictor (slot_ema, slot_phase),
//                      ppm / ppm_prev / ppm_split of the last block, FreqOffset's prominence and last_f, the sample counter, whether
//                      a strobe decoder is busy (what the next block's CGF reads as `busy`), and the magnitudes of the last estimate
//   aisref_v2_weights  Engine::setWeights on both engines (-go DD_TRAIN / DD_WEIGHT, Model.cpp:449-450), before the first push
// Pushed one V2 block at a time, the state is per block.  Nothing is copied from the reference: the private members are read
// through -fno-access-control.  Built into oracle/_ref/libaisref_afc.so and libaisrefx_afc.so by oracle/afc.mk.
#ifndef AFC_BASE
#define AFC_BASE "ref_harness.cpp"
#endif
#include AFC_BASE

extern "C" {

// channel c (0: V2_a, 1: V2_b) of a model-11 handle.  f[7] = slot_ema re, im, ppm, ppm_prev, prominence, last_f, norm2(slot_ema);
// i[4] = slot_phase, ppm_split, sample_idx, busy; mag[512] (may be NULL) = FreqOffset::magnitude.  Returns 0, -1 if no V2 model.
int aisref_v2_state(void *hv, int c, float *f, long long *i, float *mag) {
	Handle *h = (Handle *)hv;
	if (!h->mv || c < 0 || c > 1) return -1;
	V2::Engine &e = c ? h->mv->V2_b : h->mv->V2_a;
	f[0] = e.slot_ema.real();
	f[1] = e.slot_ema.imag();
	f[2] = e.ppm;
	f[3] = e.ppm_prev;
	f[4] = e.fo.prominence;
	f[5] = e.fo.last_f;
	f[6] = e.slot_ema.real() * e.slot_ema.real() + e.slot_ema.imag() * e.slot_ema.imag();
	i[0] = e.slot_phase;
	i[1] = e.ppm_split;
	i[2] = e.sample_idx;
	bool busy = false;
	for (int j = 0; j < 5; j++) busy |= e.dec[j].getState() != AIS::State::TRAINING;
	i[3] = busy;
	if (mag) memcpy(mag, e.fo.magnitude, sizeof(e.fo.magnitude));
	return 0;
}

int aisref_v2_weights(void *hv, float train, float track) {
	Handle *h = (Handle *)hv;
	if (!h->mv) return -1;
	h->mv->V2_a.setWeights(train, track);
	h->mv->V2_b.setWeights(train, track);
	return 0;
}

} // extern "C"
