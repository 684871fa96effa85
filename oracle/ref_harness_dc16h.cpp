// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// One of the reference harnesses (DC16H_BASE: ref_harness.cpp, ref_harness_x.cpp or ref_harness_disc.cpp, included unchanged) with
// one more entry point, aisref_set_format_dc16h: every later aisref_push hands its bytes to the UNMODIFIED reference as
// Format::DC16H (three 32-bit words per sample; ConvertRAW takes size / 12 samples, Utilities/StreamHelpers.cpp:120-126).  The
// harnesses' own constructors take the four formats 0 .. 3; the models do not read the device's format when they are built
// (ConvertRAW reads RAW::format per block), so a handle is created as CF32 and switched before its first push.
// Built into oracle/_ref/libaisref_dc16h.so, libaisrefx_dc16h.so and libaisrefd_dc16h.so by oracle/dc16h.mk.
#ifndef DC16H_BASE
#define DC16H_BASE "ref_harness.cpp"
#endif
#include DC16H_BASE

extern "C" void aisref_set_format_dc16h(void *p) {
	Handle *h = (Handle *)p;
	h->fmt = Format::DC16H;
	h->dev.setFormat(h->fmt);
}
