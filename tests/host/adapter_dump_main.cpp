// Test program for the -go DUMP key of ais-catcher_b200/host/ModelGPU.h: the adapter, or the reference's own model, inside the
// reference's block graph with SetKey(KEY_SETTING_DUMP, prefix) before buildModel, as CommandLine does for "-go DUMP <prefix>".
//
//   adapter_dump_test <file> <format CU8|CS16|CF32> <sample_rate> <block_samples> <model 0|1|2|3|4|11> <AB|CD|X> <prefix> [cpu]
//                     [KEY VALUE ...]
//
// Writes <prefix>_A.wav / <prefix>_B.wav (the reference writes none in X) and prints the number of messages.  With "cpu" the
// reference's CPU model runs instead, so both sides of a comparison come from one binary.  Exit code 3: a run-time failure went
// through Error() + StopRequest(); 4: a configuration error (SetKey / buildModel threw).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "Device.h"
#include "Model.h"
#include "ModelGPU.h"

static int g_stop_requests = 0;
void StopRequest() { g_stop_requests++; } // Source/Library/Common.h:72 -- the application normally defines it

namespace {
struct MemDevice : public Device::Device {
	void push(void *p, int bytes, Format f) {
		RAW r{f, p, bytes};
		Send(&r, 1, tag);
	}
};
struct Sink : public StreamIn<AIS::Message> {
	long count = 0;
	void Receive(const AIS::Message *, int len, TAG &) override { count += len; }
};
AIS::Model *cpu_model(int kind) {
	switch (kind) {
	case 0: return new AIS::ModelStandard();
	case 1: return new AIS::ModelBase();
	case 2: return new AIS::ModelDefault();
	case 3: return new AIS::ModelDiscriminator();
	case 4: return new AIS::ModelChallenger();
	default: return new AIS::ModelEngineV2();
	}
}
} // namespace

int main(int argc, char **argv) {
	if (argc < 8) {
		fprintf(stderr, "usage: %s file CU8|CS16|CF32 rate block_samples model AB|CD|X prefix [cpu] [KEY VALUE ...]\n", argv[0]);
		return 2;
	}
	const Format fmt = !strcmp(argv[2], "CF32") ? Format::CF32 : (!strcmp(argv[2], "CS16") ? Format::CS16 : Format::CU8);
	const int bps = fmt == Format::CF32 ? 8 : (fmt == Format::CS16 ? 4 : 2);
	const int rate = atoi(argv[3]), block = atoi(argv[4]), kind = atoi(argv[5]);
	const std::string mode = argv[6];
	const bool cpu = argc > 8 && !strcmp(argv[8], "cpu");
	FILE *f = fopen(argv[1], "rb");
	if (!f) { perror(argv[1]); return 2; }
	std::vector<unsigned char> data;
	unsigned char buf[65536];
	size_t n;
	while ((n = fread(buf, 1, sizeof(buf), f)) > 0) data.insert(data.end(), buf, buf + n);
	fclose(f);

	MemDevice dev;
	Sink sink;
	AIS::Model *model = nullptr;
	try {
		model = cpu ? cpu_model(kind) : new AIS::ModelGPU(kind);
		for (int i = cpu ? 9 : 8; i + 1 < argc; i += 2) {
			AIS::Keys key = AIS::KEY_SETTING_DROOP;
			if (!strcmp(argv[i], "PS_EMA")) key = AIS::KEY_SETTING_PS_EMA;
			else if (!strcmp(argv[i], "AFC_WIDE")) key = AIS::KEY_SETTING_AFC_WIDE;
			else if (!strcmp(argv[i], "DSK")) key = AIS::KEY_SETTING_DSK;
			else if (!strcmp(argv[i], "FP_DS")) key = AIS::KEY_SETTING_FP_DS;
			model->SetKey(key, argv[i + 1]);
		}
		model->SetKey(AIS::KEY_SETTING_DUMP, argv[7]);
		char ch1 = 'A', ch2 = 'B';
		if (mode == "CD") ch1 = 'C', ch2 = 'D';
		if (mode == "X") {
			model->setMode(AIS::Mode::X);
			ch1 = ch2 = 'X';
		}
		else if (mode == "CD") model->setMode(AIS::Mode::CD);
		model->buildModel(ch1, ch2, rate, false, &dev);
	}
	catch (std::exception &e) {
		fprintf(stderr, "config error: %s\n", e.what());
		delete model;
		return 4;
	}
	model->Output().out.Connect(&sink);
	const size_t step = (size_t)block * bps;
	for (size_t off = 0; off + step <= data.size() && !g_stop_requests; off += step) dev.push(data.data() + off, (int)step, fmt);
	printf("%ld\n", sink.count);
	delete model; // the dump files are completed here (WriteWAV::~WriteWAV, ~ModelGPU)
	return g_stop_requests ? 3 : 0;
}
