// Test program for ais-catcher_b200/host/ModelGPU.h on Format::DC16H buffers (three 32-bit words per sample): the adapter, or the
// reference's own model, inside the reference's block graph -- what tests/host/adapter_main.cpp does for CU8 / CF32.
//
//   adapter_dc16h_test <file of uint32 triples> <sample_rate> <block_samples> <model 0|1|2> [cpu] [odd]
//
// prints one line per message: channel|nbits|start|end|level-bits|ppm-bits|sentence[ sentence...]
// "cpu": the reference's CPU model instead of AIS::ModelGPU (A/B in one binary).  "odd": every second device buffer is 1 or 2
// words longer than the block; ConvertRAW takes size / 12 samples and drops those words (StreamHelpers.cpp:120-126), and so must
// the adapter.
// Exit code 3 = the adapter reported a run-time failure through Error() + StopRequest() (e.g. no GPU).
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
	void push(void *p, int bytes) {
		RAW r{Format::DC16H, p, bytes};
		Send(&r, 1, tag);
	}
};
struct Sink : public StreamIn<AIS::Message> {
	long count = 0;
	void Receive(const AIS::Message *m, int len, TAG &tag) override {
		for (int i = 0; i < len; i++) {
			unsigned lb, pb;
			memcpy(&lb, &tag.level, 4);
			memcpy(&pb, &tag.ppm, 4);
			printf("%c|%d|%lld|%lld|%u|%u|", m[i].getChannel(), m[i].getLength(), (long long)m[i].start_idx, (long long)m[i].end_idx, lb, pb);
			bool first = true;
			for (const auto &s : m[i].sentences()) {
				if (!first) putchar(' ');
				fwrite(s.data(), 1, s.size(), stdout);
				first = false;
			}
			putchar('\n');
			count++;
		}
	}
};
} // namespace

int main(int argc, char **argv) {
	if (argc < 5) {
		fprintf(stderr, "usage: %s file rate block_samples model [cpu] [odd]\n", argv[0]);
		return 2;
	}
	const int rate = atoi(argv[2]), block = atoi(argv[3]), kind = atoi(argv[4]);
	bool cpu = false, odd = false;
	for (int i = 5; i < argc; i++) {
		if (!strcmp(argv[i], "cpu")) cpu = true;
		if (!strcmp(argv[i], "odd")) odd = true;
	}
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
		if (cpu) model = kind == 2 ? (AIS::Model *)new AIS::ModelDefault() : (kind == 0 ? (AIS::Model *)new AIS::ModelStandard() : (AIS::Model *)new AIS::ModelBase());
		else model = new AIS::ModelGPU(kind);
		model->buildModel('A', 'B', rate, false, &dev);
	}
	catch (std::exception &e) { // what CommandLine::run does (CommandLine.cpp:752-757)
		fprintf(stderr, "config error: %s\n", e.what());
		return 4;
	}
	model->Output().out.Connect(&sink);
	size_t off = 0;
	for (int k = 0; !g_stop_requests; k++) {
		const size_t bytes = (size_t)block * 12 + ((odd && (k & 1)) ? 1 + (k / 2) % 2 : 0) * sizeof(uint32_t);
		if (off + bytes > data.size()) break;
		dev.push(data.data() + off, (int)bytes);
		off += bytes;
	}
	fprintf(stderr, "%ld messages, %d stop requests, settings: %s\n", sink.count, g_stop_requests, model->Get().c_str());
	delete model;
	return g_stop_requests ? 3 : 0;
}
