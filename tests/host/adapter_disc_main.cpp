// Test program for ais-catcher_b200/host/ModelGPU.h as the FM-discriminator input model (-m 3): the adapter inside the reference's
// own block graph, with Model::setMode called before buildModel as the Receiver does (Source/Application/Receiver.cpp:81-98).
//
//   adapter_disc_test <AB|X> <file> <CF32|CU8|CS8|CS16> <sample_rate> <block_samples> <gpu|cpu> [KEY VALUE ...]
//
// Wires MemDevice --Connection<RAW>--> AIS::ModelGPU(AISGPU_MODEL_DISCRIMINATOR) --StreamOut<Message>--> sink, or the reference's
// own ModelDiscriminator with "cpu" (an A/B in one binary), with the Receiver's default letters of the mode ("AB" / "XX").  KEY VALUE
// pairs are handed to SetKey before buildModel (-go KEY VALUE).  Prints one line per message:
// channel|nbits|start|end|level-bits|ppm-bits|sentence[ sentence...], then "class FM" or "class IQ" (getClass) on stderr.
// Exit code 3 = the adapter reported a run-time failure through Error() + StopRequest(); 4 = configuration error.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <strings.h>
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
// -go key names (CommandLine.cpp:196-234) through the reference's own key table
bool key_of(const char *name, AIS::Keys &key) {
	for (int k = 0; k < AIS::KEY_COUNT; k++) {
		const auto &cell = AIS::KeyMap[k][JSON_DICT_SETTING];
		if (cell.size() && strlen(name) == cell.size() && strncasecmp(cell.data(), name, cell.size()) == 0) {
			key = (AIS::Keys)k;
			return true;
		}
	}
	return false;
}
} // namespace

int main(int argc, char **argv) {
	if (argc < 7) {
		fprintf(stderr, "usage: %s AB|X file CF32|CU8|CS8|CS16 rate block_samples gpu|cpu [KEY VALUE ...]\n", argv[0]);
		return 2;
	}
	const bool x = strcmp(argv[1], "X") == 0;
	const std::string fs(argv[3]);
	const Format fmt = fs == "CF32" ? Format::CF32 : fs == "CS16" ? Format::CS16 : fs == "CS8" ? Format::CS8 : Format::CU8;
	const int bps = fmt == Format::CF32 ? 8 : (fmt == Format::CS16 ? 4 : 2);
	const int rate = atoi(argv[4]), block = atoi(argv[5]);
	const bool cpu = strcmp(argv[6], "cpu") == 0;
	FILE *f = fopen(argv[2], "rb");
	if (!f) { perror(argv[2]); return 2; }
	std::vector<unsigned char> data;
	unsigned char buf[65536];
	size_t n;
	while ((n = fread(buf, 1, sizeof(buf), f)) > 0) data.insert(data.end(), buf, buf + n);
	fclose(f);

	MemDevice dev;
	Sink sink;
	AIS::Model *model = cpu ? (AIS::Model *)new AIS::ModelDiscriminator() : (AIS::Model *)new AIS::ModelGPU(AISGPU_MODEL_DISCRIMINATOR);
	try {
		for (int i = 7; i + 1 < argc; i += 2) {
			AIS::Keys key;
			if (!key_of(argv[i], key)) {
				fprintf(stderr, "unknown key %s\n", argv[i]);
				return 2;
			}
			model->SetKey(key, argv[i + 1]);
		}
		model->setMode(x ? AIS::Mode::X : AIS::Mode::AB);
		model->buildModel(x ? 'X' : 'A', x ? 'X' : 'B', rate, false, &dev);
	}
	catch (std::exception &e) {
		fprintf(stderr, "config error: %s\n", e.what());
		return 4;
	}
	fprintf(stderr, "class %s\n", model->getClass() == AIS::ModelClass::FM ? "FM" : "IQ");
	model->Output().out.Connect(&sink);
	const size_t step = (size_t)block * bps;
	for (size_t off = 0; off + step <= data.size() && !g_stop_requests; off += step) dev.push(data.data() + off, (int)step, fmt);
	fprintf(stderr, "%ld messages, %d stop requests\n", sink.count, g_stop_requests);
	delete model;
	return g_stop_requests ? 3 : 0;
}
