// ModelGPU.h -- the H100 engine as one more AIS::Model of the reference application.
//
// Header-only C++11 adapter, compiled against the reference's own headers where they lie (add the reference's
// Source/* directories to the include path; nothing of the reference is copied here) and linked with libaisgpu.so
// (include/aisgpu.h).  It is the "reference-side binding" of INTEGRATION.md: the class a maintainer registers in
// Receiver::addModel (Source/Application/Receiver.cpp:155-195) next to ModelDefault / ModelStandard / ModelBase.
//
//   Model ABI      : AIS::Model (Source/DSP/Model.h:76-126): buildModel(), Output(), SetKey(), Get(), getClass()
//   Block ABI      : StreamIn<RAW>::Receive(const RAW*, int len, TAG&) (Source/Library/Stream.h:36-45), connected to
//                    `timerOn ? (*device >> timer).out : device->out` exactly as ModelFrontend does (Model.cpp:33)
//   Output         : the inherited Util::PassThrough<Message> output (Model.h:87): one AIS::Message per frame,
//                    filled the way Decoder::processData does (Source/Marine/AIS.cpp:66-96)
//   Errors         : configuration -> std::runtime_error from buildModel (Model.cpp:109-110 convention);
//                    run time -> Error() << ...; StopRequest(); (Source/Device/FileRAW.cpp:111-115 convention)
//
// A single reference receiver is a batch of ONE stream; the same engine serves thousands of streams through the C ABI
// (aisgpu_submit with n_streams > 1) -- that is where the GPU pays, see DESIGN.md.
#pragma once

#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "Model.h"   // reference Source/DSP/Model.h
#include "Logger.h"  // reference Source/Library/Logger.h
#include "aisgpu.h"

namespace AIS {

class ModelGPU : public Model, public StreamIn<RAW> {
	aisgpu_handle *engine = nullptr;
	aisgpu_config cfg;
	Message msg;
	std::vector<aisgpu_msg> frames;
	std::vector<unsigned char> fifo;  // input bytes that have not filled a whole block yet
	int granule = 64;                 // samples: every CIC stage needs an even block (DSP.cpp:94,135)
	size_t blockBytes = 0;            // every submit has this length (fixed by the first Receive, see there)
	bool failed = false;
	std::string dumpPrefix;           // -go DUMP <prefix> (Model.cpp:390-396): the 48 kHz channels to <prefix>_A.wav / _B.wav
	bool dump = false;

	static int formatOf(Format f) {
		switch (f) {
		case Format::CF32: return AISGPU_FMT_CF32;
		case Format::CU8: return AISGPU_FMT_CU8;
		case Format::CS8: return AISGPU_FMT_CS8;
		case Format::CS16: return AISGPU_FMT_CS16;
		case Format::F32_FS4: return AISGPU_FMT_F32_FS4;
		case Format::DC16H: return AISGPU_FMT_DC16H;
		default: return -1;
		}
	}
	static int bytesPerSample(int fmt) {
		return fmt == AISGPU_FMT_CF32 ? 8 : (fmt == AISGPU_FMT_DC16H ? 12 : ((fmt == AISGPU_FMT_CS16 || fmt == AISGPU_FMT_F32_FS4) ? 4 : 2));
	}

	void fail(const std::string &what) {
		if (!failed) Error() << "ModelGPU: " << what;
		failed = true;
		StopRequest();
	}

	bool ensureEngine(Format f) {
		if (engine) return formatOf(f) == cfg.format;
		const int fmt = formatOf(f);
		if (fmt < 0) return false;
		cfg.format = fmt;
		cfg.station = station;
		cfg.own_mmsi = own_mmsi;
		if (aisgpu_create(&cfg, &engine) != AISGPU_OK) {
			fail(std::string("cannot create engine: ") + aisgpu_last_error(nullptr));
			return false;
		}
		// the reference wires the dump behind FilterCIC5 in AB / CD only: in X buildModel returns before it (Model.cpp:106)
		if (dump && cfg.channel_mode == AISGPU_MODE_AB) {
			const char *prefixes[1] = { dumpPrefix.c_str() };
			if (aisgpu_dump_open(engine, prefixes) != AISGPU_OK) {
				fail(aisgpu_last_error(engine));
				return false;
			}
		}
		return true;
	}

	void publish(TAG &tag) {
		int n = 0;
		do {
			const int rc = aisgpu_poll(engine, frames.data(), (int)frames.size(), &n);
			if (rc == AISGPU_EOVERFLOW) Warning() << "ModelGPU: " << aisgpu_last_error(engine); // the surviving frames are still delivered
			else if (rc != AISGPU_OK) {
				fail(aisgpu_last_error(engine));
				return;
			}
			for (int i = 0; i < n; i++) {
				const aisgpu_msg &f = frames[i];
				msg.clear();
				if (tag.mode & 2) msg.Stamp();
				msg.setBytes(f.data, (f.nbits + 7) / 8);
				msg.setOrigin(f.channel, station, own_mmsi);
				msg.setLength(f.nbits);
				msg.setStartIdx(f.start_idx);
				msg.setEndIdx(f.end_idx);
				tag.level = f.level;
				tag.ppm = f.ppm;
				// the application's own armouring, so the process-global sequence id (Message.cpp:28-39) is shared with
				// every other model in the process; f.nmea holds the same text for hosts that are not C++
				msg.buildNMEA(tag);
				output.Receive(&msg, 1, tag);
			}
		} while (n == (int)frames.size());
	}

public:
	explicit ModelGPU(int kind = AISGPU_MODEL_DEFAULT) {
		aisgpu_default_config(&cfg);
		cfg.model = kind;
		cfg.n_streams = 1;
		frames.resize(64);
		setName(kind == AISGPU_MODEL_DEFAULT ? "AIS engine H100 (coherent)"
				: kind == AISGPU_MODEL_STANDARD ? "AIS engine H100 (FM)"
				: kind == AISGPU_MODEL_DISCRIMINATOR ? "AIS engine H100 (FM discriminator input)" : "AIS engine H100 (FM/PLL)");
	}
	~ModelGPU() override {
		if (engine) aisgpu_dump_close(engine); // completes the WAV headers, as WriteWAV::~WriteWAV does (no-op without a dump)
		aisgpu_destroy(engine);
	}

	void buildModel(char CH1, char CH2, int sample_rate, bool timerOn, Device::Device *dev) override {
		device = dev;
		if (!device) throw std::runtime_error("ModelGPU: no device");
		// AB and CD build the same chain (only the letters and the tuning differ, Receiver.cpp:81-86); X is the single-channel chain
		// (Model.cpp:35-107), whose frames carry CH1.  The FM-discriminator input model never reads the mode (Model.cpp:702-754):
		// two channels with whatever letters the receiver passes
		if (cfg.model == AISGPU_MODEL_DISCRIMINATOR || mode == Mode::AB || mode == Mode::CD) cfg.channel_mode = AISGPU_MODE_AB;
		else if (mode == Mode::X) cfg.channel_mode = AISGPU_MODE_X;
		else throw std::runtime_error("ModelGPU: only the AB, CD and X channel modes are built");
		cfg.sample_rate = sample_rate;
		cfg.channel_a = CH1;
		cfg.channel_b = CH2;
		// one RAW block of the reference's file/SDR devices is at most 24*16*16384 bytes (Device/FileRAW.h:43)
		cfg.max_chunk_samples = 24 * 16 * 16384 / 2;
		// validate the rate -> chain table now, like ModelFrontend::buildModel (Model.cpp:109-110); the engine itself is
		// created on the first block, when the device's sample format is known (ConvertRAW does the same, StreamHelpers.cpp:51)
		granule = aisgpu_chunk_granule(&cfg);
		if (granule <= 0) throw std::runtime_error(aisgpu_last_error(nullptr));
		Connection<RAW> &physical = timerOn ? (*device >> timer).out : device->out;
		physical.Connect(this);
	}

	// StreamIn<RAW>: one device buffer (Model.cpp:33; Utilities/StreamHelpers.cpp:51-57 asserts len == 1)
	void Receive(const RAW *raw, int len, TAG &tag) override {
		if (failed || len != 1 || !raw->data || raw->size <= 0) return;
		if (!ensureEngine(raw->format)) {
			if (!failed) fail("unsupported or changing sample format");
			return;
		}
		// The engine is handed blocks of ONE length: that of the device's first buffer, rounded down to the granule (the
		// reference's results depend on the block length -- Rotate renormalises and Upsample re-blocks per Receive,
		// DSP.cpp:203,309-315 -- and at interpolated rates the engine insists on a constant one).  A device that always
		// delivers that length (every file / SDR device does) is passed through without a copy; odd, short or varying
		// buffers (network sources, the last block of a file) go through a byte FIFO.
		const int bps = bytesPerSample(cfg.format);
		const unsigned char *p = (const unsigned char *)raw->data;
		size_t n = (size_t)raw->size;
		// F32_FS4: ConvertRAW drops the floats of a buffer beyond a multiple of 4 (size -= size & 3, StreamHelpers.cpp:107-108) and
		// starts the 1, j, -1, -j pattern again with the next buffer.  With them dropped here every buffer adds a whole number of
		// patterns, and the blocks below are multiples of the granule (a multiple of 4): the re-blocking keeps every sample's place.
		if (cfg.format == AISGPU_FMT_F32_FS4) n = n / 16 * 16;
		// DC16H: ConvertRAW takes size / 12 samples of a buffer (StreamHelpers.cpp:120-126); the bytes short of a sample are dropped,
		// not carried into the next buffer
		if (cfg.format == AISGPU_FMT_DC16H) n = n / 12 * 12;
		if (!blockBytes) {
			size_t samples = n / bps / granule * granule;
			if (samples < (size_t)granule) samples = (size_t)granule;
			if (samples > (size_t)cfg.max_chunk_samples / granule * granule) samples = (size_t)cfg.max_chunk_samples / granule * granule;
			blockBytes = samples * bps;
		}
		if (fifo.empty()) { // whole blocks straight from the device buffer
			while (n >= blockBytes) {
				if (aisgpu_submit(engine, p, (int)(blockBytes / bps)) != AISGPU_OK) return fail(aisgpu_last_error(engine));
				p += blockBytes;
				n -= blockBytes;
			}
		}
		if (n) {
			fifo.insert(fifo.end(), p, p + n);
			size_t off = 0;
			while (fifo.size() - off >= blockBytes) {
				if (aisgpu_submit(engine, fifo.data() + off, (int)(blockBytes / bps)) != AISGPU_OK) return fail(aisgpu_last_error(engine));
				off += blockBytes;
			}
			if (off) fifo.erase(fifo.begin(), fifo.begin() + off);
		}
		publish(tag);
	}

	Setting &SetKey(AIS::Keys key, const std::string &arg) override {
		// ModelDiscriminator has no SetKey of its own: STATION_ID / ID / OWN_MMSI, every other key "not supported" (Model.h:107-122)
		if (cfg.model == AISGPU_MODEL_DISCRIMINATOR) return Model::SetKey(key, arg);
		switch (key) {
		case AIS::KEY_SETTING_PS_EMA: cfg.ps_ema = Util::Parse::Switch(arg); break;     // ModelDefault::SetKey, Model.cpp:583-585
		case AIS::KEY_SETTING_AFC_WIDE: cfg.afc_wide = Util::Parse::Switch(arg); break; // Model.cpp:586-588
		case AIS::KEY_SETTING_DROOP: cfg.droop = Util::Parse::Switch(arg); break;       // ModelFrontend::SetKey, Model.cpp:384-386
		case AIS::KEY_SETTING_FP_DS: cfg.fp_ds = Util::Parse::Switch(arg); break;       // Model.cpp:362-365 (CU8 @1536K only, as in the reference)
		case AIS::KEY_SETTING_DSK: cfg.dsk = Util::Parse::Switch(arg); break;           // Model.cpp:377-379
		case AIS::KEY_SETTING_DUMP: // ModelFrontend::SetKey, Model.cpp:390-396; opened with the engine (ensureEngine)
			dumpPrefix = arg;
			dump = true;
			break;
		case AIS::KEY_SETTING_SOXR:
		case AIS::KEY_SETTING_SRC:
		case AIS::KEY_SETTING_MA:
			if (!Util::Parse::Switch(arg)) break; // "off" is what the engine does anyway
			throw std::runtime_error(getName() + ": setting \"" + AIS::KeyMap[key][JSON_DICT_SETTING] + "\" is not available on the GPU engine");
		default: Model::SetKey(key, arg); break; // STATION_ID, OWN_MMSI, or the reference's "not supported" error
		}
		return *this;
	}

	ModelClass getClass() override { return cfg.model == AISGPU_MODEL_DISCRIMINATOR ? ModelClass::FM : ModelClass::IQ; } // Model.h:299, 125

	std::string Get() override {
		if (cfg.model == AISGPU_MODEL_DISCRIMINATOR) return "gpu on";
		return "gpu on ps_ema " + Util::Convert::toString((bool)cfg.ps_ema) + " afc_wide " + Util::Convert::toString((bool)cfg.afc_wide) + " droop " +
			   Util::Convert::toString((bool)cfg.droop) + " fp_ds " + Util::Convert::toString((bool)cfg.fp_ds) + " dsk " + Util::Convert::toString((bool)cfg.dsk);
	}

	void setDeviceOrdinal(int d) { cfg.device = d; }
	aisgpu_handle *handle() { return engine; }
};

} // namespace AIS
