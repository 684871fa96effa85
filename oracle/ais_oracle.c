/* TEST INFRASTRUCTURE -- NOT PRODUCT CODE.  See ais_oracle.h for the parity status (PINNED).
 *
 * Plain-C restatement of the reference's IQ -> NMEA hot path, written from the
 * reference's behaviour (file:line below, all relative to /root/reference/Source),
 * block by block, with the same block boundaries, the same IEEE binary32
 * operation order and the same libm entry points (sincosf, cabsf==hypotf,
 * atan2f, log10) the strict-flags reference build links against.  Compile with
 * -fno-fast-math -ffp-contract=off (oracle/Makefile).
 *
 *   RAW -> CF32 conversion ........ Utilities/Convert.cpp:255-286, StreamHelpers.cpp:51-133
 *   Downsample2CIC5 ............... DSP/DSP.cpp:85-117
 *   FilterCIC5 .................... DSP/DSP.cpp:132-157
 *   DownsampleKFilter ............. DSP/DSP.cpp:160-189, DSP.h:181-215
 *   Upsample ...................... DSP/DSP.cpp:192-212
 *   FilterComplex / Filter ........ DSP/DSP.cpp:215-280, DSP.h:217-270
 *   FilterComplex3Tap ............. DSP/DSP.cpp:283-293, DSP.h:293-297
 *   Rotate ........................ DSP/DSP.cpp:296-316, Model.cpp:31
 *   SquareFreqOffsetCorrection .... DSP/DSP.cpp:417-489, FFT.h:36-130
 *   ScatterPLL / Deinterleave ..... DSP/DSP.h:51-118
 *   SimplePLL ..................... DSP/DSP.cpp:28-57
 *   FM / PhaseSearch(EMA) ......... DSP/Demod.cpp:27-170, Demod.h:27-31
 *   rate -> chain table ........... DSP/Model.cpp:109-356
 *   ModelBase/Standard/Default .... DSP/Model.cpp:419-438, 484-577
 *   ModelChallenger ............... DSP/Model.cpp:601-678
 *   single-channel mode at 48k .... DSP/Model.cpp:35-107 (-c X: convert >> FCIC5_a)
 *   Decoder ....................... Marine/AIS.h:91-181, AIS.cpp:33-142
 *   Message bits + NMEA ........... Marine/Message.h:181-194,264-281, Message.cpp:28-39,398-413,569-686
 */
#define _GNU_SOURCE
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "ais_oracle.h"

typedef struct { float re, im; } cf;

static const float PI_F = 3.14159265358979323846f; /* Library/Common.h:318 (a float constant) */

/* ---------- small helpers ---------- */
typedef struct { float *p; long n, cap; } fvec;
static void fv_push(fvec *v, const float *d, long n) {
	if (v->n + n > v->cap) {
		long c = v->cap ? v->cap * 2 : 4096;
		while (c < v->n + n) c *= 2;
		v->p = (float *)realloc(v->p, c * sizeof(float));
		v->cap = c;
	}
	memcpy(v->p + v->n, d, n * sizeof(float));
	v->n += n;
}
typedef struct { char *p; long n, cap; } svec;
static void sv_push(svec *v, const char *d, long n) {
	if (v->n + n > v->cap) {
		long c = v->cap ? v->cap * 2 : 4096;
		while (c < v->n + n) c *= 2;
		v->p = (char *)realloc(v->p, c);
		v->cap = c;
	}
	memcpy(v->p + v->n, d, n);
	v->n += n;
}

static cf polar1(float theta) { /* std::polar(1.0f, theta): (1*cos, 1*sin) via sincosf */
	float s, c;
	sincosf(theta, &s, &c);
	cf r = { 1.0f * c, 1.0f * s };
	return r;
}
static cf cmul(cf a, cf b) { /* std::complex<float> product, no FMA */
	cf r;
	float ac = a.re * b.re, bd = a.im * b.im, ad = a.re * b.im, bc = a.im * b.re;
	r.re = ac - bd;
	r.im = ad + bc;
	return r;
}
static float cabs1(cf a) { return hypotf(a.re, a.im); } /* std::abs(complex<float>) -> cabsf */

/* ---------- filter taps (DSP/Filters.h:24-53) ---------- */
static const float TAPS_RECEIVER[37] = {
	0.00119025f, -0.00148464f, -0.00282428f, -0.00200561f, -0.00068852f, 0.00343044f, 0.00902093f, 0.01367867f,
	0.01147965f, 0.0027259f, -0.01766614f, -0.04244429f, -0.0577468f, -0.05245161f, -0.01072754f, 0.0732564f,
	0.17643278f, 0.25582214f, 0.28200453f, 0.25582214f, 0.17643278f, 0.0732564f, -0.01072754f, -0.05245161f,
	-0.0577468f, -0.04244429f, -0.01766614f, 0.0027259f, 0.01147965f, 0.01367867f, 0.00902093f, 0.00343044f,
	-0.00068852f, -0.00200561f, -0.00282428f, -0.00148464f, 0.00119025f };
static const float TAPS_COHERENT[17] = {
	2.06995719e-06f, 3.18610148e-05f, 3.40605309e-04f, 2.52892989e-03f, 1.30411453e-02f, 4.67076746e-02f,
	1.16186141e-01f, 2.00730781e-01f, 2.40861391e-01f, 2.00730781e-01f, 1.16186141e-01f, 4.67076746e-02f,
	1.30411453e-02f, 2.52892989e-03f, 3.40605309e-04f, 3.18610148e-05f, 2.06995719e-06f };
static const float TAPS_BH_28_3[26] = {
	6.32542387e-05f, -2.90015252e-04f, -1.54206250e-03f, -1.64972455e-03f, 3.12793899e-03f, 1.09494413e-02f,
	9.04975801e-03f, -1.43685846e-02f, -4.45615933e-02f, -3.44883647e-02f, 5.53474269e-02f, 2.01827915e-01f,
	3.16534610e-01f, 3.16534610e-01f, 2.01827915e-01f, 5.53474269e-02f, -3.44883647e-02f, -4.45615933e-02f,
	-1.43685846e-02f, 9.04975801e-03f, 1.09494413e-02f, 3.12793899e-03f, -1.64972455e-03f, -1.54206250e-03f,
	-2.90015252e-04f, 6.32542387e-05f };
/* Demod.h:29-31 */
static const cf PS_PHASE[8] = {
	{ 9.9518472640441780e-01f, 9.8017143048367339e-02f }, { 9.5694033335306883e-01f, 2.9028468509743588e-01f },
	{ 8.8192125790916542e-01f, 4.7139674887287397e-01f }, { 7.7301044123076901e-01f, 6.3439329894649099e-01f },
	{ 6.3439326515712957e-01f, 7.7301046896098113e-01f }, { 4.7139671032286945e-01f, 8.8192127851457169e-01f },
	{ 2.9028464326824349e-01f, 9.5694034604181499e-01f }, { 9.8017099547459546e-02f, 9.9518473068888236e-01f } };

/* ---------- shared TAG (Library/Common.h:240-288): one per device, both channels write into it ---------- */
typedef struct { unsigned mode; float sample_lvl, level, ppm; long long sample_idx; } Tag;

/* ---------- decoder + message (Marine/AIS.*, Marine/Message.*) ---------- */
#define MAX_AIS_LENGTH 1064
#define MAX_FRAME_LENGTH (MAX_AIS_LENGTH + 16 + 7)
#define MAX_FRAME_BYTES ((MAX_FRAME_LENGTH + 7) / 8)
enum { S_TRAINING, S_STARTFLAG, S_STOPFLAG, S_DATAFCS, S_FOUND };
enum { SIG_STOP_TRAINING, SIG_START_TRAINING, SIG_RESET };

struct Chan;
typedef struct Decoder {
	struct Chan *ch;
	int idx;
	int state, lastBit, prev, position, one_seq_count;
	float level;
	long long start_idx, end_idx;
	uint8_t data[MAX_FRAME_BYTES + 4];
} Decoder;

/* ---------- demodulators ---------- */
typedef struct { float ma[16]; uint8_t bits[16]; int max_idx, rot; } PSEma;
typedef struct { float memory[16][14]; uint8_t bits[16]; int max_idx, rot, last; } PSearch;

typedef struct { float *taps; int nt; float *buffer; } FirF; /* DSP::Filter */
typedef struct { float *taps; int nt; cf *buffer; } FirC;    /* DSP::FilterComplex */

typedef struct {
	cf output[512], fft[512], rot;
	float cumsum[512];
	int count;
} Cgf;

struct Handle;
typedef struct Chan {
	struct Handle *h;
	int id; /* 0 = A (ROT.up), 1 = B (ROT.down) */
	char name;
	cf ds2[5], cic[5];
	Cgf cgf;
	FirC fc;
	FirF fr;
	cf fm_prev;
	/* ScatterPLL / Deinterleave */
	int lastSymbol;
	cf sample[5];
	float level;
	long long sample_idx;
	PSEma ema[5];
	PSearch ps[5];
	Decoder dec[10]; /* ModelChallenger: 0..4 behind the coherent branch, 5..9 (FM phase d - 5) behind the FM branch */
	/* ModelChallenger: the FM branch's Filter 37 outputs of the group of five in flight, and how far its order has stepped */
	float fm_val[5];
	int fm_n, grp_done, lvl_set;
	/* SimplePLL */
	int pll_prev;
	float pll;
	int pll_fast;
} Chan;

enum { ST_DS2, ST_US, ST_DSK, ST_FDC };
typedef struct {
	int kind;
	cf h[5];                    /* DS2 */
	float alpha, beta; cf h1, h2; /* FDC */
	float us_alpha, us_inc; cf us_a; int us_idx_out; long us_outsize; /* US */
	cf *dsk_buf; long dsk_bufsz; int dsk_idx_in, dsk_idx_out;          /* DSK */
	cf *out; long outcap;
} Stage;

enum { MODEL_STANDARD = 0, MODEL_BASE = 1, MODEL_DEFAULT = 2, MODEL_CHALLENGER = 4 };
enum { FLAG_PS_EMA = 1, FLAG_AFC_WIDE = 2, FLAG_DROOP = 4, FLAG_TAPS = 8, FLAG_MODE_X = 64 };
/* ModelChallenger's order of its ten decoders within a group of five samples (decoder d < 5: coherent phase d, d >= 5: FM phase
 * d - 5): f0 f1 f2 f3 | a0 a1 a2 a3 a4 | f4 (see chall_sample) */
static const int CHALLENGER_ORDER[10] = { 5, 6, 7, 8, 0, 1, 2, 3, 4, 9 };
#define NTAPS_C 9
#define NTAPS_F 14

typedef struct Handle {
	int model, sample_rate, format, own_mmsi;
	unsigned flags;
	int ps_ema, afc_wide, taps_on, mode_x;
	int order[10];
	int *pub; long npub, pubcap; /* the decoder that published each message not yet read (Decoder.idx) */
	Stage st[12];
	int nst;
	cf rot, mult;
	cf *up, *down; long rotcap;
	cf *conv; long convcap;
	cf omega[512];
	cf us_steps[1]; /* unused */
	Chan ch[2];
	Tag tag;
	int seq;
	long msg_count;
	svec text;
	fvec tc[NTAPS_C], tppm[NTAPS_C], tf[NTAPS_F];
	float *tmpf; long tmpfcap;
	float *tmpf2; long tmpf2cap;
	cf *tmpc; long tmpccap;
} Handle;

static void tapc(Handle *h, int t, const cf *d, int len) {
	if (!h->taps_on) return;
	fv_push(&h->tc[t], (const float *)d, 2L * len);
	fv_push(&h->tppm[t], &h->tag.ppm, 1);
}
static void tapf(Handle *h, int t, const float *d, int len) {
	if (!h->taps_on) return;
	fv_push(&h->tf[t], d, len);
}

/* ================= message / NMEA ================= */
static int msg_getbit(const uint8_t *data, int i) {
	if (i >= MAX_FRAME_LENGTH || i < 0) return 0;
	return (data[i >> 3] >> (i & 7)) & 1;
}
static void msg_setbit(uint8_t *data, int i, int b) {
	if (i >= MAX_FRAME_LENGTH || i < 0) return;
	if (b) data[i >> 3] |= (uint8_t)(1 << (i & 7));
	else data[i >> 3] &= (uint8_t)~(1 << (i & 7));
}
static unsigned msg_type(const uint8_t *d) { return d[0] >> 2; }
static unsigned msg_mmsi(const uint8_t *d) { return ((unsigned)d[1] << 22) | (d[2] << 14) | (d[3] << 6) | (d[4] >> 2); }

static int msg_validate(const uint8_t *d, int length) { /* Message.cpp:398-413 */
	static const int ml[28] = { 149, 149, 149, 168, 418, 88, 72, 56, 168, 70, 168, 72, 40, 40, 88, 92, 80, 168, 312, 70, 271, 145, 154, 160, 72, 60, 96, 168 };
	if (length == 0) return 1;
	if (length > MAX_AIS_LENGTH) return 0;
	unsigned t = msg_type(d);
	if (t < 1 || t > 28) return 0;
	if (length < ml[t - 1]) return 0;
	return 1;
}

static char msg_letter(const uint8_t *data, int length, int pos) { /* Message.cpp:643-662 */
	int start = pos * 6, end = start + 6;
	if (end > MAX_AIS_LENGTH || start < 0) return 0;
	int x = start >> 3, y = start & 7;
	unsigned w = ((unsigned)data[x] << 8) | data[x + 1];
	int l = (w >> (16 - 6 - y)) & 0x3F;
	int overrun = end - length;
	if (overrun > 0) l &= 0x3F << overrun;
	return (char)(l < 40 ? l + 48 : l + 56);
}

/* Message.cpp:569-631; seq = per-handle stand-in for the process-global counter (Message.cpp:28-39) */
static void build_nmea(Handle *h, const uint8_t *data, int length, char channel, svec *out) {
	static const char hex[] = "0123456789ABCDEF";
	int nletters = (length + 5) / 6;
	int nsent = nletters == 0 ? 1 : (nletters + 55) / 56;
	char own = (h->own_mmsi == (int)msg_mmsi(data)) ? 'O' : 'M';
	char seq = 0;
	if (nsent > 1) {
		seq = (char)(h->seq + '0');
		h->seq = (h->seq + 1) % 10;
	}
	for (int s = 0, l = 0; s < nsent; s++) {
		char p[160];
		int i = 0;
		memcpy(p, "!AIVDM,X,X,", 11);
		p[5] = own;
		p[7] = (char)(nsent + '0');
		p[9] = (char)(s + 1 + '0');
		i = 11;
		if (seq) p[i++] = seq;
		p[i++] = ',';
		if (channel != '?') p[i++] = channel;
		p[i++] = ',';
		int letters = nletters - l < 56 ? nletters - l : 56;
		for (int k = 0; k < letters; k++) p[i++] = msg_letter(data, length, l + k);
		l += letters;
		p[i++] = ',';
		p[i++] = (char)(((s == nsent - 1) ? nletters * 6 - length : 0) + '0');
		int c = 0;
		for (int k = 1; k < i; k++) c ^= (unsigned char)p[k];
		p[i++] = '*';
		p[i++] = hex[(c >> 4) & 0xF];
		p[i++] = hex[c & 0xF];
		if (s) sv_push(out, " ", 1);
		sv_push(out, p, i);
	}
}

/* ================= decoder (Marine/AIS.h:91-181, AIS.cpp) ================= */
static void dec_next_state(Decoder *d, int s, int pos);

static void dec_signal_out(Decoder *d, int sig) { /* DecoderMessage.Send: Model.cpp:434-435, 507-514, 566-573 */
	Chan *c = d->ch;
	Handle *h = c->h;
	if (h->model == MODEL_BASE) { /* connected to the SimplePLL (DSP.cpp:46-57) */
		if (sig == SIG_START_TRAINING) c->pll_fast = 1;
		else if (sig == SIG_STOP_TRAINING) c->pll_fast = 0;
		return;
	}
	if (sig != SIG_RESET) return; /* sibling decoders only act on Reset (AIS.cpp:98-108) */
	int n = h->model == MODEL_CHALLENGER ? 10 : 5; /* Model.cpp:654-673: all ten decoders of a channel are cross-connected */
	for (int j = 0; j < n; j++)
		if (j != d->idx) dec_next_state(&c->dec[j], S_TRAINING, 0);
}

static void dec_next_state(Decoder *d, int s, int pos) { /* AIS.cpp:33-53 */
	d->state = s;
	d->position = pos;
	d->one_seq_count = 0;
	switch (s) {
	case S_TRAINING: dec_signal_out(d, SIG_START_TRAINING); break;
	case S_STARTFLAG: dec_signal_out(d, SIG_STOP_TRAINING); break;
	case S_FOUND: dec_signal_out(d, SIG_RESET); break;
	default: break;
	}
}

static int dec_crc16(const Decoder *d, int len) { /* AIS.cpp:55-64 */
	const uint16_t checksum = (uint16_t)~0x0F47, poly = 0x8408;
	uint16_t crc = 0xFFFF;
	for (int i = 0; i < len; i++)
		crc = (((uint16_t)msg_getbit(d->data, i) ^ crc) & 1) ? (uint16_t)((crc >> 1) ^ poly) : (uint16_t)(crc >> 1);
	return crc == checksum;
}

static int dec_cannot_be_valid(const Decoder *d, int len) { /* AIS.cpp:111-142 */
	const int END = 24;
	if (len < 6 + END) return 0;
	int t = (int)msg_type(d->data);
	switch (len) {
	case 6 + 24: return t > 28 || t == 0;
	case 8 + 30 + 24: return msg_mmsi(d->data) > 999999999u;
	case 72 + 24: return t == 10;
	case 144 + 24: return t == 16;
	case 160 + 24: return t == 15 || t == 20 || t == 23;
	case 168 + 24: return t == 1 || t == 2 || t == 3 || t == 4 || t == 7 || t == 9 || t == 11 || t == 18 || t == 22 || t == 24 || t == 25 || t == 27 || t == 28;
	case 312 + 24: return t == 19;
	case 361 + 24: return t == 21;
	case 424 + 24: return t == 5;
	}
	(void)END;
	return 0;
}

static int dec_process(Decoder *d, int len) { /* AIS.cpp:66-96 */
	Handle *h = d->ch->h;
	Tag *tag = &h->tag;
	if (len >= 16 && dec_crc16(d, len)) {
		int nbits = len - 16;
		if ((tag->mode & 1) && tag->level != 0.0)
			tag->level = (float)(10.0f * log10(tag->level));
		/* setLength only accepts 0..MAX_AIS_LENGTH (Message.h:288-292); a longer frame keeps length 0 from clear() */
		int length = (nbits >= 0 && nbits <= MAX_AIS_LENGTH) ? nbits : 0;
		if (msg_validate(d->data, length)) {
			char buf[160];
			int n = snprintf(buf, sizeof(buf), "%c|%d|%lld|%lld|%.9g|%.9g|", d->ch->name, length, d->start_idx, d->end_idx,
							 (double)tag->level, (double)tag->ppm);
			sv_push(&h->text, buf, n);
			int nbytes = (length + 7) / 8;
			for (int b = 0; b < nbytes; b++) {
				n = snprintf(buf, sizeof(buf), "%02X", d->data[b]);
				sv_push(&h->text, buf, n);
			}
			sv_push(&h->text, "|", 1);
			build_nmea(h, d->data, length, d->ch->name, &h->text);
			sv_push(&h->text, "\n", 1);
			h->msg_count++;
			if (h->npub == h->pubcap) {
				h->pubcap = h->pubcap ? 2 * h->pubcap : 256;
				h->pub = (int *)realloc(h->pub, h->pubcap * sizeof(int));
			}
			h->pub[h->npub++] = d->idx;
		}
		return 1;
	}
	return 0;
}

static void dec_run(Decoder *d, float sample) { /* AIS.h:91-181 */
	Tag *tag = &d->ch->h->tag;
	int dd = sample > 0;
	int Bit = !(dd ^ d->prev);
	d->prev = dd;
	switch (d->state) {
	case S_TRAINING:
		if (Bit != d->lastBit) d->position++;
		else {
			if (d->position > 4) {
				d->start_idx = tag->sample_idx;
				dec_next_state(d, S_STARTFLAG, Bit ? 3 : 1);
			}
			else dec_next_state(d, S_TRAINING, 0);
		}
		break;
	case S_STARTFLAG:
		if (d->position == 7) {
			if (Bit == 0) {
				dec_next_state(d, S_DATAFCS, 0);
				d->level = 0.0f;
				memset(d->data, 0, sizeof(d->data));
			}
			else dec_next_state(d, S_TRAINING, 0);
		}
		else {
			if (Bit == 1) d->position++;
			else dec_next_state(d, S_TRAINING, 0);
		}
		break;
	case S_DATAFCS:
		msg_setbit(d->data, d->position++, Bit);
		if (tag->mode & 1) d->level += tag->sample_lvl;
		if (Bit == 1) {
			if (d->one_seq_count == 5) {
				if (tag->mode & 1) tag->level = d->level / d->position;
				d->end_idx = tag->sample_idx;
				int found = dec_process(d, d->position - 7);
				if (found) dec_next_state(d, S_FOUND, 0);
				dec_next_state(d, S_TRAINING, 0);
			}
			else d->one_seq_count++;
		}
		else {
			if (d->one_seq_count == 5) d->position--;
			d->one_seq_count = 0;
		}
		if (d->position == MAX_FRAME_LENGTH || dec_cannot_be_valid(d, d->position))
			dec_next_state(d, S_TRAINING, 0);
		break;
	default: break;
	}
	d->lastBit = Bit;
}

/* ================= demodulators (DSP/Demod.cpp) ================= */
static void prerot(int rot, cf x, float *re, float *im) { /* multiply by (1j)^rot, Demod.cpp:44-65 */
	switch (rot) {
	case 0: *re = x.re; *im = x.im; break;
	case 1: *im = x.re; *re = -x.im; break;
	case 2: *re = -x.re; *im = -x.im; break;
	default: *im = -x.re; *re = x.im; break;
	}
}

static float psema_step(PSEma *p, cf x, int nDelay) { /* Demod.cpp:39-101 */
	const float weight = 0.85f;
	float re, im;
	prerot(p->rot, x, &re, &im);
	p->rot = (p->rot + 1) & 3;
	for (int j = 0; j < 8; j++) {
		float t, a = re * PS_PHASE[j].re, b = im * PS_PHASE[j].im;
		t = a + b;
		p->bits[j] = (uint8_t)((p->bits[j] << 1) | (t > 0));
		p->ma[j] = weight * p->ma[j] + (1 - weight) * fabsf(t);
		t = a - b;
		p->bits[15 - j] = (uint8_t)((p->bits[15 - j] << 1) | (t > 0));
		p->ma[15 - j] = weight * p->ma[15 - j] + (1 - weight) * fabsf(t);
	}
	int idx = (p->max_idx - 1 + 16) & 15;
	float max_val = p->ma[idx];
	p->max_idx = idx;
	for (int q = 0; q < 2; q++) {
		idx = (idx + 1) & 15;
		if (p->ma[idx] > max_val) {
			max_val = p->ma[idx];
			p->max_idx = idx;
		}
	}
	int b2 = (p->bits[p->max_idx] >> (nDelay + 1)) & 1;
	int b1 = (p->bits[p->max_idx] >> nDelay) & 1;
	return (b1 ^ b2) ? 1.0f : -1.0f;
}

static float psearch_step(PSearch *p, cf x, int nHistory, int nDelay) { /* Demod.cpp:103-170 */
	float re, im;
	prerot(p->rot, x, &re, &im);
	p->rot = (p->rot + 1) & 3;
	for (int j = 0; j < 8; j++) {
		float a = re * PS_PHASE[j].re, b = im * PS_PHASE[j].im, t;
		t = a + b;
		p->bits[j] = (uint8_t)((p->bits[j] << 1) | (t > 0));
		p->memory[j][p->last] = fabsf(t);
		t = a - b;
		p->bits[15 - j] = (uint8_t)((p->bits[15 - j] << 1) | (t > 0));
		p->memory[15 - j][p->last] = fabsf(t);
	}
	p->last = (p->last + 1) % nHistory;
	float max_val = 0;
	int prev_max = p->max_idx;
	for (int q = 16 + prev_max - 2; q <= 16 + prev_max + 2; q++) {
		int j = q % 16;
		float avg = p->memory[j][0];
		for (int l = 1; l < nHistory; l++) avg += p->memory[j][l];
		if (avg > max_val) {
			max_val = avg;
			p->max_idx = j;
		}
	}
	int b2 = (p->bits[p->max_idx] >> (nDelay + 1)) & 1;
	int b1 = (p->bits[p->max_idx] >> nDelay) & 1;
	return (b1 ^ b2) ? 1.0f : -1.0f;
}

/* ================= per-channel back ends ================= */
/* ScatterPLL (DSP.h:95-117) -> 5 x (PhaseSearch[EMA] -> Decoder) */
static void scatter_receive(Chan *c, const cf *data, int len) {
	Handle *h = c->h;
	Tag *tag = &h->tag;
	for (int i = 0; i < len; i++) {
		c->sample[c->lastSymbol] = data[i];
		if (tag->mode & 1) c->level += data[i].re * data[i].re + data[i].im * data[i].im; /* std::norm, strict build */
		if (++c->lastSymbol == 5) {
			if (tag->mode & 1) tag->sample_lvl = c->level / 5;
			for (int j = 0; j < 5; j++) {
				tag->sample_idx = c->sample_idx++;
				float b = h->ps_ema ? psema_step(&c->ema[j], c->sample[j], 3) : psearch_step(&c->ps[j], c->sample[j], 12, 3);
				tapf(h, c->id * 5 + j, &b, 1);
				dec_run(&c->dec[j], b);
			}
			c->level = 0.0f;
			c->lastSymbol = 0;
		}
	}
}

/* FilterComplex (DSP.cpp:215-246), dot (DSP.h:224-230) */
static cf firc_dot(const FirC *f, const cf *d) {
	cf x = { 0.0f, 0.0f };
	for (int i = 0; i < f->nt; i++) {
		x.re += f->taps[i] * d[i].re;
		x.im += f->taps[i] * d[i].im;
	}
	return x;
}
static void firc_receive(Chan *c, FirC *f, const cf *data, int len, cf *output) {
	int nt = f->nt, ptr, i, j;
	if (len < nt) {
		for (j = 0; j < len; j++) {
			for (i = 1; i < nt; i++) f->buffer[i - 1] = f->buffer[i];
			f->buffer[nt - 1] = data[j];
			output[0] = firc_dot(f, f->buffer);
			tapc(c->h, 7 + c->id, output, 1);
			scatter_receive(c, output, 1);
		}
		return;
	}
	for (j = 0, ptr = nt - 1; j < nt - 1; ptr++, j++) {
		f->buffer[ptr] = data[j];
		output[j] = firc_dot(f, &f->buffer[j]);
	}
	for (i = 0; i < len - nt + 1; i++, j++) output[j] = firc_dot(f, &data[i]);
	for (ptr = 0; i < len; i++, ptr++) f->buffer[ptr] = data[i];
	tapc(c->h, 7 + c->id, output, len);
	scatter_receive(c, output, len);
}

/* SquareFreqOffsetCorrection (DSP.cpp:417-489) with FFT::Plan (FFT.h:86-131) */
static int bitrev9(int x) {
	int y = 0;
	for (int i = 0; i < 9; i++) {
		y = (y << 1) | (x & 1);
		x >>= 1;
	}
	return y;
}
static void fft512(const cf *omega, cf *x) {
	const int N = 512;
	int m = 2, m2 = 1, r = N;
	for (int s = 0; s < 9; s++) {
		int w = 0;
		r >>= 1;
		for (int j = 0; j < m2; j++) {
			cf o = omega[w];
			for (int k = 0; k < N; k += m) {
				cf t = cmul(o, x[k + j + m2]);
				cf a = x[k + j];
				x[k + j + m2].re = a.re - t.re;
				x[k + j + m2].im = a.im - t.im;
				x[k + j].re = a.re + t.re;
				x[k + j].im = a.im + t.im;
			}
			w += r;
		}
		m2 = m;
		m <<= 1;
	}
}
static float cgf_correct(Handle *h, Cgf *g) {
	const int N = 512, window = 187;
	float max_val = 0.0f, fz = -1;
	int delta = (int)(9600.0 / 48000.0 * N);
	int wi = 0;
	fft512(h->omega, g->fft);
	if (h->afc_wide) {
		int M = (int)(12500.0 / 48000.0 * N);
		int ofs = (M - delta) / 2;
		float wm = -1;
		g->cumsum[0] = 0;
		for (int i = 1; i < N; i++) {
			float p = cabs1(g->fft[(i + N / 2) % N]);
			g->cumsum[i] = g->cumsum[i - 1] + p;
		}
		for (int i = 0; i < N - M; i++) {
			float v = g->cumsum[i + M] - g->cumsum[i] + 0.6f * (cabs1(g->fft[(i + ofs + N / 2) % N]) + cabs1(g->fft[(i + ofs + delta + N / 2) % N]));
			if (v > wm) {
				wm = v;
				wi = i;
			}
		}
		wi = (wi + M / 2 - N / 2);
	}
	for (int i = wi + window; i < wi + N - window - delta; i++) {
		float hh = cabs1(g->fft[(i + N / 2) % N]) + cabs1(g->fft[(i + delta + N / 2) % N]);
		if (hh > max_val) {
			max_val = hh;
			fz = (N / 2 - (i + delta / 2.0f));
		}
	}
	float f = fz / 2.0f / N;
	cf rot_step = polar1((float)(f * 2 * PI_F));
	for (int i = 0; i < N; i++) {
		g->rot = cmul(g->rot, rot_step);
		g->output[i] = cmul(g->output[i], g->rot);
	}
	float a = cabs1(g->rot);
	g->rot.re /= a;
	g->rot.im /= a;
	return f * 48000.0f / 162.0f;
}
/* DSP::Filter (DSP.cpp:249-280) */
static float firf_dot(const FirF *f, const float *d) {
	float x = 0.0f;
	for (int i = 0; i < f->nt; i++) x += f->taps[i] * d[i];
	return x;
}

/* ModelChallenger (Model.cpp:601-678): the throttle (a one-way Deinterleave) hands each CGF output sample on alone, first to the
 * coherent branch (FilterComplex 17 -> ScatterPLL -> PhaseSearchEMA nDelay 3), then to the FM branch (FM -> Filter 37 ->
 * Deinterleave).  ScatterPLL hands a group of five out when its fifth sample arrives; Deinterleave hands FM phase j out at the
 * group's sample j.  The ten decoders step in h->order within each group: a decoder steps as soon as its input exists and every
 * decoder ahead of it in the order has stepped.  ScatterPLL writes the group's level into the tag just before the first coherent
 * decoder steps, so with the reference's order f0..f3 read the previous group's level (or the other channel's, the TAG being
 * shared) and f4 the current one. */
static void chall_sample(Chan *c, cf x) {
	Handle *h = c->h;
	Tag *tag = &h->tag;
	int taps = !h->mode_x; /* the single-channel harness records ModelChallenger's front-end taps only (ref_harness.cpp) */
	FirC *fc = &c->fc;
	for (int i = 1; i < fc->nt; i++) fc->buffer[i - 1] = fc->buffer[i]; /* DSP.cpp:219-225, len < ntaps */
	fc->buffer[fc->nt - 1] = x;
	cf y = firc_dot(fc, fc->buffer);
	if (taps) tapc(h, 7 + c->id, &y, 1);
	c->sample[c->lastSymbol++] = y;
	if (tag->mode & 1) c->level += y.re * y.re + y.im * y.im;

	cf cj = { c->fm_prev.re, -c->fm_prev.im }; /* Demod.cpp:27-37 */
	cf p = cmul(x, cj);
	float v = atan2f(p.im, p.re) / PI_F;
	c->fm_prev = x;
	if (taps) tapf(h, 10 + c->id, &v, 1);
	FirF *fr = &c->fr;
	for (int i = 1; i < fr->nt; i++) fr->buffer[i - 1] = fr->buffer[i]; /* DSP.cpp:253-259, len < ntaps */
	fr->buffer[fr->nt - 1] = v;
	v = firf_dot(fr, fr->buffer);
	if (taps) tapf(h, 12 + c->id, &v, 1);
	c->fm_val[c->fm_n++] = v;

	while (c->grp_done < 10) {
		int d = h->order[c->grp_done];
		if (d < 5) {
			if (c->lastSymbol < 5) break;
			if (!c->lvl_set && (tag->mode & 1)) tag->sample_lvl = c->level / 5;
			c->lvl_set = 1;
			tag->sample_idx = c->sample_idx + d;
			float b = psema_step(&c->ema[d], c->sample[d], 3);
			if (taps) tapf(h, c->id * 5 + d, &b, 1);
			dec_run(&c->dec[d], b);
		}
		else {
			if (d - 5 >= c->fm_n) break;
			tag->sample_idx = c->sample_idx + d - 5;
			dec_run(&c->dec[d], c->fm_val[d - 5]);
		}
		c->grp_done++;
	}
	if (c->grp_done == 10) {
		c->sample_idx += 5;
		c->level = 0.0f;
		c->lastSymbol = c->fm_n = c->grp_done = c->lvl_set = 0;
	}
}

static void cgf_receive(Chan *c, const cf *data, int len) {
	Handle *h = c->h;
	Cgf *g = &c->cgf;
	cf firout[512];
	for (int i = 0; i < len; i++) {
		g->fft[bitrev9(g->count)] = cmul(data[i], data[i]);
		g->output[g->count] = data[i];
		if (++g->count == 512) {
			h->tag.ppm = cgf_correct(h, g);
			if (h->model != MODEL_CHALLENGER || !h->mode_x) tapc(h, 5 + c->id, g->output, 512);
			if (h->model == MODEL_CHALLENGER)
				for (int k = 0; k < 512; k++) chall_sample(c, g->output[k]);
			else firc_receive(c, &c->fc, g->output, 512, firout);
			g->count = 0;
		}
	}
}


/* Deinterleave (DSP.h:65-73) -> 5 decoders ; or SimplePLL (DSP.cpp:28-44) -> 1 decoder */
static void fm_sink(Chan *c, const float *data, int len) {
	Handle *h = c->h;
	Tag *tag = &h->tag;
	if (h->model == MODEL_STANDARD) {
		for (int i = 0; i < len; i++) {
			tag->sample_idx = c->sample_idx++;
			tapf(h, c->id * 5 + c->lastSymbol, &data[i], 1);
			dec_run(&c->dec[c->lastSymbol], data[i]);
			c->lastSymbol = (c->lastSymbol + 1) % 5;
		}
	}
	else {
		for (int i = 0; i < len; i++) {
			int bit = data[i] > 0;
			if (bit != c->pll_prev) c->pll += (0.5f - c->pll) * (c->pll_fast ? 0.6f : 0.05f);
			c->pll += 0.2f;
			if (c->pll >= 1.0f) {
				tapf(h, c->id * 5, &data[i], 1);
				dec_run(&c->dec[0], data[i]);
				c->pll -= (int)c->pll;
			}
			c->pll_prev = bit;
		}
	}
}

static void firf_receive(Chan *c, FirF *f, const float *data, int len, float *output) {
	int nt = f->nt, ptr, i, j;
	if (len < nt) {
		for (j = 0; j < len; j++) {
			for (i = 1; i < nt; i++) f->buffer[i - 1] = f->buffer[i];
			f->buffer[nt - 1] = data[j];
			output[0] = firf_dot(f, f->buffer);
			tapf(c->h, 12 + c->id, output, 1);
			fm_sink(c, output, 1);
		}
		return;
	}
	for (j = 0, ptr = nt - 1; j < nt - 1; ptr++, j++) {
		f->buffer[ptr] = data[j];
		output[j] = firf_dot(f, &f->buffer[j]);
	}
	for (i = 0; i < len - nt + 1; i++, j++) output[j] = firf_dot(f, &data[i]);
	for (ptr = 0; i < len; i++, ptr++) f->buffer[ptr] = data[i];
	tapf(c->h, 12 + c->id, output, len);
	fm_sink(c, output, len);
}

static void fm_receive(Chan *c, const cf *data, int len) { /* Demod.cpp:27-37 */
	Handle *h = c->h;
	if (h->tmpfcap < len) {
		h->tmpfcap = len;
		h->tmpf = (float *)realloc(h->tmpf, len * sizeof(float));
		h->tmpf2 = (float *)realloc(h->tmpf2, len * sizeof(float));
	}
	float *out = h->tmpf;
	for (int i = 0; i < len; i++) {
		cf cj = { c->fm_prev.re, -c->fm_prev.im };
		cf p = cmul(data[i], cj);
		out[i] = atan2f(p.im, p.re) / PI_F;
		c->fm_prev = data[i];
	}
	tapf(h, 10 + c->id, out, len);
	firf_receive(c, &c->fr, out, len, h->tmpf2);
}

/* per-channel: [Downsample2CIC5 (96k->48k)] -> FilterCIC5 -> model back end (Model.cpp:341-346; single channel at 48k: 95-96) */
static void chan_receive(Chan *c, const cf *data, int len) {
	Handle *h = c->h;
	if (h->tmpccap < len) {
		h->tmpccap = len;
		h->tmpc = (cf *)realloc(h->tmpc, 2 * len * sizeof(cf));
	}
	cf *y = h->tmpc, *o = h->tmpc + len;
	int n = 0;
	cf *s = c->ds2;
	if (h->mode_x) {
		memcpy(y, data, len * sizeof(cf));
		n = len;
	}
	else
		for (int i = 0; i < len; i += 2, n++) { /* DSP.cpp:93-117 */
			cf z = data[i], r[5];
			for (int k = 0; k < 5; k++) { r[k] = z; z.re += s[k].re; z.im += s[k].im; }
			y[n].re = z.re * 0.03125f;
			y[n].im = z.im * 0.03125f;
			z = data[i + 1];
			for (int k = 0; k < 5; k++) { s[k] = z; z.re += r[k].re; z.im += r[k].im; }
		}
	s = c->cic;
	for (int i = 0; i < n; i += 2) { /* DSP.cpp:132-157 */
		cf z = y[i], r[5];
		for (int k = 0; k < 5; k++) { r[k] = z; z.re += s[k].re; z.im += s[k].im; }
		o[i].re = z.re * 0.03125f;
		o[i].im = z.im * 0.03125f;
		z = y[i + 1];
		for (int k = 0; k < 5; k++) { s[k] = z; z.re += r[k].re; z.im += r[k].im; }
		o[i + 1].re = z.re * 0.03125f;
		o[i + 1].im = z.im * 0.03125f;
	}
	tapc(h, 3 + c->id, o, n);
	if (h->model == MODEL_DEFAULT || h->model == MODEL_CHALLENGER) cgf_receive(c, o, n);
	else fm_receive(c, o, n);
}

/* Rotate (DSP.cpp:296-316) */
static void rot_receive(Handle *h, const cf *data, int len) {
	if (h->rotcap < len) {
		h->rotcap = len;
		h->up = (cf *)realloc(h->up, len * sizeof(cf));
		h->down = (cf *)realloc(h->down, len * sizeof(cf));
	}
	tapc(h, 0, data, len);
	for (int i = 0; i < len; i++) {
		float RR = data[i].re * h->rot.re, II = data[i].im * h->rot.im;
		float RI = data[i].re * h->rot.im, IR = data[i].im * h->rot.re;
		h->up[i].re = RR - II;
		h->up[i].im = IR + RI;
		h->down[i].re = RR + II;
		h->down[i].im = IR - RI;
		h->rot = cmul(h->rot, h->mult);
	}
	tapc(h, 1, h->up, len);
	chan_receive(&h->ch[0], h->up, len);
	tapc(h, 2, h->down, len);
	chan_receive(&h->ch[1], h->down, len);
	float a = cabs1(h->rot);
	h->rot.re /= a;
	h->rot.im /= a;
}

/* ================= front end stages (rate dependent) ================= */
static void stage_out_reserve(Stage *s, long n) {
	if (s->outcap < n) {
		s->out = (cf *)realloc(s->out, n * sizeof(cf));
		s->outcap = n;
	}
}

static void fe_run(Handle *h, int si, const cf *data, int len) {
	if (h->mode_x) { /* convert >> FCIC5_a: channel A's chain alone */
		tapc(h, 0, data, len);
		chan_receive(&h->ch[0], data, len);
		return;
	}
	if (si == h->nst) {
		rot_receive(h, data, len);
		return;
	}
	Stage *s = &h->st[si];
	switch (s->kind) {
	case ST_DS2: { /* DSP.cpp:93-117 */
		stage_out_reserve(s, len / 2 + 1);
		int n = 0;
		for (int i = 0; i < len; i += 2, n++) {
			cf z = data[i], r[5];
			for (int k = 0; k < 5; k++) { r[k] = z; z.re += s->h[k].re; z.im += s->h[k].im; }
			s->out[n].re = z.re * 0.03125f;
			s->out[n].im = z.im * 0.03125f;
			z = data[i + 1];
			for (int k = 0; k < 5; k++) { s->h[k] = z; z.re += r[k].re; z.im += r[k].im; }
		}
		fe_run(h, si + 1, s->out, n);
		break;
	}
	case ST_FDC: { /* DSP.cpp:283-293 */
		stage_out_reserve(s, len);
		for (int i = 0; i < len; i++) {
			cf t = { s->h1.re + data[i].re, s->h1.im + data[i].im };
			s->out[i].re = s->alpha * t.re + s->h2.re * s->beta;
			s->out[i].im = s->alpha * t.im + s->h2.im * s->beta;
			s->h1 = s->h2;
			s->h2 = data[i];
		}
		fe_run(h, si + 1, s->out, len);
		break;
	}
	case ST_US: { /* DSP.cpp:192-212 */
		if (s->us_outsize < len) {
			stage_out_reserve(s, len);
			s->us_outsize = len;
		}
		for (int i = 0; i < len; i++) {
			cf b = data[i];
			do {
				float w = 1 - s->us_alpha;
				cf o = { w * s->us_a.re + s->us_alpha * b.re, w * s->us_a.im + s->us_alpha * b.im };
				s->out[s->us_idx_out++] = o;
				s->us_alpha += s->us_inc;
				if (s->us_idx_out == len || s->us_idx_out == s->us_outsize) {
					fe_run(h, si + 1, s->out, s->us_idx_out);
					s->us_idx_out = 0;
				}
			} while (s->us_alpha < 1.0f);
			s->us_alpha -= 1.0f;
			s->us_a = b;
		}
		break;
	}
	case ST_DSK: { /* DSP.cpp:160-189 */
		const int nt = 26, K = 3, outputSize = 8192;
		if (len < nt - 1) return;
		stage_out_reserve(s, outputSize);
		if (s->dsk_bufsz < len + nt) {
			s->dsk_buf = (cf *)realloc(s->dsk_buf, (len + nt) * sizeof(cf));
			memset(s->dsk_buf + s->dsk_bufsz, 0, (len + nt - s->dsk_bufsz) * sizeof(cf));
			s->dsk_bufsz = len + nt;
		}
		int i, j;
		for (i = 0, j = nt - 1; i < len; i++, j++) s->dsk_buf[j] = data[i];
		while (s->dsk_idx_in < len) {
			cf x = { 0.0f, 0.0f };
			const cf *d = &s->dsk_buf[s->dsk_idx_in];
			for (int k = 0; k < nt; k++) {
				x.re += TAPS_BH_28_3[k] * d[k].re;
				x.im += TAPS_BH_28_3[k] * d[k].im;
			}
			s->out[s->dsk_idx_out] = x;
			if (++s->dsk_idx_out == outputSize) {
				fe_run(h, si + 1, s->out, outputSize);
				s->dsk_idx_out = 0;
			}
			s->dsk_idx_in += K;
		}
		s->dsk_idx_in -= len;
		for (j = 0, i = len - nt + 1; j < nt - 1; i++, j++) s->dsk_buf[j] = data[i];
		break;
	}
	}
}

/* Model.cpp:129-338: rate -> chain */
static int build_frontend(Handle *h) {
	static const unsigned rates[9] = { 96000, 192000, 288000, 384000, 768000, 1536000, 3072000, 6144000, 12288000 };
	int sr = h->sample_rate;
	if (sr < 96000 || sr > 12288000) return -1;
	unsigned bucket = 0;
	int interp = 0;
	for (int i = 0; i < 9; i++)
		if (rates[i] >= (unsigned)sr) {
			bucket = rates[i];
			interp = rates[i] != (unsigned)sr;
			break;
		}
	int droop = (h->flags & FLAG_DROOP) != 0;
	int n = 0;
	memset(h->st, 0, sizeof(h->st));
#define ADD(k) h->st[n++].kind = (k)
	if (bucket == 288000) {
		if (interp) ADD(ST_US);
		ADD(ST_DSK);
	}
	else {
		int k = 0;
		for (unsigned b = bucket; b > 96000; b >>= 1) k++;
		int post = k < 2 ? k : 2; /* US sits in front of the last min(k,2) DS2 stages */
		for (int i = 0; i < k - post; i++) ADD(ST_DS2);
		if (interp) ADD(ST_US);
		for (int i = 0; i < post; i++) ADD(ST_DS2);
		if (droop && k > 0) {
			float a;
			switch (bucket) {
			case 12288000: case 6144000: a = -2.0f; break;
			case 3072000: a = -1.5f; break;
			case 1536000: case 768000: a = -1.2f; break;
			case 384000: a = -1.1f; break;
			default: a = -0.8f; break;
			}
			h->st[n].alpha = a;
			h->st[n].beta = 1 - 2 * a;
			ADD(ST_FDC);
		}
	}
#undef ADD
	for (int i = 0; i < n; i++)
		if (h->st[i].kind == ST_US) {
			h->st[i].us_inc = (float)sr / (float)bucket;
			h->st[i].us_alpha = 0;
		}
	h->nst = n;
	return 0;
}

/* ================= C entry points ================= */
void *aisorc_create(int model, int sample_rate, int format, unsigned flags, int own_mmsi) {
	if (model < 0 || (model > 2 && model != MODEL_CHALLENGER) || format < 0 || format > 3) return NULL;
	if (flags & (16u | 32u)) return NULL; /* -go FP_DS / DSK: checked against the compiled reference (ref_harness.cpp) only */
	/* single-channel mode: ModelChallenger at 48k only (no US / DS2 in front), the one case pinned against the reference */
	if ((flags & FLAG_MODE_X) && (sample_rate != 48000 || model != MODEL_CHALLENGER)) return NULL;
	Handle *h = (Handle *)calloc(1, sizeof(Handle));
	h->model = model;
	h->sample_rate = sample_rate;
	h->format = format;
	h->flags = flags;
	h->own_mmsi = own_mmsi;
	h->ps_ema = (flags & FLAG_PS_EMA) != 0;
	h->afc_wide = (flags & FLAG_AFC_WIDE) != 0;
	h->taps_on = (flags & FLAG_TAPS) != 0;
	h->mode_x = (flags & FLAG_MODE_X) != 0;
	memcpy(h->order, CHALLENGER_ORDER, sizeof(h->order));
	if (!h->mode_x && build_frontend(h)) {
		free(h);
		return NULL;
	}
	h->rot.re = 1.0f;
	h->mult = polar1((float)(PI_F * 25000.0 / 48000.0)); /* Model.cpp:31 */
	for (int s = 0; s < 512; s++) /* FFT.h:81-83 */
		h->omega[s] = polar1((float)(-2.0 * PI_F) * (float)s / (float)512);
	h->tag.mode = 3;
	for (int c = 0; c < 2; c++) {
		Chan *ch = &h->ch[c];
		ch->h = h;
		ch->id = c;
		ch->name = h->mode_x ? 'X' : c ? 'B' : 'A';
		ch->cgf.rot.re = 1.0f;
		ch->fc.taps = (float *)TAPS_COHERENT;
		ch->fc.nt = 17;
		ch->fc.buffer = (cf *)calloc(34, sizeof(cf));
		ch->fr.taps = (float *)TAPS_RECEIVER;
		ch->fr.nt = 37;
		ch->fr.buffer = (float *)calloc(74, sizeof(float));
		ch->pll_fast = 1;
		for (int i = 0; i < 10; i++) {
			ch->dec[i].ch = ch;
			ch->dec[i].idx = i;
			ch->dec[i].state = S_TRAINING;
		}
	}
	return h;
}

int aisorc_push(void *hv, const void *data, long nbytes) {
	Handle *h = (Handle *)hv;
	const cf *x;
	long n;
	if (h->format == 0) {
		x = (const cf *)data;
		n = nbytes / 8;
	}
	else {
		n = h->format == 3 ? nbytes / 4 : nbytes / 2;
		if (h->convcap < n) {
			h->conv = (cf *)realloc(h->conv, n * sizeof(cf));
			h->convcap = n;
		}
		if (h->format == 1) { /* CU8, Convert.cpp:255-264 */
			const uint8_t *d = (const uint8_t *)data;
			for (long i = 0; i < n; i++) {
				h->conv[i].re = ((int)d[2 * i] - 128) / 128.0f;
				h->conv[i].im = ((int)d[2 * i + 1] - 128) / 128.0f;
			}
		}
		else if (h->format == 2) { /* CS8 */
			const int8_t *d = (const int8_t *)data;
			for (long i = 0; i < n; i++) {
				h->conv[i].re = d[2 * i] / 128.0f;
				h->conv[i].im = d[2 * i + 1] / 128.0f;
			}
		}
		else { /* CS16 */
			const int16_t *d = (const int16_t *)data;
			for (long i = 0; i < n; i++) {
				h->conv[i].re = d[2 * i] / 32768.0f;
				h->conv[i].im = d[2 * i + 1] / 32768.0f;
			}
		}
		x = h->conv;
	}
	fe_run(h, 0, x, (int)n);
	return 0;
}

static long take(fvec *v, float *dst, long max) {
	long n = v->n;
	if (dst) {
		long k = n < max ? n : max;
		memcpy(dst, v->p, k * sizeof(float));
		v->n = 0;
	}
	return n;
}
long aisorc_tap_c(void *hv, int tap, float *dst, long max) {
	if (tap < 0 || tap >= NTAPS_C) return -1;
	return take(&((Handle *)hv)->tc[tap], dst, max);
}
long aisorc_tap_ppm(void *hv, int tap, float *dst, long max) {
	if (tap < 0 || tap >= NTAPS_C) return -1;
	return take(&((Handle *)hv)->tppm[tap], dst, max);
}
long aisorc_tap_f(void *hv, int tap, float *dst, long max) {
	if (tap < 0 || tap >= NTAPS_F) return -1;
	return take(&((Handle *)hv)->tf[tap], dst, max);
}
long aisorc_msg_count(void *hv) { return ((Handle *)hv)->msg_count; }

/* The decoder that published each message aisorc_messages has not yet returned, in the same order (Decoder.idx: the phase for
 * models 0 and 2, 0 for model 1; for ModelChallenger 0..4 the coherent phases, 5..9 the FM phases).  Copies up to max and clears
 * when dst != NULL; returns the count. */
long aisorc_publishers(void *hv, int *dst, long max) {
	Handle *h = (Handle *)hv;
	long n = h->npub;
	if (dst) {
		long k = n < max ? n : max;
		memcpy(dst, h->pub, k * sizeof(int));
		h->npub = 0;
	}
	return n;
}

/* Test hook: ModelChallenger's order of its ten decoders within a group (numbered as by aisorc_publishers).  The reference's is
 * CHALLENGER_ORDER; any permutation is accepted, anything else refused (-1). */
int aisorc_challenger_order(void *hv, const int order[10]) {
	Handle *h = (Handle *)hv;
	int seen = 0;
	for (int i = 0; i < 10; i++) {
		if (order[i] < 0 || order[i] > 9 || (seen >> order[i] & 1)) return -1;
		seen |= 1 << order[i];
	}
	memcpy(h->order, order, sizeof(h->order));
	return 0;
}
long aisorc_messages(void *hv, char *dst, long max) {
	Handle *h = (Handle *)hv;
	long n = h->text.n;
	if (dst) {
		long k = n < max ? n : max;
		memcpy(dst, h->text.p, k);
		h->text.n = 0;
	}
	return n;
}
void aisorc_destroy(void *hv) {
	Handle *h = (Handle *)hv;
	if (!h) return;
	for (int i = 0; i < h->nst; i++) {
		free(h->st[i].out);
		free(h->st[i].dsk_buf);
	}
	for (int c = 0; c < 2; c++) {
		free(h->ch[c].fc.buffer);
		free(h->ch[c].fr.buffer);
	}
	for (int i = 0; i < NTAPS_C; i++) {
		free(h->tc[i].p);
		free(h->tppm[i].p);
	}
	for (int i = 0; i < NTAPS_F; i++) free(h->tf[i].p);
	free(h->up);
	free(h->down);
	free(h->conv);
	free(h->tmpf);
	free(h->tmpf2);
	free(h->tmpc);
	free(h->text.p);
	free(h->pub);
	free(h);
}
