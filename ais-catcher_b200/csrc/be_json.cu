// The record of a frame in every message format of the reference's outputs (MSGFORMAT, OutputMessage::formatInto) -- NMEA,
// NMEA_TAG, COMMUNITY_HUB, BINARY_NMEA, FULL, JSON_NMEA, and the full AIS JSON that JSONAIS::ProcessMsg builds, written by
// JSON::Serializer in the full (JSON_FULL: -o 5 and the HTTP / UDP / MQTT JSON outputs) or sparse dictionary (JSON_SPARSE) or
// annotated (JSON_ANNOTATED) -- by one formatter around one table interpreter.  The interpreter is written against a writer: the
// engine runs it on the device with the plain full-dictionary writer Out (one thread per published frame, aisgpu_poll_json); the
// host runs it with Out (aisgpu_msg_json_full) and with the dictionary-aware DOut, inside the record formatter (aisgpu_msg_format and
// the egress formatters aisgpu_msg_json / aisgpu_msg_binary).
//
// A message type is a program of field operations (U / UL / SL / E / B / TURN / text / timestamp / ETA / data / radio) in
// constant memory; the layouts with control flow (types 22, 24, 25, 26 and the application messages of 6 and 8) pick programs in
// body().  Field positions and sentinels follow ITU-R M.1371; names, order and number formatting are the reference's:
//   - integers as decimal; floats as a double, at most six decimals rounded half to even, trailing zeros trimmed, "null" outside
//     (-1e18, 1e18);
//   - a scaled field is computed in float (raw * scale + offset, the scale a float) and only then widened to double;
//   - text is 6-bit ASCII up to the first '@' (0), trailing spaces trimmed, and a field that would reach beyond bit 1064 is "";
//   - bits beyond the frame's length are read as they are in aisgpu_msg::data, and bits from 1064 on as 0.
// Types 6 and 8 (and 25 / 26 with structured data) decode every (DAC, FI) the reference decodes into fields (kAsm6 / kAsm8): flat
// layouts as programs, the ones with records, loops or formatted strings in app_special; every other (DAC, FI) prints its payload
// as "data" ("<bits>:<hex>"), as the reference does.

#include "be_json.h"
#include "fmt_text.h"
#include "json_text.h"

#include <cub/block/block_scan.cuh>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>


namespace {

#ifdef __CUDA_ARCH__
#define AJ_TAB(name) d_##name
#else
#define AJ_TAB(name) h_##name
#endif
// one table, a host and a constant-memory copy of it
#define AJ_TABLE(type, name, n, init)           \
	static const type h_##name[n] = init;       \
	__constant__ type d_##name[n] = init;

// ---- keys: the full dictionary's names, in one list ----
#define AJ_KEYS(X)                                                                                                                  \
	X(type) X(repeat) X(mmsi) X(country) X(country_code) X(status) X(status_text) X(turn_unscaled) X(turn) X(speed) X(accuracy)      \
	X(lon) X(lat) X(course) X(heading) X(second) X(maneuver) X(power) X(raim) X(radio) X(sync_state) X(slot_timeout) X(slot_offset) \
	X(utc_hour) X(utc_minute) X(slot_number) X(received_stations) X(timestamp) X(year) X(month) X(day) X(hour) X(minute) X(epfd)   \
	X(epfd_text) X(transmission_control) X(ais_version) X(imo) X(callsign) X(shipname) X(shiptype) X(shiptype_text) X(to_bow)      \
	X(to_stern) X(to_port) X(to_starboard) X(eta) X(draught) X(destination) X(dte) X(seqno) X(dest_mmsi) X(retransmit) X(dac)      \
	X(fid) X(data) X(mmsi1) X(mmsiseq1) X(mmsi2) X(mmsiseq2) X(mmsi3) X(mmsiseq3) X(mmsi4) X(mmsiseq4) X(alt) X(alt_sensor)        \
	X(assigned) X(text) X(type1_1) X(offset1_1) X(type1_2) X(offset1_2) X(type2_1) X(offset2_1) X(offset1) X(increment1)          \
	X(offset2) X(increment2) X(reserved) X(cs) X(display) X(dsc) X(band) X(msg22) X(number1) X(timeout1) X(number2) X(timeout2)    \
	X(offset3) X(number3) X(timeout3) X(increment3) X(offset4) X(number4) X(timeout4) X(increment4) X(aid_type) X(aid_type_text)   \
	X(name) X(off_position) X(aton_status) X(virtual_aid) X(channel_a) X(channel_b) X(txrx) X(dest1) X(dest2) X(ne_lon) X(ne_lat)  \
	X(sw_lon) X(sw_lat) X(addressed) X(band_a) X(band_b) X(zonesize) X(station_type) X(interval) X(quiet) X(partno) X(vendorid)    \
	X(model) X(serial) X(mothership_mmsi) X(vdes_capabilities) X(ai_available) X(gnss) X(restricted_use) X(aton_station_type)       \
	X(iala_mrn) X(dim_type) X(additional_flag) X(charted_status) X(on_station_status) X(auth_flag) X(asm_sub_app_id)                \
	X(asm_voltage_data) X(asm_current_data) X(asm_power_supply_type) X(asm_light_status) X(asm_battery_status)                     \
	X(asm_off_position_status) X(ack_required) X(text_sequence) X(requested_dac) X(requested_fid) X(persons) X(berth_type)         \
	X(berth_number) X(berth_name) X(berth_arrival_time) X(berth_departure_time) X(berth_lon) X(berth_lat) X(area_notice_type)      \
	X(area_notice_duration) X(area_notice_priority) X(area_notice_lon1) X(area_notice_lat1) X(area_notice_lon2)                    \
	X(area_notice_lat2) X(area_notice_name) X(cargo_hazard_report_type) X(cargo_hazard_class) X(cargo_hazard_category)            \
	X(cargo_hazard_id) X(cargo_hazard_quantity) X(linkage_id) X(crew_count) X(passenger_count) X(shipboard_personnel_count)        \
	X(ana_int) X(ana_ext1) X(ana_ext2) X(racon) X(health) X(stat_ext) X(station_name) X(utc_day)        \
	X(station_id) X(message_id) X(wspeed) X(wgust) X(wdir) X(barometric_pressure) X(air_temperature) X(dew_point) X(visibility_km)  \
	X(watertemp) X(water_level_type) X(waterlevel) X(reference_datum) X(reading_type) X(wind_speed_avg) X(wind_gust_speed)         \
	X(wind_direction_avg) X(water_flow) X(vts_target_id_type) X(vts_target_id) X(vts_target_lat) X(vts_target_lon)               \
	X(vts_target_cog) X(vts_target_timestamp) X(vts_target_sog) X(vin) X(length) X(beam) X(hazard) X(loaded) X(speed_q) X(course_q) \
	X(heading_q) X(wgustdir) X(airtemp) X(humidity) X(dewpoint) X(pressure) X(pressuretend) X(visgreater) X(visibility)           \
	X(leveltrend) X(cspeed) X(cdir) X(cspeed2) X(cdir2) X(cdepth2) X(cspeed3) X(cdir3) X(cdepth3) X(waveheight) X(waveperiod)      \
	X(wavedir) X(swellheight) X(swellperiod) X(swelldir) X(seastate) X(preciptype) X(salinity) X(ice) X(asm_version) X(un_country) \
	X(fairway_section) X(object_code) X(fairway_hectometre) X(bridge_clearance) X(measurement_age) X(clearance_accuracy)          \
	X(weather_report_type) X(present_weather) X(pressuretend_wmo) X(sender_classification) X(route_type) X(duration_minutes)      \
	X(waypoint_count) X(waypoints) X(sensor_report_type) X(site_id) X(report_type) X(version) X(precision) X(sensor_description)  \
	X(forecast_wspeed) X(forecast_wgust) X(forecast_wdir) X(forecast_day) X(forecast_hour) X(forecast_minute) X(forecast_duration) \
	X(un_locode) X(terminal_code) X(tugboats) X(air_draught) X(rta) X(lock_status) X(start_date) X(end_date) X(start_time)         \
	X(end_time) X(start_lon) X(start_lat) X(end_lon) X(end_lat) X(emma_warning_type) X(min_value) X(max_value) X(emma_severity)    \
	X(wind_direction) X(gauge1_id) X(gauge1_level) X(gauge2_id) X(gauge2_level) X(gauge3_id) X(gauge3_level) X(gauge4_id)          \
	X(gauge4_level) X(signal_form) X(signal_orientation) X(signal_impact) X(signal_status) X(planned_speed) X(steering_mode)       \
	X(last_port) X(next_port) X(second_port) X(tidal) X(traffic_signal) X(next_signal) X(targets) X(class) X(device) X(driver)     \
	X(hardware) X(rxtime) X(rxuxtime) X(toa) X(scaled) X(channel) X(nmea) X(signalpower) X(ppm)

enum Key : uint16_t {
#define X(n) K_##n,
	AJ_KEYS(X)
#undef X
	K_COUNT
};

struct KeyBlob {
	char s[8192];
};
#define X(n) #n "\0"
AJ_TABLE(KeyBlob, key_blob, 1, { { AJ_KEYS(X) } })
#undef X

// offsets of the key names in key_blob, found by walking the same list at compile time
struct KeyOff {
	uint16_t o[K_COUNT];
};
constexpr KeyOff make_key_off() {
	KeyOff k{};
	const char s[] = {
#define X(n) #n "\0"
		AJ_KEYS(X)
#undef X
	};
	int at = 0;
	for (int i = 0; i < K_COUNT; i++) {
		k.o[i] = (uint16_t)at;
		while (s[at]) at++;
		at++;
	}
	return k;
}
constexpr KeyOff kKeyOff = make_key_off();
AJ_TABLE(KeyOff, key_off, 1, { kKeyOff })

// ---- the texts (json_text.h, generated from the reference's output) ----
struct TextBlob {
	char s[AJ_TEXT_BLOB_SIZE + 1];
};
AJ_TABLE(TextBlob, text_blob, 1, { { AJ_TEXT_BLOB } })
AJ_TABLE(uint16_t, t_nav, AJ_NAV_STATUS_N, AJ_NAV_STATUS_INIT)
AJ_TABLE(uint16_t, t_epfd, AJ_EPFD_N, AJ_EPFD_INIT)
AJ_TABLE(uint16_t, t_ship, AJ_SHIPTYPE_N, AJ_SHIPTYPE_INIT)
AJ_TABLE(uint16_t, t_aid, AJ_AID_TYPE_N, AJ_AID_TYPE_INIT)
AJ_TABLE(uint16_t, t_cname, AJ_COUNTRY_NAME_N, AJ_COUNTRY_NAME_INIT)
AJ_TABLE(uint16_t, t_ccode, AJ_COUNTRY_CODE_N, AJ_COUNTRY_CODE_INIT)

enum TextTab : uint8_t { TT_NONE, TT_NAV, TT_EPFD, TT_SHIP, TT_AID };

// ---- the sparse names and the annotations (fmt_text.h, generated from the reference's output), in global memory ----
#ifdef __CUDA_ARCH__
#define AF_TAB(name) d_##name
#else
#define AF_TAB(name) h_##name
#endif
#define AF_TABLE(type, name, n, init)           \
	static const type h_##name[n] = init;       \
	__device__ const type d_##name[n] = init;
#define NO 0xFFFFFFFFu
static_assert(AF_KEY_N == K_COUNT, "fmt_text.h is generated from this file's key list: run tools/gen_fmt_text.py");
struct AfBlob {
	char s[AF_BLOB_SIZE + 1];
};
AF_TABLE(AfBlob, af_blob, 1, { { AF_BLOB } })
AF_TABLE(uint32_t, af_sparse, AF_KEY_N, AF_SPARSE_INIT)
AF_TABLE(uint32_t, af_unit, AF_KEY_N, AF_UNIT_INIT)
AF_TABLE(uint32_t, af_desc, AF_KEY_N, AF_DESC_INIT)
AF_TABLE(int16_t, af_lut, AF_KEY_N, AF_LUT_INIT)
AF_TABLE(int, af_lut_at, AF_NLUT, AF_LUT_AT_INIT)
AF_TABLE(int, af_lut_n, AF_NLUT, AF_LUT_N_INIT)
AF_TABLE(uint32_t, af_lut_text, AF_LUT_TEXT_N, AF_LUT_TEXT_INIT)
#undef NO

// ---- field operations ----
enum OpCode : uint8_t {
	OP_END,
	OP_U,      // unsigned, printed unless == undef
	OP_UL,     // unsigned * a (float), printed as double unless raw == undef
	OP_SL,     // signed * a (float), unless raw == (int)undef
	OP_E,      // enumeration: the number, then (tab != TT_NONE) its text under key2, "Undefined" past the table
	OP_TURN,   // rate of turn: turn_unscaled, then turn (ITU-R M.1371 ROT_AIS = 4.733 sqrt(ROT))
	OP_B,      // bool
	OP_T,      // 6-bit text of len bits
	OP_TMIN,   // 6-bit text of min(len, nbits - start) bits
	OP_TCLAMP, // 6-bit text of min(len, nbits - start) bits cut to whole characters, printed only when at least one (< 6 bits: none)
	OP_TS,     // timestamp YYYY-MM-DDTHH:MM:SSZ of 40 bits
	OP_ETA,    // MM-DDTHH:MMZ of 20 bits
	OP_DMIN,   // "<n>:<hex>" of n = min(len, nbits - start) bits, a hex digit per 4 bits from start
	OP_RADIO,  // the SOTDMA / ITDMA state of max(min(19, nbits - start), 0) bits
	OP_BRK_LE, // stop when nbits <= start
	OP_BRK_EQ, // stop when nbits == start
	OP_BEQ,    // bool: raw == undef
	OP_BITS,   // '0' / '1' string of min(128, nbits - start) bits
	OP_S,      // signed, unless == (int)undef
	OP_US,     // unsigned + (int)a as an integer, unless raw == undef
	OP_ULLT,   // unsigned * a (float), printed only when raw < undef
};

struct Op {
	uint8_t op, tab;
	uint16_t key, key2;
	int16_t start, len;
	uint32_t undef;
	float a, b; // scale and offset of UL / SL (raw * a + b, in float); the offset of US is (int)a
};

// a field with a sentinel ("not available") is written Uu / ULu / SLu, one without Un / ULn / SLn
#define NO 0xFFFFFFFFu
#define Uu(k, s, l, u) { OP_U, 0, K_##k, 0, s, l, (uint32_t)(u), 0.f }
#define Un(k, s, l) { OP_U, 0, K_##k, 0, s, l, NO, 0.f }
#define ULu(k, s, l, a, u) { OP_UL, 0, K_##k, 0, s, l, (uint32_t)(u), a }
#define ULn(k, s, l, a) { OP_UL, 0, K_##k, 0, s, l, NO, a }
#define SLu(k, s, l, a, u) { OP_SL, 0, K_##k, 0, s, l, (uint32_t)(u), a }
#define SLn(k, s, l, a) { OP_SL, 0, K_##k, 0, s, l, NO, a }
#define E_(k, s, l) { OP_E, TT_NONE, K_##k, 0, s, l, NO, 0.f }
#define Et(k, s, l, t, k2) { OP_E, t, K_##k, K_##k2, s, l, NO, 0.f }
#define B_(k, s) { OP_B, 0, K_##k, 0, s, 1, NO, 0.f }
#define T_(k, s, l) { OP_T, 0, K_##k, 0, s, l, NO, 0.f }
#define TMIN(k, s, l) { OP_TMIN, 0, K_##k, 0, s, l, NO, 0.f }
#define TCLAMP(k, s, l) { OP_TCLAMP, 0, K_##k, 0, s, l, NO, 0.f }
#define TS_(k, s) { OP_TS, 0, K_##k, 0, s, 40, NO, 0.f }
#define ETA_(k, s) { OP_ETA, 0, K_##k, 0, s, 20, NO, 0.f }
#define DMIN(k, s, l) { OP_DMIN, 0, K_##k, 0, s, l, NO, 0.f }
#define TURN_(k, s) { OP_TURN, 0, K_##k, 0, s, 8, NO, 0.f }
#define RADIO(s) { OP_RADIO, 0, 0, 0, s, 19, NO, 0.f }
#define BRK_LE(n) { OP_BRK_LE, 0, 0, 0, n, 0, NO, 0.f }
#define BRK_EQ(n) { OP_BRK_EQ, 0, 0, 0, n, 0, NO, 0.f }
#define BEQ(k, s, l, v) { OP_BEQ, 0, K_##k, 0, s, l, (uint32_t)(v), 0.f }
#define BITS(k, s) { OP_BITS, 0, K_##k, 0, s, 128, NO, 0.f }
#define S_u(k, s, l, u) { OP_S, 0, K_##k, 0, s, l, (uint32_t)(u), 0.f }
#define USu(k, s, l, off, u) { OP_US, 0, K_##k, 0, s, l, (uint32_t)(u), (float)(off) }
#define ULbu(k, s, l, a, b, u) { OP_UL, 0, K_##k, 0, s, l, (uint32_t)(u), a, b }
#define ULLT(k, s, l, a, u) { OP_ULLT, 0, K_##k, 0, s, l, (uint32_t)(u), a }
#define END { OP_END, 0, 0, 0, 0, 0, NO, 0.f }

constexpr float kDeg4 = 1 / 600000.0f;        // 1/10000 minute
constexpr float kDeg1 = 1 / 600.0f;           // 1/10 minute
constexpr float kDeg1d = (float)(1.0 / 600.0f); // the same, formed in double and narrowed (types 22 and 23)
constexpr float kDeg60 = 1 / 60000.0f;         // 1/1000 minute

// Programs.  P_* name the entry of each in kProg; application programs are relative to their first payload bit (added at run time).
enum Prog {
	P_123, P_4, P_5, P_6, P_7, P_8, P_9, P_10, P_12, P_14, P_15, P_16, P_17, P_18, P_19, P_20, P_21, P_22H, P_22A, P_22B, P_22T,
	P_23, P_24A, P_24B, P_24DIM, P_24MS, P_24X, P_25H, P_25A, P_27, P_28,
	// application messages (start = first payload bit)
	P_IALA0, P_TEXT0, P_IMO2, P_IMO3, P_IMO4, P_IMO16, P_IMO20, P_IMO23, P_IMO25, P_IMO30, P_IN55, P_UK10, P_UK20,
	P_ERI10, P_MET31, P_BRIDGE25, P_WX21, P_TEXT29, P_ROUTE27H, P_ENV26, P_MET11, P_ENV33H, P_ENV33_0, P_ENV33_1, P_ENV33_2,
	P_ENV33_3, P_ETA21, P_RTA22, P_EMMA_POS, P_EMMA_T, P_SIG40, P_EXT24, P_TIDAL32H, P_TS19, P_SLSID, P_SLSHDR, P_SLS1, P_SLS3,
	P_SLS2, P_SLS6, P_VTS16B,
	P_COUNT,
	// layouts with control flow (app_special); P_SLSID alone serves the SLS lock and specific messages
	X_VTS16 = 100, X_WX21, X_ROUTE27, X_ENV26, X_ENV33, X_EMMA23, X_WATER24, X_SWE1, X_TIDAL32, X_VTS17, X_SLS1
};

#define AJ_OPS                                                                                                                      \
	/* P_123 */ Et(status, 38, 4, TT_NAV, status_text), TURN_(turn, 42), ULu(speed, 50, 10, 0.1f, 1023), B_(accuracy, 60),         \
	SLu(lon, 61, 28, kDeg4, 108600000), SLu(lat, 89, 27, kDeg4, 54600000), ULu(course, 116, 12, 0.1f, 3600), Uu(heading, 128, 9, 511), \
	Uu(second, 137, 6, 60), E_(maneuver, 143, 2), B_(power, 147), B_(raim, 148), RADIO(149), END,                                    \
	/* P_4 */ TS_(timestamp, 38), Uu(year, 38, 14, 0), Uu(month, 52, 4, 0), Uu(day, 56, 5, 0), Uu(hour, 61, 5, 24),                   \
	Uu(minute, 66, 6, 60), Uu(second, 72, 6, 60), B_(accuracy, 78), SLu(lon, 79, 28, kDeg4, 108600000),                              \
	SLu(lat, 107, 27, kDeg4, 54600000), Et(epfd, 134, 4, TT_EPFD, epfd_text), B_(transmission_control, 138), B_(raim, 148), RADIO(149), \
	END,                                                                                                                             \
	/* P_5 */ Un(ais_version, 38, 2), Uu(imo, 40, 30, 0), T_(callsign, 70, 42), T_(shipname, 112, 120),                              \
	Et(shiptype, 232, 8, TT_SHIP, shiptype_text), Un(to_bow, 240, 9), Un(to_stern, 249, 9), Un(to_port, 258, 6),                      \
	Un(to_starboard, 264, 6), Et(epfd, 270, 4, TT_EPFD, epfd_text), ETA_(eta, 274), Uu(month, 274, 4, 0), Uu(day, 278, 5, 0),         \
	Uu(hour, 283, 5, 24), Uu(minute, 288, 6, 60), ULu(draught, 294, 8, 0.1f, 0), T_(destination, 302, 120), B_(dte, 422), END,        \
	/* P_6 */ Un(seqno, 38, 2), Un(dest_mmsi, 40, 30), B_(retransmit, 70), Un(dac, 72, 10), Un(fid, 82, 6), END,                    \
	/* P_7 */ Un(mmsi1, 40, 30), Un(mmsiseq1, 70, 2), BRK_LE(72), Un(mmsi2, 72, 30), Un(mmsiseq2, 102, 2), BRK_LE(104),              \
	Un(mmsi3, 104, 30), Un(mmsiseq3, 134, 2), BRK_LE(136), Un(mmsi4, 136, 30), Un(mmsiseq4, 166, 2), END,                            \
	/* P_8 */ Un(dac, 40, 10), Un(fid, 50, 6), END,                                                                                  \
	/* P_9 */ Uu(alt, 38, 12, 4095), Uu(speed, 50, 10, 1023), B_(accuracy, 60), SLu(lon, 61, 28, kDeg4, 108600000),                  \
	SLu(lat, 89, 27, kDeg4, 54600000), ULu(course, 116, 12, 0.1f, 3600), Uu(second, 128, 6, 60), B_(alt_sensor, 134), B_(dte, 142),   \
	B_(assigned, 146), B_(raim, 147), Un(radio, 148, 20), END,                                                                       \
	/* P_10 */ Un(dest_mmsi, 40, 30), END,                                                                                           \
	/* P_12 */ Un(seqno, 38, 2), Un(dest_mmsi, 40, 30), B_(retransmit, 70), TMIN(text, 72, 936), END,                                \
	/* P_14 */ TMIN(text, 40, 968), END,                                                                                             \
	/* P_15 */ Un(mmsi1, 40, 30), Un(type1_1, 70, 6), Un(offset1_1, 76, 12), BRK_LE(90), Un(type1_2, 90, 6), Un(offset1_2, 96, 12),   \
	BRK_LE(110), Un(mmsi2, 110, 30), Un(type2_1, 140, 6), Un(offset2_1, 146, 12), END,                                                \
	/* P_16 */ Un(mmsi1, 40, 30), Un(offset1, 70, 12), Un(increment1, 82, 10), BRK_EQ(92), Un(mmsi2, 92, 30), Un(offset2, 122, 12),  \
	Un(increment2, 134, 10), END,                                                                                                    \
	/* P_17 */ SLu(lon, 40, 18, kDeg1, 108600), SLu(lat, 58, 17, kDeg1, 54600), DMIN(data, 80, 736), END,                            \
	/* P_18 */ ULu(speed, 46, 10, 0.1f, 1023), B_(accuracy, 56), SLu(lon, 57, 28, kDeg4, 108600000), SLu(lat, 85, 27, kDeg4, 54600000), \
	ULu(course, 112, 12, 0.1f, 3600), Uu(heading, 124, 9, 511), Un(reserved, 38, 8), Uu(second, 133, 6, 60), B_(power, 139),         \
	B_(cs, 141), B_(display, 142), B_(dsc, 143), B_(band, 144), B_(msg22, 145), B_(assigned, 146), B_(raim, 147), Un(radio, 148, 20), \
	END,                                                                                                                             \
	/* P_19 */ ULu(speed, 46, 10, 0.1f, 1023), SLu(lon, 57, 28, kDeg4, 108600000), SLu(lat, 85, 27, kDeg4, 54600000),                \
	ULu(course, 112, 12, 0.1f, 3600), Uu(heading, 124, 9, 511), T_(shipname, 143, 120), Et(shiptype, 263, 8, TT_SHIP, shiptype_text), \
	Un(to_bow, 271, 9), Un(to_stern, 280, 9), Un(to_port, 289, 6), Un(to_starboard, 295, 6), Et(epfd, 301, 4, TT_EPFD, epfd_text),    \
	B_(accuracy, 56), Uu(second, 133, 6, 60), B_(raim, 305), B_(dte, 306), B_(assigned, 307), END,                                    \
	/* P_20 */ Un(offset1, 40, 12), Un(number1, 52, 4), Un(timeout1, 56, 3), Un(increment1, 59, 11), BRK_LE(99), Un(offset2, 70, 12), \
	Un(number2, 82, 4), Un(timeout2, 86, 3), Un(increment2, 89, 11), BRK_LE(129), Un(offset3, 100, 12), Un(number3, 112, 4),          \
	Un(timeout3, 116, 3), Un(increment3, 119, 11), BRK_LE(159), Un(offset4, 130, 12), Un(number4, 142, 4), Un(timeout4, 146, 3),      \
	Un(increment4, 149, 11), END,                                                                                                    \
	/* P_21 */ Et(aid_type, 38, 5, TT_AID, aid_type_text), T_(name, 43, 120), B_(accuracy, 163), SLu(lon, 164, 28, kDeg4, 108600000), \
	SLu(lat, 192, 27, kDeg4, 54600000), Un(to_bow, 219, 9), Un(to_stern, 228, 9), Un(to_port, 237, 6), Un(to_starboard, 243, 6),     \
	Et(epfd, 249, 4, TT_EPFD, epfd_text), Uu(second, 253, 6, 60), B_(off_position, 259), Un(aton_status, 260, 8), B_(raim, 268),     \
	B_(virtual_aid, 269), B_(assigned, 270), END,                                                                                    \
	/* P_22H */ Un(channel_a, 40, 12), Un(channel_b, 52, 12), Un(txrx, 64, 4), B_(power, 68), END,                                  \
	/* P_22A */ Un(dest1, 69, 30), Un(dest2, 104, 30), END,                                                                          \
	/* P_22B */ SLn(ne_lon, 69, 18, kDeg1d), SLn(ne_lat, 87, 17, kDeg1d), SLn(sw_lon, 104, 18, kDeg1d), SLn(sw_lat, 122, 17, kDeg1d), \
	END,                                                                                                                             \
	/* P_22T */ B_(addressed, 139), B_(band_a, 140), B_(band_b, 141), Un(zonesize, 142, 3), END,                                    \
	/* P_23 */ SLn(ne_lon, 40, 18, kDeg1d), SLn(ne_lat, 58, 17, kDeg1d), SLn(sw_lon, 75, 18, kDeg1d), SLn(sw_lat, 93, 17, kDeg1d),    \
	E_(station_type, 110, 4), Et(shiptype, 114, 8, TT_SHIP, shiptype_text), Un(txrx, 144, 2), E_(interval, 146, 4), Un(quiet, 150, 4), \
	END,                                                                                                                             \
	/* P_24A */ T_(shipname, 40, 120), END,                                                                                          \
	/* P_24B */ Et(shiptype, 40, 8, TT_SHIP, shiptype_text), T_(vendorid, 48, 18), Un(model, 66, 4), Un(serial, 70, 20),              \
	T_(callsign, 90, 42), END,                                                                                                       \
	/* P_24DIM */ Un(to_bow, 132, 9), Un(to_stern, 141, 9), Un(to_port, 150, 6), Un(to_starboard, 156, 6), END,                    \
	/* P_24MS */ Un(mothership_mmsi, 132, 30), END,                                                                                 \
	/* P_24X */ Et(epfd, 162, 4, TT_EPFD, epfd_text), Un(vdes_capabilities, 166, 2), END,                                           \
	/* P_25H */ B_(addressed, 38), B_(ai_available, 39), END,                                                                        \
	/* P_25A */ Un(dest_mmsi, 40, 30), END,                                                                                          \
	/* P_27 */ B_(accuracy, 38), B_(raim, 39), Et(status, 40, 4, TT_NAV, status_text), SLu(lon, 44, 18, kDeg1, 108600),              \
	SLu(lat, 62, 17, kDeg1, 54600), Uu(speed, 79, 6, 63), Uu(course, 85, 9, 511), Un(gnss, 94, 1), END,                              \
	/* P_28 */ Uu(second, 38, 6, 60), SLu(lon, 44, 28, kDeg4, 108600000), SLu(lat, 72, 27, kDeg4, 54600000), Un(restricted_use, 99, 2), \
	Un(aton_station_type, 101, 3), BEQ(virtual_aid, 101, 3, 4), Et(aid_type, 104, 7, TT_AID, aid_type_text), Un(iala_mrn, 111, 17),  \
	Un(dim_type, 128, 4), Un(to_bow, 132, 9), Un(to_stern, 141, 11), B_(additional_flag, 152), B_(charted_status, 153),               \
	Un(on_station_status, 154, 4), Un(aton_status, 158, 8), B_(auth_flag, 167), END,                                                  \
	/* P_IALA0: IALA buoy monitor */ Un(asm_sub_app_id, 0, 16), ULn(asm_voltage_data, 16, 12, 0.1f), ULn(asm_current_data, 28, 10, 0.1f), \
	B_(asm_power_supply_type, 38), B_(asm_light_status, 39), B_(asm_battery_status, 40), B_(asm_off_position_status, 41), END,        \
	/* P_TEXT0: text, 6-bit */ B_(ack_required, 0), Un(text_sequence, 1, 11), TMIN(text, 12, 924), END,                            \
	/* P_IMO2: interrogation */ Un(requested_dac, 0, 10), Un(requested_fid, 10, 6), END,                                             \
	/* P_IMO3: interrogation for a DAC */ Un(requested_dac, 0, 10), END,                                                             \
	/* P_IMO4: capability reply */ BITS(ai_available, 0), END,                                                                       \
	/* P_IMO16: persons on board */ Uu(persons, 0, 13, 8191), END,                                                                   \
	/* P_IMO20: berthing data */ Un(berth_type, 0, 4), Uu(berth_number, 4, 10, 0), T_(berth_name, 14, 84),                          \
	Uu(berth_arrival_time, 98, 20, 0), Uu(berth_departure_time, 118, 20, 0), SLn(berth_lon, 138, 25, kDeg4),                         \
	SLn(berth_lat, 163, 24, kDeg4), END,                                                                                             \
	/* P_IMO23: area notice */ Un(area_notice_type, 0, 7), Uu(area_notice_duration, 7, 13, 0), B_(area_notice_priority, 20),        \
	SLn(area_notice_lon1, 21, 25, kDeg4), SLn(area_notice_lat1, 46, 24, kDeg4), SLn(area_notice_lon2, 70, 25, kDeg4),                 \
	SLn(area_notice_lat2, 95, 24, kDeg4), TCLAMP(area_notice_name, 119, 360), END,                                                    \
	/* P_IMO25: dangerous cargo */ Un(cargo_hazard_report_type, 0, 8), Un(cargo_hazard_class, 8, 4), Un(cargo_hazard_category, 12, 4), \
	Uu(cargo_hazard_id, 16, 13, 0), ULn(cargo_hazard_quantity, 29, 10, 0.1f), END,                                                    \
	/* P_IMO30: text, addressed */ Uu(linkage_id, 0, 10, 0), TCLAMP(text, 10, 930), END,                                             \
	/* P_IN55: persons on board (inland) */ Uu(crew_count, 0, 8, 255), Uu(passenger_count, 8, 13, 8191),                            \
	Uu(shipboard_personnel_count, 21, 8, 255), END,                                                                                  \
	/* P_UK10: AtoN monitor */ ULn(ana_int, 0, 10, 0.05f), ULn(ana_ext1, 10, 10, 0.05f), ULn(ana_ext2, 20, 10, 0.05f),              \
	Un(racon, 30, 2), Un(health, 34, 1), Un(stat_ext, 35, 8), B_(off_position, 43), END,                                             \
	/* P_UK20: buoy position */ T_(station_name, 0, 204), Uu(utc_day, 204, 5, 0), Uu(utc_hour, 209, 5, 24), Uu(utc_minute, 214, 6, 60), \
	SLu(lon, 220, 28, kDeg4, 1810000), SLu(lat, 248, 27, kDeg4, 910000), B_(off_position, 275), END,                               \
	/* P_ERI10: inland static and voyage data */ T_(vin, 0, 48), ULn(length, 48, 13, 0.1f), ULn(beam, 61, 10, 0.1f),               \
	Un(shiptype, 71, 14), Un(hazard, 85, 3), ULn(draught, 88, 11, 0.01f), Un(loaded, 99, 2), B_(speed_q, 101), B_(course_q, 102),    \
	B_(heading_q, 103), END,                                                                                                         \
	/* P_MET31: meteorological / hydrological data */ SLn(lon, 0, 25, kDeg60), SLn(lat, 25, 24, kDeg60), B_(accuracy, 49),          \
	Uu(day, 50, 5, 0), Uu(hour, 55, 5, 24), Uu(minute, 60, 6, 60), Uu(wspeed, 66, 7, 127), Uu(wgust, 73, 7, 127),                   \
	Uu(wdir, 80, 9, 360), Uu(wgustdir, 89, 9, 360), SLu(airtemp, 98, 11, 0.1f, -1024), Uu(humidity, 109, 7, 101),                    \
	SLu(dewpoint, 116, 10, 0.1f, 501), USu(pressure, 126, 9, 799, 511), Uu(pressuretend, 135, 2, 3), B_(visgreater, 137),            \
	ULu(visibility, 138, 7, 0.1f, 127), ULbu(waterlevel, 145, 12, 0.01f, -10.0f, 4001), Uu(leveltrend, 157, 2, 3),                   \
	ULu(cspeed, 159, 8, 0.1f, 255), Uu(cdir, 167, 9, 360), ULu(cspeed2, 176, 8, 0.1f, 255), Uu(cdir2, 184, 9, 360),                  \
	Uu(cdepth2, 193, 5, 31), ULu(cspeed3, 198, 8, 0.1f, 255), Uu(cdir3, 206, 9, 360), Uu(cdepth3, 215, 5, 31),                       \
	ULu(waveheight, 220, 8, 0.1f, 255), Uu(waveperiod, 228, 6, 63), Uu(wavedir, 234, 9, 360), ULu(swellheight, 243, 8, 0.1f, 255),   \
	Uu(swellperiod, 251, 6, 63), Uu(swelldir, 257, 9, 360), Uu(seastate, 266, 4, 13), SLu(watertemp, 270, 10, 0.1f, 501),            \
	Uu(preciptype, 280, 3, 7), ULLT(salinity, 283, 9, 0.1f, 510), Uu(ice, 292, 2, 3), END,                                           \
	/* P_BRIDGE25: bridge clearance */ Un(asm_version, 0, 3), T_(un_country, 3, 12), Uu(fairway_section, 15, 17, 0),               \
	T_(object_code, 32, 30), Uu(fairway_hectometre, 62, 17, 0), Uu(bridge_clearance, 79, 14, 0), Uu(measurement_age, 93, 10, 722),   \
	Uu(clearance_accuracy, 103, 5, 0), END,                                                                                          \
	/* P_WX21: weather observation, non-WMO variant */ T_(station_name, 1, 120), SLu(lon, 121, 25, kDeg60, 10860000),               \
	SLu(lat, 146, 24, kDeg60, 5460000), Uu(day, 170, 5, 0), Uu(hour, 175, 5, 24), Uu(minute, 180, 6, 60),                           \
	Uu(present_weather, 186, 4, 8), B_(visgreater, 190), ULu(visibility, 191, 7, 0.1f, 127), Uu(humidity, 198, 7, 101),               \
	Uu(wspeed, 205, 7, 127), Uu(wdir, 212, 9, 360), USu(pressure, 221, 9, 799, 403), Uu(pressuretend_wmo, 230, 4, 15),               \
	SLu(airtemp, 234, 11, 0.1f, -1024), SLu(watertemp, 245, 10, 0.1f, 501), Uu(waveperiod, 255, 6, 63),                             \
	ULu(waveheight, 261, 8, 0.1f, 255), Uu(wavedir, 269, 9, 360), ULu(swellheight, 278, 8, 0.1f, 255), Uu(swelldir, 286, 9, 360),    \
	Uu(swellperiod, 295, 6, 63), END,                                                                                                \
	/* P_TEXT29: text description */ Uu(linkage_id, 0, 10, 0), TCLAMP(text, 10, 966), END,                                        \
	/* P_ROUTE27H: route information */ Uu(linkage_id, 0, 10, 0), Un(sender_classification, 10, 3), Un(route_type, 13, 5),        \
	Uu(month, 18, 4, 0), Uu(day, 22, 5, 0), Uu(hour, 27, 5, 24), Uu(minute, 32, 6, 60), Uu(duration_minutes, 38, 18, 262143),        \
	Uu(waypoint_count, 56, 5, 0), END,                                                                                               \
	/* P_ENV26: environmental, first report's header */ Un(sensor_report_type, 0, 4), Uu(day, 4, 5, 0), Uu(hour, 9, 5, 24),        \
	Uu(minute, 14, 6, 60), Un(site_id, 20, 7), END,                                                                                  \
	/* P_MET11: meteorological / hydrological data, old layout */ SLu(lat, 0, 24, kDeg60, 8388607), SLu(lon, 24, 25, kDeg60, 16777215), \
	Uu(day, 49, 5, 0), Uu(hour, 54, 5, 24), Uu(minute, 59, 6, 60), Uu(wspeed, 65, 7, 127), Uu(wgust, 72, 7, 127), Uu(wdir, 79, 9, 511), \
	Uu(wgustdir, 88, 9, 511), ULbu(airtemp, 97, 11, 0.1f, -60.0f, 2047), Uu(humidity, 108, 7, 127),                                   \
	ULbu(dewpoint, 115, 10, 0.1f, -20.0f, 1023), USu(pressure, 125, 9, 800, 511), Uu(pressuretend, 134, 2, 3),                       \
	ULu(visibility, 136, 8, 0.1f, 255), ULbu(waterlevel, 144, 9, 0.1f, -10.0f, 511), Uu(leveltrend, 153, 2, 3),                      \
	ULu(cspeed, 155, 8, 0.1f, 255), Uu(cdir, 163, 9, 511), ULu(cspeed2, 172, 8, 0.1f, 255), Uu(cdir2, 180, 9, 511),                  \
	Uu(cdepth2, 189, 5, 31), ULu(cspeed3, 194, 8, 0.1f, 255), Uu(cdir3, 202, 9, 511), Uu(cdepth3, 211, 5, 31),                       \
	ULu(waveheight, 216, 8, 0.1f, 255), Uu(waveperiod, 224, 6, 63), Uu(wavedir, 230, 9, 511), ULu(swellheight, 239, 8, 0.1f, 255),   \
	Uu(swellperiod, 247, 6, 63), Uu(swelldir, 253, 9, 511), Uu(seastate, 262, 4, 13), ULbu(watertemp, 266, 10, 0.1f, -10.0f, 1023),  \
	Uu(preciptype, 276, 3, 7), ULu(salinity, 279, 9, 0.1f, 511), Uu(ice, 288, 2, 3), END,                                           \
	/* P_ENV33H: environmental sensor report header */ Un(report_type, 0, 4), Uu(day, 4, 5, 0), Uu(hour, 9, 5, 24),                \
	Uu(minute, 14, 6, 60), Un(site_id, 20, 7), END,                                                                                  \
	/* P_ENV33_0: site location */ Un(version, 0, 6), SLn(lon, 6, 28, kDeg4), SLn(lat, 34, 27, kDeg4), Un(precision, 61, 3),      \
	S_u(alt, 64, 12, -4096), END,                                                                                                    \
	/* P_ENV33_1: station id */ T_(name, 0, 84), END,                                                                                \
	/* P_ENV33_2: wind */ Uu(wspeed, 0, 7, 127), Uu(wgust, 7, 7, 127), Uu(wdir, 14, 9, 360), Uu(wgustdir, 23, 9, 360),                \
	Un(sensor_description, 33, 2), Uu(forecast_wspeed, 35, 7, 127), Uu(forecast_wgust, 42, 7, 127), Uu(forecast_wdir, 49, 9, 360),    \
	Uu(forecast_day, 58, 5, 0), Uu(forecast_hour, 63, 5, 24), Uu(forecast_minute, 68, 6, 60), Uu(forecast_duration, 74, 8, 255), END, \
	/* P_ENV33_3: water level */ Un(water_level_type, 0, 1), SLu(waterlevel, 1, 16, 0.01f, -32768), Un(leveltrend, 17, 2),          \
	Un(reference_datum, 19, 5), END,                                                                                                 \
	/* P_ETA21: inland ETA */ T_(un_country, 0, 12), T_(un_locode, 12, 18), T_(fairway_section, 30, 30), T_(terminal_code, 60, 30),  \
	T_(fairway_hectometre, 90, 30), ETA_(eta, 120), Uu(tugboats, 140, 3, 7), ULu(air_draught, 143, 12, 0.01f, 0), END,                \
	/* P_RTA22: inland RTA */ T_(un_country, 0, 12), T_(un_locode, 12, 18), T_(fairway_section, 30, 30), T_(terminal_code, 60, 30),  \
	T_(fairway_hectometre, 90, 30), ETA_(rta, 120), Uu(lock_status, 140, 2, 3), END,                                                  \
	/* P_EMMA_POS: EMMA warning area */ SLn(start_lon, 56, 28, kDeg4), SLn(start_lat, 84, 27, kDeg4), SLn(end_lon, 111, 28, kDeg4),  \
	SLn(end_lat, 139, 27, kDeg4), Un(emma_warning_type, 166, 4), END,                                                                \
	/* P_EMMA_T */ Un(emma_severity, 188, 2), Un(wind_direction, 190, 4), END,                                                       \
	/* P_SIG40: signal status */ SLn(lon, 0, 28, kDeg4), SLn(lat, 28, 27, kDeg4), Un(signal_form, 55, 4),                          \
	Un(signal_orientation, 59, 9), Un(signal_impact, 68, 3), Un(signal_status, 71, 30), END,                                          \
	/* P_EXT24: extended static data */ Uu(linkage_id, 0, 10, 0), ULu(air_draught, 10, 13, 0.1f, 0), T_(last_port, 23, 30),       \
	T_(next_port, 53, 30), T_(second_port, 83, 30), END,                                                                             \
	/* P_TIDAL32H: tidal window */ Uu(month, 0, 4, 0), Uu(day, 4, 5, 0), END,                                                        \
	/* P_TS19: marine traffic signal */ Uu(linkage_id, 0, 10, 0), T_(station_name, 10, 120), SLn(lon, 130, 25, kDeg60),            \
	SLn(lat, 155, 24, kDeg60), Un(traffic_signal, 181, 5), Uu(hour, 186, 5, 24), Uu(minute, 191, 6, 60), Un(next_signal, 197, 5), END, \
	/* P_SLSID: SLS message id */ Un(message_id, 2, 6), END,                                                                         \
	/* P_SLSHDR: SLS report header (relative to the report) */ Uu(month, 0, 4, 0), Uu(day, 4, 5, 0), Uu(hour, 9, 5, 24),           \
	Uu(minute, 14, 6, 60), T_(station_id, 20, 42), SLu(lon, 62, 25, kDeg60, 10800000), SLu(lat, 87, 24, kDeg60, 5400000), END,        \
	/* P_SLS1: weather station */ ULn(wspeed, 111, 10, 0.1f), ULn(wgust, 121, 10, 0.1f), Uu(wdir, 131, 9, 511),                    \
	Uu(barometric_pressure, 140, 14, 16383), SLu(air_temperature, 154, 10, 0.1f, -512), SLu(dew_point, 164, 10, 0.1f, -512),          \
	ULn(visibility_km, 174, 8, 0.1f), SLu(watertemp, 182, 10, 0.1f, -512), END,                                                       \
	/* P_SLS3: water level */ Un(water_level_type, 111, 1), SLu(waterlevel, 112, 16, 0.01f, -32768), Un(reference_datum, 128, 2),    \
	Un(reading_type, 130, 2), END,                                                                                                   \
	/* P_SLS2: wind */ ULn(wind_speed_avg, 111, 10, 0.1f), ULn(wind_gust_speed, 121, 10, 0.1f), Uu(wind_direction_avg, 131, 9, 511), END, \
	/* P_SLS6: water flow */ Uu(water_flow, 111, 14, 16383), END,                                                                    \
	/* P_VTS16B: VTS target after its id */ SLn(vts_target_lat, 48, 24, kDeg60), SLn(vts_target_lon, 72, 25, kDeg60),               \
	Uu(vts_target_cog, 97, 9, 360), Uu(vts_target_timestamp, 106, 6, 60), Uu(vts_target_sog, 112, 8, 255), END

constexpr Op kOps[] = { AJ_OPS };
constexpr int kNOps = (int)(sizeof(kOps) / sizeof(kOps[0]));
AJ_TABLE(Op, ops, kNOps, { AJ_OPS })

struct ProgIdx {
	int16_t at[P_COUNT];
};
constexpr ProgIdx make_prog_idx() {
	ProgIdx p{};
	int k = 0;
	p.at[0] = 0;
	for (int i = 0; i < kNOps && k + 1 < P_COUNT; i++)
		if (kOps[i].op == OP_END) p.at[++k] = (int16_t)(i + 1);
	return p;
}
constexpr ProgIdx kProgIdx = make_prog_idx();
static_assert(kProgIdx.at[P_COUNT - 1] > 0, "one END per program");
AJ_TABLE(ProgIdx, prog_idx, 1, { kProgIdx })

// The application messages of types 6 (addressed) and 8 (broadcast): (DAC, FI) -> program (< P_COUNT) or layout with control flow
// (X_*, app_special).  Anything else is printed as "data".
struct Asm {
	int16_t dac, fid, prog;
};
#define ASM6                                                                                                                        \
	{ 0, 0, P_IALA0 }, { 1, 0, P_TEXT0 }, { 1, 2, P_IMO2 }, { 1, 3, P_IMO3 }, { 1, 4, P_IMO4 }, { 1, 16, P_IMO16 }, { 1, 40, P_IMO16 }, \
	{ 1, 20, P_IMO20 }, { 1, 23, P_IMO23 }, { 1, 25, P_IMO25 }, { 1, 28, X_ROUTE27 }, { 1, 32, X_TIDAL32 }, { 1, 30, P_IMO30 }, { 210, 0, P_TEXT0 },  \
	{ 248, 0, P_TEXT0 }, { 353, 0, P_TEXT0 }, { 200, 21, P_ETA21 }, { 200, 22, P_RTA22 }, { 200, 55, P_IN55 }, { 235, 10, P_UK10 },               \
	{ 250, 10, P_UK10 }, { 366, 10, P_UK10 }, { 235, 20, P_UK20 }, { 316, 1, X_SLS1 }, { 366, 1, X_SLS1 }, { 316, 2, P_SLSID },   \
	{ 366, 2, P_SLSID }, { 316, 32, P_SLSID }, { 366, 32, P_SLSID }
#define ASM8                                                                                                                        \
	{ 1, 0, P_TEXT0 }, { 1, 16, X_VTS16 }, { 1, 20, P_IMO20 }, { 1, 22, P_IMO23 }, { 1, 23, P_IMO23 }, { 1, 24, P_EXT24 }, { 1, 25, P_IMO25 },    \
	{ 210, 0, P_TEXT0 }, { 248, 0, P_TEXT0 }, { 353, 0, P_TEXT0 }, { 200, 10, P_ERI10 }, { 200, 23, X_EMMA23 }, { 200, 24, X_WATER24 }, { 200, 40, P_SIG40 },  \
	{ 200, 55, P_IN55 }, { 1, 31, P_MET31 }, { 200, 25, P_BRIDGE25 }, { 1, 21, X_WX21 }, { 1, 29, P_TEXT29 }, { 1, 27, X_ROUTE27 }, { 1, 19, P_TS19 }, { 1, 17, X_VTS17 },     \
	{ 1, 26, X_ENV26 }, { 1, 11, P_MET11 }, { 235, 10, P_UK10 }, { 250, 10, P_UK10 }, { 366, 10, P_UK10 }, { 316, 1, X_SLS1 }, { 366, 1, X_SLS1 }, \
	{ 316, 2, P_SLSID }, { 366, 2, P_SLSID }, { 316, 32, P_SLSID }, { 366, 32, P_SLSID }, { 367, 33, X_ENV33 }, { 265, 1, X_SWE1 }
constexpr Asm kAsm6[] = { ASM6 }, kAsm8[] = { ASM8 };
constexpr int kNAsm6 = (int)(sizeof(kAsm6) / sizeof(Asm)), kNAsm8 = (int)(sizeof(kAsm8) / sizeof(Asm));
AJ_TABLE(Asm, asm6, kNAsm6, { ASM6 })
AJ_TABLE(Asm, asm8, kNAsm8, { ASM8 })

const int kMaxBits = 1064;  // MAX_AIS_LENGTH
const int kMaxBytes = 133;  // the bytes of a message; the rest reads as 0
const int kBufBytes = 144;

// ---- output ----
struct Out {
	char *p, *end;
	bool full;
	__host__ __device__ Out(char *b, int cap) : p(b), end(b + cap), full(false) {}
	__host__ __device__ void ch(char c) {
		if (p < end) *p++ = c;
		else full = true;
	}
	__host__ __device__ void raw(const char *s, int n) {
		for (int i = 0; i < n; i++) ch(s[i]);
	}
	__host__ __device__ void cstr(const char *s) {
		while (*s) ch(*s++);
	}
	__host__ __device__ void u64(unsigned long long v) {
		char t[20];
		int n = 0;
		do {
			t[n++] = (char)('0' + (int)(v % 10));
			v /= 10;
		} while (v);
		while (n) ch(t[--n]);
	}
	__host__ __device__ void i64(long long v) {
		if (v < 0) {
			ch('-');
			u64(0ULL - (unsigned long long)v);
		}
		else u64((unsigned long long)v);
	}
	// JSON::Writer's float: six decimals rounded half to even, trailing zeros trimmed, "null" outside (-1e18, 1e18)
	__host__ __device__ void f64(double v) {
		if (!(v > -1e18 && v < 1e18)) {
			raw("null", 4);
			return;
		}
		if (v < 0) {
			ch('-');
			v = -v;
		}
		long long whole = (long long)v;
		const double fd = (v - (double)whole) * 1000000.0;
		int frac = (int)(fd + 0.5);
		if ((double)frac - fd == 0.5 && (frac & 1)) frac--;
		if (frac >= 1000000) {
			whole++;
			frac -= 1000000;
		}
		u64((unsigned long long)whole);
		if (frac == 0) return;
		char d[6];
		for (int i = 5; i >= 0; i--) {
			d[i] = (char)('0' + frac % 10);
			frac /= 10;
		}
		int n = 6;
		while (d[n - 1] == '0') n--;
		ch('.');
		raw(d, n);
	}
	// a JSON string body: ", \ and control characters escaped as the Writer escapes them
	__host__ __device__ void esc(const char *s, int n) {
		for (int i = 0; i < n; i++) {
			const unsigned char c = (unsigned char)s[i];
			if (c == '"') raw("\\\"", 2);
			else if (c == '\\') raw("\\\\", 2);
			else if (c >= 0x20) ch((char)c);
			else if (c == '\b') raw("\\b", 2);
			else if (c == '\f') raw("\\f", 2);
			else if (c == '\n') raw("\\n", 2);
			else if (c == '\r') raw("\\r", 2);
			else if (c == '\t') raw("\\t", 2);
			else {
				const char *hex = "0123456789abcdef";
				raw("\\u00", 4);
				ch(hex[c >> 4]);
				ch(hex[c & 15]);
			}
		}
	}
	__host__ __device__ void qstr(const char *s) {
		ch('"');
		int n = 0;
		while (s[n]) n++;
		esc(s, n);
		ch('"');
	}
	__host__ __device__ void key(int k) {
		const char *s = AJ_TAB(key_blob)[0].s + AJ_TAB(key_off)[0].o[k];
		raw(",\"", 2);
		cstr(s);
		raw("\":", 2);
	}
	__host__ __device__ void kbool(int k, bool b) {
		key(k);
		if (b) raw("true", 4);
		else raw("false", 5);
	}
};

// ---- the message ----
struct Msg {
	uint8_t d[kBufBytes];
	int nbits;
	__host__ __device__ unsigned u(int start, int len) const {
		if (start < 0 || start + len > kMaxBits) return 0;
		const int x = start >> 3, y = start & 7;
		const unsigned long long w = ((unsigned long long)d[x] << 32) | ((unsigned long long)d[x + 1] << 24) |
									 ((unsigned long long)d[x + 2] << 16) | ((unsigned long long)d[x + 3] << 8) | d[x + 4];
		const unsigned mask = len >= 32 ? 0xFFFFFFFFu : ((1u << len) - 1u);
		return (unsigned)(w >> (40 - y - len)) & mask;
	}
	__host__ __device__ int s(int start, int len) const {
		unsigned v = u(start, len);
		if (v & (1u << (len - 1))) v |= ~0u << len;
		return (int)v;
	}
	__host__ __device__ unsigned c6(int bit) const { return ((((unsigned)d[bit >> 3] << 8) | d[(bit >> 3) + 1]) >> (10 - (bit & 7))) & 0x3F; }
	__host__ __device__ unsigned mmsi() const { return ((unsigned)d[1] << 22) | ((unsigned)d[2] << 14) | ((unsigned)d[3] << 6) | (d[4] >> 2); }
};

__host__ __device__ void put_text(Out &o, const Msg &m, int k, int start, int len) {
	o.key(k);
	o.ch('"');
	if (!(start < 0 || len <= 0 || start + len > kMaxBits)) {
		const int nch = (len + 5) / 6;
		int n = 0, last = 0;
		for (; n < nch; n++) {
			unsigned c = m.c6(start + 6 * n);
			if (!c) break;
			if (c != 32 && c != 0) last = n + 1; // ' ' is 6-bit 32
		}
		for (int i = 0; i < last; i++) {
			unsigned c = m.c6(start + 6 * i);
			if (!(c & 32)) c |= 64;
			if (c == '"' || c == '\\') o.ch('\\');
			o.ch((char)c);
		}
	}
	o.ch('"');
}

__host__ __device__ void put_tab_text(Out &o, int k, int tab, unsigned v) {
	const uint16_t *t = nullptr;
	unsigned n = 0;
	switch (tab) {
	case TT_NAV: t = AJ_TAB(t_nav), n = AJ_NAV_STATUS_N; break;
	case TT_EPFD: t = AJ_TAB(t_epfd), n = AJ_EPFD_N; break;
	case TT_SHIP: t = AJ_TAB(t_ship), n = AJ_SHIPTYPE_N; break;
	default: t = AJ_TAB(t_aid), n = AJ_AID_TYPE_N; break;
	}
	o.key(k);
	o.qstr(v < n ? AJ_TAB(text_blob)[0].s + t[v] : "Undefined");
}

// ProcessRadio: the 19-bit SOTDMA / ITDMA communication state
__host__ __device__ void put_radio(Out &o, const Msg &m, int start, int len) {
	const unsigned r = m.u(start, len);
	o.key(K_radio);
	if (r == 0 || len != 19) {
		o.ch('0');
		return;
	}
	o.u64(r);
	const unsigned sync = (r >> 17) & 3, to = (r >> 14) & 7, sub = r & 0x3FFF;
	o.key(K_sync_state);
	o.u64(sync);
	o.key(K_slot_timeout);
	o.u64(to);
	if (to == 0) {
		o.key(K_slot_offset);
		o.u64(sub);
	}
	else if (to == 1) {
		const unsigned hh = (sub >> 9) & 0x1F, mm = (sub >> 2) & 0x7F;
		if (hh < 24 && mm < 60) {
			o.key(K_utc_hour);
			o.u64(hh);
			o.key(K_utc_minute);
			o.u64(mm);
		}
	}
	else if (to == 2 || to == 4 || to == 6) {
		o.key(K_slot_number);
		o.u64(sub);
	}
	else {
		o.key(K_received_stations);
		o.u64(sub);
	}
}

__host__ __device__ void put2(Out &o, unsigned v) {
	o.ch((char)('0' + v / 10));
	o.ch((char)('0' + v % 10));
}

// runs program p with bit positions offset by base
__host__ __device__ void run(Out &o, const Msg &m, int p, int base) {
	const Op *ops = AJ_TAB(ops);
	for (int i = AJ_TAB(prog_idx)[0].at[p];; i++) {
		const Op f = ops[i];
		const int st = f.start + base;
		switch (f.op) {
		case OP_END: return;
		case OP_U: {
			const unsigned v = m.u(st, f.len);
			if (v != f.undef) {
				o.key(f.key);
				o.i64((int)v);
			}
			break;
		}
		case OP_UL: {
			const unsigned v = m.u(st, f.len);
			if (v != f.undef) {
				o.key(f.key);
				o.f64((double)(v * f.a + f.b));
			}
			break;
		}
		case OP_ULLT: {
			const unsigned v = m.u(st, f.len);
			if (v < f.undef) {
				o.key(f.key);
				o.f64((double)(v * f.a));
			}
			break;
		}
		case OP_US: {
			const unsigned v = m.u(st, f.len);
			if (v != f.undef) {
				o.key(f.key);
				o.i64((int)(v + (int)f.a));
			}
			break;
		}
		case OP_S: {
			const int v = m.s(st, f.len);
			if (v != (int)f.undef) {
				o.key(f.key);
				o.i64(v);
			}
			break;
		}
		case OP_SL: {
			const int v = m.s(st, f.len);
			if (v != (int)f.undef) {
				o.key(f.key);
				o.f64((double)(v * f.a + f.b));
			}
			break;
		}
		case OP_E: {
			const unsigned v = m.u(st, f.len);
			o.key(f.key);
			o.i64((int)v);
			if (f.tab != TT_NONE) put_tab_text(o, f.key2, f.tab, v);
			break;
		}
		case OP_TURN: {
			const int v = m.s(st, 8);
			o.key(K_turn_unscaled);
			o.i64(v);
			if (v > -127 && v < 127) {
				double r = v / 4.733;
				r = v < 0 ? -r * r : r * r;
				o.key(f.key);
				o.i64((int)(r + 0.5));
			}
			else if (v != -128) {
				o.key(f.key);
				o.i64(v);
			}
			break;
		}
		case OP_B: o.kbool(f.key, m.u(st, 1) != 0); break;
		case OP_BEQ: o.kbool(f.key, m.u(st, f.len) == f.undef); break;
		case OP_T: put_text(o, m, f.key, st, f.len); break;
		case OP_TMIN: {
			const int rest = m.nbits - st;
			put_text(o, m, f.key, st, rest < f.len ? rest : f.len);
			break;
		}
		case OP_TCLAMP: {
			int n = m.nbits - st;
			if (n < 6) n = 0;
			if (n > f.len) n = f.len;
			n -= n % 6;
			if (n > 0) put_text(o, m, f.key, st, n);
			break;
		}
		case OP_TS: {
			o.key(f.key);
			o.ch('"');
			const unsigned y = m.u(st, 14);
			o.ch((char)('0' + y / 1000));
			o.ch((char)('0' + (y / 100) % 10));
			put2(o, y % 100);
			o.ch('-');
			put2(o, m.u(st + 14, 4));
			o.ch('-');
			put2(o, m.u(st + 18, 5));
			o.ch('T');
			put2(o, m.u(st + 23, 5));
			o.ch(':');
			put2(o, m.u(st + 28, 6));
			o.ch(':');
			put2(o, m.u(st + 34, 6));
			o.cstr("Z\"");
			break;
		}
		case OP_ETA: {
			o.key(f.key);
			o.ch('"');
			put2(o, m.u(st, 4));
			o.ch('-');
			put2(o, m.u(st + 4, 5));
			o.ch('T');
			put2(o, m.u(st + 9, 5));
			o.ch(':');
			put2(o, m.u(st + 14, 6));
			o.cstr("Z\"");
			break;
		}
		case OP_DMIN: {
			const int rest = m.nbits - st, n = rest < f.len ? rest : f.len;
			o.key(f.key);
			o.ch('"');
			o.i64(n);
			o.ch(':');
			for (int b = st; b < st + n; b += 4) {
				const unsigned c = m.u(b, 4);
				o.ch((char)(c < 10 ? c + '0' : c + 'a' - 10));
			}
			o.ch('"');
			break;
		}
		case OP_RADIO: {
			int n = m.nbits - st;
			n = n < 19 ? n : 19;
			put_radio(o, m, st, n > 0 ? n : 0);
			break;
		}
		case OP_BRK_LE: if (m.nbits <= f.start) return; break;
		case OP_BRK_EQ: if (m.nbits == f.start) return; break;
		case OP_BITS: {
			const int rest = m.nbits - st, n = rest < 128 ? rest : 128;
			o.key(f.key);
			o.ch('"');
			for (int b = 0; b < n; b++) o.ch(m.u(st + b, 1) ? '1' : '0');
			o.ch('"');
			break;
		}
		}
	}
}

// printf("%.<prec>f", v): the exact binary value of v rounded to prec decimals, ties to even, "-" for any negative v
__host__ __device__ void put_fixed(Out &o, double v, int prec) {
	if (signbit(v)) {
		o.ch('-');
		v = -v;
	}
	int e;
	const double fr = frexp(v, &e); // v = fr * 2^e, fr in [0.5, 1)
	const unsigned long long mant = (unsigned long long)ldexp(fr, 53);
	e -= 53; // v = mant * 2^e exactly
	unsigned long long p10 = 1;
	for (int i = 0; i < prec; i++) p10 *= 10;
	unsigned __int128 q;
	if (v == 0.0) q = 0;
	else if (e >= 0) q = ((unsigned __int128)mant << e) * p10; // not reached for the values printed here (|v| < 2^11)
	else if (-e >= 100) q = 0;
	else {
		const unsigned __int128 P = (unsigned __int128)mant * p10;
		const int sh = -e;
		q = P >> sh;
		const unsigned __int128 r = P - (q << sh), half = (unsigned __int128)1 << (sh - 1);
		if (r > half || (r == half && (q & 1))) q++;
	}
	o.u64((unsigned long long)(q / p10));
	if (prec > 0) {
		o.ch('.');
		char d[20];
		unsigned long long f = (unsigned long long)(q % p10);
		for (int i = prec - 1; i >= 0; i--) {
			d[i] = (char)('0' + f % 10);
			f /= 10;
		}
		o.raw(d, prec);
	}
}

// the layouts of application messages with control flow
__host__ __device__ void app_special(Out &o, const Msg &m, int x, int start) {
	switch (x) {
	case X_VTS16: { // VTS targets: an id of 2 x 6-bit text or a number, then the target's position and motion
		if (m.nbits < start + 120) return;
		const unsigned id_type = m.u(start, 2);
		o.key(K_vts_target_id_type);
		o.u64(id_type);
		if (id_type == 2) put_text(o, m, K_vts_target_id, start + 2, 42);
		else {
			const unsigned long long id = ((unsigned long long)m.u(start + 2, 10) << 32) | m.u(start + 12, 32);
			if (id <= 0x7FFFFFFFull) {
				o.key(K_vts_target_id);
				o.u64(id);
			}
		}
		run(o, m, P_VTS16B, start);
		return;
	}
	case X_WX21: { // weather observation from a ship: only the non-WMO variant has fields
		const unsigned variant = m.u(start, 1);
		o.key(K_weather_report_type);
		o.u64(variant);
		if (variant == 0) run(o, m, P_WX21, start);
		return;
	}
	case X_ROUTE27: { // route information: up to 16 waypoints of 55 bits as "lat,lon;..."
		run(o, m, P_ROUTE27H, start);
		int n = (int)m.u(start + 56, 5);
		if (n > 16) n = 16;
		const int avail = m.nbits - (start + 61);
		if (n * 55 > avail) n = avail > 0 ? avail / 55 : 0;
		if (n <= 0) return;
		o.key(K_waypoints);
		o.ch('"');
		for (int i = 0; i < n; i++) {
			const int base = start + 61 + i * 55;
			if (i) o.ch(';');
			put_fixed(o, (double)m.s(base + 28, 27) / 600000.0, 6);
			o.ch(',');
			put_fixed(o, (double)m.s(base, 28) / 600000.0, 6);
		}
		o.ch('"');
		return;
	}
	case X_ENV26: // environmental: the first report's header, when it is all there
		if (m.nbits >= start + 27) run(o, m, P_ENV26, start);
		return;
	case X_ENV33: { // environmental sensor report: header, then the body of report types 0-3
		if (m.nbits < start + 27) return;
		const unsigned rt = m.u(start, 4);
		run(o, m, P_ENV33H, start);
		if (m.nbits < start + 112 || rt > 3) return;
		run(o, m, P_ENV33_0 + (int)rt, start + 27);
		return;
	}
	case X_EMMA23: { // EMMA warning: dates YYYYMMDD and times HHMM when valid, the area, signed magnitudes
		for (int k = 0; k < 2; k++) {
			const int b = start + 17 * k;
			const unsigned y = m.u(b, 8), mo = m.u(b + 8, 4), d = m.u(b + 12, 5);
			if (y > 0 && mo > 0 && d > 0) {
				o.key(k ? K_end_date : K_start_date);
				o.ch('"');
				o.u64(2000 + y);
				put2(o, mo);
				put2(o, d);
				o.ch('"');
			}
		}
		for (int k = 0; k < 2; k++) {
			const unsigned hh = m.u(start + 34 + 11 * k, 5), mm = m.u(start + 39 + 11 * k, 6);
			if (hh < 24 && mm < 60) {
				o.key(k ? K_end_time : K_start_time);
				o.ch('"');
				put2(o, hh);
				put2(o, mm);
				o.ch('"');
			}
		}
		run(o, m, P_EMMA_POS, start);
		for (int k = 0; k < 2; k++) {
			const unsigned mag = m.u(start + 171 + 9 * k, 8);
			if (mag != 255) {
				o.key(k ? K_max_value : K_min_value);
				o.i64(m.u(start + 170 + 9 * k, 1) ? -(int)mag : (int)mag);
			}
		}
		run(o, m, P_EMMA_T, start);
		return;
	}
	case X_WATER24: { // water levels of up to four gauges; a gauge id of 0 is no gauge
		put_text(o, m, K_un_country, start, 12);
		for (int i = 0; i < 4; i++) {
			const int b = start + 12 + 25 * i;
			const unsigned id = m.u(b, 11);
			if (!id) continue;
			o.key(K_gauge1_id + 2 * i);
			o.u64(id);
			o.key(K_gauge1_level + 2 * i);
			o.i64((m.u(b + 11, 1) ? 1 : -1) * (int)m.u(b + 12, 13));
		}
		return;
	}
	case X_SWE1: { // route: first waypoint, up to 6 delta-coded legs, an absolute last leg with planned speed and steering mode
		const int len = m.nbits;
		if (len - start < 56) return;
		int p = start + 56, nlegs = (len - p - 72) / 64;
		if (nlegs < 0) nlegs = 0;
		if (nlegs > 6) nlegs = 6;
		const int pl = p + 64 * nlegs;
		const bool last = len - pl >= 72;
		if (last) {
			const unsigned sp = m.u(pl + 1, 10);
			if (sp != 0) {
				o.key(K_planned_speed);
				o.f64((double)(sp * 0.1f + 0.0f));
			}
			o.key(K_steering_mode);
			o.u64(m.u(pl + 66, 2));
		}
		double lon = m.s(start + 1, 28) / 600000.0, lat = m.s(start + 29, 27) / 600000.0;
		o.key(K_waypoints);
		o.ch('"');
		put_fixed(o, lat, 6);
		o.ch(',');
		put_fixed(o, lon, 6);
		for (int i = 0; i < nlegs; i++, p += 64) {
			lon += m.s(p + 20, 22) / 600000.0;
			lat += m.s(p + 42, 22) / 600000.0;
			o.ch(';');
			put_fixed(o, lat, 6);
			o.ch(',');
			put_fixed(o, lon, 6);
		}
		if (last) {
			o.ch(';');
			put_fixed(o, m.s(p + 39, 27) / 600000.0, 6);
			o.ch(',');
			put_fixed(o, m.s(p + 11, 28) / 600000.0, 6);
		}
		o.ch('"');
		return;
	}
	case X_TIDAL32: { // tidal window: three prediction points "lat,lon,dir,speed"; points off the globe are left out
		run(o, m, P_TIDAL32H, start);
		const int lon_b[3] = { 9, 97, 174 }, lat_b[3] = { 34, 122, 199 }, dir_b[3] = { 80, 157, 245 }, spd_b[3] = { 89, 166, 254 };
		bool any = false;
		for (int i = 0; i < 3; i++) {
			const int lo = m.s(start + lon_b[i], 25), la = m.s(start + lat_b[i], 24);
			if (lo > 10800000 || lo < -10800000 || la > 5400000 || la < -5400000) continue;
			if (!any) {
				o.key(K_tidal);
				o.ch('"');
			}
			else o.ch(';');
			any = true;
			const unsigned dir = m.u(start + dir_b[i], 9), spd = m.u(start + spd_b[i], 8);
			put_fixed(o, la / 60000.0, 5);
			o.ch(',');
			put_fixed(o, lo / 60000.0, 5);
			o.ch(',');
			o.i64(dir == 360 ? -1 : (int)dir);
			o.ch(',');
			put_fixed(o, spd == 255 ? -1.0 : spd * 0.1, 1);
		}
		if (any) o.ch('"');
		return;
	}
	case X_VTS17: { // VTS-generated targets: up to four of 120 bits as "id,lat,lon,cog,sog;..."
		int n = (m.nbits - start) / 120;
		if (n > 4) n = 4;
		if (n <= 0) return;
		o.key(K_targets);
		o.ch('"');
		for (int i = 0; i < n; i++) {
			const int b = start + 120 * i;
			char id[7];
			int e = 7;
			for (int k = 0; k < 7; k++) {
				const unsigned c = m.u(b + 2 + 6 * k, 6);
				id[k] = (char)(c < 32 ? c + 64 : c);
			}
			while (e > 0 && (id[e - 1] == '@' || id[e - 1] == ' ')) e--;
			if (i) o.ch(';');
			o.esc(id, e);
			o.ch(',');
			put_fixed(o, m.s(b + 48, 24) / 60000.0, 5);
			o.ch(',');
			put_fixed(o, m.s(b + 72, 25) / 60000.0, 5);
			o.ch(',');
			o.u64(m.u(b + 97, 9));
			o.ch(',');
			o.u64(m.u(b + 112, 8));
		}
		o.ch('"');
		return;
	}
	case X_SLS1: { // SLS meteorological / hydrological: message id, then one report when the frame holds all of it
		run(o, m, P_SLSID, start);
		const unsigned id = m.u(start + 2, 6);
		const int rpt = start + 8;
		int body = -1;
		if (id == 1 && m.nbits >= rpt + 192) body = P_SLS1;
		else if (id == 3 && m.nbits >= rpt + 144) body = P_SLS3;
		else if (id == 2 && m.nbits >= rpt + 144) body = P_SLS2;
		else if (id == 6 && m.nbits >= rpt + 144) body = P_SLS6;
		if (body < 0) return;
		run(o, m, P_SLSHDR, rpt);
		run(o, m, body, rpt);
		return;
	}
	}
}

// the application message of a type 6 (addressed) / 8 (broadcast) layout
__host__ __device__ void app(Out &o, const Msg &m, bool addressed) {
	const int start = addressed ? 88 : 56;
	const unsigned dac = m.u(addressed ? 72 : 40, 10), fid = m.u(addressed ? 82 : 50, 6);
	const Asm *t = addressed ? AJ_TAB(asm6) : AJ_TAB(asm8);
	const int n = addressed ? kNAsm6 : kNAsm8;
	for (int i = 0; i < n; i++)
		if ((unsigned)t[i].dac == dac && (unsigned)t[i].fid == fid) {
			if (t[i].prog < P_COUNT) run(o, m, t[i].prog, start);
			else app_special(o, m, t[i].prog, start);
			return;
		}
	const int rest = m.nbits - start, lim = addressed ? 920 : 952, len = rest < lim ? rest : lim;
	o.key(K_data);
	o.ch('"');
	o.i64(len);
	o.ch(':');
	for (int b = start; b < start + len; b += 4) {
		const unsigned c = m.u(b, 4);
		o.ch((char)(c < 10 ? c + '0' : c + 'a' - 10));
	}
	o.ch('"');
}

__host__ __device__ void country(Out &o, const Msg &m) {
	const unsigned mmsi = m.mmsi();
	unsigned mid = mmsi;
	while (mid > 1000) mid /= 10;
	if (mid == 111) {
		mid = mmsi;
		while (mid > 1000000) mid /= 10;
		mid %= 1000;
	}
	else if (mid / 10 == 99 || mid / 10 == 98) {
		mid = mmsi;
		while (mid > 100000) mid /= 10;
		mid %= 1000;
	}
	if (mid > 100 && mid < 1000 && AJ_TAB(t_cname)[mid] != 0xFFFF) {
		o.key(K_country);
		o.qstr(AJ_TAB(text_blob)[0].s + AJ_TAB(t_cname)[mid]);
		o.key(K_country_code);
		o.qstr(AJ_TAB(text_blob)[0].s + AJ_TAB(t_ccode)[mid]);
	}
}

// everything after the engine prefix
__host__ __device__ void body(Out &o, const Msg &m, const aisgpu_msg *src, int mode, int station) {
	o.cstr(",\"channel\":\"");
	o.esc(&src->channel, 1);
	o.cstr("\",\"nmea\":[");
	const int ns = src->n_sentences < 0 ? 0 : (src->n_sentences > 4 ? 4 : src->n_sentences);
	for (int i = 0; i < ns; i++) {
		if (i) o.ch(',');
		o.ch('"');
		int len = src->nmea_len[i];
		len = len < 0 ? 0 : (len > 100 ? 100 : len);
		o.esc(src->nmea[i], len);
		o.ch('"');
	}
	o.ch(']');
	if (mode & 1) {
		if (src->level != 1024.0f) {
			o.cstr(",\"signalpower\":");
			o.f64((double)src->level);
		}
		if (src->ppm != 1024.0f) {
			o.cstr(",\"ppm\":");
			o.f64((double)src->ppm);
		}
	}
	if (station) {
		o.cstr(",\"station_id\":");
		o.i64(station);
	}
	if (m.nbits > 0) {
		o.key(K_type);
		o.i64((int)m.u(0, 6));
		o.key(K_repeat);
		o.i64((int)m.u(6, 2));
		o.key(K_mmsi);
		o.i64((int)m.u(8, 30));
		if (mode & 4) country(o, m);
	}
	const unsigned type = m.d[0] >> 2;
	switch (type) {
	case 1: case 2: case 3: run(o, m, P_123, 0); break;
	case 4: case 11: run(o, m, P_4, 0); break;
	case 5: run(o, m, P_5, 0); break;
	case 6:
		run(o, m, P_6, 0);
		app(o, m, true);
		break;
	case 7: case 13: run(o, m, P_7, 0); break;
	case 8:
		run(o, m, P_8, 0);
		app(o, m, false);
		break;
	case 9: run(o, m, P_9, 0); break;
	case 10: run(o, m, P_10, 0); break;
	case 12: run(o, m, P_12, 0); break;
	case 14: run(o, m, P_14, 0); break;
	case 15: run(o, m, P_15, 0); break;
	case 16: run(o, m, P_16, 0); break;
	case 17: run(o, m, P_17, 0); break;
	case 18: run(o, m, P_18, 0); break;
	case 19: run(o, m, P_19, 0); break;
	case 20: run(o, m, P_20, 0); break;
	case 21: run(o, m, P_21, 0); break;
	case 22:
		run(o, m, P_22H, 0);
		run(o, m, m.u(139, 1) ? P_22A : P_22B, 0);
		run(o, m, P_22T, 0);
		break;
	case 23: run(o, m, P_23, 0); break;
	case 24:
		o.key(K_partno);
		o.i64((int)m.u(38, 2));
		if (m.u(38, 2) == 0) run(o, m, P_24A, 0);
		else {
			run(o, m, P_24B, 0);
			run(o, m, m.mmsi() / 10000000 == 98 ? P_24MS : P_24DIM, 0);
			if (m.nbits >= 168) run(o, m, P_24X, 0);
		}
		break;
	case 25: case 26: {
		run(o, m, P_25H, 0);
		const bool addressed = m.u(38, 1), structured = m.u(39, 1);
		if (addressed) run(o, m, P_25A, 0);
		if (structured) {
			o.key(K_dac);
			o.i64((int)m.u(addressed ? 72 : 40, 10));
			o.key(K_fid);
			o.i64((int)m.u(addressed ? 82 : 50, 6));
			app(o, m, addressed);
		}
		if (type == 26 && m.nbits - 20 >= 40) put_radio(o, m, m.nbits - 20 + 1, 19);
		break;
	}
	case 27: run(o, m, P_27, 0); break;
	case 28: run(o, m, P_28, 0); break;
	default: break;
	}
}

// Message::getRxTime / Convert::toTimeStr: YYYYMMDDHHMMSS (UTC) of the whole seconds, times before the epoch as the epoch
__host__ __device__ void put_rxtime(Out &o, long long us) {
	long long t = us / 1000000;
	if (t < 0) t = 0;
	const int sec = (int)(t % 60), mn = (int)(t / 60 % 60), hr = (int)(t / 3600 % 24);
	const int z = (int)(t / 86400) + 719468, era = (z >= 0 ? z : z - 146096) / 146097;
	const unsigned doe = (unsigned)(z - era * 146097), yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
	const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100), mp = (5 * doy + 2) / 153;
	const int day = (int)(doy - (153 * mp + 2) / 5 + 1), mon = (int)(mp + (mp < 10 ? 3 : -9));
	const int year = (int)yoe + era * 400 + (mon <= 2);
	const int parts[7] = { year / 100, year % 100, mon, day, hr, mn, sec };
	for (int v : parts) put2(o, (unsigned)v);
}

// printf("%g", (double)f) as glibc prints it: the exact binary value rounded to six significant digits, ties to even; exponent
// form when the decimal exponent after that rounding is below -4 or at least 6; trailing zeros trimmed.  The value is m * 2^e
// with a 24-bit m; it is written as the integer M = m * 2^e (e >= 0) or m * 5^-e (e < 0, the decimal point -e digits from the
// right), at most 371 bits, whose decimal digits give the rounding exactly.
__host__ __device__ void put_g(Out &o, float f) {
	uint32_t b;
	memcpy(&b, &f, 4);
	const int bexp = (int)((b >> 23) & 0xFF);
	uint32_t man = b & 0x7FFFFF;
	if (b >> 31) o.ch('-');
	if (bexp == 0xFF) {
		o.cstr(man ? "nan" : "inf");
		return;
	}
	if (bexp == 0 && man == 0) {
		o.ch('0');
		return;
	}
	int e2 = -149;
	if (bexp) {
		man |= 0x800000;
		e2 = bexp - 150;
	}
	uint32_t L[12];
	int nl = 1;
	L[0] = man;
	auto mul = [&](uint32_t k) {
		unsigned long long c = 0;
		for (int i = 0; i < nl; i++) {
			c += (unsigned long long)L[i] * k;
			L[i] = (uint32_t)c;
			c >>= 32;
		}
		if (c) L[nl++] = (uint32_t)c;
	};
	int q = 0; // the value is M * 10^q
	if (e2 >= 0)
		for (int k = e2; k > 0; k -= 31) mul(1u << (k < 31 ? k : 31));
	else {
		for (int k = -e2; k > 0; k -= 13) {
			uint32_t p5 = 1;
			for (int j = 0; j < (k < 13 ? k : 13); j++) p5 *= 5;
			mul(p5);
		}
		q = e2;
	}
	char dg[120]; // M's decimal digits, least significant first
	int nd = 0;
	while (nl > 0) {
		unsigned long long r = 0;
		for (int i = nl - 1; i >= 0; i--) {
			const unsigned long long cur = (r << 32) | L[i];
			L[i] = (uint32_t)(cur / 1000000000u);
			r = cur % 1000000000u;
		}
		while (nl > 0 && L[nl - 1] == 0) nl--;
		for (int j = 0; j < 9 && (nl > 0 || r > 0); j++) {
			dg[nd++] = (char)(r % 10);
			r /= 10;
		}
	}
	int E = nd - 1 + q; // decimal exponent of the leading digit
	long K = 0;          // the six significant digits
	for (int j = 0; j < 6; j++) K = K * 10 + (j < nd ? dg[nd - 1 - j] : 0);
	if (nd > 6) {
		const int d6 = dg[nd - 7];
		bool rest = false;
		for (int j = 0; j < nd - 7; j++) rest |= dg[j] != 0;
		if (d6 > 5 || (d6 == 5 && (rest || (K & 1)))) K++;
		if (K == 1000000) {
			K = 100000;
			E++;
		}
	}
	char k6[6];
	for (int j = 5; j >= 0; j--) {
		k6[j] = (char)('0' + K % 10);
		K /= 10;
	}
	int last = 5;
	while (last > 0 && k6[last] == '0') last--;
	if (E < -4 || E >= 6) {
		o.ch(k6[0]);
		if (last > 0) {
			o.ch('.');
			o.raw(k6 + 1, last);
		}
		o.ch('e');
		o.ch(E < 0 ? '-' : '+');
		const int a = E < 0 ? -E : E;
		if (a >= 100) o.ch((char)('0' + a / 100));
		put2(o, (unsigned)(a % 100));
	}
	else if (E >= 0) {
		o.raw(k6, E + 1);
		if (last > E) {
			o.ch('.');
			o.raw(k6 + E + 1, last - E);
		}
	}
	else {
		o.raw("0.", 2);
		for (int j = 0; j < -E - 1; j++) o.ch('0');
		o.raw(k6, last + 1);
	}
}

__host__ __device__ int n_sent(const aisgpu_msg *src) { return src->n_sentences < 0 ? 0 : (src->n_sentences > 4 ? 4 : src->n_sentences); }
__host__ __device__ int sent_len(const aisgpu_msg *src, int i) {
	const int l = src->nmea_len[i];
	return l < 0 ? 0 : (l > 100 ? 100 : l);
}

// ---- the sparse and the annotated JSON: the full line rewritten member by member ----
// Every member of the full line is a key of AJ_KEYS; a key is found by its name through an open-addressing hash table built at
// compile time from the same list.
enum Dict : uint8_t { D_SPARSE, D_ANNOTATED };
constexpr int kHashN = 1024;
__host__ __device__ constexpr unsigned key_hash(const char *s, int n) {
	unsigned h = 2166136261u; // FNV-1a
	for (int i = 0; i < n; i++) h = (h ^ (unsigned char)s[i]) * 16777619u;
	return h;
}
struct KeyHash {
	int16_t k[kHashN];
};
constexpr KeyHash make_key_hash() {
	KeyHash t{};
	const char s[] = {
#define X(n) #n "\0"
		AJ_KEYS(X)
#undef X
	};
	for (int i = 0; i < kHashN; i++) t.k[i] = -1;
	for (int k = 0; k < K_COUNT; k++) {
		const char *name = s + kKeyOff.o[k];
		int n = 0;
		while (name[n]) n++;
		unsigned h = key_hash(name, n) % kHashN;
		while (t.k[h] >= 0) h = (h + 1) % kHashN;
		t.k[h] = (int16_t)k;
	}
	return t;
}
AJ_TABLE(KeyHash, key_hash_tab, 1, { make_key_hash() })

// the key named s[0, n), or -1
__host__ __device__ int find_key(const char *s, int n) {
	const char *blob = AJ_TAB(key_blob)[0].s;
	for (unsigned h = key_hash(s, n) % kHashN;; h = (h + 1) % kHashN) {
		const int k = AJ_TAB(key_hash_tab)[0].k[h];
		if (k < 0) return -1;
		const char *name = blob + AJ_TAB(key_off)[0].o[k];
		int i = 0;
		while (i < n && name[i] == s[i]) i++;
		if (i == n && !name[n]) return k;
	}
}

// The full line in[0, n) (a flat object: numbers, strings, booleans, null and one array of strings) written in dictionary d, as
// JSON::Serializer writes the same members: sparse -- each key renamed, a key without a sparse name left out with its value;
// annotated -- each value as {"value":v[,"unit":..][,"description":..][,"text":..]}, "text" being the key's lookup entry for a
// number's integer part (a number's value: the lookup keys hold integers).
__host__ __device__ void rewrite(Out &o, const char *in, int n, int d) {
	const char *blob = AF_TAB(af_blob)[0].s;
	o.ch('{');
	bool first = true;
	int i = 1;
	while (i < n && in[i] != '}') {
		if (in[i] == ',') i++;
		const int ks = i + 1;
		int ke = ks;
		while (ke < n && in[ke] != '"') ke++;
		const int vs = ke + 2; // past '":'
		int ve = vs, depth = 0;
		bool str = false;
		for (; ve < n; ve++) {
			const char c = in[ve];
			if (str) {
				if (c == '\\') ve++;
				else if (c == '"') str = false;
			}
			else if (c == '"') str = true;
			else if (c == '[') depth++;
			else if (c == ']') depth--;
			else if ((c == ',' || c == '}') && depth == 0) break;
		}
		i = ve;
		const int k = find_key(in + ks, ke - ks);
		if (d == D_SPARSE) {
			const char *name = k >= 0 ? blob + AF_TAB(af_sparse)[k] : "";
			if (!*name) continue;
			if (!first) o.ch(',');
			o.ch('"');
			o.cstr(name);
			o.raw("\":", 2);
			o.raw(in + vs, ve - vs);
		}
		else {
			if (!first) o.ch(',');
			o.raw(in + ks - 1, ke - ks + 3); // "key":
			o.raw("{\"value\":", 9);
			o.raw(in + vs, ve - vs);
			if (k >= 0) {
				const uint32_t u = AF_TAB(af_unit)[k], ds = AF_TAB(af_desc)[k];
				if (u != 0xFFFFFFFFu) {
					o.raw(",\"unit\":\"", 9);
					o.cstr(blob + u);
					o.ch('"');
				}
				if (ds != 0xFFFFFFFFu) {
					o.raw(",\"description\":\"", 16);
					o.cstr(blob + ds);
					o.ch('"');
				}
				const int t = AF_TAB(af_lut)[k];
				const char c0 = in[vs];
				if (t >= 0 && ((c0 >= '0' && c0 <= '9') || c0 == '-')) {
					long long v = 0;
					for (int j = c0 == '-' ? vs + 1 : vs; j < ve && in[j] >= '0' && in[j] <= '9' && v < 1000000; j++) v = v * 10 + (in[j] - '0');
					if (c0 == '-') v = -v;
					if (v >= 0 && v < AF_TAB(af_lut_n)[t]) {
						o.raw(",\"text\":\"", 9);
						o.cstr(blob + AF_TAB(af_lut_text)[AF_TAB(af_lut_at)[t] + (int)v]);
						o.ch('"');
					}
				}
			}
			o.ch('}');
		}
		first = false;
	}
	o.ch('}');
}

// seconds from microseconds the way getNMEAJSON prints rxuxtime / toa: integer when whole (Message.cpp:121-137)
__host__ __device__ void usec(Out &o, long long t) {
	if (t % 1000000 != 0) o.f64((double)t / 1000000.0);
	else o.i64(t / 1000000);
}

// AIS::Message::getNMEAJSON (Message.cpp:93-191); rxtime_us: the frame's stamp
__host__ __device__ void nmea_json(Out &o, const aisgpu_msg *m, const FmtCtx &c, long long rxtime_us) {
	o.cstr("{\"class\":\"AIS\",\"device\":\"AIS-catcher\",\"version\":");
	o.i64(c.version);
	o.cstr(",\"driver\":");
	o.i64(c.driver);
	o.cstr(",\"hardware\":");
	o.qstr(c.hardware);
	o.cstr(",\"channel\":\"");
	o.ch(m->channel);
	o.cstr("\",\"repeat\":");
	o.i64(m->data[0] & 3); // Message::repeat(), Message.h:186-189
	if (c.include_ssl) {
		o.cstr(",\"ssc\":");
		o.i64(m->start_idx);
		o.cstr(",\"sl\":");
		o.i64(m->end_idx - m->start_idx);
	}
	if (c.status) {
		o.cstr(",\"msg_status\":");
		o.i64(c.status);
	}
	if (c.mode & 2) {
		o.cstr(",\"rxuxtime\":");
		usec(o, rxtime_us);
	}
	if (c.toa_us != 0) {
		o.cstr(",\"toa\":");
		usec(o, c.toa_us);
	}
	if (c.uuid[0]) {
		o.cstr(",\"uuid\":\"");
		o.cstr(c.uuid); // copied verbatim, as the reference does
		o.ch('"');
	}
	if (c.ipv4) {
		o.cstr(",\"ipv4\":");
		o.i64((long long)c.ipv4);
	}
	if (c.mode & 1) {
		o.cstr(",\"signalpower\":");
		if (m->level == 1024.0f) o.cstr("null"); // LEVEL_UNDEFINED
		else o.f64((double)m->level);
		o.cstr(",\"ppm\":");
		if (m->ppm == 1024.0f) o.cstr("null"); // PPM_UNDEFINED
		else o.f64((double)m->ppm);
	}
	if (c.station) {
		o.cstr(",\"station_id\":");
		o.i64(c.station);
	}
	if (m->nbits > 0) {
		const unsigned mmsi = ((unsigned)m->data[1] << 22) | ((unsigned)m->data[2] << 14) | ((unsigned)m->data[3] << 6) | ((unsigned)m->data[4] >> 2);
		o.cstr(",\"mmsi\":");
		o.i64((long long)mmsi); // Message.h:191-194
		o.cstr(",\"type\":");
		o.i64(m->data[0] >> 2);
	}
	o.cstr(",\"nmea\":[");
	for (int i = 0; i < n_sent(m); i++) {
		if (i) o.ch(',');
		o.ch('"');
		o.raw(m->nmea[i], sent_len(m, i));
		o.ch('"');
	}
	o.cstr("]}");
	o.cstr(c.suffix);
}

// AIS::Message::getBinaryNMEA (Message.cpp:287-396): 0xAC 0x00 <flags> | the rest byte-stuffed: '\n' -> AD AE, '\r' -> AD AF,
// 0xAD -> AD AD | '\n'; nothing for a length outside [0, 1064].  start: where the record began (the CRC covers it).
__host__ __device__ void binary(Out &o, const char *start, const aisgpu_msg *m, long long rxtime_us, bool crc) {
	if (m->nbits < 0 || m->nbits > kMaxBits) return;
	const int nbytes = (m->nbits + 7) / 8;
	auto put = [&](unsigned b) {
		b &= 0xffu;
		if (b == '\n' || b == '\r' || b == 0xad) {
			o.ch((char)0xad);
			o.ch((char)(b == '\n' ? 0xae : b == '\r' ? 0xaf : 0xad));
		}
		else o.ch((char)b);
	};
	o.ch((char)0xac);
	o.ch((char)0x00);
	unsigned flags = 0;
	if (m->level != 1024.0f && m->ppm != 1024.0f) flags |= 1u;
	if (crc) flags |= 2u;
	o.ch((char)flags);
	for (int i = 0; i < 8; i++) put((unsigned)((unsigned long long)rxtime_us >> ((7 - i) * 8))); // big-endian time stamp
	if (flags & 1u) {
		const int level10 = (int)(m->level * 10.0f);
		put((unsigned)(level10 >> 8));
		put((unsigned)level10);
		const int ppm10 = (int)(m->ppm * 10.0f);
		put((unsigned)(int8_t)ppm10);
	}
	o.ch(m->channel); // these two are written unescaped by the reference (Message.cpp:376-377)
	o.ch((char)((m->nbits >> 8) & 0xff));
	put((unsigned)m->nbits);
	for (int i = 0; i < nbytes; i++) put(m->data[i]);
	if (crc && !o.full) { // CRC-16/ARC style (reflected 0xA001, init 0xFFFF) over everything written so far, escapes included
		unsigned cr = 0xffffu;
		for (const unsigned char *q = (const unsigned char *)start; q < (const unsigned char *)o.p; q++) {
			cr ^= *q;
			for (int j = 0; j < 8; j++) cr = (cr & 1u) ? (cr >> 1) ^ 0xa001u : cr >> 1;
		}
		put(cr >> 8);
		put(cr);
	}
	o.ch('\n');
}

// AIS::Message::getNMEATagBlock (Message.cpp:198-285) with the engine's group counter: groups = the multi-sentence frames before
// this one
__host__ __device__ void tag_block(Out &o, const aisgpu_msg *m, const FmtCtx &c, long long rxtime_us, long long groups) {
	const int total = n_sent(m);
	const int group = total > 1 ? (int)(groups % 9999) + 1 : 0;
	for (int seq = 1; seq <= total; seq++) {
		char tb[96];
		Out t(tb, (int)sizeof(tb));
		t.raw("s:s", 3);
		t.i64(c.station);
		t.raw(",c:", 3);
		t.f64((double)rxtime_us / 1000000.0);
		if (total > 1) {
			t.raw(",g:", 3);
			t.i64(seq);
			t.ch('-');
			t.i64(total);
			t.ch('-');
			t.i64(group);
		}
		const int n = (int)(t.p - tb);
		unsigned x = 0;
		for (int i = 0; i < n; i++) x ^= (unsigned char)tb[i];
		o.ch('\\');
		o.raw(tb, n);
		o.ch('*');
		o.ch("0123456789ABCDEF"[(x >> 4) & 15]);
		o.ch("0123456789ABCDEF"[x & 15]);
		o.ch('\\');
		o.raw(m->nmea[seq - 1], sent_len(m, seq - 1));
		o.raw("\r\n", 2);
	}
}

// the screen's annotated sentences (OutputMessage::formatInto, MsgOut.h:73-106)
__host__ __device__ void full_text(Out &o, const aisgpu_msg *m, const FmtCtx &c, long long rxtime_us) {
	for (int i = 0; i < n_sent(m); i++) {
		o.raw(m->nmea[i], sent_len(m, i));
		o.raw(" ( ", 3);
		if (m->nbits > 0) {
			o.cstr("MSG: ");
			o.u64(m->data[0] >> 2);
			o.cstr(", REPEAT: ");
			o.u64(m->data[0] & 3);
			o.cstr(", MMSI: ");
			o.u64(((unsigned)m->data[1] << 22) | ((unsigned)m->data[2] << 14) | ((unsigned)m->data[3] << 6) | ((unsigned)m->data[4] >> 2));
		}
		else o.cstr("empty");
		if ((c.mode & 1) && m->ppm != 1024.0f && m->level != 1024.0f) {
			o.cstr(", signalpower: ");
			put_g(o, m->level);
			o.cstr(", ppm: ");
			put_g(o, m->ppm);
		}
		if (c.mode & 2) {
			o.cstr(", timestamp: ");
			put_rxtime(o, rxtime_us);
		}
		if (c.station) {
			o.cstr(", ID: ");
			o.i64(c.station);
		}
		o.raw(")\n", 2);
	}
}

// one full-JSON line: the prefix with the time members of rxtime_us where the mode prints them (JSONAIS.cpp:1101-1106), body, '}';
// its length, or -2 when it does not fit in cap
__host__ __device__ int line(const aisgpu_msg *src, const FmtCtx &c, long long rxtime_us, char *out, int cap) {
	Msg m;
	for (int i = 0; i < kBufBytes; i++) m.d[i] = i < kMaxBytes ? src->data[i] : 0;
	m.nbits = (src->nbits >= 0 && src->nbits <= kMaxBits) ? src->nbits : 0; // Message::setLength ignores other lengths
	Out o(out, cap);
	o.raw(c.prefix, c.prefix_time);
	if (c.mode & 2) {
		o.cstr(",\"rxtime\":\"");
		put_rxtime(o, rxtime_us); // Message::getRxTime
		o.cstr("\",\"rxuxtime\":");
		o.f64((double)rxtime_us / 1000000.0);
	}
	o.raw(c.prefix + c.prefix_time, c.prefix_len - c.prefix_time);
	body(o, m, src, c.mode, c.station);
	o.ch('}');
	return o.full ? -2 : (int)(o.p - out);
}

// The record of one frame in c.fmt (OutputMessage::formatInto, MsgOut.h:58-122, and OutputMessage::Receive for the JSON formats):
// its length, or -2 when it does not fit in cap.  ordinal: the frames published before it; groups: the multi-sentence ones among
// them; rxtime_us: its stamp.  JSON_SPARSE and JSON_ANNOTATED write the full line into scratch (scap bytes) first and rewrite it
// into out.
__host__ __device__ int record(const aisgpu_msg *src, const FmtCtx &c, long long rxtime_us, long long ordinal, long long groups, char *out,
							   int cap, char *scratch, int scap) {
	Out o(out, cap);
	switch (c.fmt) {
	case AISGPU_MSGFORMAT_NMEA:
		for (int i = 0; i < n_sent(src); i++) {
			o.raw(src->nmea[i], sent_len(src, i));
			o.cstr(c.suffix);
		}
		break;
	case AISGPU_MSGFORMAT_NMEA_TAG: tag_block(o, src, c, rxtime_us, groups); break;
	case AISGPU_MSGFORMAT_COMMUNITY_HUB:
		if (ordinal % 100 == 0) nmea_json(o, src, c, rxtime_us);
		else binary(o, out, src, rxtime_us, false);
		break;
	case AISGPU_MSGFORMAT_BINARY_NMEA: binary(o, out, src, rxtime_us, c.crc != 0); break;
	case AISGPU_MSGFORMAT_FULL: full_text(o, src, c, rxtime_us); break;
	case AISGPU_MSGFORMAT_JSON_NMEA: nmea_json(o, src, c, rxtime_us); break;
	case AISGPU_MSGFORMAT_JSON_FULL: {
		const int n = line(src, c, rxtime_us, out, cap);
		if (n < 0) return -2;
		o.p += n;
		o.cstr(c.suffix);
		break;
	}
	default: {
		const int n = line(src, c, rxtime_us, scratch, scap);
		if (n < 0) return -2;
		rewrite(o, scratch, n, c.fmt == AISGPU_MSGFORMAT_JSON_SPARSE ? D_SPARSE : D_ANNOTATED);
		o.cstr(c.suffix);
		break;
	}
	}
	return o.full ? -2 : (int)(o.p - out);
}

// groups[i] = base + the multi-sentence frames of the batch before frame i; total[3] = those of the whole batch (one block, tiles of
// 256 frames: an exclusive scan with a carried sum)
__global__ void __launch_bounds__(256) k_fmt_groups(const aisgpu_msg *__restrict__ msgs, int n, long long base,
													long long *__restrict__ groups, long long *__restrict__ total) {
	typedef cub::BlockScan<long long, 256> Scan;
	__shared__ typename Scan::TempStorage ts;
	__shared__ long long s_carry;
	if (threadIdx.x == 0) s_carry = base;
	__syncthreads();
	for (int t0 = 0; t0 < n; t0 += 256) {
		const int i = t0 + threadIdx.x;
		const long long f = i < n && msgs[i].n_sentences > 1 ? 1 : 0;
		long long ex, agg;
		Scan(ts).ExclusiveSum(f, ex, agg);
		if (i < n) groups[i] = s_carry + ex;
		__syncthreads();
		if (threadIdx.x == 0) s_carry += agg;
		__syncthreads();
	}
	if (threadIdx.x == 0) total[3] = s_carry - base;
}

// record i (frame ordinal + i) into the first cap bytes of its slot, the rest of the slot its scratch; its length into len[i].  The
// context is ctx[0], or with per_stream that of the frame's stream (a receiver table); the time is stamps[i] (an engine with a
// clock), else the context's
__global__ void k_fmt_records(const aisgpu_msg *__restrict__ msgs, const long long *__restrict__ stamps, int n, const FmtCtx *__restrict__ ctx,
							  int per_stream, long long ordinal, const long long *__restrict__ groups, char *__restrict__ slots, int slot, int cap,
							  int *__restrict__ len) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	char *s = slots + (size_t)i * slot;
	const FmtCtx &c = ctx[per_stream ? msgs[i].stream : 0];
	len[i] = record(msgs + i, c, stamps ? stamps[i] : c.rxtime_us, ordinal + i, groups[i], s, cap, s + cap, slot - cap);
}

// Where each record goes: record i is kept when the records of its submit up to and including it fit in cap bytes, and kept
// records are packed in frame order.  A submit that began in an earlier batch has already used carry bytes (records of the first
// submit of the batch count from -carry).  One block walks the batch in tiles of 256 frames twice: the running sum of every
// record, then the running sum of the kept ones.  keep[i] = its bytes, -1 when it is dropped.
__global__ void __launch_bounds__(256) k_fmt_place(const int *__restrict__ len, const int *__restrict__ seg, int n, long long cap,
												   long long carry, long long *__restrict__ psum, long long *__restrict__ off,
												   int *__restrict__ keep, long long *__restrict__ total) {
	typedef cub::BlockScan<long long, 256> Scan;
	__shared__ typename Scan::TempStorage ts;
	__shared__ long long s_carry, s_kept;
	if (threadIdx.x == 0) {
		s_carry = 0;
		s_kept = 0;
	}
	__syncthreads();
	for (int t0 = 0; t0 < n; t0 += 256) {
		const int i = t0 + threadIdx.x;
		const long long b = i < n ? (long long)(len[i] > 0 ? len[i] : 0) : 0; // a record too long for its slot (never: see the slot) is ""
		long long incl, agg;
		Scan(ts).InclusiveSum(b, incl, agg);
		if (i < n) psum[i] = s_carry + incl;
		__syncthreads();
		if (threadIdx.x == 0) s_carry += agg;
		__syncthreads();
	}
	if (threadIdx.x == 0) s_carry = 0;
	__syncthreads();
	for (int t0 = 0; t0 < n; t0 += 256) {
		const int i = t0 + threadIdx.x;
		long long k = 0;
		bool kept = false;
		if (i < n) {
			const long long before = seg[i] > 0 ? psum[seg[i] - 1] : -carry;
			kept = psum[i] - before <= cap;
			k = kept ? psum[i] - (i > 0 ? psum[i - 1] : 0) : 0;
		}
		long long ex, agg;
		Scan(ts).ExclusiveSum(k, ex, agg);
		if (i < n) {
			keep[i] = kept ? (int)k : -1;
			off[i] = s_carry + ex;
		}
		const int nk = __syncthreads_count(kept);
		if (threadIdx.x == 0) {
			s_carry += agg;
			s_kept += nk;
		}
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		total[0] = s_carry;
		total[1] = s_kept;
		total[2] = psum[n - 1] - (seg[n - 1] > 0 ? psum[seg[n - 1] - 1] : -carry); // bytes of the last submit so far, for the next batch
	}
}

// One warp per kept record: its bytes from the slot to the packed text.
__global__ void k_fmt_copy(const char *__restrict__ slots, int slot, const int *__restrict__ keep, const long long *__restrict__ off,
						   int n, char *__restrict__ text) {
	const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	if (i >= n || keep[i] <= 0) return;
	const int l = keep[i];
	const char *s = slots + (size_t)i * slot;
	char *d = text + off[i];
	for (int c = lane; c < l; c += 32) d[c] = s[c];
}

} // namespace

int fmt_record_host(const aisgpu_msg *m, const FmtCtx *c, long long ordinal, long long groups, char *out, int cap) {
	const bool rewritten = c->fmt == AISGPU_MSGFORMAT_JSON_SPARSE || c->fmt == AISGPU_MSGFORMAT_JSON_ANNOTATED;
	std::vector<char> scratch(rewritten ? (size_t)c->prefix_len + kAjTimeMax + 4096 : 0);
	const int n = record(m, *c, c->rxtime_us, ordinal, groups, out, cap, scratch.data(), (int)scratch.size());
	return n < 0 ? AISGPU_EOVERFLOW : n;
}

AjPrefix aj_prefix(const aisgpu_tag *tag) {
	std::string s(256 + (tag->hardware ? strlen(tag->hardware) * 6 : 0), '\0');
	Out o(&s[0], (int)s.size());
	o.cstr("{\"class\":\"AIS\",\"device\":\"AIS-catcher\",\"version\":");
	o.i64(tag->version);
	o.cstr(",\"driver\":");
	o.i64(tag->driver);
	o.cstr(",\"hardware\":");
	o.qstr(tag->hardware ? tag->hardware : "");
	const int time_at = (int)(o.p - &s[0]);
	if (tag->toa_us) {
		o.cstr(",\"toa\":");
		o.f64((double)tag->toa_us / 1000000.0);
	}
	o.cstr(",\"scaled\":true");
	s.resize((size_t)(o.p - &s[0]));
	return AjPrefix{ s, time_at };
}

cudaError_t fmt_launch(const aisgpu_msg *d_msgs, const long long *d_stamps, int n, const FmtCtx *d_ctx, int per_stream, long long ordinal, long long groups, long long *d_groups,
					   char *d_slots, int slot, int cap, int *d_len, const int *d_seg, long long budget, long long carry,
					   long long *d_psum, long long *d_off, int *d_keep, long long *d_total, char *d_text, cudaStream_t st) {
	if (n <= 0) return cudaSuccess;
	k_fmt_groups<<<1, 256, 0, st>>>(d_msgs, n, groups, d_groups, d_total);
	k_fmt_records<<<(n + 127) / 128, 128, 0, st>>>(d_msgs, d_stamps, n, d_ctx, per_stream, ordinal, d_groups, d_slots, slot, cap, d_len);
	k_fmt_place<<<1, 256, 0, st>>>(d_len, d_seg, n, budget, carry, d_psum, d_off, d_keep, d_total);
	k_fmt_copy<<<(n + 7) / 8, 256, 0, st>>>(d_slots, slot, d_keep, d_off, n, d_text);
	return cudaGetLastError();
}

// the context of a tag: NULL strings as "" (suffix as given: NULL is none); prefix: aj_prefix(tag), which must outlive the context
FmtCtx fmt_ctx(const aisgpu_tag *tag, int fmt, const char *suffix, const AjPrefix &prefix) {
	FmtCtx c;
	c.fmt = fmt;
	c.version = tag->version;
	c.driver = tag->driver;
	c.mode = tag->mode;
	c.station = tag->station;
	c.status = tag->status;
	c.include_ssl = tag->include_ssl;
	c.crc = 0;
	c.ipv4 = tag->ipv4;
	c.rxtime_us = tag->rxtime_us;
	c.toa_us = tag->toa_us;
	c.hardware = tag->hardware ? tag->hardware : "";
	c.uuid = tag->uuid ? tag->uuid : "";
	c.suffix = suffix ? suffix : "";
	c.prefix = prefix.text.data();
	c.prefix_len = (int)prefix.text.size();
	c.prefix_time = prefix.time_at;
	return c;
}

extern "C" int aisgpu_msg_json_full(const aisgpu_msg *m, const aisgpu_tag *tag, char *out, int cap) {
	if (!m || !tag || !out || cap <= 0) return AISGPU_EINVAL;
	const AjPrefix p = aj_prefix(tag);
	const FmtCtx c = fmt_ctx(tag, AISGPU_MSGFORMAT_JSON_FULL, tag->suffix, p);
	return fmt_record_host(m, &c, 0, 0, out, cap);
}

extern "C" int aisgpu_msg_format(const aisgpu_msg *m, const aisgpu_tag *tag, int msgformat, aisgpu_format_state *st, char *out, int cap) {
	if (!m || !tag || !out || cap <= 0 || msgformat < AISGPU_MSGFORMAT_NMEA || msgformat > AISGPU_MSGFORMAT_JSON_ANNOTATED)
		return AISGPU_EINVAL;
	const AjPrefix p = aj_prefix(tag);
	const FmtCtx c = fmt_ctx(tag, msgformat, tag->suffix ? tag->suffix : "\r\n", p);
	const int n = fmt_record_host(m, &c, st ? st->records : 0, st ? st->groups : 0, out, cap);
	if (n >= 0 && st) {
		st->records++;
		if (m->n_sentences > 1) st->groups++;
	}
	return n;
}
