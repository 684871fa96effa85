/* TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
 *
 * Plain-C restatement of the reference's IQ -> NMEA hot path (see ais_oracle.c
 * for the file:line map).  Same C entry points as oracle/ref_harness.cpp so the
 * Python side (oracle/oracle.py) can swap one for the other.
 *
 * Parity status: PINNED.  The reference holds no golden vectors for this path
 * (SURVEY.md 4 / 8c), so the restatement is pinned against outputs of the
 * reference itself: tests/test_oracle_port_vs_ref.py compares every tap and
 * every message of this port bit-for-bit with oracle/_ref/libaisref.so (the
 * unmodified reference sources compiled with strict IEEE flags), and
 * tests/golden/ holds committed vectors generated from that library by
 * tests/golden/make_golden.py for machines where /root/reference is absent.
 */
#ifndef AIS_ORACLE_H
#define AIS_ORACLE_H

#ifdef __cplusplus
extern "C" {
#endif

void *aisorc_create(int model, int sample_rate, int format, unsigned flags, int own_mmsi);
int aisorc_push(void *h, const void *data, long nbytes);
long aisorc_tap_c(void *h, int tap, float *dst, long max);
long aisorc_tap_ppm(void *h, int tap, float *dst, long max);
long aisorc_tap_f(void *h, int tap, float *dst, long max);
long aisorc_msg_count(void *h);
long aisorc_messages(void *h, char *dst, long max);
long aisorc_publishers(void *h, int *dst, long max);
int aisorc_challenger_order(void *h, const int order[10]);
void aisorc_destroy(void *h);

#ifdef __cplusplus
}
#endif
#endif
