// The full AIS JSON of published frames (be_json.cu): the host-side view aisgpu.cu needs.
#pragma once
#include "../../include/aisgpu.h"

#include <cuda_runtime.h>
#include <string>

// The part of every line that depends only on the tag (class .. hardware, rxtime / rxuxtime, toa, "scaled"), ending in
// "scaled":true -- built once per engine and copied in front of every line.
std::string aj_prefix(const aisgpu_tag *tag);

// One line for m into out (cap bytes), without newline: its length, or AISGPU_EOVERFLOW when it does not fit.
int aj_line_host(const aisgpu_msg *m, const char *prefix, int prefix_len, int mode, int station, char *out, int cap);

// The device side of one batch of n published frames (already in d_msgs), three launches on st:
//   - line i into the slot d_slots + i * slot, its length into d_len[i] (-2: longer than slot);
//   - the placement: line i and its newline are kept when the lines of its submit up to and including it fit in cap bytes (d_seg[i]
//     = index of the first frame of frame i's submit; carry = the bytes the batch's first submit used in earlier batches);
//     d_keep[i] = the bytes it takes (0: dropped), d_off[i] = where, d_total[0] = all of them, d_total[1] the lines kept and
//     d_total[2] the bytes of the batch's last submit so far (d_psum: scratch, n);
//   - the kept lines packed, newline-terminated, into d_text.
// Returns the launch error, if any.
cudaError_t aj_launch(const aisgpu_msg *d_msgs, int n, const char *d_prefix, int prefix_len, int mode, int station, char *d_slots,
					  int slot, int *d_len, const int *d_seg, long long cap, long long carry, long long *d_psum, long long *d_off, int *d_keep,
					  long long *d_total, char *d_text, cudaStream_t st);
