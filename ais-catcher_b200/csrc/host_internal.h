// Hooks the host-side units of libaisgpu.so (feeder.cpp) use besides the public ABI; defined in aisgpu.cu, not part of include/aisgpu.h.
#pragma once
#include "../../include/aisgpu.h"
extern "C" {
const aisgpu_config *aisgpu_internal_config(aisgpu_handle *h);
int aisgpu_internal_inputs(aisgpu_handle *h); // the rows a submit holds: n_streams, or n_streams / per_input (aisgpu_set_tunings)
void aisgpu_internal_set_error(aisgpu_handle *h, const char *msg); // h == NULL: the error aisgpu_last_error(NULL) returns
int aisgpu_internal_grouped(aisgpu_handle *h); // 1 for a member of an engine group or a leader with members
}
