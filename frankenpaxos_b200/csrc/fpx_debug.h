/* fpx_debug.h -- test and profiling aids of libfpx.so.  They are not part of the C ABI of include/fpx.h and
 * get no JNI stub; fpx_engine.cu defines them (comments there), frankenpaxos_b200/_lib.py binds them from here. */
#ifndef FPX_DEBUG_H
#define FPX_DEBUG_H

#include <stdint.h>

#include "../../include/fpx.h"

#ifdef __cplusplus
extern "C" {
#endif

int fpx_debug_phase_times(fpx_engine* e, unsigned long long* acceptor8, unsigned long long* tally8);
int fpx_debug_set_tally_path(fpx_engine* e, int32_t path);
int fpx_debug_last_paths(fpx_engine* e, int32_t* out);
int fpx_debug_set_acceptor_segments(fpx_engine* e, int32_t segments);
int fpx_debug_set_tally_max_sub(fpx_engine* e, int32_t votes);
int fpx_debug_set_counters(fpx_engine* e, uint32_t seq_base, uint32_t rseq_base, uint32_t rng_seq_base,
                           uint32_t vm_tag);
int fpx_debug_get_counters(fpx_engine* e, uint32_t* out);
int fpx_debug_epaxos_set_counters(fpx_epaxos* e, uint32_t tag, uint32_t seq_base);
int fpx_debug_epaxos_get_counters(fpx_epaxos* e, uint32_t* out);

#ifdef __cplusplus
}
#endif

#endif /* FPX_DEBUG_H */
