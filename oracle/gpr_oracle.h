/*
 * gpr_oracle.h — CPU restatement of gpu-pruner's idle decision.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this; nothing in the product path (gpu-pruner_b200/, libgpr.so) links, imports
 * or calls it.
 *
 * PARITY UNPINNED: the reference holds no golden vectors, known-answer tests or fixtures for
 * this path (its 11 template tests, gpu-pruner/src/main.rs:572-740, assert only on query
 * TEXT), and the arithmetic itself runs in an external Prometheus server of unpinned version
 * (gpu-pruner/src/main.rs:397), not in the reference.  This file therefore restates PromQL
 * semantics for the one expression in gpu-pruner/src/query.promql.j2:1-44 plus the Rust-side
 * dedup and age gate, and is cross-checked against an independent numpy restatement
 * (oracle/oracle_np.py) and the hand-derived known-answer vectors K1..K14 (SURVEY.md §8(c)).
 */
#ifndef GPR_ORACLE_H_
#define GPR_ORACLE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* counts[0] = idle series in non-vetoed pods (QueryResponse.num_pods, main.rs:418),
 * counts[1] = candidate pods, counts[2] = decided pods                                   */

/* max_over_time over one series' window, evaluated in float64 as Prometheus does.
 * NaN in the dense row = "no sample at this step".  Returns NaN iff no sample present.   */
double gpo_max_over_time(const float *row, uint32_t n_samples);

/* Whole decision for pods [0, n_pods).  Any output pointer may be NULL.  row_stride 0 =
 * n_samples.  power_threshold 0.0 / NaN or power == NULL => no veto clause.               */
int gpo_decide(const float *util, const float *power, const uint8_t *eligible,
               const int64_t *created_ts, int64_t cutoff_ts, uint32_t n_pods, uint32_t n_gpus,
               uint32_t n_samples, uint64_t row_stride, double power_threshold,
               uint32_t *decision_bits, uint32_t *candidate_bits, float *series_max,
               uint64_t counts[3]);

/* Same, over contiguous pod ranges on n_threads POSIX threads (the timed CPU baseline).   */
int gpo_decide_mt(int n_threads, const float *util, const float *power, const uint8_t *eligible,
                  const int64_t *created_ts, int64_t cutoff_ts, uint32_t n_pods, uint32_t n_gpus,
                  uint32_t n_samples, uint64_t row_stride, double power_threshold,
                  uint32_t *decision_bits, uint32_t *candidate_bits, float *series_max,
                  uint64_t counts[3]);

/* Synthetic DCGM universe (SURVEY.md §8(d); exact recipe in DESIGN.md §synthetic).        */
float gpo_synth_cell(uint64_t seed, int plane, uint64_t series, uint32_t t, uint32_t n_samples);
uint8_t gpo_synth_eligible_pod(uint64_t seed, uint64_t pod);
int gpo_synth_fill(int n_threads, uint64_t seed, int plane, float *dst, uint64_t pod_offset,
                   uint32_t n_pods, uint32_t n_gpus, uint32_t n_samples, uint64_t row_stride);
int gpo_synth_eligible(uint64_t seed, uint8_t *dst, uint64_t pod_offset, uint32_t n_pods);

/* Decision over a synthetic universe WITHOUT materialising it: each thread regenerates one
 * row at a time into a private buffer.  Used for parity at sizes that do not fit host RAM
 * and as the streaming CPU baseline.  use_power / use_elig select the optional clauses.    */
int gpo_decide_synth(int n_threads, uint64_t seed, uint64_t pod_offset, uint32_t n_pods,
                     uint32_t n_gpus, uint32_t n_samples, int use_power, double power_threshold,
                     int use_elig, uint32_t *decision_bits, uint32_t *candidate_bits,
                     uint64_t counts[3]);
/* Same, plus the window max of every util series (series_max[p * n_gpus + g], may be NULL) and the pods the
 * power clause vetoes (veto_bits, may be NULL): together they check every row of a window, also rows that
 * change no verdict bit.                                                                    */
int gpo_decide_synth_ex(int n_threads, uint64_t seed, uint64_t pod_offset, uint32_t n_pods,
                        uint32_t n_gpus, uint32_t n_samples, int use_power, double power_threshold,
                        int use_elig, uint32_t *decision_bits, uint32_t *candidate_bits,
                        float *series_max, uint32_t *veto_bits, uint64_t counts[3]);

/* CPUs this process may run on (affinity-mask aware) */
int gpo_hardware_threads(void);
/* Timed baseline only: pin pool worker i to the i-th allowed CPU (takes effect at each worker's next
 * job), so that windows filled by gpo_synth_fill are NUMA-local to the thread that reduces them. */
void gpo_pool_pin(int on);

#ifdef __cplusplus
}
#endif
#endif
