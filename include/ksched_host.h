/*
 * ksched_host — the string-level entry points: the host layer ABOVE the flat C-ABI of ksched.h. Link with -lksched -lkmodel
 * (libkmodel.so: problems / results, no CUDA; libksched.so: everything that solves).
 *
 * ksched.h is what a Go encoder would bind (flat structs, no strings). This header is the other way to bind the library:
 * hand it the reference's objects as they are — pods, provisioners, instance types, state nodes as one JSON document
 * (the field names of karpenter-core_b200/host/loader.cc, which mirror v1.Pod / v1alpha5.Provisioner /
 * cloudprovider.InstanceType / state.Node) — and let the library's own host layer (host/encoder.cc) do the work
 * provisioner.go:237-296 and scheduler.go:42-78 do before Solve. Every decision still runs on the GPU through ksched_*;
 * without a CUDA device every call here fails with KSCHED_ERR_NO_DEVICE (there is no CPU path).
 *
 * Reference entry points replaced:
 *   kh_scheduler_solve        (*Scheduler).Solve                      provisioning/scheduling/scheduler.go:96
 *   kh_rank_candidates        candidateNodes + sortAndFilterCandidates deprovisioning/helpers.go:171-249, consolidation.go:85-118
 *   kh_cluster_* / kh_consolidate          computeConsolidation + firstNNodeConsolidationOption
 *                                                                       consolidation.go:190-274, multinodeconsolidation.go:74-114
 *   kh_consolidate_single     SingleNodeConsolidation.ComputeCommand   singlenodeconsolidation.go:43-84 (every command taken as valid)
 *   kh_cluster_validate       Validation.IsValid + ValidateCommand     validation.go:63-172
 *   kh_consolidate_validated  MultiNodeConsolidation.ComputeCommand    multinodeconsolidation.go:41-70
 *   kh_consolidate_single_validated  SingleNodeConsolidation.ComputeCommand with validation  singlenodeconsolidation.go:43-84
 *
 * Conventions: opaque pointers are owned by the caller and freed with the matching *_free / *_close; int returns are
 * KSCHED_OK (0) or a negative KSCHED_ERR_* (ksched.h) unless stated; the message of the last failure on the calling thread
 * is kh_scheduler_error() (kh_last_error() for the loader). Actions: 0 do nothing, 1 delete, 2 replace, 3 retry (a command
 * failed validation, deprovisioning/types.go). Instance types are named by their index in the problem's instanceTypes list, nodes by their
 * index in its nodes list.
 */
#ifndef KSCHED_HOST_H
#define KSCHED_HOST_H

#include "ksched.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kh_problem kh_problem;  /* the inputs of NewScheduler + Solve (host/model.h: kmodel::Problem) */
typedef struct kh_result kh_result;    /* ([]*Node, []*ExistingNode) of one Solve (host/model.h: kmodel::Result) */
typedef struct kh_cluster kh_cluster;  /* one consolidation pass: candidates ranked, cluster resident on the device */

/* ---- problems and results */
/* NULL on a parse error: kh_last_error(). Pod (anti-)affinity terms, required and preferred, of pending, bound and daemonset
 * pods: {labelSelector, namespaces[], namespaceSelector, topologyKey}. A namespaceSelector ({} selects every namespace) is
 * resolved as buildNamespaceList does (topology.go:326-347) against the document's top-level namespaces[] {name, labels},
 * the cluster's Namespace objects. Refused here: a namespaceSelector in a document without namespaces[], one that
 * metav1.LabelSelectorAsSelector rejects (an operator other than In / NotIn / Exists / DoesNotExist, In / NotIn without
 * values, Exists / DoesNotExist with values, an invalid label key or value), duplicate namespace names, and a pod or
 * Namespace named "<no namespace>" (the loader's name for a selector that resolved to no namespace). */
kh_problem* kh_problem_from_json(const char* text);
void kh_problem_free(kh_problem* p);
const char* kh_last_error(void);
long long kh_parse_quantity(const char* s);         /* k8s resource.Quantity -> milli-units */
kh_result* kh_result_new(void);
void kh_result_free(kh_result* r);
const char* kh_result_error(const kh_result* r);
long long kh_result_num_pods(const kh_result* r);
long long kh_result_num_new_nodes(const kh_result* r);
long long kh_result_num_existing(const kh_result* r);
void kh_result_assign(const kh_result* r, int* out);  /* [pods] -1 | existing node | existing + new node index */
void kh_result_relax(const kh_result* r, int* out);   /* [pods] successful Preferences.Relax calls */
long long kh_result_new_node_options(const kh_result* r, long long node, int* out, long long cap); /* InstanceTypeOptions, input order */
long long kh_result_to_json(const kh_result* r, char* buf, long long cap); /* everything, incl. requirements, requests, launch choice */

/* ---- the device */
int kh_set_device(int ordinal);   /* CUDA device of this process's scheduler handle (default 0) */
const char* kh_scheduler_error(void);
int kh_nccl_init(const void* id128, int rank, int world); /* communicator for kh_allgather_i32 (id: ksched_nccl_unique_id) */
int kh_allgather_i32(const int* send, int n, int* recv);  /* one ncclAllGather, recv holds world * n */

/* ---- Scheduler.Solve. candidates: node indices whose pods are rescheduled and which are not offered as existing nodes
 * (simulateScheduling, deprovisioning/helpers.go:42-93); none for provisioning. */
int kh_scheduler_solve(const kh_problem* p, const int* candidates, int n_candidates, kh_result* out);

/* ---- deprovisioning: ranking. order = node indices by ascending disruption cost (ties: list order), cost parallel.
 * Returns the number of candidates or a negative error. With "deriveCandidates": false in the problem the nodes' own
 * candidate / disruptionCost fields are taken and only ordered. */
int kh_rank_candidates(const kh_problem* p, int* order, double* cost, int cap);

/* ---- deprovisioning: the simulator. Open once per pass; every probe is one entry of a ksched_simulate_batch call against
 * the device-resident cluster (resident = 0: the snapshot refused the cluster and each probe is a freshly encoded
 * ksched_solve instead - same answers, slower). */
kh_cluster* kh_cluster_open(const kh_problem* p, int* resident, int* n_candidates);
void kh_cluster_close(kh_cluster* c);
int kh_cluster_candidates(const kh_cluster* c, int* nodes, int cap); /* disruption order */
/* computeConsolidation for n_sets candidate sets; set q = sets[set_off[q] .. set_off[q+1]) as positions in the disruption
 * order; multi != 0 applies the multi-node caller's filterOutSameType. actions[q]; the replacement options of set q go to
 * options[q * options_stride ...], n_options[q] of them. */
int kh_cluster_probe_sets(kh_cluster* c, const int* sets, const int* set_off, int n_sets, int multi, int* actions, int* options, int options_stride,
                          int* n_options);

/* MultiNodeConsolidation.firstNNodeConsolidationOption. out4 = [action, nodes removed (a prefix of the disruption order),
 * simulations, n_options]; probes / probe_actions = the binary search's trace. */
int kh_consolidate(const kh_problem* p, int* out4, int* options, int options_cap, int* probes, int* probe_actions, int probes_cap, int* n_probes);
/* SingleNodeConsolidation.ComputeCommand over positions [first, last) of the disruption order (last < 0: all), `batch`
 * independent simulations per device call. out4 = [action, winning position or -1, simulations, n_options]; *node = the
 * node the command removes. */
int kh_consolidate_single(const kh_problem* p, int first, int last, int batch, int* out4, int* node, int* options, int options_cap);

/* ---- deprovisioning: validation against the cluster as it stands when the consolidation TTL ends (`after`; the wait itself
 * is the caller's). Every validation of one ComputeCommand reads one snapshot of `after` (DESIGN.md section 6, R7), resident
 * on a device handle of its own and opened at the first command that needs validation. Validation candidates:
 * candidateNodes(after, Validation.ShouldDeprovision) in node-list order, matched to the command's nodes by name. */
/* Validation.IsValid of n_sets commands of an open session, in one ksched_simulate_batch call. Command q = the candidates
 * at positions sets[set_off[q] .. set_off[q+1]), actions[q] (1 or 2) and options[q * options_stride ...] (n_options[q]) -
 * what kh_cluster_probe_sets returns. valid[q] = 1 / 0. The session keeps the snapshot of `after` until it closes or is
 * handed a different problem (told apart by a process-unique problem id, not by address). */
int kh_cluster_validate(kh_cluster* c, const kh_problem* after, const int* sets, const int* set_off, int n_sets, const int* actions, const int* options,
                        int options_stride, const int* n_options, int* valid);
/* MultiNodeConsolidation.ComputeCommand: the search of kh_consolidate on `before`, then one validation against `after`; a
 * command that fails it becomes retry, out4 = [3, 0, simulations, 0]. *verdict = 1 valid, 0 invalid, -1 none run. */
int kh_consolidate_validated(const kh_problem* before, const kh_problem* after, int* out4, int* options, int options_cap, int* probes,
                             int* probe_actions, int probes_cap, int* n_probes, int* verdict);
/* SingleNodeConsolidation.ComputeCommand: as kh_consolidate_single, but each batch's actionable commands are validated
 * together against `after` and the first valid one wins; none, after a failed validation, is retry (3). trace / trace_valid =
 * positions validated and verdicts up to and including the winner, *n_trace of them; *failed_validation = a validation failed.
 * Shares [first, last) merge as: the first share with a winner wins; with none, retry when any share failed a validation. */
int kh_consolidate_single_validated(const kh_problem* before, const kh_problem* after, int first, int last, int batch, int* out4, int* node,
                                    int* options, int options_cap, int* trace, int* trace_valid, int trace_cap, int* n_trace, int* failed_validation);

/* ---- an encoding's volume claims (tests): `enc` is an encoding of kh_encode / kh_encode_cluster. Tracked claim `id` as
 * "driver claim" into out[cap], in id order (ksched.h: ksched_class_volumes); -1 when there is no such claim or it does not
 * fit. */
int kh_encoded_volume_claim(const void* enc, int id, char* out, int cap);

/* ---- self-test of the encoder's value classes (CPU, no device): random wide keys and requirement pairs, the exact string
 * algebra against the collapsed masks (host form and region form). Returns the number of mismatches. */
int kh_value_class_selftest(unsigned seed, int iters);

#ifdef __cplusplus
}
#endif
#endif /* KSCHED_HOST_H */
