/*
 * ksched — H100-native (sm_90a) drop-in for Karpenter's provisioning scheduler hot path.
 *
 * C-ABI boundary: plain pointers and sizes only. A cgo shim in the reference would marshal the
 * arguments of scheduling.NewScheduler (pkg/controllers/provisioning/scheduling/scheduler.go:42-45)
 * into ksched_catalog + ksched_problem, call ksched_solve in place of (*Scheduler).Solve
 * (scheduler.go:96), and rebuild []*Node / []*ExistingNode from ksched_result (INTEGRATION.md shows
 * the stub). Every buffer is caller-allocated and caller-owned; the library keeps no pointer to caller
 * memory after a call returns (cgo pointer rules). Unschedulable pods are data (assign = -1), never
 * errors — Solve itself never fails in the reference (scheduler.go:132).
 *
 * Encoding (done by the caller; karpenter-core_b200/host/encoder.cc is the C++ version):
 *  - label keys are dictionary ids; up to KSCHED_MAX_KEYS "mask keys", each with <= 63 distinct values,
 *    one bit per value. kubernetes.io/hostname and node.kubernetes.io/instance-type are NOT mask keys:
 *    a node's hostname is its slot index, an instance-type requirement is a bitset over types.
 *  - a requirement mirrors pkg/scheduling/requirement.go:36-42: {complement, values}; `values` are the members
 *    (complement=0) or the excluded members (complement=1). Gt/Lt bounds travel as excluded REGION bits
 *    (ksched_key_regions below), so the device algebra is pure mask arithmetic.
 *  - resource quantities are int64 milli-units (k8s resource.Quantity, exact for whole milli values).
 *  - instance types ("columns") are supplied in ascending (cheapest available offering price, input
 *    index) order; type_input_index maps back to the caller's slice order (lo.Filter keeps input order,
 *    node.go:138).
 */
#ifndef KSCHED_H
#define KSCHED_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KSCHED_ABI_VERSION 4
#define KSCHED_MAX_RES_EXT 24 /* resources beyond the KSCHED_MAX_RES row slots (ksched_catalog.n_res_ext) */
#define KSCHED_MAX_KEYS 16
#define KSCHED_MAX_RES 8
#define KSCHED_MAX_TEMPLATES 64 /* ksched_type_row.template_members is one bit per template */
#define KSCHED_ROW_WORDS 32 /* canonical 256-byte rows (SURVEY.md 8d: B_pod = B_col = 256 B) */
#define KSCHED_KEY_HOSTNAME 255
#define KSCHED_NONE 0xFFFFFFFFu
#define KSCHED_HOSTNAME_TABLE (-2) /* hostname_reqs[i][1]: the admitted existing slots are row i of problem.hostname_slots */
#define KSCHED_ITYPE_UNLISTED 0xFFFFFFFEu /* problem.existing_itype: an instance-type label that names no type of the catalog */

/* error codes (negative) */
#define KSCHED_OK 0
#define KSCHED_ERR_INVALID -1     /* bad argument / inconsistent sizes */
#define KSCHED_ERR_UNSUPPORTED -2 /* problem uses a feature the encoding cannot express (fail loudly) */
#define KSCHED_ERR_CUDA -3
#define KSCHED_ERR_NCCL -4
#define KSCHED_ERR_NO_DEVICE -5
#define KSCHED_ERR_OVERFLOW -6 /* a capacity bound (max new nodes, queue) was exceeded */

/* meta word of a requirement set (16 keys): bit k of each 16-bit field */
#define KSCHED_META_PRESENT_SHIFT 0
#define KSCHED_META_COMPLEMENT_SHIFT 16
#define KSCHED_META_HASGT_SHIFT 32
#define KSCHED_META_HASLT_SHIFT 48

/* A set of requirements over the mask keys: replaces scheduling.Requirements (requirements.go:33). */
typedef struct ksched_reqset {
  uint64_t values[KSCHED_MAX_KEYS];
  uint64_t meta;
} ksched_reqset; /* 136 bytes */

/* Integer bounds (Gt/Lt, requirement.go:58-66) of one reqset in the HOST algebra (csrc/reqmask.cuh); only read where meta
 * has HASGT/HASLT. Nothing that crosses the C-ABI carries them: see ksched_key_regions. */
typedef struct ksched_bounds {
  int64_t gt[KSCHED_MAX_KEYS];
  int64_t lt[KSCHED_MAX_KEYS];
} ksched_bounds;

/*
 * Region form of Gt/Lt — how bounded requirements cross the C-ABI and live on the device.
 * For one key let t[0] < ... < t[m-1] be every threshold any Gt/Lt requirement of the problem names. They cut the integers
 * that are NOT dictionary values into m+1 regions R0 = (-inf,t0), Ri = (t[i-1],t[i]), Rm = (t[m-1],+inf); region Ri is bit
 * region_shift+i of the key's 64-bit value word, right above the real dictionary values. A complement requirement with bounds
 * {excluded E, >gt, <lt} (requirement.go:36-42) is handed over as complement=1 with
 *     values = E  |  every real dictionary value outside (gt,lt) (non-integers included)  |  every region outside (gt,lt)
 * and the HASGT/HASLT meta bits clear. Then Intersection's max(gt)/min(lt)/"drop members outside the bounds"
 * (requirement.go:120-143) is the plain union / and-not of the masks, "gt >= lt -> DoesNotExist" (:124-126) is "all regions
 * excluded", Has(v) is the bit test, and the excluded set proper (for Operator(), :186-197) is
 * values & above[low] & below[high] with low / high the number of excluded regions at either end.
 * A key also gets region bits (m = 0: one region) when some instance type carries a complement requirement on it
 * (NotIn / Exists / Gt / Lt): the region bits are what a complement node requirement and a complement type have in common.
 * Keys with neither have region_mask 0 and nothing changes for them.
 * A caller that builds its own dictionary may collapse a wide key the same way the host encoder does (DESIGN.md §3, value
 * classes): values that no requirement, label, threshold or topology domain of the problem names, and that appear only in
 * instance types' In requirements or existing nodes' labels, can be replaced by one representative per class (unnamed
 * integers of one region Ri, unnamed non-integers), kept as an ordinary dictionary value. The answers do not change.
 * Likewise a key that only templates name (no pod, daemonset, topology term, node filter or bound pod's anti-affinity term
 * names it; neither zone nor capacity-type) needs no mask key at all: its node requirement is always the template's own, so
 * it only decides which instance types a template admits, and can be folded into ksched_type_row.template_members. The
 * caller then renders the template's requirement on that key into each new node's requirements itself (DESIGN.md §3,
 * template-only keys).
 */
#define KSCHED_MAX_THRESHOLDS 7
typedef struct ksched_key_regions {
  uint64_t region_mask;  /* n_thresholds+1 contiguous bits, or 0 */
  int32_t region_shift;  /* bit of R0 */
  int32_t n_thresholds;
  int64_t thresholds[KSCHED_MAX_THRESHOLDS];   /* ascending */
  uint64_t above[KSCHED_MAX_THRESHOLDS + 1];   /* above[i]: real values admitted when the i lowest regions are excluded (above[0] = all) */
  uint64_t below[KSCHED_MAX_THRESHOLDS + 1];   /* below[j]: ... when the j highest regions are excluded (below[0] = all) */
} ksched_key_regions;

/*
 * 256-byte pod-class row. One row per class of pods that are indistinguishable to the scheduler
 * (same requests, requirements, tolerations, host ports, topology terms); every relaxation level
 * (preferences.go:36-56) of a pod is its own class, chained by relax_next.
 * Replaces: resources.RequestsForPods (utils/resources/resources.go:25), NewPodRequirements
 * (requirements.go:61), Taints.Tolerates (taints.go:28), HostPortUsage entries (hostportusage.go:118).
 */
typedef struct ksched_pod_row {
  int64_t requests[KSCHED_MAX_RES]; /* includes pods: 1000 */
  uint64_t values[KSCHED_MAX_KEYS]; /* NewPodRequirements on the mask keys */
  uint64_t meta;
  uint64_t tolerated_taintsets; /* bit s: pod tolerates every taint of taint set s (s < 64; see problem.class_tolerated_ext) */
  uint64_t hostport_conflicts;  /* host-port entries this pod's ports clash with (hostportusage.go:45-57); entries < 64 (see
                                   problem.class_hostport_conflicts_ext) */
  uint64_t hostport_entries;    /* host-port entries this pod reserves (entries < 64) */
  uint32_t res_present;         /* bit r: resource r is a key of the pod's request map */
  uint32_t relax_next;          /* class after one successful Relax, or KSCHED_NONE */
  uint32_t itype_req;           /* index into problem.itype_req_sets (instance-type key), or KSCHED_NONE */
  uint32_t hostname_req;        /* index into problem.hostname_reqs, or KSCHED_NONE */
  uint32_t topo_begin, topo_end; /* range in problem.class_topo (groups that constrain / record this class) */
  uint64_t reserved;            /* must hold the row's own index in problem.classes */
} ksched_pod_row; /* 256 bytes */

/* 256-byte instance-type column. Replaces cloudprovider.InstanceType (cloudprovider/types.go:72-85). */
typedef struct ksched_type_row {
  int64_t allocatable[KSCHED_MAX_RES]; /* Capacity - Overhead.Total(), types.go:87-89; 0 where absent */
  uint64_t values[KSCHED_MAX_KEYS];
  uint64_t meta;
  uint64_t offerings;        /* bit s: an AVAILABLE offering exists in offering slot s (node.go:151-159; ksched_catalog.zone_slots) */
  uint64_t template_members; /* bit v: type is in template v's GetInstanceTypes list (and meets its template-only keys) */
  double min_price;          /* cheapest available offering */
  uint32_t res_present;      /* resources present in Capacity */
  uint32_t input_index;      /* position in the caller's instance-type slice */
  uint64_t reserved[3];
} ksched_type_row; /* 256 bytes */

typedef struct ksched_template {
  ksched_reqset reqs;               /* NewMachineTemplate requirements (machinetemplate.go:46-62) */
  int64_t daemon_requests[KSCHED_MAX_RES]; /* getDaemonOverhead (scheduler.go:250-267); includes pods */
  uint32_t daemon_res_present;
  uint32_t taintset;                /* index of this template's taint set, < 64 */
  int32_t has_limits;               /* provisioner.Spec.Limits != nil */
  uint32_t limit_present;           /* resources that are keys of the limits map */
  int64_t remaining[KSCHED_MAX_RES]; /* remainingResources after calculateExistingMachines */
} ksched_template;

/* dictionary facts the kernels need */
typedef struct ksched_keyinfo {
  uint64_t dict_mask;   /* bits of the values that exist for this key */
  uint64_t int_mask;    /* values that parse as integers (strconv.Atoi), for Gt/Lt */
  int32_t well_known;   /* key is in v1alpha5.WellKnownLabels (requirements.go:125) */
  int32_t is_zone;      /* topology.kubernetes.io/zone */
  int32_t is_capacity_type; /* karpenter.sh/capacity-type */
  int32_t pad;
} ksched_keyinfo;

typedef struct ksched_catalog {
  int32_t n_keys, n_res, n_types, n_templates;
  const ksched_keyinfo* keys;      /* [n_keys]; dict_mask = the REAL values (region bits are added by the library) */
  const ksched_key_regions* key_regions; /* [n_keys] or NULL (no key has region bits) */
  const int64_t* key_int_values;   /* [n_keys][64] integer value of dictionary entry, where int_mask set; may be NULL */
  const ksched_type_row* types;    /* [n_types], price order */
  const ksched_bounds* type_bounds; /* must be NULL: bounded requirements arrive in region form */
  const int64_t* type_capacity;    /* [n_types][KSCHED_MAX_RES] Capacity (limits bookkeeping, scheduler.go:273-309) */
  const ksched_template* templates; /* [n_templates], weight order (v1alpha5/provisioner.go:132) */
  const ksched_bounds* template_bounds; /* must be NULL (region form) */
  /* Launch choice (the step after the path: fake/cloudprovider.go:74-84 orders the surviving options by their cheapest
     compatible offering, cloudprovider/types.go:128-145 picks that offering). [n_types][64], one entry per offering slot s
     (see zone_slots): (rank of the offering's price among all distinct prices of the catalog) << 16 | position in the type's
     Offerings list << 8 | s, for AVAILABLE offerings (the smallest such key when several offerings share a slot); ~0
     elsewhere. NULL: ksched_result.launch is not filled. */
  const uint64_t* offering_keys;
  /* Ext resources: resources from the 9th on (at most KSCHED_MAX_RES_EXT). n_res keeps its meaning (the <= 8 row slots), so
     no reader of the rows indexes past them. Only pod classes request ext resources: no daemonset, provisioner limit or
     existing node's remaining daemon overhead names one (the caller assigns the slots so). 0 / NULL: none. */
  int32_t n_res_ext;
  int32_t pad_ext;
  const int64_t* type_alloc_ext;   /* [n_types][n_res_ext] allocatable of ext resource x (0 where the type lacks it) */
  /* Offering slots: bit s of ksched_type_row.offerings and entry s of offering_keys stand for one (capacity type, zone) pair
     of dictionary ids (without a zone or capacity-type mask key every offering counts as value 0 of that key). Both NULL: slot
     = ct*16 + zone, which holds zone ids below 16 and capacity-type ids below 4. Otherwise zone_slots[z] is the set of slots
     whose zone is value z and ct_slots[c] the set whose capacity type is value c, so the slot of pair (c, z) is
     zone_slots[z] & ct_slots[c]. Every slot belongs to exactly one zone and one capacity type, and every offerings bit of
     every type is a slot of the tables; ksched_load_catalog answers KSCHED_ERR_INVALID otherwise. The host encoder numbers
     the distinct pairs of available offerings in ascending (capacity-type id, zone id) order (DESIGN.md §3). */
  const uint64_t* zone_slots; /* [64] or NULL */
  const uint64_t* ct_slots;   /* [64] or NULL */
} ksched_catalog;

/* Existing (real / in-flight) node: NewExistingNode, existingnode.go:41-75. */
typedef struct ksched_existing_node {
  ksched_reqset reqs;                 /* NewLabelRequirements(node.Labels) on the mask keys */
  int64_t available[KSCHED_MAX_RES];  /* state.Node.Available(), state/node.go:113 */
  int64_t requests[KSCHED_MAX_RES];   /* remaining daemonset overhead, clamped >= 0 */
  uint32_t available_present, requests_present;
  uint32_t taintset;
  uint32_t itype;                     /* node's instance-type label as a type column, or KSCHED_NONE */
  uint64_t hostport_entries;          /* entries already reserved by bound pods (entries < 64; see problem.existing_hostport_ext) */
  uint64_t label_keys_other;          /* reserved */
} ksched_existing_node;

/*
 * CSI volume limits of existing nodes (scheduling/volumeusage.go:33-131, checked by ExistingNode.Add, existingnode.go:88-96).
 * The API Gets of VolumeUsage.validate (:133-190: claim -> storage class / bound volume -> CSI driver) are the caller's; what
 * crosses the ABI is counting. Only drivers that some existing node limits matter (<= KSCHED_MAX_VOLUME_DRIVERS). A claim that
 * exactly one pod of (batch + bound pods) mounts is counted (priv / used); a claim several pods share is a TRACKED id, one bit
 * of a mask, so that mounting it twice on a node counts once (volumes.union, :55-70). When that rule would track more than 64
 * claims, a claim is tracked only when two different pods mount it and one of them is a pod of the batch; a claim only bound
 * pods mount stays in each node's used[]. Ids 0-63 are bits of shared / mounted / volume_driver_mask[d], ids from 64 on bits
 * of the problem's *_volumes_*_ext tables (see class_volumes_shared_ext). Pod p fits node e iff for every limited driver d:
 *   used[d] + popcount over all words of ((mounted | shared) & volume_driver_mask[d]) + priv[d] <= limit[d].
 * A node that already exceeds a limit accepts nobody (Exceeds walks the node's own drivers too, :101-112): the caller marks it
 * by an `available` vector no pod fits.
 */
#define KSCHED_MAX_VOLUME_DRIVERS 4
typedef struct ksched_class_volumes {
  uint64_t shared;                          /* tracked claims the pods of this class mount */
  uint16_t priv[KSCHED_MAX_VOLUME_DRIVERS]; /* claims only this pod mounts, per limited driver */
} ksched_class_volumes;
typedef struct ksched_node_volumes {
  uint64_t mounted;                         /* tracked claims already mounted on the node */
  int32_t used[KSCHED_MAX_VOLUME_DRIVERS];  /* mounted claims that are not tracked ids, per driver */
  int32_t limit[KSCHED_MAX_VOLUME_DRIVERS]; /* CSINode allocatable count, -1 = the node has no limit for the driver */
} ksched_node_volumes;

/* topology group: TopologyGroup, topologygroup.go:53-64 */
typedef struct ksched_topo_group {
  uint8_t type;      /* 0 spread, 1 pod affinity, 2 pod anti-affinity */
  uint8_t key;       /* mask key index or KSCHED_KEY_HOSTNAME */
  uint8_t inverse;   /* lives in Topology.inverseTopologies (topology.go:47) */
  uint8_t dormant;   /* created only by Topology.Update after a relaxation (topology.go:86-117): it records nothing and
                        knows no hostname registered before the first pod that owns it is relaxed */
  int32_t max_skew;
  uint32_t filter_begin, filter_end; /* TopologyNodeFilter terms in problem.filter_terms; empty = always matches */
  uint64_t registered;               /* mask-key groups: domains the group knows (universe + recorded) */
  int32_t extra_nonzero_domains;     /* hostname groups: counted domains that are not schedulable node slots */
  int32_t pad2;
} ksched_topo_group;

/* one (class, group) relation */
#define KSCHED_TOPO_CONSTRAINS 1 /* group is owned by the class, or is an inverse group selecting it (topology.go:351-364) */
#define KSCHED_TOPO_SELECTS 2    /* TopologyGroup.selects(pod), topologygroup.go:246 */
#define KSCHED_TOPO_RECORDS 4    /* group in Topology.topologies and selects the class (topology.go:122-135) */
#define KSCHED_TOPO_RECORDS_INVERSE 8 /* inverse group owned by the class (topology.go:138-142) */
#define KSCHED_TOPO_HOST_EXTRA 16 /* hostname affinity group the class constrains: its hostname requirement admits a domain with a
                                     count that is no existing slot (ksched_topo_group.extra_nonzero_domains), so the group's
                                     options for the class are never empty (topologygroup.go:202-231) */
typedef struct ksched_class_topo {
  uint32_t group;
  uint32_t flags;
} ksched_class_topo;

typedef struct ksched_problem {
  int32_t n_pods, n_classes, n_existing, n_groups;
  const ksched_pod_row* classes;     /* [n_classes] */
  const ksched_bounds* class_bounds; /* must be NULL (region form) */
  const uint32_t* pod_class;         /* [n_pods] initial class of every pod, caller order */
  const int64_t* pod_timestamp;      /* [n_pods] creationTimestamp seconds (queue.go:100) */
  const uint32_t* pod_uid_rank;      /* [n_pods] rank of the pod's UID in ascending string order (queue.go:108) */
  const ksched_existing_node* existing; /* [n_existing], caller order */
  const ksched_bounds* existing_bounds; /* must be NULL (region form) */
  const ksched_topo_group* groups;   /* [n_groups] */
  const int32_t* group_domain_counts; /* [n_groups][64] initial per-domain counts of mask-key groups (countDomains) */
  const int32_t* group_existing_counts; /* [n_groups][n_existing] initial counts of hostname groups per existing node */
  const ksched_class_topo* class_topo; /* ranges referenced by pod rows */
  int32_t n_class_topo;
  const ksched_reqset* filter_terms;  /* TopologyNodeFilter requirement sets */
  int32_t n_filter_terms;
  const uint64_t* itype_req_sets;     /* [n_itype_reqs][type_words]: allowed types per instance-type requirement */
  const uint8_t* itype_req_complement; /* [n_itype_reqs] 1 = NotIn/Exists form (allows types outside the catalog) */
  int32_t n_itype_reqs;
  const int32_t* hostname_reqs;       /* [n_hostname_reqs][2]: {complement, existing node slot or -1 (= none of ours)}, or
                                         {admits new nodes (0/1), KSCHED_HOSTNAME_TABLE}: see hostname_slots */
  int32_t n_hostname_reqs;
  int32_t max_new_nodes;              /* capacity for new nodes (<= n_pods) */
  int32_t write_feasibility;          /* also copy the dense feasibility bitmask back (result.feasibility) */
  int32_t count_nodes_visited;        /* keep the exact nodes_visited statistic (one extra pass over the in-flight nodes per pod) */
  /* CSI volume limits; both NULL when no pod of the batch mounts a claim of a driver that some existing node limits */
  const ksched_class_volumes* class_volumes;   /* [n_classes] */
  const ksched_node_volumes* existing_volumes; /* [n_existing] */
  uint64_t volume_driver_mask[KSCHED_MAX_VOLUME_DRIVERS]; /* tracked claim ids by driver */
  /* Taint sets beyond the 64 of ksched_pod_row.tolerated_taintsets. Templates and existing nodes share one id space of taint
     sets; template sets must have ids below 64 (ksched_load_catalog refuses others), so only existing nodes may carry an id
     s >= 64. Bit (s - 64) % 64 of word [class][(s - 64) / 64] says that the class tolerates every taint of set s.
     NULL (0 words) when every set id is below 64; ksched_upload refuses an existing node whose id the table does not cover. */
  const uint64_t* class_tolerated_ext; /* [n_classes][n_tolerated_ext_words] */
  int32_t n_tolerated_ext_words;
  int32_t pad_ext;
  /* Ext resources (ksched_catalog.n_res_ext). They are not bits of ksched_pod_row.res_present: code that walks that mask
     indexes the 8 row slots. All three NULL when n_res_ext is 0. */
  const int64_t* class_requests_ext;      /* [n_classes][n_res_ext] request (ceiling over init containers) */
  const uint32_t* class_res_ext_present;  /* [n_classes] bit x: ext resource x is a key of the class's request map */
  const int64_t* existing_available_ext;  /* [n_existing][n_res_ext] state.Node.Available() (0 where the node lacks it) */
  /* Host-port entries beyond the 64 of ksched_pod_row.hostport_conflicts / hostport_entries and
     ksched_existing_node.hostport_entries. Entry e >= 64 is bit (e - 64) % 64 of word (e - 64) / 64 of a row of these tables;
     entries 0-63 stay in the row and node words. Relaxed classes are classes and have rows too. All three NULL and the count 0
     when every entry is below 64; ksched_upload answers KSCHED_ERR_INVALID when the tables and the count disagree. */
  const uint64_t* class_hostport_conflicts_ext; /* [n_classes][n_hostport_ext_words] */
  const uint64_t* class_hostport_entries_ext;   /* [n_classes][n_hostport_ext_words] */
  const uint64_t* existing_hostport_ext;        /* [n_existing][n_hostport_ext_words] (may be NULL when n_existing is 0) */
  int32_t n_hostport_ext_words;
  int32_t pad_hostport;
  /* Hostname requirements beyond the {complement, slot} pair (In / NotIn one value, Exists): value lists, several
     requirements on one pod, DoesNotExist, Gt / Lt. An entry i of hostname_reqs whose second word is KSCHED_HOSTNAME_TABLE
     admits existing slot e iff bit e % 64 of hostname_slots[i][e / 64] is set, and a new node iff hostname_reqs[i][0] is 1 (a
     new node's hostname is a placeholder). Rows of pair entries hold the slots the pair admits; the kernels read the pair.
     filter_term_hostname[f] is the hostname part of filter term f, an entry of hostname_reqs, or KSCHED_NONE; it is NULL
     when no term names the hostname. Both tables NULL and the count 0 when no entry needs them; ksched_upload answers
     KSCHED_ERR_INVALID when the tables and the count disagree. */
  const uint64_t* hostname_slots;        /* [n_hostname_reqs][n_hostname_words] */
  const uint32_t* filter_term_hostname;  /* [n_filter_terms] (needs hostname_slots) */
  int32_t n_hostname_words;
  int32_t pad_hostname;
  /* Topology node filter terms that name node.kubernetes.io/instance-type. Every value is an entry of itype_req_sets /
     itype_req_complement, or KSCHED_NONE for "no requirement on the key". filter_term_itype[f] is the instance-type part of
     filter term f. template_itype[v] is the requirement a new node of template v starts from (its provisioner's, from
     NewMachineTemplate). existing_itype[e] is existing node e's requirement In [its instance-type label]; a label that is no
     type of the catalog is KSCHED_ITYPE_UNLISTED. Pods' instance-type requirements intersect into these as they are added,
     and a filter term's part is tested against the result with Intersects. All three NULL when no filter term names the
     key (existing_itype may also be NULL without existing nodes); ksched_upload answers KSCHED_ERR_INVALID otherwise. */
  const uint32_t* filter_term_itype;     /* [n_filter_terms] */
  const uint32_t* template_itype;        /* [catalog n_templates] */
  const uint32_t* existing_itype;        /* [n_existing] */
  /* Tracked volume claims beyond the 64 of ksched_class_volumes.shared, ksched_node_volumes.mounted and volume_driver_mask.
     Claim t >= 64 is bit (t - 64) % 64 of word (t - 64) / 64 of a row of these tables; claims 0-63 stay in the words. Relaxed
     classes are classes and have rows too. All three NULL and the count 0 when at most 64 claims are tracked, and they need
     class_volumes / existing_volumes; ksched_upload answers KSCHED_ERR_INVALID when the tables and the count disagree. */
  const uint64_t* class_volumes_shared_ext;     /* [n_classes][n_volume_ext_words] */
  const uint64_t* existing_volumes_mounted_ext; /* [n_existing][n_volume_ext_words] */
  const uint64_t* volume_driver_mask_ext;       /* [KSCHED_MAX_VOLUME_DRIVERS][n_volume_ext_words] */
  int32_t n_volume_ext_words;
  int32_t pad_volume;
} ksched_problem;

typedef struct ksched_new_node {
  int32_t template_index;
  int32_t pod_count;
  int64_t requests[KSCHED_MAX_RES];
  uint32_t requests_present;
  uint32_t pad;
  ksched_reqset reqs; /* final requirements on the mask keys (hostname removed, node.go:111-115) */
} ksched_new_node;

/* What the cloud provider would launch for a new node: the option whose cheapest compatible AVAILABLE offering is
   cheapest (ties: provider input order), and that offering (ties: Offerings list order). */
typedef struct ksched_launch_choice {
  int32_t type_column;    /* column (price order) of the chosen instance type, -1 if the node has no option */
  int32_t offering_slot;  /* the offering's slot (ksched_catalog.zone_slots) */
  uint32_t price_rank;    /* rank of the offering's price (see ksched_catalog.offering_keys) */
  uint32_t offering_index; /* position of that offering in the instance type's Offerings list */
} ksched_launch_choice;

typedef struct ksched_result {
  int32_t* assign;       /* [n_pods] -1 | existing slot | n_existing + new node index (creation order) */
  int32_t* relax_level;  /* [n_pods] successful Relax calls */
  int32_t* place_seq;    /* [n_pods] order in which the pod was committed (-1 if never) */
  ksched_new_node* new_nodes; /* [max_new_nodes] */
  uint64_t* new_node_types;   /* [max_new_nodes][type_words] surviving InstanceTypeOptions bitset (price order) */
  ksched_reqset* existing_reqs; /* [n_existing] final requirements, or NULL */
  uint64_t* feasibility; /* [n_pods][n_templates][type_words] dense pods x columns bitmask, or NULL */
  uint64_t* best_column; /* [n_pods] min over feasible columns of (f32 price bits << 32 | template << 24 | type), or NULL */
  int32_t n_new_nodes;
  int32_t n_unscheduled;
  int64_t nodes_visited; /* candidate nodes examined, reference scan order (SURVEY.md 8d K2 bytes) */
  int64_t add_calls;     /* queue pops = Scheduler.add calls */
  ksched_launch_choice* launch; /* [max_new_nodes] or NULL (needs ksched_catalog.offering_keys) */
  /* Ext resources of the new nodes (ksched_catalog.n_res_ext), or NULL: [max_new_nodes][n_res_ext] requests and
     [max_new_nodes] presence masks (bit x: ext resource x is a key of the node's request map). */
  int64_t* new_node_requests_ext;
  uint32_t* new_node_requests_ext_present;
} ksched_result;

/*
 * Device-resident cluster snapshot for the consolidation simulator (deprovisioning/helpers.go:42-115, the state it reads:
 * controllers/state/cluster.go:74-103, state/node.go:113-143). One consolidation pass simulates many candidate sets against the
 * same cluster; the cluster crosses the ABI ONCE, as a superset problem:
 *   existing = every owned, not-deleting node - the candidates too - with ALL its pods bound (available, host ports, volumes);
 *   pods     = the pending pods first, then every reschedulable pod of every candidate node, node by node;
 *   pod_node = the existing slot a pod is bound to (-1 = pending: part of every simulation).
 * A simulation names the existing slots it removes: their pods form the batch, the slots accept nobody, the rest of the cluster
 * is what the superset says.
 * Topology (problem->n_groups > 0): the superset's initial group counters count NO pod of the batch (topology.go:66-70); a pod
 * that stays on its node in a simulation is counted again on the device from the tables below - countDomains
 * (topology.go:231-276: namespace + selector per class, node label + TopologyNodeFilter per node) and the inverse
 * anti-affinity groups of bound pods (topology.go:183-227). A cluster with groups but without these tables is refused with
 * KSCHED_ERR_UNSUPPORTED.
 */
#define KSCHED_COUNT_DOMAINS 0 /* a group in Topology.topologies counts the bound pod (countDomains) */
#define KSCHED_COUNT_INVERSE 1 /* an inverse anti-affinity group the bound pod owns (updateInverseAffinities) */
typedef struct ksched_count_rel {
  uint32_t group;
  uint8_t kind;   /* KSCHED_COUNT_* */
  uint8_t times;  /* how many of the pod's terms hash to this group */
  uint16_t pad;
} ksched_count_rel;
typedef struct ksched_cluster {
  const ksched_problem* problem;
  const int32_t* pod_node; /* [problem->n_pods] */
  /* topology tables (all NULL when problem->n_groups == 0) */
  const uint32_t* class_count_begin;      /* [n_classes + 1] ranges in class_count */
  const ksched_count_rel* class_count;
  const int8_t* node_domain;              /* [n_keys][n_existing] dictionary id of the node's label value, -1 = no such label */
  const uint8_t* node_has_hostname_label; /* [n_existing] */
  const uint32_t* group_filter_match;     /* [n_groups][(n_existing + 31) / 32] bit e: TopologyNodeFilter.Matches(node e) */
} ksched_cluster;

typedef struct ksched_candidate_set {
  const int32_t* nodes;     /* existing slots removed by this simulation (the candidates, helpers.go:52-68), distinct */
  int32_t n_nodes;
  int32_t pad;
  const int64_t* remaining; /* [n_templates][KSCHED_MAX_RES] provisioner limits left with the removed nodes' capacity given back
                               (scheduler.go:221-248 only subtracts the nodes that stay), or NULL = as in the catalog */
} ksched_candidate_set;

/* What computeConsolidation reads of one simulation (consolidation.go:190-274). A simulation stops as soon as a second new
   node is opened - len(newNodes) != 1 means "do nothing" whatever the rest of the batch does (:214-224) - so n_new_nodes >= 2
   comes with n_unscheduled > 0 for the pods that were never tried. */
typedef struct ksched_sim_result {
  int32_t n_pods;        /* size of the batch */
  int32_t n_unscheduled;
  int32_t n_new_nodes;
  int32_t error;         /* 0, or a negative ksched error of this simulation (capacity overflow ...) */
  ksched_new_node node0; /* the first new node, valid when n_new_nodes >= 1 */
} ksched_sim_result;

/*
 * Candidate ranking for deprovisioning: disruption cost per node and the order consolidation tries the nodes in
 * (deprovisioning/helpers.go:125-165,275-287 disruptionCost / GetPodEvictionCost / calculateLifetimeRemaining,
 * consolidation.go:85-103 sortAndFilterCandidates). What needs strings or the API server stays with the caller and arrives as
 * flags: node_eligible (candidateNodes' label / annotation filters, helpers.go:171-222, consolidation.go:104-118) and the
 * "blocks eviction" pod flag (PDB with no disruptions left, do-not-evict: helpers.go:339-366, pdblimits.go:55-68).
 */
#define KSCHED_RANK_HAS_DELETION_COST 1
#define KSCHED_RANK_HAS_PRIORITY 2
#define KSCHED_RANK_BLOCKS_EVICTION 4
typedef struct ksched_rank_input {
  int32_t n_nodes, n_pods;
  const int32_t* pod_offsets;      /* [n_nodes + 1] pods of node n = [pod_offsets[n], pod_offsets[n+1]), in the node's pod-list order */
  const double* pod_deletion_cost; /* [n_pods] controller.kubernetes.io/pod-deletion-cost */
  const int32_t* pod_priority;     /* [n_pods] Spec.Priority */
  const uint8_t* pod_flags;        /* [n_pods] KSCHED_RANK_* */
  const uint8_t* node_eligible;    /* [n_nodes] */
  const double* node_age_seconds;  /* [n_nodes] clock.Since(node.CreationTimestamp) */
  const double* node_ttl_seconds;  /* [n_nodes] provisioner.Spec.TTLSecondsUntilExpired, < 0 = nil */
  const double* node_cost;         /* NULL, or [n_nodes] disruption costs computed elsewhere: only filter + order */
} ksched_rank_input;

typedef struct ksched_timings {
  double upload_us, sort_us, feasibility_us, pack_us, download_us, total_us, allreduce_us;
  int64_t feasibility_bytes; /* P*256 + C*256 + P*C/8 (SURVEY.md 8d) for the last solve */
  int64_t pack_steps;
  int32_t feasibility_launches, pack_launches, sort_launches;
  int32_t pad;
  int64_t h2d_bytes, d2h_bytes; /* host<->device bytes moved by the last ksched_solve (upload + download) */
  double class_feasibility_us;  /* ksched_run_feasibility_only: the per-class row evaluations that precede the dense-matrix kernel */
} ksched_timings;

typedef struct ksched_handle ksched_handle;

int ksched_abi_version(void);
/* number of CUDA devices visible, or a negative error */
int ksched_device_count(void);
/* Bind a handle to one CUDA device. One handle = one stream, single-threaded; handles are independent. */
int ksched_create(int device_ordinal, ksched_handle** out);
void ksched_destroy(ksched_handle* h);
const char* ksched_last_error(const ksched_handle* h);
/* words (uint64) per instance-type bitset for n_types types */
int ksched_type_words(int n_types);

/* Upload the instance-type catalog + templates and build the bit-sliced type tables (amortised across solves). */
int ksched_load_catalog(ksched_handle* h, const ksched_catalog* catalog);
/* Column sharding for multi-GPU feasibility: this handle owns types [begin, end) (SURVEY.md 8e). Default: all. */
int ksched_set_shard(ksched_handle* h, int rank, int world);
/* The [begin, end) range of 32-bit column words rank owns out of n_words32 (pure host arithmetic, no device needed). */
int ksched_shard_range(int n_words32, int rank, int world, int* begin, int* end);
/* NCCL: rank 0 calls ksched_nccl_unique_id, the host distributes the 128 bytes, every rank calls ksched_nccl_init. */
int ksched_nccl_unique_id(void* out128);
int ksched_nccl_init(ksched_handle* h, const void* id128, int rank, int world);
/* One ncclAllGather of `bytes` bytes per rank on the handle's communicator (host buffers; recv holds world * bytes): the
   exchange step of a sharded consolidation pass (each rank's simulation verdicts). Call ksched_set_shard(h, 0, 1) after
   ksched_nccl_init when the communicator is only used for this (no column sharding of the feasibility matrix). */
int ksched_allgather(ksched_handle* h, const void* send, size_t bytes, void* recv);

/* Scheduler.Solve: host buffers in, host buffers out; stream-synchronised before returning. */
int ksched_solve(ksched_handle* h, const ksched_problem* problem, ksched_result* result);

/* Device-resident benchmarking of the same path: upload once, then time kernels only. */
int ksched_upload(ksched_handle* h, const ksched_problem* problem);
int ksched_run_resident(ksched_handle* h, int flush_l2);
int ksched_download(ksched_handle* h, const ksched_problem* problem, ksched_result* result);
int ksched_run_feasibility_only(ksched_handle* h, int flush_l2, float* elapsed_us);

/* Consolidation simulator on a device-resident cluster snapshot: upload once, then any number of simulations. A handle holds
   one snapshot: ksched_upload (and ksched_solve through it) reuses the snapshot's buffers and drops it, after which
   ksched_simulate_batch fails with KSCHED_ERR_INVALID until the next ksched_load_cluster. Keep a snapshot that must survive
   other work on a handle of its own. */
int ksched_load_cluster(ksched_handle* h, const ksched_cluster* cluster);
/* results[n_sets]; node0_types[n_sets][type_words] = surviving InstanceTypeOptions of each simulation's first new node.
   The simulations run back to back on the handle's stream with one synchronisation at the end. */
int ksched_simulate_batch(ksched_handle* h, const ksched_candidate_set* sets, int n_sets, ksched_sim_result* results, uint64_t* node0_types);

/* order[0..*n_candidates) = node indices by ascending disruption cost (ties: input order), cost[i] = cost of order[i]. */
int ksched_rank_candidates(ksched_handle* h, const ksched_rank_input* in, int32_t* order, double* cost, int32_t* n_candidates);

int ksched_get_timings(const ksched_handle* h, ksched_timings* out);

#ifdef __cplusplus
}
#endif
#endif /* KSCHED_H */
