// catalog.cuh - device view of the catalog (bit-sliced column tables) and the helpers every kernel shares.
// Part of the single translation unit ksched.cu (included inside its anonymous namespace, in this order: catalog.cuh,
// feasibility_kernel.cuh, topology.cuh, pack_kernel.cuh); not a standalone header.
#pragma once

// ------------------------------------------------------------------------------------------------
// Device-side catalog: instance-type columns as bit-sliced tables (one bit per column, u32 words).
// ------------------------------------------------------------------------------------------------
struct DevCatalog {
  int n_keys, n_res, n_types, n_templates, W32;
  const ksched_keyinfo* keys;        // [n_keys]
  const int64_t* key_int_values;     // [n_keys][64]
  const ksched_key_regions* key_regions;  // [n_keys] or nullptr: region form of Gt/Lt (ksched.h); keys[k].dict_mask includes the region bits
  const ksched_template* templates;  // [n_templates]
  const ksched_type_row* types;      // [n_types]
  const int64_t* capacity;           // [n_types][8]
  const float* price32;              // [n_types]
  const int16_t* valrow;             // [n_keys*64] row in valset or -1
  const uint32_t* valset;            // [rows][W32] type has a positive requirement on key containing value
  const uint32_t* absent;            // [n_keys][W32] type has no requirement on key
  const uint32_t* negempty;          // [n_keys][W32] type requirement on key is DoesNotExist
  uint32_t type_relevant;            // bit k: some type defines key k
  const int16_t* offrow;             // [64] row in offset table or -1
  const uint32_t* offset;            // [rows][W32] type has an available offering in the row's slot
  const uint32_t* anyoffer;          // [W32]
  const uint64_t* slots;             // [128] zone value -> its offering slots, then capacity-type value -> its slots (ksched.h)
  uint64_t zone_used, ct_used;       // zone / capacity-type values that own a slot
  uint64_t all_slots;                // every slot of the tables
  uint64_t offer_used;               // slots with an offset row
  const uint32_t* member;            // [n_templates][W32]
  const int64_t* alloc_sorted;       // [n_res][n_types] ascending
  const uint32_t* fitset;            // [n_res][n_types+1][W32]  rank -> types with alloc >= alloc_sorted[rank]
  const int32_t* perm_desc;          // [n_res][n_types] types by descending allocatable
  const int64_t* alloc_rt;           // [n_res][n_types] allocatable, resource-major
  const uint32_t* domset;            // [n_types][W32] types whose allocatable vector (first 4 resources) is dominated by the row's type
  int zone_key, ct_key;
  // bit d of pin_neutral[k]: narrowing a node's requirement on key k to the single value d can never remove an instance type
  // of any template (every member type admits d on k, and - for the zone / capacity-type keys - has an available offering
  // for d combined with every value of the other key). Built by ksched_load_catalog; lets the pack kernel's class-run loop
  // accept a topology-spread placement that pins a node's domain without re-filtering its options.
  uint64_t pin_neutral[KSCHED_MAX_KEYS];
  const uint64_t* offer_keys;        // [n_types][64] launch-choice keys (ksched_catalog.offering_keys) or nullptr
  const uint32_t* input_index;       // [n_types] provider input order of the column
  int n_res_ext;                     // ext resources (ksched.h: ksched_catalog.n_res_ext), 0 = none
  const int64_t* alloc_ext;          // [n_types][n_res_ext] or nullptr
};

// Fits (resources.go:138-145) on the ext resources: the types of column word w of `word` whose allocatable holds
// node[x] + pod[x] for every ext resource x of `present` (node: the node's ext sums, nullptr for a fresh node; an allocatable
// the type lacks counts as 0). Only classes that request an ext resource call it, so a per-type loop is enough; out of line,
// so that the pack kernel's paths for other classes keep their code size.
__device__ __noinline__ uint32_t ext_fit_word(const DevCatalog& c, const int64_t* node, const int64_t* pod, uint32_t present, uint32_t word, int w) {
  uint32_t out = word;
  for (uint32_t m = word; m; m &= m - 1) {
    const int b = __ffs(m) - 1;
    const int64_t* a = c.alloc_ext + (size_t)(w * 32 + b) * c.n_res_ext;
    for (uint32_t p = present; p; p &= p - 1) {
      const int x = __ffs(p) - 1;
      if ((node ? node[x] : 0) + pod[x] > a[x]) { out &= ~(1u << b); break; }
    }
  }
  return out;
}

__device__ __forceinline__ KeyMeta key_meta(const DevCatalog& c, int k) {
  return KeyMeta{c.keys[k].int_mask, c.key_int_values ? c.key_int_values + (size_t)k * 64 : nullptr, c.key_regions ? c.key_regions + k : nullptr};
}

// number of types with alloc_r < q  (lower bound)
__device__ __forceinline__ int fit_rank(const int64_t* alloc_sorted, int n_types, int r, int64_t q) {
  const int64_t* a = alloc_sorted + (size_t)r * n_types;
  int lo = 0, hi = n_types;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] < q) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Column set {t : instanceType.Requirements.Intersects(node) holds on key k} for one u32 word
// (requirements.go:189-206 with the type as receiver). `allowed` = dictionary values the node requirement
// admits, `neg` = its operator is NotIn/DoesNotExist.
__device__ __forceinline__ uint32_t key_typeset_word(const DevCatalog& c, int k, uint64_t allowed, bool neg, int w) {
  uint32_t s = c.absent[(size_t)k * c.W32 + w];
  if (neg) s |= c.negempty[(size_t)k * c.W32 + w];
  uint64_t m = allowed;
  while (m) {
    int b = __ffsll((long long)m) - 1;
    m &= m - 1;
    int row = c.valrow[k * 64 + b];
    if (row >= 0) s |= c.valset[(size_t)row * c.W32 + w];
  }
  return s;
}
// hasOffering (node.go:151-159) for one word: slots = the offering slots the node's zone / capacity-type requirements admit
// (ksched::admitted_slots)
__device__ __forceinline__ uint32_t offer_word(const DevCatalog& c, uint64_t slots, bool unconstrained, int w) {
  if (unconstrained) return c.anyoffer[w];
  uint32_t s = 0;
  for (uint64_t m = slots & c.offer_used; m; m &= m - 1) s |= c.offset[(size_t)c.offrow[__ffsll((long long)m) - 1] * c.W32 + w];
  return s;
}
// admitted offering slots of a node from its zone / capacity-type allowed value bits
__device__ __forceinline__ uint64_t node_slots(const DevCatalog& c, uint64_t zallowed, uint64_t callowed) {
  return ksched::admitted_slots(c.slots, c.zone_used, c.ct_used, c.all_slots, zallowed, callowed);
}

