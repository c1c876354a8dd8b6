// Launch choice for a finished new node (SURVEY section 8f-2): the step right after Scheduler.Solve.
//   instance type: the surviving option whose cheapest compatible AVAILABLE offering is cheapest — the order the fake
//     cloud provider sorts by before it takes element 0 (cloudprovider/fake/cloudprovider.go:74-84); ties keep the
//     provider's input order (canonical rule R4: sort.Slice treated as a stable sort);
//   offering: Offerings.Available().Requirements(reqs).Cheapest() (cloudprovider/types.go:128-145); lo.MinBy keeps the
//     first minimum, i.e. Offerings list order.
// Shared by the device kernel and (host instantiation) the CPU tests of the encoder's offering table.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define KS_LHD __host__ __device__ __forceinline__
#else
#define KS_LHD inline
#endif

namespace ksched {

constexpr uint64_t kNoOffering = ~0ull;

KS_LHD int ctz64(uint64_t m) {
#if defined(__CUDA_ARCH__)
  return __ffsll((long long)m) - 1;
#else
  return __builtin_ctzll(m);
#endif
}

// Offering slot tables (ksched.h: ksched_catalog.zone_slots / ct_slots) of the ct*16 + zone layout: zone z < 16 owns the
// slots ct*16 + z, capacity type c < 4 the slots c*16 + z.
KS_LHD void formula_slot_tables(uint64_t* zone_slots, uint64_t* ct_slots) {
  for (int v = 0; v < 64; ++v) {
    zone_slots[v] = v < 16 ? 0x0001000100010001ull << v : 0;
    ct_slots[v] = v < 4 ? 0xFFFFull << (16 * v) : 0;
  }
}

// Union of the slots of `values` in one table (value -> its slots); used = values that own a slot, all = every slot. Every
// slot belongs to exactly one value, so a set that takes in every used value owns every slot.
KS_LHD uint64_t slot_union(const uint64_t* table, uint64_t used, uint64_t all, uint64_t values) {
  values &= used;
  if (values == used) return all;
  uint64_t s = 0;
  for (; values; values &= values - 1) s |= table[ctz64(values)];
  return s;
}

// The slots whose zone is one of `zones` and whose capacity type is one of `cts` (dictionary value bits): the offerings a
// node's zone / capacity-type requirements admit (Offerings.Requirements, types.go:120-126). tables = zone_slots[64] then
// ct_slots[64].
KS_LHD uint64_t admitted_slots(const uint64_t* tables, uint64_t zone_used, uint64_t ct_used, uint64_t all, uint64_t zones, uint64_t cts) {
  return slot_union(tables, zone_used, all, zones) & slot_union(tables + 64, ct_used, all, cts);
}

// min over the admitted offering slots; keys64 = the type's 64 table entries
KS_LHD uint64_t offering_min_key(const uint64_t* keys64, uint64_t slots) {
  uint64_t best = kNoOffering;
  for (; slots; slots &= slots - 1) {
    const uint64_t k = keys64[ctz64(slots)];
    best = k < best ? k : best;
  }
  return best;
}
// ordering key of an option: (price rank of its cheapest compatible offering, provider input order)
KS_LHD uint64_t option_key(uint64_t offering_key, uint32_t input_index) { return ((offering_key >> 16) << 32) | input_index; }

}  // namespace ksched
