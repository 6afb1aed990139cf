// lookup.cuh -- K15's string table view and probe, shared by lookup.cu (StringLookup) and text.cu (K16: TextVectorization
// looks its tokens up in the table of its inner StringLookup).
//
// The probe of a string b[0, len): SipHash-2-4 of the bytes under the table's key (siphash.cuh) is both the home slot
// (masked to cap - 1) and the fingerprint; linear probing from there compares the fingerprint, then the length, then the
// bytes.  lookup.cu owns the key (LK_K0 / LK_K1) and the slot rule.
#pragma once
#include "common.cuh"
#include "siphash.cuh"

namespace tfrs {

struct LkTable {
  int* slots;
  unsigned long long cmask;             // cap - 1
  const long long* keys;                // I64 keys [V]
  const uint8_t* bytes;                 // BYTES keys
  const long long* offsets;             // BYTES offsets [V + 1]
  unsigned long long* fp;               // BYTES fingerprints [V]
  long long V;
  int has_mask;
  long long mask;                       // I64 mask value
  const uint8_t* mask_bytes;            // BYTES mask token
  long long mask_len;
};

__device__ __forceinline__ bool lk_bytes_equal(const uint8_t* a, const uint8_t* b, long long n) {
  for (long long k = 0; k < n; ++k)
    if (a[k] != b[k]) return false;
  return true;
}

__device__ __forceinline__ uint64_t lk_fingerprint(const uint8_t* b, long long len, uint64_t k0, uint64_t k1) {
  const uint8_t* p = nullptr;
  Msg m;
  bytes_msg(m, b, len, &p);
  return siphash(m, p, k0, k1);
}

// Probes a BYTES table for the string b[0, len): hit(p) for vocabulary position p, or miss() when it is not there.
template <typename Hit, typename Miss>
__device__ __forceinline__ void lk_probe_bytes(const LkTable& t, const uint8_t* b, long long len, uint64_t k0, uint64_t k1,
                                               Hit hit, Miss miss) {
  const unsigned long long h = lk_fingerprint(b, len, k0, k1);
  unsigned long long s = h & t.cmask;
  for (;;) {
    const int p = __ldg(t.slots + s);
    if (p < 0) {
      miss();
      break;
    }
    if (__ldg(t.fp + p) == h) {
      const long long c0 = __ldg(t.offsets + p);
      if (__ldg(t.offsets + p + 1) - c0 == len && lk_bytes_equal(t.bytes + c0, b, len)) { hit(p); break; }
    }
    s = (s + 1) & t.cmask;
  }
}

// lookup.cu: the device view of a table descriptor (checked; TFRS_ERR_INVALID_ARG with the error text on a bad one), and
// the SipHash key of string tables.
int lk_table(const tfrs_lookup_table* d, LkTable* t, const char* what);
extern const uint64_t lk_string_key[2];

}  // namespace tfrs
