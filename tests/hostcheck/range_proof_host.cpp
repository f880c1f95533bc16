// Test-only: compiles the DEVICE per-range rules of the range-proof check (phant_b200/csrc/range_proof.cuh) as HOST code, so
// that the exact statements the GPU runs per entry and per proof item can be compared with tests/range_proof_oracle.py on a
// machine without a GPU.  Built as a shared object by tests/test_range_proof_header_host.py; nothing in the product links or
// loads this.
#include <stdint.h>
#define __device__
#define __forceinline__ inline
#include "../../phant_b200/csrc/range_proof.cuh"

using namespace phant;

// entries (n x 32 keys, n + 1 value offsets) of one range: 1 when every entry passes the entry checks
extern "C" int hr_entries_ok(const uint8_t* keys, const uint64_t* val_off, uint32_t n, const uint8_t* origin, int whole)
{
    for (uint32_t i = 0; i < n; ++i)
        if (!rp_entry_ok(keys + 32ull * i, i ? keys + 32ull * (i - 1) : nullptr, origin, whole != 0, val_off[i + 1] - val_off[i])) return 0;
    return 1;
}
extern "C" void hr_last(const uint8_t* last_entry, uint8_t* out) { rp_last(last_entry, out); }
// bit 0: inside [origin, last]; bit 1: above last
extern "C" int hr_classify(const uint8_t* key, uint32_t depth, const uint8_t* origin, const uint8_t* last)
{
    return (rp_inside(key, depth, origin, last) ? 1 : 0) | (rp_above(key, last) ? 2 : 0);
}
