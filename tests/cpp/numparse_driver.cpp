// Host build of kolibrie_b200/csrc/kb_numparse.cuh (the parse the device numeric side table runs), for tests/test_numparse_cpu.py.
// stdin: u64 n, then n times (u64 len, len bytes). stdout: n records of (u32 route, u64 f64 bits, u32 is_i32, i32 value); the bits of a
// NUM_SLOW string are those slow_f64 computes, as kb_dict_numeric_derive's second kernel does.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kb_numparse.cuh"

static const kb_np::Tables kTables = {
    {
#include "kb_pow5.inc"
    },
    KB_NP_POW10_INIT,
    KB_NP_IPOW10_INIT,
};

template <class T> static bool get(T* v) { return fread(v, sizeof(T), 1, stdin) == 1; }

int main() {
    uint64_t n = 0;
    if (!get(&n)) return 2;
    std::vector<uint8_t> buf;
    static kb_np::Decimal dec;
    for (uint64_t k = 0; k < n; k++) {
        uint64_t len = 0;
        if (!get(&len)) return 2;
        buf.resize(len + 1);
        if (len && fread(buf.data(), 1, len, stdin) != len) return 2;
        uint64_t bits = 0;
        const uint32_t route = kb_np::parse_f64(buf.data(), len, &kTables, &bits);
        if (route == kb_np::NUM_SLOW) bits = kb_np::slow_f64(buf.data(), len, &dec);
        int32_t v = 0;
        const uint32_t ok = kb_np::parse_i32(buf.data(), len, &v) ? 1u : 0u;
        fwrite(&route, 4, 1, stdout);
        fwrite(&bits, 8, 1, stdout);
        fwrite(&ok, 4, 1, stdout);
        fwrite(&v, 4, 1, stdout);
    }
    return 0;
}
