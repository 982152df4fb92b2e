// Host run of kb_device.cuh's mix32 (__host__ __device__), for tests/test_hash_mirror_cpu.py: one decimal u32 per line on stdin, its
// mix32 per line on stdout. Needs no device.
#include <cstdio>

#include "../../kolibrie_b200/csrc/kb_device.cuh"

int main() {
    unsigned long long v;
    while (scanf("%llu", &v) == 1) printf("%u\n", kb::mix32((kb::u32)v));
    return 0;
}
