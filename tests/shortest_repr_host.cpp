// Test-only host build of the device float formatter (v2e_b200/csrc/shortest_repr.cuh): compiled by
// tests/test_sinks_text.py with the system C++ compiler into a temporary directory, never into libv2e_b200.so.
#include <stdint.h>
#include <string.h>

#include "../v2e_b200/csrc/shortest_repr.cuh"

// repr(float(v[i])) + '\n' for every i, concatenated into out (24 + 1 bytes per value at most). Returns the bytes
// written, or -1 - i if value i wrote a different number of bytes than repr_length promised.
extern "C" int64_t repr_lines_f32(const float *v, int64_t n, char *out) {
    int64_t o = 0;
    for (int64_t i = 0; i < n; ++i) {
        const double d = (double)v[i];
        uint64_t bits;
        memcpy(&bits, &d, sizeof bits);
        const v2e_repr::Repr r = v2e_repr::repr_prepare(bits);
        const int32_t len = v2e_repr::repr_length(r);
        if (v2e_repr::repr_write(r, out + o) != len) return -1 - i;
        o += len;
        out[o++] = '\n';
    }
    return o;
}
