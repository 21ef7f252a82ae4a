// Host build of the exact accumulator (redner_b200/csrc/rb_exact.cuh) for tests/test_exact_sum_cpu.py.
// Reads lines "<normalise_every> <n> <bits> ... <bits>" (float bit patterns in hex), adds the n floats into one accumulator in the
// given order (normalising after every normalise_every adds, 0: never) and prints "<float bits> <double bits>" of the rounded sum.
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "../redner_b200/csrc/rb_exact.cuh"

int main() {
    long long every, n;
    while (scanf("%lld %lld", &every, &n) == 2) {
        long long acc[RB_EXACT_WORDS] = {0};
        for (long long i = 0; i < n; i++) {
            unsigned u;
            if (scanf("%x", &u) != 1) return 1;
            exact_add_serial(acc, exact_float(u));
            if (every > 0 && (i + 1) % every == 0) exact_normalise(acc);
        }
        const double d = exact_to_double(acc);
        unsigned long long db;
        memcpy(&db, &d, 8);
        printf("%08x %016llx\n", exact_bits(exact_to_float(acc)), db);
    }
    return 0;
}
