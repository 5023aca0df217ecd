// Exhaustive check of the runtime-constant exact division used by spatial_tap_uv (bevy_hikari_b200/csrc/hk_spatial_taps.cuh):
//     q = x * y;  r = fma(-q, C, x);  result = fma(r, y, q)      with y = RN(1 / C) computed once on the host
// against IEEE x / C for EVERY float x (all 2^32 bit patterns) and a list of image extents C.
// build: g++ -O2 -march=x86-64-v3 -ffp-contract=off -fopenmp tools/check_runtime_division.cpp -o /tmp/divcheck/check
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

int main(int argc, char** argv) {
    int failures = 0;
    for (int a = 1; a < argc; ++a) {
        const float C = (float)atoi(argv[a]);
        const float y = 1.0f / C;
        unsigned long long bad = 0, bad_normal = 0;
#pragma omp parallel for reduction(+ : bad, bad_normal) schedule(static)
        for (long long i = 0; i < (1ll << 32); ++i) {
            uint32_t u = (uint32_t)i;
            float x;
            memcpy(&x, &u, 4);
            if (x != x) continue;
            float q = x * y;
            float r = fmaf(-q, C, x);
            float fast = fmaf(r, y, q);
            float exact = x / C;
            uint32_t fb, eb;
            memcpy(&fb, &fast, 4);
            memcpy(&eb, &exact, 4);
            if (fb != eb && !(fast != fast && exact != exact)) {
                bad += 1;
                if (fabsf(exact) >= 1.17549435e-38f && fabsf(x) < 3.0e38f) bad_normal += 1;
            }
        }
        printf("C = %6d: %llu of 2^32 inputs differ (%llu with a normal quotient and finite x)\n", (int)C, bad, bad_normal);
        failures += bad_normal != 0;
    }
    return failures;
}
