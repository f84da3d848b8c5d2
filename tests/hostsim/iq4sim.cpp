// iq4sim.cpp — TEST INFRASTRUCTURE.  Compiles llama-box_b200/csrc/mmq_wide32.cuh — the stage load and unpack the int8 tile kernel
// (mmq_tc32.cu) runs for IQ4_NL / IQ4_XS weights, and the q8_K arithmetic of its IQ4_XS activation image — with the host compiler, so
// tests/test_mmq_iq4_hostsim.py checks them against the C oracle on the CPU.  Not linked into any product library.
//
// Built as a shared library for the comparisons, and with -DIQ4SIM_MAIN (under AddressSanitizer) as a program that unpacks every stage of
// rows held in allocations of exactly the row's size, so a load past the row's last byte is reported.
#include "../../llama-box_b200/csrc/mmq_wide32.cuh"

#include <stdio.h>
#include <stdlib.h>

long xf_misaligned = 0;

extern "C" {
// every stage of one native row (k % 256 == 0): q[k] int8 in element order, sc[k / 32] the per-block scale word; returns the count of
// misaligned loads (0)
long sim_iq4_unpack_row(int type, const uint8_t * row, int64_t k, int8_t * q, uint32_t * sc) {
    xf_misaligned = 0;
    for (int64_t s = 0; s < k / 128; s++) {
        uint32_t w[18], qq[8];
        if (type == XF_IQ4_NL) w32_load<XF_IQ4_NL>(row, s, w); else w32_load<XF_IQ4_XS>(row, s, w);
        for (int b = 0; b < 4; b++) {
            sc[4 * s + b] = type == XF_IQ4_NL ? w32_unpack<XF_IQ4_NL>(w, s, b, qq) : w32_unpack<XF_IQ4_XS>(w, s, b, qq);
            memcpy(q + 128 * s + 32 * b, qq, 32);
        }
    }
    return xf_misaligned;
}

// one column quantised to q8_K the way the tile kernel's IQ4_XS quantiser does it: per super-block the first element of largest |x|
// (the warp's reduction), then w32_q8k_quant8 on each run of 8 elements.  q[k] int8, d[k / 256]
void sim_q8k_column(const float * x, int64_t k, int8_t * q, float * d) {
    for (int64_t sb = 0; sb < k / 256; sb++) {
        const float * xs = x + 256 * sb;
        float am = 0.0f; int ai = 0;
        for (int j = 0; j < 256; j++) { const float a = fabsf(xs[j]); if (a > am) { am = a; ai = j; } }
        for (int l = 0; l < 32; l++) {
            float v[8]; uint32_t lo, hi;
            for (int j = 0; j < 8; j++) v[j] = xs[8 * l + j];
            d[sb] = w32_q8k_quant8(v, xs[ai], am, lo, hi);
            memcpy(q + 256 * sb + 8 * l, &lo, 4); memcpy(q + 256 * sb + 8 * l + 4, &hi, 4);
        }
    }
}
}

#ifdef IQ4SIM_MAIN
// iq4sim <type> <k> <rows> <seed>: random rows, each copied into a malloc of exactly its size, every stage unpacked
int main(int argc, char ** argv) {
    if (argc != 5) return 2;
    const int type = atoi(argv[1]); const int64_t k = atoll(argv[2]); const int rows = atoi(argv[3]);
    srand((unsigned)atoi(argv[4]));
    const int64_t rb = type == XF_IQ4_NL ? k / 32 * 18 : k / 256 * 136;
    int8_t * q = (int8_t *)malloc(k); uint32_t * sc = (uint32_t *)malloc(k / 32 * 4);
    long sum = 0, mis = 0;
    for (int r = 0; r < rows; r++) {
        uint8_t * row = (uint8_t *)aligned_alloc(8, (size_t)rb);        // rb is a multiple of 8: no slack after the row
        for (int64_t i = 0; i < rb; i++) row[i] = (uint8_t)rand();
        mis += sim_iq4_unpack_row(type, row, k, q, sc);
        for (int64_t i = 0; i < k; i++) sum += q[i];
        free(row);
    }
    printf("ok rows %d k %lld misaligned %ld checksum %ld\n", rows, (long long)k, mis, sum);
    free(q); free(sc);
    return mis != 0;
}
#endif
