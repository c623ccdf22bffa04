// kj_emu_format.cpp -- TEST INFRASTRUCTURE ONLY: the output-line code of kj_classify_files (kaiju_b200/csrc/kj_format.h) compiled for the CPU.
// Compiled by tests/test_format_lines.py.
#include <stdio.h>
#include <stdlib.h>
#include "../../kaiju_b200/csrc/kj_format.h"

extern "C" {
// The lines of reads [0, n) into out: the length pass (lens[r]), then the write pass by a group of nl lanes run one after another (nl = 32:
// the lane-strided copy of kj_fmt_write's warp).  Returns the bytes written; aborts if a lane's length disagrees with the length pass.
uint64_t kjfmt_lines(const KjFmtIn* in, uint64_t n, uint32_t nl, char* out, uint32_t* lens) {
    uint64_t pos = 0;
    for (uint64_t r = 0; r < n; r++) {
        const uint32_t len = kj_fmt_line(*in, r, nullptr, 0, 1); lens[r] = len;
        for (uint32_t lane = 0; lane < nl; lane++) if (kj_fmt_line(*in, r, out + pos, lane, nl) != len) { fprintf(stderr, "kjfmt: lane length differs\n"); abort(); }
        pos += len;
    }
    return pos;
}
int kjfmt_status(const KjFmtIn* in, uint64_t r) { return kj_fmt_status(*in, r); }
uint32_t kjfmt_self_score(uint32_t c) { return kj_fmt_self_score(c); }
}
