// Host check of the block word layout helpers of kivi_decode.cuh against the layout its header comment states:
//   word w of a block: chunk c = w / (128 slabs), slab sl = (w / 128) % slabs, lane = (w % 128) / 4 = 4 g8 + t, r = w % 4;
//   low / high 16 bits, field j: code of (inner 16c + 2t + 8 (r >> 1) + {0, 1}, outer sl * 16F + 16j + g8 + 8 (r & 1)).
// Prints the number of violations (0 = pass).
#include <cstdio>
#include <vector>

#include "../kivi_b200/csrc/kivi_decode.cuh"

using namespace kivi;

int main() {
    long bad = 0;
    for (int bits : {2, 4}) {
        const int F = 16 / bits, slab_rows = 16 * F, slabs = 128 / slab_rows, words = 8 * slabs * 128;
        if (lay_code_bytes(bits) != 4 * words) ++bad;
        std::vector<int> hits(128 * 128, 0);
        for (int w = 0; w < words; ++w) {
            const int c = w / (128 * slabs), sl = (w / 128) % slabs, lane = (w % 128) / 4, r = w % 4;
            const int g8 = lane >> 2, t = lane & 3;
            const int i0 = 16 * c + 2 * t + 8 * (r >> 1), o0 = sl * slab_rows + g8 + 8 * (r & 1);
            const WordPos p = lay_word_pos(bits, w);                       // the inverse
            if (p.i0 != i0 || p.o0 != o0) ++bad;
            for (int par = 0; par < 2; ++par)
                for (int j = 0; j < F; ++j) {
                    const int i = i0 + par, o = o0 + 16 * j;
                    ++hits[i * 128 + o];
                    if (lay_word_off(bits, i, o) != 4 * w || lay_bit_pos(bits, i, o) != 16 * par + bits * j) ++bad;
                    // the two independent parts (the K flush passes slab and row < 16)
                    if (lay_word_inner(bits, i) + lay_word_row(sl, o % 16) != w) ++bad;
                }
        }
        for (int h : hits) bad += h != 1;                                   // every element in exactly one field
        for (int g : {32, 64, 128})
            for (int i0 = 0; i0 < 128; i0 += 2)
                for (int G = 0; G < 128 / g; ++G) {                         // the 8-byte { z, z', s, s' } meta pair
                    const int m = lay_meta_pair_off(bits, g, i0, G);
                    if (m != lay_zero_off(bits, g, i0, G) || m + 2 != lay_zero_off(bits, g, i0 + 1, G) ||
                        m + 4 != lay_scale_off(bits, g, i0, G) || m + 6 != lay_scale_off(bits, g, i0 + 1, G) || m % 8 != 0)
                        ++bad;
                }
    }
    printf("%ld\n", bad);
    return bad != 0;
}
