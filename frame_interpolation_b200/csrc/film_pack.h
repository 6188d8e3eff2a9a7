// Weight layout of the persistent 3x3 kernel (film_conv3x3_tc.cu) for a source whose 64-channel chunks hold data in
// their first 16-channel k-step only (the fusion side tensor: 10 of 64 channels).  The kernel issues k-step 0 alone of
// each of that source's nine taps, so a [cout x 64] K block per tap would carry 48 channels of zeros.  Instead each
// chunk gets one K block per dx column: the three dy taps' 16-channel slices at K offsets 0 / 16 / 32, zeros in the
// fourth k-step -- 3 blocks per chunk instead of 9, with the same issued k-steps.  Host code only (no CUDA), so the
// layout can be checked without a GPU.
#pragma once
#include <stdint.h>

#include <vector>

namespace film {

// per_tap: [cout][ktot], K order (source, chunk, tap, channel) with nine dx-major taps (t = 3 dx + dy) and `chunk`
// channels per block.  Sources with packed[s] != 0 are repacked as above (chunk must be 64); the others are copied.
// Returns [cout][ktot_out].
inline std::vector<uint16_t> pack_dx_blocks(const std::vector<uint16_t>& per_tap, int cout, int ktot, int chunk,
                                            const std::vector<int>& src_chunks, const std::vector<int>& packed,
                                            int& ktot_out) {
  ktot_out = ktot;
  for (size_t s = 0; s < src_chunks.size(); ++s)
    if (packed[s]) ktot_out -= src_chunks[s] * 6 * chunk;
  std::vector<uint16_t> out((size_t)cout * ktot_out, 0);
  for (int n = 0; n < cout; ++n) {
    const uint16_t* src = per_tap.data() + (size_t)n * ktot;
    uint16_t* dst = out.data() + (size_t)n * ktot_out;
    for (size_t s = 0; s < src_chunks.size(); ++s)
      for (int ch = 0; ch < src_chunks[s]; ++ch, src += 9 * chunk) {
        if (!packed[s]) {
          for (int k = 0; k < 9 * chunk; ++k) *dst++ = src[k];
          continue;
        }
        for (int t = 0; t < 9; ++t)
          for (int c = 0; c < 16; ++c) dst[(t / 3) * chunk + (t % 3) * 16 + c] = src[t * chunk + c];
        dst += 3 * chunk;
      }
  }
  return out;
}

// Weight layout of the folded Cout = 32 pixels-on-N form of the persistent 3x3 kernel: one M = 64 operand holds two dy
// taps of one dx column.  per_tap: [32][ktot] in the K order above.  Each (chunk, dx) gets two [64 x chunk] K blocks:
// rows 0-31 tap dy = -1 and rows 32-63 tap dy = 0, then zero rows 0-31 and rows 32-63 tap dy = +1 (the kernel reads it
// at the dy = 0 box offset, so its 17 tile rows stay inside the box).  Returns [64][ktot * 2 / 3].
inline std::vector<uint16_t> pack_dy_pairs(const std::vector<uint16_t>& per_tap, int ktot, int chunk) {
  const int ktot_out = ktot / 9 * 6;
  std::vector<uint16_t> out((size_t)64 * ktot_out, 0);
  for (int g = 0; g < ktot / (9 * chunk); ++g)
    for (int dx = 0; dx < 3; ++dx)
      for (int n = 0; n < 32; ++n)
        for (int c = 0; c < chunk; ++c) {
          const uint16_t* src = per_tap.data() + (size_t)n * ktot + (size_t)(g * 9 + 3 * dx) * chunk + c;
          uint16_t* dst = out.data() + (size_t)(g * 6 + 2 * dx) * chunk + c;
          dst[(size_t)n * ktot_out] = src[0];                                // dy = -1
          dst[(size_t)(32 + n) * ktot_out] = src[chunk];                     // dy = 0
          dst[(size_t)(32 + n) * ktot_out + chunk] = src[2 * chunk];         // dy = +1
        }
  return out;
}

}  // namespace film
