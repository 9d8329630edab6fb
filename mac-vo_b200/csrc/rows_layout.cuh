// Padded pixel-row layouts of the decoder's tensor-core convolutions (csrc/gru_conv_tc.cu, csrc/conv_tc.cu).
//
// Activations between the decoder's convolutions are fp16 rows of C channels, one row per pixel, stored with zero padding so
// that a convolution tap is a ROW OFFSET and a tile of 128 consecutive rows never needs edge handling:
//
//   layout U ("universal", 2 zero pixels on every side): image b, pixel (y, x) ->
//       row  GUARD + (b (H + 4) + y + 2) (W + 4) + x + 2          tap (dy, dx) -> + dy (W + 4) + dx
//     used by the 3x3 and 1x1 convolutions and by the GRU's 1x5 pass.
//   layout V (the GRU's 5x1 pass: columns are the contiguous lines): image b, pixel (y, x) ->
//       row  GUARD + (b W + x) (H + 4) + y + 2                     tap dy -> + dy
//
// Buffers are allocated zeroed once (macvo_rows_count rows) and the kernels only ever write pixel rows, so the padding stays
// zero. GUARD leading rows keep the first tile's halo inside the allocation.
#pragma once

namespace macvo_rows {

constexpr int GUARD = 2;
constexpr int TILE_M = 128;

__host__ __device__ inline long long urow(int b, int y, int x, int height, int width) {
    return (long long)GUARD + ((long long)b * (height + 4) + y + 2) * (width + 4) + x + 2;
}
__host__ __device__ inline long long vrow(int b, int y, int x, int height, int width) {
    return (long long)GUARD + ((long long)b * width + x) * (height + 4) + y + 2;
}
// padded pixel count (rows between the guards) and allocation size in rows (rounded up to a multiple of 256 rows, + guards)
__host__ __device__ inline int padded_pixels(int batch, int height, int width, int vertical) {
    return vertical ? batch * width * (height + 4) : batch * (height + 4) * (width + 4);
}
__host__ __device__ inline long long alloc_rows(int batch, int height, int width, int vertical) {
    const int pairs = (padded_pixels(batch, height, width, vertical) + 2 * TILE_M - 1) / (2 * TILE_M);
    return (long long)pairs * 2 * TILE_M + 32;
}

}  // namespace macvo_rows
