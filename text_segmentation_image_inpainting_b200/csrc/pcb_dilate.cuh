// pcb_dilate.cuh -- cv2.dilate(mask, np.ones((10, 10))) of one T x T output tile in shared memory, shared by the inpainting
// data path (inpaint_data.cu) and the text-removal holes (text_removal.cu).
//
// cv2's anchor of an even 10 x 10 kernel is (5, 5): output pixel (y, x) is the max over rows y-5 .. y+4 and columns x-5 .. x+4.
// Pixels outside the image do not take part (cv2's default border for dilate), so the caller loads them as 0.  The tile is
// held with that halo: `hole[ly][lx]` is image pixel (y0 - 5 + ly, x0 - 5 + lx); the max is separable, a 10-wide row max
// into `rmax`, then a 10-high column max per output pixel.
#pragma once
#include <stdint.h>

namespace dil {

constexpr int BEFORE = 5;          // halo rows / columns before the tile
constexpr int AFTER = 4;           // and after it

template <int T>
struct Tile {
    static constexpr int HT = T + BEFORE + AFTER;
    uint8_t hole[HT][HT];          // the thresholded mask over tile + halo, 0 / 1
    uint8_t rmax[HT][T];           // its 10-wide row max
};

// rmax[ly][lx] = max(hole[ly][lx .. lx + 9]) for the whole tile; the caller syncs before and after
template <int T>
__device__ __forceinline__ void row_max(Tile<T> &t, int tid, int nthreads) {
    for (int q = tid; q < Tile<T>::HT * T; q += nthreads) {
        const int ly = q / T, lx = q - ly * T;
        uint8_t m = 0;
#pragma unroll
        for (int d = 0; d < BEFORE + AFTER + 1; ++d) m |= t.hole[ly][lx + d];
        t.rmax[ly][lx] = m;
    }
}

// the dilated value of tile pixel (ly, lx): max(rmax[ly .. ly + 9][lx])
template <int T>
__device__ __forceinline__ uint8_t col_max(const Tile<T> &t, int ly, int lx) {
    uint8_t m = 0;
#pragma unroll
    for (int d = 0; d < BEFORE + AFTER + 1; ++d) m |= t.rmax[ly + d][lx];
    return m;
}

}  // namespace dil
