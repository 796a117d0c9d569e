// Receiver coverage stage of the batch decoder (decoder option "coverage", DESIGN.md §8): the greatest range heard in
// every 5-degree bearing sector, for each of nine altitude bands - az_map_model (python/az_map.py:35-82) fed as
// az_map_output.output (az_map.py:187-202) feeds it, kept on the device across calls.
//
//   amb_coverage_kernel  one thread per record: a counted record does one shared atomicMax with the IEEE bits of its
//                        range on its own (row, col) cell of the block's grid; after the barrier one thread per cell
//                        takes the running maximum over bands 0..col of its row (rule 4: every band from col up) and
//                        issues one global atomicMax when it is non-zero.
//
// Non-negative finite doubles order like their bit patterns as unsigned integers, and a counted range is > 0, so the
// maxima are exact and do not depend on the order of the records or on how the stream is cut into calls.
#pragma once

#include <string.h>

#define AMB_COVERAGE_CELLS (AMB_COVERAGE_ROWS * AMB_COVERAGE_BANDS)

// The cell row * AMB_COVERAGE_BANDS + col a record updates (include/airmodes_b200.h rules 1-3), and the bits of its
// range in *bits; -1 for a record that does not count or whose range is not > 0 (rule 4 then changes nothing).
AMB_HD int amb_coverage_cell(const amb_fields& r, unsigned long long* bits)
{
    if (r.status & (AMB_FS_NOT_QUEUED | AMB_FS_NO_HANDLER)) return -1;
    if (r.df != 17 || (r.bds != 0x05 && r.bds != 0x06) || !(r.status & AMB_FS_HAS_RANGE)) return -1;
    const double range = r.range;
    if (!(range > 0.0)) return -1;
    const int alt = r.bds == 0x06 ? 0 : r.altitude;               // az_map.py:196 / parseBDS05's decode_alt(alt, False)
    const int bands[AMB_COVERAGE_BANDS] = AMB_COVERAGE_ALTITUDES;
    int col = 0;                                                   // az_map.py:60-63: the first band >= alt, else the last
    while (col < AMB_COVERAGE_BANDS - 1 && alt > bands[col]) col++;
    const long long t = (long long)(r.bearing + 2.5);              // az_map.py:66 with npoints = 72: the double sum,
    const int row = (int)(t / 5 % AMB_COVERAGE_ROWS);              // truncated, then divided as an integer
    memcpy(bits, &range, sizeof range);
    return row * AMB_COVERAGE_BANDS + col;
}

__global__ void __launch_bounds__(256) amb_coverage_kernel(const amb_fields* __restrict__ fields, int n,
                                                           unsigned long long* __restrict__ grid)
{
    __shared__ unsigned long long s[AMB_COVERAGE_CELLS];
    for (int i = threadIdx.x; i < AMB_COVERAGE_CELLS; i += blockDim.x) s[i] = 0ull;
    __syncthreads();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) {
        unsigned long long bits;
        const int cell = amb_coverage_cell(fields[k], &bits);
        if (cell >= 0) atomicMax(&s[cell], bits);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < AMB_COVERAGE_CELLS; i += blockDim.x) {
        const int row0 = i - i % AMB_COVERAGE_BANDS;
        unsigned long long m = 0ull;
        for (int j = row0; j <= i; j++) m = s[j] > m ? s[j] : m;
        if (m) atomicMax(&grid[i], m);
    }
}

// Enqueue the stage for the n records on stream s: one launch. Returns 1, or -1 with *err set.
static int amb_coverage_launch(const amb_fields* fields, int n, unsigned long long* grid, cudaStream_t s, cudaError_t* err)
{
    AMB_LAUNCH((amb_coverage_kernel), (n + 255) / 256, 256, 0, s, fields, n, grid);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 1 : -1;
}
