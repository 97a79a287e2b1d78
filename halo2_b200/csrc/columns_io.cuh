// K25: resident polynomials from and to the caller's device memory (h2_poly_upload_dev / h2_poly_download_dev), every
// column of a call in one launch.
//
// The grid covers (column, element): blockIdx.y is the column, the x dimension its elements.  Column c's resident buffer
// comes from the call's column table (col_table, as the batched transforms get theirs), its caller pointer and length
// from the IoCol entries right behind the pointers.  Import reads the caller's element, converts it from `repr` to
// Montgomery form with fe_to_mont -- the conversion h2_poly_upload runs (convert_field) -- and stores it in the
// resident buffer; export is the reverse, fe_from_mont into the caller's buffer.  Montgomery data is a plain copy.
//
// No range check: like h2_poly_upload, every 256-bit input is taken as it is, values >= p and all-ones bytes included, and
// the bytes equal those of the host path for the same 32-byte elements.  fe_load / fe_store move two uint4, so both
// sides must be 16-byte aligned; the entry points refuse other pointers before anything is launched.
#pragma once
#include "field.cuh"

namespace h2 {

struct IoCol {           // one column of a call: the caller's elements and how many of them move
    uint64_t ptr;        // device address of the caller's first element
    uint64_t len;
};

template <class P> struct ColumnsIO {
    // element i of one column; to_dev: caller -> resident, else resident -> caller
    static H2_HD void body(fe *res, const IoCol &io, int to_dev, int canon, uint64_t i) {
        if (i >= io.len) return;
        fe *caller = reinterpret_cast<fe *>(io.ptr);
        if (to_dev) {
            const fe x = fe_load(caller + i);
            fe_store(res + i, canon ? fe_to_mont<P>(x) : x);
        } else {
            const fe x = fe_load(res + i);
            fe_store(caller + i, canon ? fe_from_mont<P>(x) : x);
        }
    }
};

#if defined(__CUDACC__)
// columns [col0, col0 + gridDim.y) of the table; grid.x covers the longest of them
template <class P> __global__ void __launch_bounds__(256) columns_io_kernel(fe *const *res, const IoCol *io, uint32_t col0, int to_dev, int canon) {
    const uint32_t c = col0 + blockIdx.y;
    ColumnsIO<P>::body(res[c], io[c], to_dev, canon, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
#endif

}  // namespace h2
