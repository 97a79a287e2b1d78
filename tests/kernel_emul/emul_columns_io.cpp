// TEST-ONLY serial execution of K25 (columns_io.cuh): h2_poly_upload_dev / h2_poly_download_dev's kernel over its whole grid,
// (longest column / 256) x count blocks of 256 threads, blocks visited in reverse so that no column relies on another's order.
#include <cstring>
#include <vector>
#include "columns_io.cuh"
using namespace h2;

template <class P> static void run(int to_dev, int canon, uint64_t count, uint8_t *const *res, uint8_t *const *caller, const uint64_t *lens) {
    std::vector<IoCol> io(count);
    uint64_t longest = 0;
    for (uint64_t c = 0; c < count; c++) {
        io[c] = {(uint64_t)(uintptr_t)caller[c], lens[c]};
        if (lens[c] > longest) longest = lens[c];
    }
    const uint64_t blocks = (longest + 255) / 256;
    for (uint64_t c = count; c-- > 0;)
        for (uint64_t b = blocks; b-- > 0;)
            for (uint64_t t = 0; t < 256; t++) ColumnsIO<P>::body(reinterpret_cast<fe *>(res[c]), io[c], to_dev, canon, b * 256 + t);
}
extern "C" int emu_columns_io(int field, int to_dev, int canon, uint64_t count, uint8_t *const *res, uint8_t *const *caller, const uint64_t *lens) {
    if (field == 0) run<FpParams>(to_dev, canon, count, res, caller, lens);
    else run<FqParams>(to_dev, canon, count, res, caller, lens);
    return 0;
}
// convert_field's per-element conversion (util_kernels.cuh convert_kernel), the one h2_poly_upload / h2_poly_download run:
// n elements in place, to Montgomery form (to_mont) or back
extern "C" int emu_convert(int field, int to_mont, uint64_t n, uint8_t *a) {
    for (uint64_t i = 0; i < n; i++) {
        fe x;
        memcpy(x.v, a + 32 * i, 32);
        if (field == 0) x = to_mont ? fe_to_mont<FpParams>(x) : fe_from_mont<FpParams>(x);
        else x = to_mont ? fe_to_mont<FqParams>(x) : fe_from_mont<FqParams>(x);
        memcpy(a + 32 * i, x.v, 32);
    }
    return 0;
}
