/* The reference's Assembly (plonk/permutation/keygen.rs:24-100) restated in C: TEST INFRASTRUCTURE ONLY, like
 * halo2_oracle.c.  Built on its own by oracle/assembly.py into oracle/_build/libassembly_oracle.so. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

/* ---------------------------------------------------------------- Assembly::new + Assembly::copy (plonk/permutation/keygen.rs:24-100)
 * The reference's sequential copy loop over m copies (four uint32 each: left column, left row, right column, right row, in
 * synthesis order) on cols permutation columns of 2^k rows; a cell (c, r) is the flat index c * 2^k + r.  out_mapping:
 * cols * 2^k (column, row) pairs, the final `mapping`.  Returns 0, or 1 (a column outside the permutation,
 * Error::ColumnNotInPermutation) / 2 (a row outside the domain, Error::BoundsFailure) with *bad = the index of the first
 * bad copy; out_mapping is then not written.  Used as the oracle of the device assembly and as its timed CPU baseline. */
int orc_assembly(const uint32_t *copies, size_t m, uint32_t cols, uint32_t k, uint32_t *out_mapping, size_t *bad) {
    const uint64_t n = 1ull << k, N = (uint64_t)cols << k;
    uint32_t *mapping = (uint32_t *)malloc(sizeof(uint32_t) * (N ? N : 1)), *aux = (uint32_t *)malloc(sizeof(uint32_t) * (N ? N : 1));
    uint32_t *sizes = (uint32_t *)malloc(sizeof(uint32_t) * (N ? N : 1));
    for (uint64_t v = 0; v < N; v++) { mapping[v] = aux[v] = (uint32_t)v; sizes[v] = 1; }              /* :25-43 */
    int rc = 0;
    for (size_t i = 0; i < m && !rc; i++) {
        const uint32_t *c = copies + 4 * i;
        if (c[0] >= cols || c[2] >= cols) { rc = 1; *bad = i; break; }                                     /* :51-60 */
        if (c[1] >= n || c[3] >= n) { rc = 2; *bad = i; break; }                                           /* :63-67 */
        const uint32_t left = (uint32_t)(c[0] * n + c[1]), right = (uint32_t)(c[2] * n + c[3]);
        uint32_t lc = aux[left], rcy = aux[right];
        if (lc == rcy) continue;                                                                            /* :71-77 */
        if (sizes[lc] < sizes[rcy]) { uint32_t t = lc; lc = rcy; rcy = t; }                                  /* :79-81 */
        sizes[lc] += sizes[rcy];                                                                            /* :84 */
        uint32_t j = rcy;
        do { aux[j] = lc; j = mapping[j]; } while (j != rcy);                                               /* :85-92 */
        const uint32_t t = mapping[left]; mapping[left] = mapping[right]; mapping[right] = t;              /* :94-96 */
    }
    if (!rc)
        for (uint64_t v = 0; v < N; v++) { out_mapping[2 * v] = (uint32_t)(mapping[v] >> k); out_mapping[2 * v + 1] = (uint32_t)(mapping[v] & (n - 1)); }
    free(mapping); free(aux); free(sizes);
    return rc;
}
