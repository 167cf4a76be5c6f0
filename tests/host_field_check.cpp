// Host path of renegade_b200/csrc/ff.cuh (the #else branches: 64-bit CIOS fe_mul, fe_add, fe_sub, and fe_sqr /
// fe_mul_add2 / fe_mul_sub2 built on them), run over operands chosen by tests/test_host_field_cpu.py, which checks the
// results against Python integers.  This path runs every MSM's host Horner and affine normalisation and the transcript.
//   host_field_check FIELD IN OUT    FIELD 0 = Fr, 1 = Fq
// IN holds n (uint64) then the n a's and the n b's (32-byte little-endian Montgomery residues).  OUT receives six arrays
// of n elements: a*b, a+b, a-b, a^2, a*b + a'*b', a*b - a'*b', where a', b' are element n - 1 - i.
#include <cstdint>
#include <cstdio>
#include <vector>
#include "ec.cuh"
using namespace b200;

template <class C>
static void run(const std::vector<fe>& a, const std::vector<fe>& b, std::vector<fe>& out) {
    const size_t n = a.size();
    out.resize(6 * n);
    for (size_t i = 0; i < n; ++i) {
        const size_t j = n - 1 - i;
        out[i] = fe_mul<C>(a[i], b[i]);
        out[n + i] = fe_add<C>(a[i], b[i]);
        out[2 * n + i] = fe_sub<C>(a[i], b[i]);
        out[3 * n + i] = fe_sqr<C>(a[i]);
        out[4 * n + i] = fe_mul_add2<C>(a[i], b[i], a[j], b[j]);
        out[5 * n + i] = fe_mul_sub2<C>(a[i], b[i], a[j], b[j]);
    }
}

int main(int argc, char** argv) {
    if (argc != 4) {
        fprintf(stderr, "usage: %s FIELD IN OUT\n", argv[0]);
        return 2;
    }
    FILE* f = fopen(argv[2], "rb");
    uint64_t n = 0;
    if (!f || fread(&n, 8, 1, f) != 1) return 2;
    std::vector<fe> a(n), b(n), out;
    if (fread(a.data(), sizeof(fe), n, f) != n || fread(b.data(), sizeof(fe), n, f) != n) return 2;
    fclose(f);
    if (argv[1][0] == '0') run<FrCfg>(a, b, out);
    else run<FqCfg>(a, b, out);
    f = fopen(argv[3], "wb");
    if (!f || fwrite(out.data(), sizeof(fe), out.size(), f) != out.size()) return 2;
    fclose(f);
    return 0;
}
