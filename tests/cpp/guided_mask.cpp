// Host-only: the eligibility mask of guided matching, computed by the same __host__ __device__ function the kernels use
// (popsift_b200/csrc/k_guided.h).  No CUDA, no library.
//
//   guided_mask <in> <out>
//   in:  int32 model (0: homography, 1: fundamental), float32 t, float32 m[9] (row-major, left -> right),
//        int32 n_l, float32 left[n_l][2], int32 n_r, float32 right[n_r][2]   (pixels, little-endian)
//   out: uint8 mask[n_l][n_r], 1 where right point j is eligible for left point i
#include "k_guided.h"

#include <cstdio>
#include <vector>

namespace {

template <typename T>
bool get(FILE* f, T* v, size_t n) { return fread(v, sizeof(T), n, f) == n; }

template <int MODEL>
void mask(const float (&m)[9], float t2, const std::vector<float>& l, const std::vector<float>& r, std::vector<unsigned char>& out)
{
    const size_t nl = l.size() / 2, nr = r.size() / 2;
    for (size_t i = 0; i < nl; ++i)
        for (size_t j = 0; j < nr; ++j)
            out[i * nr + j] = psb::guided_eligible<MODEL>(m, t2, l[2 * i], l[2 * i + 1], r[2 * j], r[2 * j + 1]) ? 1 : 0;
}

} // namespace

int main(int argc, char** argv)
{
    if (argc != 3) { fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror(argv[1]); return 1; }
    int32_t model = 0, nl = 0, nr = 0;
    float t = 0.0f, m[9];
    std::vector<float> l, r;
    bool ok = get(f, &model, 1) && get(f, &t, 1) && get(f, m, 9) && get(f, &nl, 1) && nl >= 0;
    if (ok) { l.resize((size_t)nl * 2); ok = get(f, l.data(), l.size()) && get(f, &nr, 1) && nr >= 0; }
    if (ok) { r.resize((size_t)nr * 2); ok = get(f, r.data(), r.size()); }
    fclose(f);
    if (!ok || (model != 0 && model != 1)) { fprintf(stderr, "%s: bad input\n", argv[1]); return 1; }
    const float t2 = t * t;
    std::vector<unsigned char> out((size_t)nl * nr);
    if (model == 0) mask<psb::kGuidedH>(m, t2, l, r, out);
    else mask<psb::kGuidedF>(m, t2, l, r, out);
    FILE* o = fopen(argv[2], "wb");
    if (!o) { perror(argv[2]); return 1; }
    const bool w = fwrite(out.data(), 1, out.size(), o) == out.size();
    fclose(o);
    return w ? 0 : 1;
}
