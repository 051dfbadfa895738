// PopSift::describe through the C++ API: one frame is extracted, then described at its own keypoints, with describe
// and enqueue jobs interleaved in one FIFO:
//   enqueue(frame) -> describe(frame, one keypoint per descriptor, given angles) -> enqueue(frame)
//   -> describe(frame, one keypoint per Feature, computeOrientations) -> enqueue(frame)
// The frame is extracted once through the C ABI; the keypoints carry each Feature's octave and, as level, the extremum's
// lpos (ps_debug_extrema, whose index is the Feature index).  Every descriptor must be bit-identical to the extraction's, the
// orientations too, and every enqueue job must return the first one's features (as sorted rows).
// Usage: describe_check W H frame.raw      prints "OK <features> <descriptors>" or a FAIL line
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <memory>
#include <vector>

namespace {

struct Result {
    std::vector<popsift::Feature> feat;
    std::vector<popsift::Descriptor> desc;
    std::vector<int> first;   // index of each Feature's first descriptor
};

Result take(SiftJob* job)
{
    Result r;
    std::unique_ptr<popsift::FeaturesHost> f(job->get());
    delete job;
    if (!f) return r;
    const int nf = f->getFeatureCount(), nd = f->getDescriptorCount();
    r.feat.assign(f->getFeatures(), f->getFeatures() + nf);
    r.desc.assign(f->getDescriptors(), f->getDescriptors() + nd);
    for (int i = 0; i < nf; ++i) r.first.push_back(r.feat[i].num_ori > 0 ? (int)(r.feat[i].desc[0] - f->getDescriptors()) : -1);
    return r;
}

bool same_desc(const popsift::Descriptor& a, const popsift::Descriptor& b) { return std::memcmp(&a, &b, sizeof(a)) == 0; }

// an extraction as sorted (octave, x, y, sigma, angle, descriptor) rows: the order of detected extrema is not fixed
std::vector<std::vector<float>> canonical(const Result& r)
{
    std::vector<std::vector<float>> rows;
    for (size_t i = 0; i < r.feat.size(); ++i)
        for (int k = 0; k < r.feat[i].num_ori; ++k) {
            const popsift::Feature& f = r.feat[i];
            std::vector<float> row = {(float)f.debug_octave, f.xpos, f.ypos, f.sigma, f.orientation[k]};
            const float* d = r.desc[r.first[i] + k].features;
            row.insert(row.end(), d, d + 128);
            rows.push_back(row);
        }
    std::sort(rows.begin(), rows.end());
    return rows;
}

} // namespace

int main(int argc, char** argv)
{
    if (argc < 4) { std::fprintf(stderr, "usage: describe_check W H frame.raw\n"); return 2; }
    const int w = std::atoi(argv[1]), h = std::atoi(argv[2]);
    std::vector<unsigned char> img((size_t)w * h);
    std::ifstream in(argv[3], std::ios::binary);
    in.read(reinterpret_cast<char*>(img.data()), img.size());
    if (!in) { std::fprintf(stderr, "short read\n"); return 2; }

    // the extraction, and its extrema's levels, from the C ABI (same default configuration)
    ps_config c;
    ps_config_default(&c);
    ps_ctx* ctx = ps_create(0, &c, w, h, 1);
    if (!ctx) { std::printf("FAIL ps_create: %s\n", ps_last_error(nullptr)); return 1; }
    int32_t nf = 0, nd = 0;
    if (ps_submit_u8(ctx, 0, img.data(), w, h) != PS_OK || ps_counts(ctx, 0, &nf, &nd) != PS_OK) {
        std::printf("FAIL C-ABI run: %s\n", ps_last_error(ctx)); return 1;
    }
    std::vector<ps_extremum> ext((size_t)nf);
    std::vector<ps_feature> pf((size_t)nf);
    Result base;
    base.desc.resize((size_t)nd);
    static_assert(sizeof(ps_feature) == sizeof(popsift::Feature) && sizeof(ps_descriptor) == sizeof(popsift::Descriptor), "layouts");
    ps_descriptor* pd = reinterpret_cast<ps_descriptor*>(base.desc.data());
    if (ps_download(ctx, 0, pf.data(), pd) != PS_OK || ps_debug_extrema(ctx, 0, ext.data(), nf) != nf) {
        std::printf("FAIL C-ABI download: %s\n", ps_last_error(ctx)); return 1;
    }
    ps_destroy(ctx);
    for (const ps_feature& f : pf) {
        popsift::Feature g;
        std::memcpy(&g, &f, sizeof(g));
        base.feat.push_back(g);
        base.first.push_back(f.num_ori > 0 ? (int)(f.desc[0] - pd) : -1);
    }
    if (nf < 100) { std::printf("FAIL extraction: %d features\n", nf); return 1; }

    popsift::Config config;
    PopSift sift(config, popsift::Config::ExtractingMode, PopSift::ByteImages, 0);
    std::vector<popsift::Keypoint> per_desc, per_feat;
    for (int i = 0; i < nf; ++i) {
        const popsift::Feature& f = base.feat[i];
        for (int k = 0; k < f.num_ori; ++k)
            per_desc.push_back(popsift::Keypoint{f.xpos, f.ypos, f.sigma, f.orientation[k], f.debug_octave, ext[i].lpos});
        per_feat.push_back(popsift::Keypoint{f.xpos, f.ypos, f.sigma, 0.0f, f.debug_octave, ext[i].lpos});
    }
    // all five jobs in the queue before the first result is read
    SiftJob* jobs[5] = {sift.enqueue(w, h, img.data()), sift.describe(w, h, img.data(), per_desc),
                        sift.enqueue(w, h, img.data()), sift.describe(w, h, img.data(), per_feat, true),
                        sift.enqueue(w, h, img.data())};
    Result r[5];
    for (int q = 0; q < 5; ++q) r[q] = take(jobs[q]);
    const std::vector<std::vector<float>> base_rows = canonical(base);
    for (int q : {0, 2, 4})
        if (canonical(r[q]) != base_rows) { std::printf("FAIL enqueue job %d\n", q); return 1; }
    // given angles: one Feature and one descriptor per keypoint, the extraction's descriptor bit for bit
    if (r[1].feat.size() != per_desc.size() || r[1].desc.size() != base.desc.size()) { std::printf("FAIL describe sizes\n"); return 1; }
    for (size_t d = 0; d < per_desc.size(); ++d) {
        const popsift::Feature& f = r[1].feat[d];
        if (f.num_ori != 1 || f.orientation[0] != per_desc[d].orientation || f.xpos != per_desc[d].xpos || r[1].first[d] != (int)d
            || !same_desc(r[1].desc[d], base.desc[d])) { std::printf("FAIL describe (given angles) keypoint %zu\n", d); return 1; }
    }
    // computed orientations: the extraction's Features (orientations and descriptors), in the same order
    if (r[3].feat.size() != base.feat.size() || r[3].desc.size() != base.desc.size()) { std::printf("FAIL describe (orientations) sizes\n"); return 1; }
    for (int i = 0; i < nf; ++i) {
        const popsift::Feature &a = r[3].feat[i], &b = base.feat[i];
        if (a.num_ori != b.num_ori || a.debug_octave != b.debug_octave || std::memcmp(a.orientation, b.orientation, sizeof(a.orientation)) != 0)
            { std::printf("FAIL describe (orientations) feature %d\n", i); return 1; }
        for (int k = 0; k < a.num_ori; ++k)
            if (!same_desc(r[3].desc[r[3].first[i] + k], base.desc[base.first[i] + k])) { std::printf("FAIL describe (orientations) descriptor %d/%d\n", i, k); return 1; }
    }
    sift.uninit();
    std::printf("OK %d %d\n", nf, nd);
    return 0;
}
