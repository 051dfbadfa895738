// popsift::Feature / FeaturesHost -- containers and the text format of the reference
// (reference src/popsift/features.cu:25-110,310-338): one line per (feature, orientation):
//   x y 1/sigma^2 0 1/sigma^2 d0 .. d127
#include "popsift/features.h"
#include "pinned_pool.h"
#include "popsift_b200.h"
#include "popsift_b200_guided.h"
#include "popsift_b200_retrieval.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>
#include <cstdlib>
#include <iomanip>
#include <map>
#include <mutex>
#include <new>
#include <stdexcept>

namespace popsift {

FeaturesBase::FeaturesBase() : _num_ext(0), _num_ori(0) {}
FeaturesBase::~FeaturesBase() = default;

FeaturesHost::FeaturesHost() : _ext(nullptr), _ori(nullptr) {}
FeaturesHost::FeaturesHost(int num_ext, int num_ori) : _ext(nullptr), _ori(nullptr) { reset(num_ext, num_ori); }

FeaturesHost::~FeaturesHost()
{
    popsift::detail::pinned_pool().put(_ext);
    popsift::detail::pinned_pool().put(_ori);
}

void FeaturesHost::reset(int num_ext, int num_ori)
{
    popsift::detail::pinned_pool().put(_ext); _ext = nullptr;
    popsift::detail::pinned_pool().put(_ori); _ori = nullptr;
    _ext = static_cast<Feature*>(popsift::detail::pinned_pool().get((size_t)(num_ext > 0 ? num_ext : 1) * sizeof(Feature)));
    _ori = static_cast<Descriptor*>(popsift::detail::pinned_pool().get((size_t)(num_ori > 0 ? num_ori : 1) * sizeof(Descriptor)));
    if (!_ext || !_ori) throw std::runtime_error("Runtime error:\n    Failed to (re)allocate memory for downloading features");
    setFeatureCount(num_ext);
    setDescriptorCount(num_ori);
}

// ---- FeaturesDev (reference features.cu:127-163): device arrays through the C ABI's allocator

FeaturesDev::FeaturesDev() : _ext(nullptr), _ori(nullptr), _rev(nullptr) {}
FeaturesDev::FeaturesDev(int num_ext, int num_ori) : _ext(nullptr), _ori(nullptr), _rev(nullptr) { reset(num_ext, num_ori); }

FeaturesDev::~FeaturesDev()
{
    ps_dev_free(_ext);
    ps_dev_free(_ori);
    ps_dev_free(_rev);
}

void FeaturesDev::reset(int num_ext, int num_ori)
{
    ps_dev_free(_ext); _ext = nullptr;
    ps_dev_free(_ori); _ori = nullptr;
    ps_dev_free(_rev); _rev = nullptr;
    _ext = static_cast<Feature*>(ps_dev_alloc((size_t)(num_ext > 0 ? num_ext : 1) * sizeof(Feature)));
    _ori = static_cast<Descriptor*>(ps_dev_alloc((size_t)(num_ori > 0 ? num_ori : 1) * sizeof(Descriptor)));
    _rev = static_cast<int*>(ps_dev_alloc((size_t)(num_ori > 0 ? num_ori : 1) * sizeof(int)));
    if (!_ext || !_ori || !_rev) throw std::runtime_error("Runtime error:\n    Failed to allocate device memory for features");
    setFeatureCount(num_ext);
    setDescriptorCount(num_ori);
}

namespace {

// squared distance in the reference's float32 evaluation order (features.cu:165-185): lane k of a warp holds floats
// 4k..4k+3, computes x*x + y*y + z*z + w*w (SASS: FMUL, FFMA, FFMA, FFMA), then a shuffle-down tree 16, 8, 4, 2, 1
float warp_order_sq_dist(const Descriptor& l, const Descriptor& r)
{
    float lane[32];
    for (int k = 0; k < 32; ++k) {
        const float dx = l.features[4 * k] - r.features[4 * k], dy = l.features[4 * k + 1] - r.features[4 * k + 1];
        const float dz = l.features[4 * k + 2] - r.features[4 * k + 2], dw = l.features[4 * k + 3] - r.features[4 * k + 3];
        float v = dx * dx;
        v = std::fmaf(dy, dy, v);
        v = std::fmaf(dz, dz, v);
        v = std::fmaf(dw, dw, v);
        lane[k] = v;
    }
    for (int s = 16; s > 0; s >>= 1)
        for (int k = 0; k < s; ++k) lane[k] = lane[k] + lane[k + s];
    return lane[0];
}

} // namespace

// reference features.cu:282-304: 2-nearest-neighbour search of every descriptor of *this among `other`'s, then one
// line per descriptor on stdout (show_distance, features.cu:229-277: a device printf there, a host printf here).
// The search runs on the device (ps_match: wgmma tensor-core pass + exact re-rank, or the CUDA-core kernel for small sets).
void FeaturesDev::match(FeaturesDev* other)
{
    if (!other) throw std::runtime_error("FeaturesDev::match: null argument");
    const int l_len = getDescriptorCount(), r_len = other->getDescriptorCount();
    if (l_len <= 0 || r_len <= 0) return;
    const std::vector<int> m = matchIndices(other);
    std::vector<Descriptor> lo((size_t)l_len), ro((size_t)r_len);
    std::vector<int> lrev((size_t)l_len), rrev((size_t)r_len);
    if (ps_dev_to_host(lo.data(), _ori, lo.size() * sizeof(Descriptor)) != PS_OK ||
        ps_dev_to_host(ro.data(), other->_ori, ro.size() * sizeof(Descriptor)) != PS_OK ||
        ps_dev_to_host(lrev.data(), _rev, lrev.size() * sizeof(int)) != PS_OK ||
        ps_dev_to_host(rrev.data(), other->_rev, rrev.size() * sizeof(int)) != PS_OK)
        throw std::runtime_error("FeaturesDev::match: device -> host copy failed");
    for (int i = 0; i < l_len; ++i) {
        const int b1 = m[3 * (size_t)i], b2 = m[3 * (size_t)i + 1];
        const float d1 = warp_order_sq_dist(lo[i], ro[b1]), d2 = warp_order_sq_dist(lo[i], ro[b2]);
        std::printf("%s feat %4d [%4d] matches feat %4d [%4d] ( 2nd feat %4d [%4d] ) dist %.3f vs %.3f\n",
                    m[3 * (size_t)i + 2] ? "accept" : "reject", lrev[i], i, rrev[b1], b1, rrev[b2], b2, d1, d2);
    }
    std::fflush(stdout);
}

// the match matrix of the reference's compute_distance as a host vector: 3 ints (best, second, accept) per descriptor
std::vector<int> FeaturesDev::matchIndices(FeaturesDev* other, int flags)
{
    if (!other) throw std::runtime_error("FeaturesDev::matchIndices: null argument");
    const int l_len = getDescriptorCount(), r_len = other->getDescriptorCount();
    std::vector<int> m((size_t)std::max(l_len, 0) * 3, 0);
    if (l_len <= 0) return m;
    int32_t* d_out = static_cast<int32_t*>(ps_dev_alloc(m.size() * sizeof(int32_t)));
    if (!d_out) throw std::runtime_error("FeaturesDev::match: failed to allocate device memory");
    const int dev = std::max(0, ps_pointer_device(_ori));
    int rc = ps_match(dev, reinterpret_cast<const ps_descriptor*>(_ori), l_len, reinterpret_cast<const ps_descriptor*>(other->_ori),
                      r_len, d_out, flags);
    if (rc == PS_OK) rc = ps_dev_to_host(m.data(), d_out, m.size() * sizeof(int32_t));
    ps_dev_free(d_out);
    if (rc != PS_OK) throw std::runtime_error(std::string("FeaturesDev::match failed: ") + ps_last_error(nullptr));
    return m;
}

std::vector<std::vector<int>> matchPairs(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs, int flags)
{
    std::vector<const ps_descriptor*> d_sets(sets.size());
    std::vector<int32_t> n_desc(sets.size());
    for (size_t i = 0; i < sets.size(); ++i) {
        if (!sets[i]) throw std::runtime_error("popsift::matchPairs: null set");
        d_sets[i] = reinterpret_cast<const ps_descriptor*>(sets[i]->getDescriptors());
        n_desc[i] = sets[i]->getDescriptorCount();
    }
    std::vector<int32_t> flat(2 * pairs.size());
    std::vector<std::vector<int>> out(pairs.size());
    size_t rows = 0;
    for (size_t p = 0; p < pairs.size(); ++p) {
        const int l = pairs[p].first, r = pairs[p].second;
        if (l < 0 || (size_t)l >= sets.size() || r < 0 || (size_t)r >= sets.size()) throw std::runtime_error("popsift::matchPairs: set index out of range");
        flat[2 * p] = l; flat[2 * p + 1] = r;
        out[p].assign((size_t)std::max(n_desc[l], 0) * 3, 0);
        rows += out[p].size() / 3;
    }
    if (rows == 0) return out;
    int32_t* d_out = static_cast<int32_t*>(ps_dev_alloc(rows * 3 * sizeof(int32_t)));
    if (!d_out) throw std::runtime_error("popsift::matchPairs: failed to allocate device memory");
    int dev = 0;
    for (size_t i = 0; i < sets.size(); ++i)
        if (n_desc[i] > 0) { dev = std::max(0, ps_pointer_device(d_sets[i])); break; }
    int rc = ps_match_batch(dev, (int)sets.size(), d_sets.data(), n_desc.data(), (int)pairs.size(), flat.data(), d_out, flags);
    size_t row = 0;
    for (size_t p = 0; p < pairs.size() && rc == PS_OK; ++p) {
        rc = ps_dev_to_host(out[p].data(), d_out + 3 * row, out[p].size() * sizeof(int32_t));
        row += out[p].size() / 3;
    }
    ps_dev_free(d_out);
    if (rc != PS_OK) throw std::runtime_error(std::string("popsift::matchPairs failed: ") + ps_last_error(nullptr));
    return out;
}

std::vector<std::vector<int>> matchPairsU8(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs, int flags)
{
    std::vector<int32_t> n_desc(sets.size());
    for (size_t i = 0; i < sets.size(); ++i) {
        if (!sets[i]) throw std::runtime_error("popsift::matchPairsU8: null set");
        n_desc[i] = std::max(sets[i]->getDescriptorCount(), 0);
    }
    std::vector<int32_t> flat(2 * pairs.size());
    std::vector<std::vector<int>> out(pairs.size());
    size_t rows = 0;
    for (size_t p = 0; p < pairs.size(); ++p) {
        const int l = pairs[p].first, r = pairs[p].second;
        if (l < 0 || (size_t)l >= sets.size() || r < 0 || (size_t)r >= sets.size()) throw std::runtime_error("popsift::matchPairsU8: set index out of range");
        flat[2 * p] = l; flat[2 * p + 1] = r;
        out[p].assign((size_t)n_desc[l] * 3, 0);
        rows += out[p].size() / 3;
    }
    if (rows == 0) return out;
    int dev = 0;
    for (size_t i = 0; i < sets.size(); ++i)
        if (n_desc[i] > 0) { dev = std::max(0, ps_pointer_device(sets[i]->getDescriptors())); break; }
    // the 8-bit copies of every set (cudaMalloc: 256-byte aligned) and the result rows
    std::vector<void*> owned;
    auto release = [&]() { for (void* p : owned) ps_dev_free(p); };
    std::vector<const uint8_t*> d_sets(sets.size(), nullptr);
    int rc = PS_OK;
    for (size_t i = 0; i < sets.size() && rc == PS_OK; ++i) {
        if (n_desc[i] == 0) continue;
        uint8_t* q = static_cast<uint8_t*>(ps_dev_alloc((size_t)n_desc[i] * 128));
        if (!q) { release(); throw std::runtime_error("popsift::matchPairsU8: failed to allocate device memory"); }
        owned.push_back(q);
        d_sets[i] = q;
        rc = ps_descriptors_to_u8(dev, reinterpret_cast<const ps_descriptor*>(sets[i]->getDescriptors()), n_desc[i], q);
    }
    int32_t* d_out = rc == PS_OK ? static_cast<int32_t*>(ps_dev_alloc(rows * 3 * sizeof(int32_t))) : nullptr;
    if (rc == PS_OK && !d_out) { release(); throw std::runtime_error("popsift::matchPairsU8: failed to allocate device memory"); }
    if (d_out) owned.push_back(d_out);
    if (rc == PS_OK) rc = ps_match_u8_batch(dev, (int)sets.size(), d_sets.data(), n_desc.data(), (int)pairs.size(), flat.data(), d_out, flags);
    size_t row = 0;
    for (size_t p = 0; p < pairs.size() && rc == PS_OK; ++p) {
        rc = ps_dev_to_host(out[p].data(), d_out + 3 * row, out[p].size() * sizeof(int32_t));
        row += out[p].size() / 3;
    }
    release();
    if (rc != PS_OK) throw std::runtime_error(std::string("popsift::matchPairsU8 failed: ") + ps_last_error(nullptr));
    return out;
}

std::vector<PairGeometry> verifyPairs(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                      const std::vector<std::vector<int>>& matches, const VerifyParams& params)
{
    if (matches.size() != pairs.size()) throw std::runtime_error("popsift::verifyPairs: one match list per pair expected");
    std::vector<const ps_feature*> d_feat(sets.size());
    std::vector<const int32_t*> d_rev(sets.size());
    std::vector<int32_t> n_desc(sets.size());
    for (size_t i = 0; i < sets.size(); ++i) {
        if (!sets[i]) throw std::runtime_error("popsift::verifyPairs: null set");
        d_feat[i] = reinterpret_cast<const ps_feature*>(sets[i]->getFeatures());
        d_rev[i] = sets[i]->getReverseMap();
        n_desc[i] = std::max(sets[i]->getDescriptorCount(), 0);
    }
    std::vector<int32_t> flat(2 * pairs.size()), start(pairs.size()), n_corr(pairs.size(), 0);
    size_t rows = 0;
    for (size_t p = 0; p < pairs.size(); ++p) {
        const int l = pairs[p].first, r = pairs[p].second;
        if (l < 0 || (size_t)l >= sets.size() || r < 0 || (size_t)r >= sets.size()) throw std::runtime_error("popsift::verifyPairs: set index out of range");
        if (matches[p].size() != (size_t)n_desc[l] * 3) throw std::runtime_error("popsift::verifyPairs: match rows do not fit the left set");
        flat[2 * p] = l; flat[2 * p + 1] = r;
        start[p] = (int32_t)rows;
        rows += (size_t)n_desc[l];
    }
    std::vector<PairGeometry> out(pairs.size());
    for (PairGeometry& g : out) { std::fill(g.model, g.model + 9, 0.0f); g.n_inliers = 0; }
    if (pairs.empty()) return out;
    int dev = 0;
    for (size_t i = 0; i < sets.size(); ++i)
        if (n_desc[i] > 0) { dev = std::max(0, ps_pointer_device(d_feat[i])); break; }
    // device buffers: match rows, correspondences (16-byte rows), source rows, masks; models and counts per pair
    const size_t nr = std::max<size_t>(rows, 1);
    std::vector<void*> owned;
    auto release = [&]() { for (void* p : owned) ps_dev_free(p); };
    auto alloc = [&](size_t bytes) {
        void* p = ps_dev_alloc(bytes);
        if (!p) { release(); throw std::runtime_error("popsift::verifyPairs: failed to allocate device memory"); }
        owned.push_back(p);
        return p;
    };
    int32_t* d_match = static_cast<int32_t*>(alloc(nr * 3 * sizeof(int32_t)));
    float* d_corr = static_cast<float*>(alloc(nr * 4 * sizeof(float)));
    int32_t* d_src = static_cast<int32_t*>(alloc(nr * sizeof(int32_t)));
    uint8_t* d_mask = static_cast<uint8_t*>(alloc(nr));
    float* d_models = static_cast<float*>(alloc(pairs.size() * 9 * sizeof(float)));
    int32_t* d_n = static_cast<int32_t*>(alloc(pairs.size() * sizeof(int32_t)));
    int rc = PS_OK;
    for (size_t p = 0; p < pairs.size() && rc == PS_OK; ++p)
        if (!matches[p].empty())
            rc = ps_host_to_dev(d_match + 3 * (size_t)start[p], matches[p].data(), matches[p].size() * sizeof(int32_t));
    if (rc == PS_OK)
        rc = ps_match_correspondences(dev, (int)sets.size(), d_feat.data(), d_rev.data(), n_desc.data(), (int)pairs.size(), flat.data(),
                                      d_match, d_corr, d_src, n_corr.data());
    ps_verify_params prm;
    prm.model = params.model;
    prm.n_samples = params.n_samples;
    prm.threshold = params.threshold;
    prm.refine = params.refine ? 1 : 0;
    prm.seed = params.seed;
    if (rc == PS_OK)
        rc = ps_verify_batch(dev, (int)pairs.size(), d_corr, start.data(), n_corr.data(), &prm, d_models, d_n, d_mask, nullptr);
    std::vector<float> models(pairs.size() * 9);
    std::vector<int32_t> counts(pairs.size()), src(rows);
    std::vector<uint8_t> mask(rows);
    if (rc == PS_OK) rc = ps_dev_to_host(models.data(), d_models, models.size() * sizeof(float));
    if (rc == PS_OK) rc = ps_dev_to_host(counts.data(), d_n, counts.size() * sizeof(int32_t));
    if (rc == PS_OK && rows) rc = ps_dev_to_host(src.data(), d_src, rows * sizeof(int32_t));
    if (rc == PS_OK && rows) rc = ps_dev_to_host(mask.data(), d_mask, rows);
    release();
    if (rc != PS_OK) throw std::runtime_error(std::string("popsift::verifyPairs failed: ") + ps_last_error(nullptr));
    for (size_t p = 0; p < pairs.size(); ++p) {
        std::copy(models.begin() + 9 * p, models.begin() + 9 * (p + 1), out[p].model);
        out[p].n_inliers = counts[p];
        for (int k = 0; k < n_corr[p]; ++k)
            if (mask[(size_t)start[p] + k]) out[p].inlier_rows.push_back(src[(size_t)start[p] + k]);
    }
    return out;
}

namespace {

// matchPairsGuided / matchPairsGuidedU8: the C ABI call on the sets' descriptors (float) or their 8-bit copies
std::vector<std::vector<int>> match_guided(const char* name, bool u8, const std::vector<FeaturesDev*>& sets,
                                           const std::vector<std::pair<int, int>>& pairs, const std::vector<PairGeometry>& geometry,
                                           const VerifyParams& params, int flags)
{
    const std::string who = std::string("popsift::") + name;
    if (geometry.size() != pairs.size()) throw std::runtime_error(who + ": one geometry per pair expected");
    std::vector<const ps_feature*> d_feat(sets.size());
    std::vector<const int32_t*> d_rev(sets.size());
    std::vector<int32_t> n_desc(sets.size());
    for (size_t i = 0; i < sets.size(); ++i) {
        if (!sets[i]) throw std::runtime_error(who + ": null set");
        d_feat[i] = reinterpret_cast<const ps_feature*>(sets[i]->getFeatures());
        d_rev[i] = sets[i]->getReverseMap();
        n_desc[i] = std::max(sets[i]->getDescriptorCount(), 0);
    }
    std::vector<int32_t> flat(2 * pairs.size());
    std::vector<std::vector<int>> out(pairs.size());
    size_t rows = 0;
    for (size_t p = 0; p < pairs.size(); ++p) {
        const int l = pairs[p].first, r = pairs[p].second;
        if (l < 0 || (size_t)l >= sets.size() || r < 0 || (size_t)r >= sets.size()) throw std::runtime_error(who + ": set index out of range");
        flat[2 * p] = l; flat[2 * p + 1] = r;
        out[p].assign((size_t)n_desc[l] * 3, 0);
        rows += out[p].size() / 3;
    }
    if (rows == 0) return out;
    int dev = 0;
    for (size_t i = 0; i < sets.size(); ++i)
        if (n_desc[i] > 0) { dev = std::max(0, ps_pointer_device(sets[i]->getDescriptors())); break; }
    std::vector<void*> owned;
    auto release = [&]() { for (void* p : owned) ps_dev_free(p); };
    auto alloc = [&](size_t bytes) {
        void* p = ps_dev_alloc(bytes);
        if (!p) { release(); throw std::runtime_error(who + ": failed to allocate device memory"); }
        owned.push_back(p);
        return p;
    };
    std::vector<float> models(pairs.size() * 9);
    for (size_t p = 0; p < pairs.size(); ++p) std::copy(geometry[p].model, geometry[p].model + 9, models.begin() + 9 * p);
    float* d_models = static_cast<float*>(alloc(models.size() * sizeof(float)));
    int32_t* d_out = static_cast<int32_t*>(alloc(rows * 3 * sizeof(int32_t)));
    int rc = ps_host_to_dev(d_models, models.data(), models.size() * sizeof(float));
    if (u8) {
        // the 8-bit copies of every set (cudaMalloc: 256-byte aligned)
        std::vector<const uint8_t*> d_sets(sets.size(), nullptr);
        for (size_t i = 0; i < sets.size() && rc == PS_OK; ++i) {
            if (n_desc[i] == 0) continue;
            uint8_t* q = static_cast<uint8_t*>(alloc((size_t)n_desc[i] * 128));
            d_sets[i] = q;
            rc = ps_descriptors_to_u8(dev, reinterpret_cast<const ps_descriptor*>(sets[i]->getDescriptors()), n_desc[i], q);
        }
        if (rc == PS_OK)
            rc = ps_match_u8_guided_batch(dev, (int)sets.size(), d_sets.data(), d_feat.data(), d_rev.data(), n_desc.data(), (int)pairs.size(),
                                          flat.data(), d_models, params.model, params.threshold, d_out, flags);
    } else {
        std::vector<const ps_descriptor*> d_sets(sets.size());
        for (size_t i = 0; i < sets.size(); ++i) d_sets[i] = reinterpret_cast<const ps_descriptor*>(sets[i]->getDescriptors());
        if (rc == PS_OK)
            rc = ps_match_guided_batch(dev, (int)sets.size(), d_sets.data(), d_feat.data(), d_rev.data(), n_desc.data(), (int)pairs.size(),
                                       flat.data(), d_models, params.model, params.threshold, d_out, flags);
    }
    size_t row = 0;
    for (size_t p = 0; p < pairs.size() && rc == PS_OK; ++p) {
        rc = ps_dev_to_host(out[p].data(), d_out + 3 * row, out[p].size() * sizeof(int32_t));
        row += out[p].size() / 3;
    }
    release();
    if (rc != PS_OK) throw std::runtime_error(who + " failed: " + ps_last_error(nullptr));
    return out;
}

} // namespace

std::vector<std::vector<int>> matchPairsGuided(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                               const std::vector<PairGeometry>& geometry, const VerifyParams& params, int flags)
{
    return match_guided("matchPairsGuided", false, sets, pairs, geometry, params, flags);
}

std::vector<std::vector<int>> matchPairsGuidedU8(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                                 const std::vector<PairGeometry>& geometry, const VerifyParams& params, int flags)
{
    return match_guided("matchPairsGuidedU8", true, sets, pairs, geometry, params, flags);
}

void FeaturesHost::pin() {}
void FeaturesHost::unpin() {}

void FeaturesHost::print(std::ostream& ostr, bool write_as_uchar) const
{
    for (int i = 0; i < size(); i++) _ext[i].print(ostr, write_as_uchar);
}

std::ostream& operator<<(std::ostream& ostr, const FeaturesHost& f)
{
    f.print(ostr, false);
    return ostr;
}

void Feature::print(std::ostream& ostr, bool write_as_uchar) const
{
    const float sigval = 1.0f / (sigma * sigma);
    for (int o = 0; o < num_ori; o++) {
        ostr << xpos << " " << ypos << " " << sigval << " 0 " << sigval << " ";
        if (write_as_uchar) {
            for (int i = 0; i < 128; i++) ostr << roundf(desc[o]->features[i]) << " ";
        } else {
            ostr << std::setprecision(3);
            for (int i = 0; i < 128; i++) ostr << desc[o]->features[i] << " ";
            ostr << std::setprecision(6);
        }
        ostr << std::endl;
    }
}

std::ostream& operator<<(std::ostream& ostr, const Feature& f)
{
    f.print(ostr, false);
    return ostr;
}

namespace {

// the device pointers and counts of FeaturesDev sets, and the device of the first non-empty one
int vlad_sets(const char* fn, const std::vector<FeaturesDev*>& sets, std::vector<const ps_descriptor*>& d_sets, std::vector<int32_t>& n_desc)
{
    d_sets.resize(sets.size());
    n_desc.resize(sets.size());
    int dev = -1;
    for (size_t i = 0; i < sets.size(); ++i) {
        if (!sets[i]) throw std::runtime_error(std::string(fn) + ": null set");
        d_sets[i] = reinterpret_cast<const ps_descriptor*>(sets[i]->getDescriptors());
        n_desc[i] = sets[i]->getDescriptorCount();
        if (dev < 0 && n_desc[i] > 0) dev = std::max(0, ps_pointer_device(d_sets[i]));
    }
    return std::max(dev, 0);
}

// a device buffer freed at scope exit
struct DevBuf {
    void* p;
    explicit DevBuf(size_t bytes, const char* fn) : p(ps_dev_alloc(std::max<size_t>(bytes, 16)))
    {
        if (!p) throw std::runtime_error(std::string(fn) + ": failed to allocate device memory");
    }
    ~DevBuf() { ps_dev_free(p); }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
};

void check(int rc, const char* fn, const char* entry)
{
    if (rc != PS_OK) throw std::runtime_error(std::string(fn) + ": " + entry + " failed: " + ps_last_error(nullptr));
}

} // namespace

std::vector<float> vladCodebook(const std::vector<FeaturesDev*>& sets, const VladParams& params, int flags)
{
    const char* fn = "popsift::vladCodebook";
    std::vector<const ps_descriptor*> d_sets;
    std::vector<int32_t> n_desc;
    const int dev = vlad_sets(fn, sets, d_sets, n_desc);
    const int k = std::max(params.k, 0);
    DevBuf c((size_t)k * 128 * sizeof(float), fn);
    check(ps_vlad_train(dev, (int)sets.size(), d_sets.data(), n_desc.data(), params.k, params.iters, params.seed,
                        static_cast<float*>(c.p), flags), fn, "ps_vlad_train");
    std::vector<float> out((size_t)k * 128);
    check(ps_dev_to_host(out.data(), c.p, out.size() * sizeof(float)), fn, "ps_dev_to_host");
    return out;
}

std::vector<float> vladEncode(const std::vector<FeaturesDev*>& sets, const std::vector<float>& codebook, int flags)
{
    const char* fn = "popsift::vladEncode";
    if (codebook.empty() || codebook.size() % 128) throw std::runtime_error(std::string(fn) + ": the codebook is not k x 128 floats");
    std::vector<const ps_descriptor*> d_sets;
    std::vector<int32_t> n_desc;
    const int dev = vlad_sets(fn, sets, d_sets, n_desc);
    const int k = (int)(codebook.size() / 128);
    std::vector<float> out(sets.size() * codebook.size());
    if (sets.empty()) return out;
    DevBuf c(codebook.size() * sizeof(float), fn), v(out.size() * sizeof(float), fn);
    check(ps_host_to_dev(c.p, codebook.data(), codebook.size() * sizeof(float)), fn, "ps_host_to_dev");
    check(ps_vlad_encode(dev, (int)sets.size(), d_sets.data(), n_desc.data(), k, static_cast<const float*>(c.p),
                         static_cast<float*>(v.p), nullptr, flags), fn, "ps_vlad_encode");
    check(ps_dev_to_host(out.data(), v.p, out.size() * sizeof(float)), fn, "ps_dev_to_host");
    return out;
}

std::vector<std::pair<int, int>> retrievePairs(const std::vector<float>& vectors, int n, int m)
{
    const char* fn = "popsift::retrievePairs";
    if (n < 0 || (n > 0 && vectors.size() % (size_t)n)) throw std::runtime_error(std::string(fn) + ": vectors.size() is not a multiple of n");
    std::vector<std::pair<int, int>> out;
    if (n == 0) return out;
    const int dim = (int)(vectors.size() / n);
    DevBuf v(vectors.size() * sizeof(float), fn), nb((size_t)n * std::max(m, 1) * sizeof(int32_t), fn), sc((size_t)n * std::max(m, 1) * sizeof(float), fn);
    check(ps_host_to_dev(v.p, vectors.data(), vectors.size() * sizeof(float)), fn, "ps_host_to_dev");
    check(ps_retrieve_pairs(0 <= ps_pointer_device(v.p) ? ps_pointer_device(v.p) : 0, n, static_cast<const float*>(v.p), dim, m,
                            static_cast<int32_t*>(nb.p), static_cast<float*>(sc.p)), fn, "ps_retrieve_pairs");
    std::vector<int32_t> nbr((size_t)n * m);
    check(ps_dev_to_host(nbr.data(), nb.p, nbr.size() * sizeof(int32_t)), fn, "ps_dev_to_host");
    for (int i = 0; i < n; ++i)
        for (int q = 0; q < m; ++q) {
            const int j = nbr[(size_t)i * m + q];
            if (j >= 0 && j != i) out.push_back({std::min(i, j), std::max(i, j)});
        }
    std::sort(out.begin(), out.end());
    out.erase(std::unique(out.begin(), out.end()), out.end());
    return out;
}

} // namespace popsift
