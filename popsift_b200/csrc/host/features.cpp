// popsift::Feature / FeaturesHost -- containers and the text format of the reference
// (reference src/popsift/features.cu:25-110,310-338): one line per (feature, orientation):
//   x y 1/sigma^2 0 1/sigma^2 d0 .. d127
#include "popsift/features.h"
#include "pinned_pool.h"
#include "popsift_b200.h"
#include "popsift_b200_guided.h"
#include "popsift_b200_pose.h"
#include "popsift_b200_retrieval.h"
#include "popsift_b200_tracks.h"
#include "popsift_b200_triangulate.h"
#include "popsift_b200_bundle.h"
#include "popsift_b200_global.h"
#include "popsift_b200_viewgraph.h"
#include "popsift_b200_twoview.h"
#include "popsift_b200_depth.h"
#include "popsift_b200_mesh.h"
#include "popsift_b200_render.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>
#include <cstdlib>
#include <iomanip>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <optional>
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

// a device buffer freed at scope exit
struct DevBuf {
    void* p;
    explicit DevBuf(size_t bytes, const std::string& fn) : p(ps_dev_alloc(std::max<size_t>(bytes, 16)))
    {
        if (!p) throw std::runtime_error(fn + ": failed to allocate device memory");
    }
    ~DevBuf() { ps_dev_free(p); }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
};

// throws "<who>[: <entry>] failed: <last C ABI error>" unless rc is PS_OK
void check(int rc, const std::string& who, const char* entry = nullptr)
{
    if (rc != PS_OK) throw std::runtime_error(who + (entry ? std::string(": ") + entry : std::string()) + " failed: " + ps_last_error(nullptr));
}

// the C ABI arguments of a batched call over FeaturesDev sets: each set's device arrays and descriptor count, the device
// of the first non-empty set, the pair list flattened with each pair's first output row, and the rows of all pairs
struct Batch {
    std::string who;
    std::vector<const ps_descriptor*> desc;
    std::vector<const ps_feature*> feat;
    std::vector<const int32_t*> rev;
    std::vector<int32_t> n_desc;
    int dev = 0;
    std::vector<int32_t> flat;
    std::vector<size_t> start;
    size_t rows = 0, descs = 0;   // descs: the descriptors of all sets

    Batch(const char* name, const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs)
        : who(std::string("popsift::") + name), desc(sets.size()), feat(sets.size()), rev(sets.size()), n_desc(sets.size()),
          flat(2 * pairs.size()), start(pairs.size())
    {
        int first = -1;
        for (size_t i = 0; i < sets.size(); ++i) {
            if (!sets[i]) throw std::runtime_error(who + ": null set");
            desc[i] = reinterpret_cast<const ps_descriptor*>(sets[i]->getDescriptors());
            feat[i] = reinterpret_cast<const ps_feature*>(sets[i]->getFeatures());
            rev[i] = sets[i]->getReverseMap();
            n_desc[i] = sets[i]->getDescriptorCount();
            if (n_desc[i] > 0 && first < 0) first = (int)i;
            descs += (size_t)std::max(n_desc[i], 0);
        }
        if (first >= 0) dev = std::max(0, ps_pointer_device(desc[first]));
        for (size_t p = 0; p < pairs.size(); ++p) {
            const int l = pairs[p].first, r = pairs[p].second;
            if (l < 0 || (size_t)l >= sets.size() || r < 0 || (size_t)r >= sets.size()) throw std::runtime_error(who + ": set index out of range");
            flat[2 * p] = l; flat[2 * p + 1] = r;
            start[p] = rows;
            rows += pair_rows(p);
        }
    }

    size_t pair_rows(size_t p) const { return (size_t)std::max(n_desc[flat[2 * p]], 0); }

    // the caller's rows of every pair (3 ints per left descriptor) into d (rows x 3 int32 of device memory)
    void upload(const std::vector<std::vector<int>>& matches, int32_t* d) const
    {
        if (matches.size() != start.size()) throw std::runtime_error(who + ": one match list per pair expected");
        for (size_t p = 0; p < start.size(); ++p)
            if (matches[p].size() != pair_rows(p) * 3) throw std::runtime_error(who + ": match rows do not fit the left set");
        for (size_t p = 0; p < start.size(); ++p)
            if (!matches[p].empty()) check(ps_host_to_dev(d + 3 * start[p], matches[p].data(), matches[p].size() * sizeof(int32_t)), who);
    }

    // the 8-bit copies of all sets, back to back in q (128-byte rows keep every set 16-byte aligned)
    std::vector<const uint8_t*> to_u8(uint8_t* q) const
    {
        std::vector<const uint8_t*> u8(n_desc.size(), nullptr);
        for (size_t i = 0; i < n_desc.size(); ++i) {
            if (n_desc[i] <= 0) continue;
            check(ps_descriptors_to_u8(dev, desc[i], n_desc[i], q), who);
            u8[i] = q;
            q += (size_t)n_desc[i] * 128;
        }
        return u8;
    }

    // the result rows (best, second, accept) on the device, downloaded and split by pair
    std::vector<std::vector<int>> download(const int32_t* d_out) const
    {
        std::vector<int> all(rows * 3);
        check(ps_dev_to_host(all.data(), d_out, all.size() * sizeof(int32_t)), who);
        std::vector<std::vector<int>> out(start.size());
        for (size_t p = 0; p < out.size(); ++p)
            out[p].assign(all.begin() + 3 * start[p], all.begin() + 3 * (start[p] + pair_rows(p)));
        return out;
    }
};

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
    const char* who = "FeaturesDev::match";
    DevBuf d_out(m.size() * sizeof(int32_t), who);
    const int dev = std::max(0, ps_pointer_device(_ori));
    check(ps_match(dev, reinterpret_cast<const ps_descriptor*>(_ori), l_len, reinterpret_cast<const ps_descriptor*>(other->_ori), r_len,
                   static_cast<int32_t*>(d_out.p), flags), who);
    check(ps_dev_to_host(m.data(), d_out.p, m.size() * sizeof(int32_t)), who);
    return m;
}

namespace {

// matchPairs, matchPairsU8 (u8), matchPairsGuided and matchPairsGuidedU8 (geometry non-null): the C ABI call on the sets'
// descriptors or on their 8-bit copies
std::vector<std::vector<int>> match_pairs(const char* name, bool u8, const std::vector<FeaturesDev*>& sets,
                                          const std::vector<std::pair<int, int>>& pairs, const std::vector<PairGeometry>* geometry,
                                          const VerifyParams* params, int flags)
{
    if (geometry && geometry->size() != pairs.size()) throw std::runtime_error(std::string("popsift::") + name + ": one geometry per pair expected");
    const Batch b(name, sets, pairs);
    if (b.rows == 0) return std::vector<std::vector<int>>(pairs.size());
    DevBuf d_out(b.rows * 3 * sizeof(int32_t), b.who);
    int32_t* out = static_cast<int32_t*>(d_out.p);
    std::optional<DevBuf> d_models, q;
    if (geometry) {
        std::vector<float> models(pairs.size() * 9);
        for (size_t p = 0; p < pairs.size(); ++p) std::copy((*geometry)[p].model, (*geometry)[p].model + 9, models.begin() + 9 * p);
        d_models.emplace(models.size() * sizeof(float), b.who);
        check(ps_host_to_dev(d_models->p, models.data(), models.size() * sizeof(float)), b.who);
    }
    std::vector<const uint8_t*> d_u8;
    if (u8) d_u8 = b.to_u8(static_cast<uint8_t*>(q.emplace(b.descs * 128, b.who).p));
    const int n_sets = (int)sets.size(), n_pairs = (int)pairs.size();
    int rc;
    if (!geometry)
        rc = u8 ? ps_match_u8_batch(b.dev, n_sets, d_u8.data(), b.n_desc.data(), n_pairs, b.flat.data(), out, flags)
                : ps_match_batch(b.dev, n_sets, b.desc.data(), b.n_desc.data(), n_pairs, b.flat.data(), out, flags);
    else {
        const float* m = static_cast<const float*>(d_models->p);
        rc = u8 ? ps_match_u8_guided_batch(b.dev, n_sets, d_u8.data(), b.feat.data(), b.rev.data(), b.n_desc.data(), n_pairs, b.flat.data(),
                                           m, params->model, params->threshold, out, flags)
                : ps_match_guided_batch(b.dev, n_sets, b.desc.data(), b.feat.data(), b.rev.data(), b.n_desc.data(), n_pairs, b.flat.data(),
                                        m, params->model, params->threshold, out, flags);
    }
    check(rc, b.who);
    return b.download(out);
}

} // namespace

std::vector<std::vector<int>> matchPairs(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs, int flags)
{
    return match_pairs("matchPairs", false, sets, pairs, nullptr, nullptr, flags);
}

std::vector<std::vector<int>> matchPairsU8(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs, int flags)
{
    return match_pairs("matchPairsU8", true, sets, pairs, nullptr, nullptr, flags);
}

std::vector<std::vector<int>> matchPairsGuided(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                               const std::vector<PairGeometry>& geometry, const VerifyParams& params, int flags)
{
    return match_pairs("matchPairsGuided", false, sets, pairs, &geometry, &params, flags);
}

std::vector<std::vector<int>> matchPairsGuidedU8(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                                 const std::vector<PairGeometry>& geometry, const VerifyParams& params, int flags)
{
    return match_pairs("matchPairsGuidedU8", true, sets, pairs, &geometry, &params, flags);
}

std::vector<PairGeometry> verifyPairs(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                      const std::vector<std::vector<int>>& matches, const VerifyParams& params)
{
    if (matches.size() != pairs.size()) throw std::runtime_error("popsift::verifyPairs: one match list per pair expected");
    const Batch b("verifyPairs", sets, pairs);
    std::vector<PairGeometry> out(pairs.size());
    for (PairGeometry& g : out) { std::fill(g.model, g.model + 9, 0.0f); g.n_inliers = 0; }
    // device buffers: match rows, correspondences (16-byte rows), source rows, masks; models and counts per pair
    const size_t nr = std::max<size_t>(b.rows, 1), np = pairs.size();
    DevBuf match(nr * 3 * sizeof(int32_t), b.who);
    b.upload(matches, static_cast<int32_t*>(match.p));
    if (pairs.empty()) return out;
    DevBuf corr(nr * 4 * sizeof(float), b.who), src(nr * sizeof(int32_t), b.who), mask(nr, b.who),
        models(np * 9 * sizeof(float), b.who), counts(np * sizeof(int32_t), b.who);
    std::vector<int32_t> start(b.start.begin(), b.start.end()), n_corr(np, 0);
    check(ps_match_correspondences(b.dev, (int)sets.size(), b.feat.data(), b.rev.data(), b.n_desc.data(), (int)np, b.flat.data(),
                                   static_cast<const int32_t*>(match.p), static_cast<float*>(corr.p), static_cast<int32_t*>(src.p), n_corr.data()),
          b.who);
    ps_verify_params prm;
    prm.model = params.model;
    prm.n_samples = params.n_samples;
    prm.threshold = params.threshold;
    prm.refine = params.refine ? 1 : 0;
    prm.seed = params.seed;
    check(ps_verify_batch(b.dev, (int)np, static_cast<const float*>(corr.p), start.data(), n_corr.data(), &prm, static_cast<float*>(models.p),
                          static_cast<int32_t*>(counts.p), static_cast<uint8_t*>(mask.p), nullptr),
          b.who);
    std::vector<float> h_models(np * 9);
    std::vector<int32_t> h_counts(np), h_src(b.rows);
    std::vector<uint8_t> h_mask(b.rows);
    check(ps_dev_to_host(h_models.data(), models.p, h_models.size() * sizeof(float)), b.who);
    check(ps_dev_to_host(h_counts.data(), counts.p, h_counts.size() * sizeof(int32_t)), b.who);
    check(ps_dev_to_host(h_src.data(), src.p, b.rows * sizeof(int32_t)), b.who);
    check(ps_dev_to_host(h_mask.data(), mask.p, b.rows), b.who);
    for (size_t p = 0; p < np; ++p) {
        std::copy(h_models.begin() + 9 * p, h_models.begin() + 9 * (p + 1), out[p].model);
        out[p].n_inliers = h_counts[p];
        for (int k = 0; k < n_corr[p]; ++k)
            if (h_mask[b.start[p] + k]) out[p].inlier_rows.push_back(h_src[b.start[p] + k]);
    }
    return out;
}

std::vector<TwoViewPose> relativePoses(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                       const std::vector<std::vector<int>>& matches, const std::vector<Camera>& cameras,
                                       const PoseParams& params)
{
    if (matches.size() != pairs.size()) throw std::runtime_error("popsift::relativePoses: one match list per pair expected");
    if (cameras.size() != sets.size()) throw std::runtime_error("popsift::relativePoses: one camera per set expected");
    const Batch b("relativePoses", sets, pairs);
    std::vector<TwoViewPose> out(pairs.size());
    for (TwoViewPose& g : out) {
        std::fill(g.E, g.E + 9, 0.0f); std::fill(g.F, g.F + 9, 0.0f); std::fill(g.R, g.R + 9, 0.0f); std::fill(g.t, g.t + 3, 0.0f);
        g.n_inliers = g.n_front = 0;
    }
    const size_t nr = std::max<size_t>(b.rows, 1), np = pairs.size();
    DevBuf match(nr * 3 * sizeof(int32_t), b.who);
    b.upload(matches, static_cast<int32_t*>(match.p));
    if (pairs.empty()) return out;
    DevBuf corr(nr * 4 * sizeof(float), b.who), src(nr * sizeof(int32_t), b.who), mask(nr, b.who), two(np * sizeof(ps_two_view), b.who);
    std::vector<int32_t> start(b.start.begin(), b.start.end()), n_corr(np, 0);
    check(ps_match_correspondences(b.dev, (int)sets.size(), b.feat.data(), b.rev.data(), b.n_desc.data(), (int)np, b.flat.data(),
                                   static_cast<const int32_t*>(match.p), static_cast<float*>(corr.p), static_cast<int32_t*>(src.p), n_corr.data()),
          b.who);
    std::vector<ps_camera> cams(2 * np);
    for (size_t p = 0; p < np; ++p)
        for (int k = 0; k < 2; ++k) {
            const Camera& c = cameras[k ? pairs[p].second : pairs[p].first];
            cams[2 * p + k] = ps_camera{c.fx, c.fy, c.cx, c.cy};
        }
    ps_pose_params prm{};
    prm.n_samples = params.n_samples;
    prm.threshold = params.threshold;
    prm.refine = params.refine ? 1 : 0;
    prm.seed = params.seed;
    check(ps_relative_pose_batch(b.dev, (int)np, static_cast<const float*>(corr.p), start.data(), n_corr.data(), cams.data(), &prm,
                                 static_cast<ps_two_view*>(two.p), static_cast<uint8_t*>(mask.p), nullptr, nullptr),
          b.who);
    std::vector<ps_two_view> h_two(np);
    std::vector<int32_t> h_src(b.rows);
    std::vector<uint8_t> h_mask(b.rows);
    check(ps_dev_to_host(h_two.data(), two.p, np * sizeof(ps_two_view)), b.who);
    check(ps_dev_to_host(h_src.data(), src.p, b.rows * sizeof(int32_t)), b.who);
    check(ps_dev_to_host(h_mask.data(), mask.p, b.rows), b.who);
    for (size_t p = 0; p < np; ++p) {
        const ps_two_view& v = h_two[p];
        TwoViewPose& g = out[p];
        std::copy(v.E, v.E + 9, g.E); std::copy(v.F, v.F + 9, g.F); std::copy(v.R, v.R + 9, g.R); std::copy(v.t, v.t + 3, g.t);
        g.n_inliers = v.n_inliers;
        g.n_front = v.n_front;
        for (int k = 0; k < n_corr[p]; ++k) {
            const uint8_t m = h_mask[b.start[p] + k];
            if (m & 1) g.inlier_rows.push_back(h_src[b.start[p] + k]);
            if (m & 2) g.front_rows.push_back(h_src[b.start[p] + k]);
        }
    }
    return out;
}

std::vector<TwoViewGeometry> twoViewGeometries(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                               const std::vector<std::vector<int>>& matches, const std::vector<Camera>& cameras,
                                               const PoseParams& params, const TwoViewConfigParams& config)
{
    if (matches.size() != pairs.size()) throw std::runtime_error("popsift::twoViewGeometries: one match list per pair expected");
    if (cameras.size() != sets.size()) throw std::runtime_error("popsift::twoViewGeometries: one camera per set expected");
    const Batch b("twoViewGeometries", sets, pairs);
    std::vector<TwoViewGeometry> out(pairs.size());
    for (TwoViewGeometry& g : out) {
        TwoViewPose& v = g.pose;
        std::fill(v.E, v.E + 9, 0.0f); std::fill(v.F, v.F + 9, 0.0f); std::fill(v.R, v.R + 9, 0.0f); std::fill(v.t, v.t + 3, 0.0f);
        v.n_inliers = v.n_front = 0;
    }
    const size_t nr = std::max<size_t>(b.rows, 1), np = pairs.size();
    DevBuf match(nr * 3 * sizeof(int32_t), b.who);
    b.upload(matches, static_cast<int32_t*>(match.p));
    if (pairs.empty()) return out;
    DevBuf corr(nr * 4 * sizeof(float), b.who), src(nr * sizeof(int32_t), b.who), hmask(nr, b.who), fmask(nr, b.who), emask(nr, b.who),
        mask(nr, b.who), hom(np * 9 * sizeof(float), b.who), fund(np * 9 * sizeof(float), b.who), hn(np * sizeof(int32_t), b.who),
        fn(np * sizeof(int32_t), b.who), ess(np * sizeof(ps_two_view), b.who), two(np * sizeof(ps_two_view), b.who);
    std::vector<int32_t> start(b.start.begin(), b.start.end()), n_corr(np, 0);
    check(ps_match_correspondences(b.dev, (int)sets.size(), b.feat.data(), b.rev.data(), b.n_desc.data(), (int)np, b.flat.data(),
                                   static_cast<const int32_t*>(match.p), static_cast<float*>(corr.p), static_cast<int32_t*>(src.p), n_corr.data()),
          b.who);
    std::vector<ps_camera> cams(2 * np);
    for (size_t p = 0; p < np; ++p)
        for (int k = 0; k < 2; ++k) {
            const Camera& c = cameras[k ? pairs[p].second : pairs[p].first];
            cams[2 * p + k] = ps_camera{c.fx, c.fy, c.cx, c.cy};
        }
    const float* d_corr = static_cast<const float*>(corr.p);
    ps_verify_params vp{};
    vp.n_samples = params.n_samples;
    vp.threshold = params.threshold;
    vp.refine = params.refine ? 1 : 0;
    vp.seed = params.seed;
    vp.model = PS_GEOM_HOMOGRAPHY;
    check(ps_verify_batch(b.dev, (int)np, d_corr, start.data(), n_corr.data(), &vp, static_cast<float*>(hom.p), static_cast<int32_t*>(hn.p),
                          static_cast<uint8_t*>(hmask.p), nullptr),
          b.who);
    vp.model = PS_GEOM_FUNDAMENTAL;
    check(ps_verify_batch(b.dev, (int)np, d_corr, start.data(), n_corr.data(), &vp, static_cast<float*>(fund.p), static_cast<int32_t*>(fn.p),
                          static_cast<uint8_t*>(fmask.p), nullptr),
          b.who);
    ps_pose_params pp{};
    pp.n_samples = params.n_samples;
    pp.threshold = params.threshold;
    pp.refine = params.refine ? 1 : 0;
    pp.seed = params.seed;
    check(ps_relative_pose_batch(b.dev, (int)np, d_corr, start.data(), n_corr.data(), cams.data(), &pp, static_cast<ps_two_view*>(ess.p),
                                 static_cast<uint8_t*>(emask.p), nullptr, nullptr),
          b.who);
    ps_two_view_config_params cp{};
    cp.min_inliers = config.min_inliers;
    cp.threshold = params.threshold;
    cp.min_ef_ratio = config.min_ef_ratio;
    cp.max_h_ratio = config.max_h_ratio;
    cp.min_rotation_ratio = config.min_rotation_ratio;
    std::vector<ps_two_view_info> info(np);
    check(ps_two_view_config_batch(b.dev, (int)np, d_corr, start.data(), n_corr.data(), cams.data(), static_cast<const ps_two_view*>(ess.p),
                                   static_cast<const uint8_t*>(emask.p), static_cast<const int32_t*>(fn.p), static_cast<const float*>(hom.p),
                                   static_cast<const uint8_t*>(hmask.p), &cp, static_cast<ps_two_view*>(two.p), static_cast<uint8_t*>(mask.p),
                                   nullptr, info.data()),
          b.who, "ps_two_view_config_batch");
    std::vector<ps_two_view> h_two(np);
    std::vector<int32_t> h_src(b.rows);
    std::vector<uint8_t> h_mask(b.rows);
    check(ps_dev_to_host(h_two.data(), two.p, np * sizeof(ps_two_view)), b.who);
    check(ps_dev_to_host(h_src.data(), src.p, b.rows * sizeof(int32_t)), b.who);
    check(ps_dev_to_host(h_mask.data(), mask.p, b.rows), b.who);
    for (size_t p = 0; p < np; ++p) {
        const ps_two_view& v = h_two[p];
        TwoViewGeometry& g = out[p];
        std::copy(v.E, v.E + 9, g.pose.E); std::copy(v.F, v.F + 9, g.pose.F); std::copy(v.R, v.R + 9, g.pose.R); std::copy(v.t, v.t + 3, g.pose.t);
        g.pose.n_inliers = v.n_inliers;
        g.pose.n_front = v.n_front;
        for (int k = 0; k < n_corr[p]; ++k) {
            const uint8_t m = h_mask[b.start[p] + k];
            if (m & 1) g.pose.inlier_rows.push_back(h_src[b.start[p] + k]);
            if (m & 2) g.pose.front_rows.push_back(h_src[b.start[p] + k]);
        }
        const ps_two_view_info& in = info[p];
        g.config = in.config;
        std::copy(in.normal, in.normal + 3, g.normal);
        g.tri_angle = in.tri_angle;
        g.n_e = in.n_e; g.n_f = in.n_f; g.n_h = in.n_h; g.n_rotation = in.n_rotation;
    }
    return out;
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

std::vector<float> vladCodebook(const std::vector<FeaturesDev*>& sets, const VladParams& params, int flags)
{
    const Batch b("vladCodebook", sets, {});
    const int k = std::max(params.k, 0);
    DevBuf c((size_t)k * 128 * sizeof(float), b.who);
    check(ps_vlad_train(b.dev, (int)sets.size(), b.desc.data(), b.n_desc.data(), params.k, params.iters, params.seed,
                        static_cast<float*>(c.p), flags), b.who, "ps_vlad_train");
    std::vector<float> out((size_t)k * 128);
    check(ps_dev_to_host(out.data(), c.p, out.size() * sizeof(float)), b.who, "ps_dev_to_host");
    return out;
}

std::vector<float> vladEncode(const std::vector<FeaturesDev*>& sets, const std::vector<float>& codebook, int flags)
{
    const char* fn = "popsift::vladEncode";
    if (codebook.empty() || codebook.size() % 128) throw std::runtime_error(std::string(fn) + ": the codebook is not k x 128 floats");
    const Batch b("vladEncode", sets, {});
    const int k = (int)(codebook.size() / 128);
    std::vector<float> out(sets.size() * codebook.size());
    if (sets.empty()) return out;
    DevBuf c(codebook.size() * sizeof(float), fn), v(out.size() * sizeof(float), fn);
    check(ps_host_to_dev(c.p, codebook.data(), codebook.size() * sizeof(float)), fn, "ps_host_to_dev");
    check(ps_vlad_encode(b.dev, (int)sets.size(), b.desc.data(), b.n_desc.data(), k, static_cast<const float*>(c.p),
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
    check(ps_retrieve_pairs(std::max(0, ps_pointer_device(v.p)), n, static_cast<const float*>(v.p), dim, m,
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

namespace {

// both buildTracks: the match rows on the device, then the correspondences -- the inlier rows of `geometry`, or (none
// given) those ps_match_correspondences gathers -- and ps_tracks_from_matches over them without a mask
Tracks build_tracks(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                    const std::vector<std::vector<int>>& matches, const std::vector<PairGeometry>* geometry, int min_length)
{
    if (geometry && geometry->size() != pairs.size()) throw std::runtime_error("popsift::buildTracks: one geometry per pair expected");
    const Batch b("buildTracks", sets, pairs);
    const size_t nr = std::max<size_t>(b.rows, 1), np = pairs.size();
    DevBuf match(nr * 3 * sizeof(int32_t), b.who), src(nr * sizeof(int32_t), b.who);
    b.upload(matches, static_cast<int32_t*>(match.p));
    std::vector<int32_t> n_corr(np, 0);
    if (geometry) {
        std::vector<int32_t> h_src(b.rows);
        for (size_t p = 0; p < np; ++p) {
            const std::vector<int>& in = (*geometry)[p].inlier_rows;
            if (in.size() > b.pair_rows(p)) throw std::runtime_error(b.who + ": more inlier rows than left descriptors");
            std::copy(in.begin(), in.end(), h_src.begin() + b.start[p]);
            n_corr[p] = (int32_t)in.size();
        }
        check(ps_host_to_dev(src.p, h_src.data(), h_src.size() * sizeof(int32_t)), b.who);
    } else if (np > 0) {
        DevBuf corr(nr * 4 * sizeof(float), b.who);
        check(ps_match_correspondences(b.dev, (int)sets.size(), b.feat.data(), b.rev.data(), b.n_desc.data(), (int)np, b.flat.data(),
                                       static_cast<const int32_t*>(match.p), static_cast<float*>(corr.p), static_cast<int32_t*>(src.p),
                                       n_corr.data()),
              b.who);
    }
    std::vector<int32_t> n_feat(sets.size());
    std::vector<size_t> off(sets.size() + 1, 0);
    for (size_t i = 0; i < sets.size(); ++i) {
        n_feat[i] = sets[i]->getFeatureCount();
        off[i + 1] = off[i] + (size_t)std::max(n_feat[i], 0);
    }
    const size_t N = off.back();
    DevBuf track_of(N * sizeof(int32_t), b.who), track_start((N / std::max(min_length, 2) + 1) * sizeof(int32_t), b.who),
        members(N * sizeof(int32_t), b.who);
    ps_track_counts c;
    check(ps_tracks_from_matches(b.dev, (int)sets.size(), n_feat.data(), b.rev.data(), b.n_desc.data(), (int)np, b.flat.data(),
                                 static_cast<const int32_t*>(match.p), static_cast<const int32_t*>(src.p), n_corr.data(), nullptr,
                                 min_length, static_cast<int32_t*>(track_of.p), static_cast<int32_t*>(track_start.p),
                                 static_cast<int32_t*>(members.p), &c),
          b.who, "ps_tracks_from_matches");
    Tracks t;
    t.start.resize((size_t)c.n_tracks + 1);
    std::vector<int32_t> mem((size_t)c.n_members), of(N);
    check(ps_dev_to_host(t.start.data(), track_start.p, t.start.size() * sizeof(int32_t)), b.who);
    check(ps_dev_to_host(mem.data(), members.p, mem.size() * sizeof(int32_t)), b.who);
    check(ps_dev_to_host(of.data(), track_of.p, of.size() * sizeof(int32_t)), b.who);
    for (const int32_t g : mem) {
        const size_t s = (size_t)(std::upper_bound(off.begin(), off.end(), (size_t)g) - off.begin()) - 1;
        t.set.push_back((int)s);
        t.feature.push_back((int)(g - off[s]));
    }
    for (size_t i = 0; i < sets.size(); ++i) t.track_of.emplace_back(of.begin() + off[i], of.begin() + off[i + 1]);
    t.n_components = c.n_components;
    t.n_conflicting = c.n_conflicting;
    t.n_short = c.n_short;
    return t;
}

} // namespace

Tracks buildTracks(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                   const std::vector<std::vector<int>>& matches, const std::vector<PairGeometry>& geometry, int min_length)
{
    return build_tracks(sets, pairs, matches, &geometry, min_length);
}

Tracks buildTracks(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                   const std::vector<std::vector<int>>& matches, int min_length)
{
    return build_tracks(sets, pairs, matches, nullptr, min_length);
}

TrackPoints triangulateTracks(const std::vector<FeaturesDev*>& sets, const Tracks& tracks, const std::vector<Camera>& cameras,
                              const std::vector<Rigid>& poses, const TriangulateParams& params)
{
    const Batch b("triangulateTracks", sets, {});
    if (cameras.size() != sets.size()) throw std::runtime_error(b.who + ": one camera per set expected");
    if (poses.size() != sets.size()) throw std::runtime_error(b.who + ": one pose per set expected");
    if (tracks.start.empty() || tracks.set.size() != tracks.feature.size() || (size_t)tracks.start.back() != tracks.set.size())
        throw std::runtime_error(b.who + ": malformed tracks");
    std::vector<int32_t> n_feat(sets.size());
    std::vector<int64_t> off(sets.size() + 1, 0);
    for (size_t i = 0; i < sets.size(); ++i) {
        n_feat[i] = sets[i]->getFeatureCount();
        off[i + 1] = off[i] + std::max(n_feat[i], 0);
    }
    const size_t nt = tracks.start.size() - 1, nm = tracks.set.size();
    std::vector<int32_t> mem(nm);
    for (size_t k = 0; k < nm; ++k) {
        const int s = tracks.set[k], f = tracks.feature[k];
        if (s < 0 || (size_t)s >= sets.size() || f < 0 || f >= n_feat[s]) throw std::runtime_error(b.who + ": track member out of range");
        mem[k] = (int32_t)(off[s] + f);
    }
    std::vector<ps_camera> cams(sets.size());
    std::vector<ps_rigid> rig(sets.size());
    for (size_t i = 0; i < sets.size(); ++i) {
        cams[i] = ps_camera{cameras[i].fx, cameras[i].fy, cameras[i].cx, cameras[i].cy};
        std::copy(poses[i].R, poses[i].R + 9, rig[i].R);
        std::copy(poses[i].t, poses[i].t + 3, rig[i].t);
    }
    ps_triangulate_params prm{};
    prm.max_error = params.max_error;
    prm.min_angle = params.min_angle;
    prm.min_views = params.min_views;
    prm.n_samples = params.n_samples;
    prm.refine_iters = params.refine_iters;
    prm.seed = params.seed;
    DevBuf start(tracks.start.size() * sizeof(int32_t), b.who), members(nm * sizeof(int32_t), b.who);
    DevBuf pts(std::max<size_t>(nt, 1) * sizeof(ps_track_point), b.who), mask(nm, b.who), err(nm * sizeof(float), b.who);
    check(ps_host_to_dev(start.p, tracks.start.data(), tracks.start.size() * sizeof(int32_t)), b.who);
    check(ps_host_to_dev(members.p, mem.data(), nm * sizeof(int32_t)), b.who);
    ps_triangulate_counts c;
    check(ps_triangulate_tracks(b.dev, (int)sets.size(), n_feat.data(), b.feat.data(), cams.data(), rig.data(), (int)nt,
                                static_cast<const int32_t*>(start.p), static_cast<const int32_t*>(members.p), (int)nm, &prm,
                                static_cast<ps_track_point*>(pts.p), static_cast<uint8_t*>(mask.p), static_cast<float*>(err.p), &c),
          b.who, "ps_triangulate_tracks");
    TrackPoints out;
    std::vector<ps_track_point> h(nt);
    out.mask.resize(nm);
    out.obs_error.resize(nm);
    check(ps_dev_to_host(h.data(), pts.p, nt * sizeof(ps_track_point)), b.who);
    check(ps_dev_to_host(out.mask.data(), mask.p, nm), b.who);
    check(ps_dev_to_host(out.obs_error.data(), err.p, nm * sizeof(float)), b.who);
    out.points.resize(nt);
    for (size_t t = 0; t < nt; ++t) {
        TrackPoint& p = out.points[t];
        std::copy(h[t].X, h[t].X + 3, p.X);
        p.error = h[t].error;
        p.angle = h[t].angle;
        p.n_inliers = h[t].n_inliers;
        p.status = h[t].status;
    }
    std::copy(c.n_status, c.n_status + 5, out.n_status);
    out.n_inlier_obs = c.n_inlier_obs;
    return out;
}

std::pair<std::vector<Rigid>, BundleReport> bundleAdjust(const std::vector<FeaturesDev*>& sets, const Tracks& tracks,
                                                         const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
                                                         const std::vector<bool>& fixed, TrackPoints& points, const BundleParams& params)
{
    const Batch b("bundleAdjust", sets, {});
    if (cameras.size() != sets.size()) throw std::runtime_error(b.who + ": one camera per set expected");
    if (poses.size() != sets.size()) throw std::runtime_error(b.who + ": one pose per set expected");
    if (fixed.size() != sets.size()) throw std::runtime_error(b.who + ": one fixed flag per set expected");
    if (tracks.start.empty() || tracks.set.size() != tracks.feature.size() || (size_t)tracks.start.back() != tracks.set.size())
        throw std::runtime_error(b.who + ": malformed tracks");
    const size_t nt = tracks.start.size() - 1, nm = tracks.set.size();
    if (points.points.size() != nt || points.mask.size() != nm) throw std::runtime_error(b.who + ": points do not match the tracks");
    std::vector<int32_t> n_feat(sets.size());
    std::vector<int64_t> off(sets.size() + 1, 0);
    for (size_t i = 0; i < sets.size(); ++i) {
        n_feat[i] = sets[i]->getFeatureCount();
        off[i + 1] = off[i] + std::max(n_feat[i], 0);
    }
    std::vector<int32_t> mem(nm);
    for (size_t k = 0; k < nm; ++k) {
        const int s = tracks.set[k], f = tracks.feature[k];
        if (s < 0 || (size_t)s >= sets.size() || f < 0 || f >= n_feat[s]) throw std::runtime_error(b.who + ": track member out of range");
        mem[k] = (int32_t)(off[s] + f);
    }
    std::vector<ps_camera> cams(sets.size());
    std::vector<ps_rigid> rig(sets.size()), out(sets.size());
    std::vector<uint8_t> fix(sets.size());
    for (size_t i = 0; i < sets.size(); ++i) {
        cams[i] = ps_camera{cameras[i].fx, cameras[i].fy, cameras[i].cx, cameras[i].cy};
        std::copy(poses[i].R, poses[i].R + 9, rig[i].R);
        std::copy(poses[i].t, poses[i].t + 3, rig[i].t);
        fix[i] = fixed[i] ? 1 : 0;
    }
    std::vector<ps_track_point> h(nt);
    for (size_t t = 0; t < nt; ++t) {
        const TrackPoint& p = points.points[t];
        std::copy(p.X, p.X + 3, h[t].X);
        h[t].error = p.error;
        h[t].angle = p.angle;
        h[t].n_inliers = p.n_inliers;
        h[t].status = p.status;
    }
    ps_bundle_params prm{};
    prm.loss = params.loss;
    prm.max_iters = params.max_iters;
    prm.cg_max_iters = params.cg_max_iters;
    prm.scale_set = params.scale_set;
    prm.scale_axis = params.scale_axis;
    prm.loss_scale = params.loss_scale;
    prm.function_tol = params.function_tol;
    prm.cg_tol = params.cg_tol;
    prm.initial_lambda = params.initial_lambda;
    DevBuf start(tracks.start.size() * sizeof(int32_t), b.who), members(nm * sizeof(int32_t), b.who);
    DevBuf pts(std::max<size_t>(nt, 1) * sizeof(ps_track_point), b.who), mask(nm, b.who), err(nm * sizeof(float), b.who);
    check(ps_host_to_dev(start.p, tracks.start.data(), tracks.start.size() * sizeof(int32_t)), b.who);
    check(ps_host_to_dev(members.p, mem.data(), nm * sizeof(int32_t)), b.who);
    check(ps_host_to_dev(pts.p, h.data(), nt * sizeof(ps_track_point)), b.who);
    check(ps_host_to_dev(mask.p, points.mask.data(), nm), b.who);
    ps_bundle_report r;
    check(ps_bundle_adjust(b.dev, (int)sets.size(), n_feat.data(), b.feat.data(), cams.data(), rig.data(), (int)nt,
                           static_cast<const int32_t*>(start.p), static_cast<const int32_t*>(members.p), (int)nm,
                           static_cast<ps_track_point*>(pts.p), static_cast<const uint8_t*>(mask.p), fix.data(), &prm, out.data(),
                           static_cast<float*>(err.p), &r),
          b.who, "ps_bundle_adjust");
    check(ps_dev_to_host(h.data(), pts.p, nt * sizeof(ps_track_point)), b.who);
    points.obs_error.resize(nm);
    check(ps_dev_to_host(points.obs_error.data(), err.p, nm * sizeof(float)), b.who);
    for (size_t t = 0; t < nt; ++t) {
        TrackPoint& p = points.points[t];
        std::copy(h[t].X, h[t].X + 3, p.X);
        p.error = h[t].error;
        p.angle = h[t].angle;
    }
    std::pair<std::vector<Rigid>, BundleReport> res;
    res.first.resize(sets.size());
    for (size_t i = 0; i < sets.size(); ++i) {
        std::copy(out[i].R, out[i].R + 9, res.first[i].R);
        std::copy(out[i].t, out[i].t + 3, res.first[i].t);
    }
    BundleReport& R = res.second;
    R.initial_cost = r.initial_cost;
    R.final_cost = r.final_cost;
    R.iterations = r.iterations;
    R.accepted = r.accepted;
    R.cg_iterations = r.cg_iterations;
    R.termination = r.termination;
    R.n_obs = r.n_obs;
    R.n_points = r.n_points;
    R.n_free_cams = r.n_free_cams;
    return res;
}

Rotations rotationAveraging(int n_sets, const std::vector<std::pair<int, int>>& pairs, const std::vector<TwoViewPose>& poses,
                            const RotationParams& params)
{
    const std::string who = "popsift::rotationAveraging";
    if (n_sets < 0) throw std::runtime_error(who + ": n_sets < 0");
    if (poses.size() != pairs.size()) throw std::runtime_error(who + ": one relative pose per pair expected");
    const size_t np = pairs.size();
    std::vector<ps_two_view> rec(np);
    std::vector<int32_t> flat(2 * np);
    for (size_t p = 0; p < np; ++p) {
        rec[p] = ps_two_view{};
        std::copy(poses[p].R, poses[p].R + 9, rec[p].R);
        std::copy(poses[p].t, poses[p].t + 3, rec[p].t);
        rec[p].n_inliers = poses[p].n_inliers;
        rec[p].n_front = poses[p].n_front;
        flat[2 * p] = pairs[p].first;
        flat[2 * p + 1] = pairs[p].second;
    }
    DevBuf d(std::max<size_t>(np, 1) * sizeof(ps_two_view), who);
    if (np) check(ps_host_to_dev(d.p, rec.data(), np * sizeof(ps_two_view)), who);
    ps_rotation_params prm{};
    prm.loss = params.loss;
    prm.max_iters = params.max_iters;
    prm.cg_max_iters = params.cg_max_iters;
    prm.min_inliers = params.min_inliers;
    prm.loss_scale = params.loss_scale;
    prm.step_tol = params.step_tol;
    prm.cg_tol = params.cg_tol;
    std::vector<double> R(9 * (size_t)std::max(n_sets, 1));
    std::vector<uint8_t> reg(std::max(n_sets, 1));
    Rotations out;
    out.pair_error.resize(np);
    ps_rotation_report r;
    check(ps_rotation_averaging(0, n_sets, (int)np, flat.data(), static_cast<const ps_two_view*>(d.p), &prm, R.data(), reg.data(),
                                out.pair_error.data(), &r),
          who, "ps_rotation_averaging");
    out.R.resize(n_sets);
    out.registered.resize(n_sets);
    for (int i = 0; i < n_sets; ++i) {
        std::copy(&R[9 * (size_t)i], &R[9 * (size_t)i] + 9, out.R[i].R);
        out.registered[i] = reg[i] != 0;
    }
    RotationReport& o = out.report;
    o.initial_cost = r.initial_cost;
    o.final_cost = r.final_cost;
    o.iterations = r.iterations;
    o.cg_iterations = r.cg_iterations;
    o.n_pairs = r.n_pairs;
    o.n_registered = r.n_registered;
    o.termination = r.termination;
    return out;
}

// the C ABI arguments of a depth call: images, cameras, poses, refs and the source CSR
struct DepthCall {
    std::vector<ps_image> img;
    std::vector<ps_camera> cam;
    std::vector<ps_rigid> pose;
    std::vector<int32_t> refs, start, src;
    DepthCall(const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
              const std::vector<int>& r, const std::vector<std::vector<int>>& sources, const std::string& who)
    {
        if (cameras.size() != images.size() || poses.size() != images.size())
            throw std::runtime_error(who + ": one camera and one pose per image expected");
        if (sources.size() != r.size()) throw std::runtime_error(who + ": one source list per reference expected");
        for (const DeviceImage& im : images) img.push_back(ps_image{im.data, im.pitch, im.width, im.height});
        for (const Camera& c : cameras) cam.push_back(ps_camera{c.fx, c.fy, c.cx, c.cy});
        for (const Rigid& p : poses) {
            ps_rigid q;
            std::copy(p.R, p.R + 9, q.R);
            std::copy(p.t, p.t + 3, q.t);
            pose.push_back(q);
        }
        refs.assign(r.begin(), r.end());
        start.push_back(0);
        for (const auto& s : sources) {
            src.insert(src.end(), s.begin(), s.end());
            start.push_back((int32_t)src.size());
        }
    }
    // the reference's image size, 0 x 0 for an index the C ABI refuses
    std::pair<int, int> size(size_t j) const
    {
        const int r = refs[j];
        return r >= 0 && r < (int)img.size() ? std::make_pair(img[r].width, img[r].height) : std::make_pair(0, 0);
    }
};

DepthMaps depthMaps(const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
                    const std::vector<int>& refs, const std::vector<std::vector<int>>& sources,
                    const std::vector<std::pair<float, float>>& ranges, const DepthParams& params, int device)
{
    const std::string who = "popsift::depthMaps";
    const DepthCall a(images, cameras, poses, refs, sources, who);
    if (ranges.size() != refs.size()) throw std::runtime_error(who + ": one depth range per reference expected");
    const size_t nr = refs.size();
    std::vector<float> rng;
    for (const auto& r : ranges) rng.insert(rng.end(), {r.first, r.second});
    std::vector<std::unique_ptr<DevBuf>> bufs;
    std::vector<float*> d_depth, d_cost;
    std::vector<uint8_t*> d_nsrc;
    for (size_t j = 0; j < nr; ++j) {
        const auto wh = a.size(j);
        const size_t n = (size_t)wh.first * wh.second;
        bufs.emplace_back(new DevBuf(n * 4, who));
        d_depth.push_back(static_cast<float*>(bufs.back()->p));
        bufs.emplace_back(new DevBuf(n * 4, who));
        d_cost.push_back(static_cast<float*>(bufs.back()->p));
        bufs.emplace_back(new DevBuf(n, who));
        d_nsrc.push_back(static_cast<uint8_t*>(bufs.back()->p));
    }
    const ps_depth_params prm{params.n_depths, params.radius, params.top_k, params.min_sources, params.max_cost, params.min_var};
    ps_depth_report rep;
    check(ps_depth_maps(device, (int)images.size(), a.img.data(), a.cam.data(), a.pose.data(), (int)nr, a.refs.data(), rng.data(),
                        a.start.data(), a.src.data(), &prm, d_depth.data(), d_cost.data(), d_nsrc.data(), &rep),
          who, "ps_depth_maps");
    DepthMaps out;
    out.n_candidates = rep.n_candidates;
    out.n_depths = rep.n_depths;
    out.maps.resize(nr);
    for (size_t j = 0; j < nr; ++j) {
        DepthMap& m = out.maps[j];
        m.width = a.size(j).first;
        m.height = a.size(j).second;
        const size_t n = (size_t)m.width * m.height;
        m.depth.resize(n);
        m.cost.resize(n);
        m.n_src.resize(n);
        check(ps_dev_to_host(m.depth.data(), d_depth[j], n * 4), who);
        check(ps_dev_to_host(m.cost.data(), d_cost[j], n * 4), who);
        check(ps_dev_to_host(m.n_src.data(), d_nsrc[j], n), who);
    }
    return out;
}

DensePoints filterDepthMaps(const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
                            const std::vector<int>& refs, const std::vector<std::vector<int>>& sources, const DepthMaps& maps,
                            const DepthFilterParams& params, int device)
{
    const std::string who = "popsift::filterDepthMaps";
    const DepthCall a(images, cameras, poses, refs, sources, who);
    const size_t nr = refs.size();
    if (maps.maps.size() != nr) throw std::runtime_error(who + ": one depth map per reference expected");
    std::vector<std::unique_ptr<DevBuf>> bufs;
    std::vector<const float*> d_depth;
    std::vector<uint8_t*> d_nc;
    size_t cap = 0;
    for (size_t j = 0; j < nr; ++j) {
        const DepthMap& m = maps.maps[j];
        const size_t n = (size_t)m.width * m.height;
        if (a.size(j) != std::make_pair(m.width, m.height) || m.depth.size() != n)
            throw std::runtime_error(who + ": a depth map does not match its reference image");
        bufs.emplace_back(new DevBuf(n * 4, who));
        if (n) check(ps_host_to_dev(bufs.back()->p, m.depth.data(), n * 4), who);
        d_depth.push_back(static_cast<const float*>(bufs.back()->p));
        bufs.emplace_back(new DevBuf(n, who));
        d_nc.push_back(static_cast<uint8_t*>(bufs.back()->p));
        cap += n;
    }
    DevBuf d_pts(cap * sizeof(ps_dense_point), who);
    const ps_depth_filter_params prm{params.max_reproj_error, params.max_depth_diff, params.min_consistent, 0};
    ps_depth_filter_report rep;
    check(ps_depth_filter(device, (int)images.size(), a.img.data(), a.cam.data(), a.pose.data(), (int)nr, a.refs.data(), a.start.data(),
                          a.src.data(), d_depth.data(), &prm, d_nc.data(), static_cast<ps_dense_point*>(d_pts.p), &rep),
          who, "ps_depth_filter");
    DensePoints out;
    out.n_tested = rep.n_tested;
    out.n_consistent.resize(nr);
    for (size_t j = 0; j < nr; ++j) {
        out.n_consistent[j].resize(maps.maps[j].depth.size());
        check(ps_dev_to_host(out.n_consistent[j].data(), d_nc[j], out.n_consistent[j].size()), who);
    }
    std::vector<ps_dense_point> pts((size_t)rep.n_points);
    if (!pts.empty()) check(ps_dev_to_host(pts.data(), d_pts.p, pts.size() * sizeof(ps_dense_point)), who);
    out.points.resize(pts.size());
    for (size_t i = 0; i < pts.size(); ++i) {
        DensePoint& q = out.points[i];
        std::copy(pts[i].X, pts[i].X + 3, q.X);
        q.ref = pts[i].ref;
        q.x = pts[i].x;
        q.y = pts[i].y;
        q.n_consistent = pts[i].n_consistent;
        q.grey = pts[i].grey;
    }
    return out;
}

namespace {

ps_volume c_volume(const DeviceVolume& v)
{
    ps_volume c;
    std::copy(v.origin(), v.origin() + 3, c.origin);
    c.voxel = v.voxel();
    c.nx = v.nx();
    c.ny = v.ny();
    c.nz = v.nz();
    c.pad_ = 0;
    c.tsdf = v.tsdf();
    c.weight = v.weight();
    c.grey = v.grey();
    return c;
}

} // namespace

DeviceVolume::DeviceVolume(const double origin[3], double voxel, int nx, int ny, int nz, int device)
    : _voxel(voxel), _n{nx, ny, nz}, _device(device)
{
    const std::string who = "popsift::DeviceVolume";
    std::copy(origin, origin + 3, _origin);
    if (nx < 2 || ny < 2 || nz < 2 || nx > 2048 || ny > 2048 || nz > 2048)
        throw std::runtime_error(who + ": dimensions must lie in 2 .. 2048");
    const size_t bytes = (size_t)nx * ny * nz * sizeof(float);
    _tsdf = static_cast<float*>(ps_dev_alloc(bytes));
    _weight = static_cast<float*>(ps_dev_alloc(bytes));
    _grey = static_cast<float*>(ps_dev_alloc(bytes));
    try {
        if (!_tsdf || !_weight || !_grey) throw std::runtime_error(who + ": failed to allocate device memory");
        clearVolume(*this);
    } catch (...) {
        ps_dev_free(_tsdf);
        ps_dev_free(_weight);
        ps_dev_free(_grey);
        throw;
    }
}

DeviceVolume::~DeviceVolume()
{
    ps_dev_free(_tsdf);
    ps_dev_free(_weight);
    ps_dev_free(_grey);
}

void clearVolume(DeviceVolume& volume)
{
    const ps_volume c = c_volume(volume);
    check(ps_volume_clear(volume.device(), &c), "popsift::clearVolume", "ps_volume_clear");
}

TsdfReport integrateDepthMaps(DeviceVolume& volume, const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras,
                              const std::vector<Rigid>& poses, const std::vector<DepthMap>& maps,
                              const std::vector<std::vector<std::uint8_t>>& masks, const TsdfParams& params)
{
    const std::string who = "popsift::integrateDepthMaps";
    const size_t n = images.size();
    if (cameras.size() != n || poses.size() != n || maps.size() != n)
        throw std::runtime_error(who + ": one camera, one pose and one depth map per image expected");
    const bool use_masks = params.min_consistent > 0;
    if (use_masks && masks.size() != n) throw std::runtime_error(who + ": one mask per image expected");
    // the images, cameras and poses in the C ABI's layouts (DepthCall with every set its own reference)
    std::vector<int> refs(n);
    for (size_t v = 0; v < n; ++v) refs[v] = (int)v;
    const DepthCall a(images, cameras, poses, refs, std::vector<std::vector<int>>(n), who);
    std::vector<std::unique_ptr<DevBuf>> bufs;
    std::vector<const float*> d_depth;
    std::vector<const uint8_t*> d_mask;
    for (size_t v = 0; v < n; ++v) {
        const size_t px = (size_t)std::max(images[v].width, 0) * (size_t)std::max(images[v].height, 0);
        if (maps[v].width != images[v].width || maps[v].height != images[v].height || maps[v].depth.size() != px)
            throw std::runtime_error(who + ": a depth map does not match its image");
        bufs.emplace_back(new DevBuf(px * 4, who));
        if (px) check(ps_host_to_dev(bufs.back()->p, maps[v].depth.data(), px * 4), who);
        d_depth.push_back(static_cast<const float*>(bufs.back()->p));
        if (use_masks) {
            if (masks[v].size() != px) throw std::runtime_error(who + ": a mask does not match its image");
            bufs.emplace_back(new DevBuf(px, who));
            if (px) check(ps_host_to_dev(bufs.back()->p, masks[v].data(), px), who);
            d_mask.push_back(static_cast<const uint8_t*>(bufs.back()->p));
        }
    }
    const ps_volume c = c_volume(volume);
    const ps_tsdf_params prm{params.trunc, params.min_consistent};
    ps_tsdf_report rep;
    check(ps_tsdf_integrate(volume.device(), (int)n, a.img.data(), a.cam.data(), a.pose.data(), d_depth.data(),
                            use_masks ? d_mask.data() : nullptr, &prm, &c, &rep),
          who, "ps_tsdf_integrate");
    TsdfReport out;
    out.n_updates = rep.n_updates;
    out.n_voxels_touched = rep.n_voxels_touched;
    return out;
}

Mesh extractMesh(const DeviceVolume& volume, const MeshParams& params)
{
    const std::string who = "popsift::extractMesh";
    const ps_volume c = c_volume(volume);
    const ps_mesh_params prm{params.min_weight, 0};
    ps_mesh_report rep;
    const int rc = ps_tsdf_mesh(volume.device(), &c, &prm, 0, 0, nullptr, nullptr, &rep);
    if (rc != PS_ERR_OVERFLOW) check(rc, who, "ps_tsdf_mesh");
    Mesh out;
    out.n_cells = rep.n_cells;
    if (rc == PS_OK) return out;   // no triangles
    if (rep.n_vertices < 0 || rep.n_vertices >= 0x80000000LL)
        throw std::runtime_error(who + ": the mesh has 2^31 vertices or more");
    DevBuf d_v((size_t)rep.n_vertices * sizeof(ps_mesh_vertex), who), d_t((size_t)rep.n_triangles * 3 * sizeof(int32_t), who);
    check(ps_tsdf_mesh(volume.device(), &c, &prm, rep.n_vertices, rep.n_triangles, static_cast<ps_mesh_vertex*>(d_v.p),
                       static_cast<int32_t*>(d_t.p), &rep),
          who, "ps_tsdf_mesh");
    out.vertices.resize((size_t)rep.n_vertices);
    out.triangles.resize((size_t)rep.n_triangles * 3);
    static_assert(sizeof(MeshVertex) == sizeof(ps_mesh_vertex), "vertex layout");
    if (!out.vertices.empty()) check(ps_dev_to_host(out.vertices.data(), d_v.p, out.vertices.size() * sizeof(MeshVertex)), who);
    if (!out.triangles.empty()) check(ps_dev_to_host(out.triangles.data(), d_t.p, out.triangles.size() * sizeof(int)), who);
    return out;
}

namespace {

// a mesh on the device for the render calls
struct DeviceMesh {
    DevBuf v, t;
    int64_t nv, nt;
    DeviceMesh(const Mesh& mesh, const std::string& who)
        : v(mesh.vertices.size() * sizeof(ps_mesh_vertex), who), t(mesh.triangles.size() * sizeof(int32_t), who),
          nv((int64_t)mesh.vertices.size()), nt((int64_t)mesh.triangles.size() / 3)
    {
        if (mesh.triangles.size() % 3) throw std::runtime_error(who + ": three vertex indices per triangle expected");
        if (nv) check(ps_host_to_dev(v.p, mesh.vertices.data(), (size_t)nv * sizeof(ps_mesh_vertex)), who);
        if (nt) check(ps_host_to_dev(t.p, mesh.triangles.data(), (size_t)nt * 3 * sizeof(int32_t)), who);
    }
};

std::vector<ps_camera> c_cameras(const std::vector<Camera>& cameras)
{
    std::vector<ps_camera> out;
    for (const Camera& c : cameras) out.push_back(ps_camera{c.fx, c.fy, c.cx, c.cy});
    return out;
}

std::vector<ps_rigid> c_rigids(const std::vector<Rigid>& poses)
{
    std::vector<ps_rigid> out(poses.size());
    for (size_t i = 0; i < poses.size(); ++i) {
        std::copy(poses[i].R, poses[i].R + 9, out[i].R);
        std::copy(poses[i].t, poses[i].t + 3, out[i].t);
    }
    return out;
}

// ps_mesh_render into device maps (bufs: depth, triangle per view)
ps_render_report render_dev(const DeviceMesh& m, const std::vector<ps_camera>& cam, const std::vector<ps_rigid>& pose,
                            const std::vector<int32_t>& sizes, float z_near, std::vector<std::unique_ptr<DevBuf>>& bufs,
                            std::vector<float*>& d_depth, std::vector<int32_t*>& d_tri, int device, const std::string& who)
{
    const size_t n = cam.size();
    for (size_t v = 0; v < n; ++v) {
        const size_t px = (size_t)std::max(sizes[2 * v], 0) * (size_t)std::max(sizes[2 * v + 1], 0);
        bufs.emplace_back(new DevBuf(px * 4, who));
        d_depth.push_back(static_cast<float*>(bufs.back()->p));
        bufs.emplace_back(new DevBuf(px * 4, who));
        d_tri.push_back(static_cast<int32_t*>(bufs.back()->p));
    }
    const ps_render_params prm{z_near, 0};
    ps_render_report rep;
    check(ps_mesh_render(device, (int)n, sizes.data(), cam.data(), pose.data(), static_cast<const ps_mesh_vertex*>(m.v.p), m.nv,
                         static_cast<const int32_t*>(m.t.p), m.nt, &prm, d_depth.data(), d_tri.data(), &rep),
          who, "ps_mesh_render");
    return rep;
}

} // namespace

RenderedMesh renderMesh(const Mesh& mesh, const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
                        const std::vector<std::pair<int, int>>& sizes, const RenderParams& params, int device)
{
    const std::string who = "popsift::renderMesh";
    const size_t n = sizes.size();
    if (cameras.size() != n || poses.size() != n) throw std::runtime_error(who + ": one camera, one pose and one size per view expected");
    static_assert(sizeof(MeshVertex) == sizeof(ps_mesh_vertex), "vertex layout");
    const DeviceMesh m(mesh, who);
    std::vector<int32_t> sz;
    for (const auto& s : sizes) sz.insert(sz.end(), {s.first, s.second});
    std::vector<std::unique_ptr<DevBuf>> bufs;
    std::vector<float*> d_depth;
    std::vector<int32_t*> d_tri;
    const ps_render_report rep = render_dev(m, c_cameras(cameras), c_rigids(poses), sz, params.z_near, bufs, d_depth, d_tri, device, who);
    RenderedMesh out;
    out.n_drawn = rep.n_drawn;
    out.n_big = rep.n_big;
    out.n_covered = rep.n_covered;
    out.maps.resize(n);
    for (size_t v = 0; v < n; ++v) {
        RenderMap& r = out.maps[v];
        r.width = sizes[v].first;
        r.height = sizes[v].second;
        const size_t px = (size_t)r.width * r.height;
        r.depth.resize(px);
        r.triangle.resize(px);
        check(ps_dev_to_host(r.depth.data(), d_depth[v], px * 4), who);
        check(ps_dev_to_host(r.triangle.data(), d_tri[v], px * 4), who);
    }
    return out;
}

TexturedMesh textureMesh(const Mesh& mesh, const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras,
                         const std::vector<Rigid>& poses, const TextureParams& params, int device)
{
    const std::string who = "popsift::textureMesh";
    const size_t n = images.size();
    if (cameras.size() != n || poses.size() != n) throw std::runtime_error(who + ": one camera and one pose per image expected");
    const DeviceMesh m(mesh, who);
    const std::vector<ps_camera> cam = c_cameras(cameras);
    const std::vector<ps_rigid> pose = c_rigids(poses);
    std::vector<ps_image> img;
    std::vector<int32_t> sz;
    for (const DeviceImage& im : images) {
        img.push_back(ps_image{im.data, im.pitch, im.width, im.height});
        sz.insert(sz.end(), {im.width, im.height});
    }
    std::vector<std::unique_ptr<DevBuf>> bufs;
    std::vector<float*> d_depth;
    std::vector<int32_t*> d_tri;
    render_dev(m, cam, pose, sz, params.z_near, bufs, d_depth, d_tri, device, who);
    TexturedMesh out;
    out.cell = params.cell;
    out.cells_per_row = params.cells_per_row;
    if (out.cells_per_row == 0 && params.cell > 0)
        out.cells_per_row = std::max(1, std::min((int)std::ceil(std::sqrt((double)std::max<int64_t>(m.nt, 1))), 65535 / params.cell));
    if (out.cells_per_row < 1) throw std::runtime_error(who + ": cells_per_row must be >= 1");
    out.width = out.cells_per_row * params.cell;
    out.height = (int)((m.nt + out.cells_per_row - 1) / out.cells_per_row) * params.cell;
    DevBuf d_atlas((size_t)std::max(out.width, 0) * std::max(out.height, 0), who), d_view((size_t)m.nt * 4, who);
    const ps_texture_params prm{params.cell, out.cells_per_row, params.depth_tol, params.min_cos, params.z_near, 0};
    ps_texture_report rep;
    std::vector<const float*> c_depth(d_depth.begin(), d_depth.end());
    check(ps_mesh_texture(device, (int)n, img.data(), cam.data(), pose.data(), c_depth.data(), static_cast<const ps_mesh_vertex*>(m.v.p), m.nv,
                          static_cast<const int32_t*>(m.t.p), m.nt, &prm, static_cast<uint8_t*>(d_atlas.p), static_cast<int32_t*>(d_view.p),
                          &rep),
          who, "ps_mesh_texture");
    out.n_viewed = rep.n_viewed;
    out.n_fallback = rep.n_fallback;
    out.atlas.resize((size_t)out.width * out.height);
    out.view.resize((size_t)m.nt);
    if (!out.atlas.empty()) check(ps_dev_to_host(out.atlas.data(), d_atlas.p, out.atlas.size()), who);
    if (!out.view.empty()) check(ps_dev_to_host(out.view.data(), d_view.p, out.view.size() * 4), who);
    return out;
}

ViewGraph filterViewGraph(int n_sets, const std::vector<std::pair<int, int>>& pairs, const std::vector<TwoViewPose>& poses,
                          const ViewGraphParams& params)
{
    const std::string who = "popsift::filterViewGraph";
    if (n_sets < 0) throw std::runtime_error(who + ": n_sets < 0");
    if (poses.size() != pairs.size()) throw std::runtime_error(who + ": one relative pose per pair expected");
    const size_t np = pairs.size();
    std::vector<ps_two_view> rec(np);
    std::vector<int32_t> flat(2 * np);
    for (size_t p = 0; p < np; ++p) {
        rec[p] = ps_two_view{};
        std::copy(poses[p].R, poses[p].R + 9, rec[p].R);
        std::copy(poses[p].t, poses[p].t + 3, rec[p].t);
        rec[p].n_inliers = poses[p].n_inliers;
        rec[p].n_front = poses[p].n_front;
        flat[2 * p] = pairs[p].first;
        flat[2 * p + 1] = pairs[p].second;
    }
    DevBuf d(std::max<size_t>(np, 1) * sizeof(ps_two_view), who);
    if (np) check(ps_host_to_dev(d.p, rec.data(), np * sizeof(ps_two_view)), who);
    ps_view_graph_params prm{};
    prm.min_inliers = params.min_inliers;
    prm.min_consistent = params.min_consistent;
    prm.keep_untested = params.keep_untested ? 1 : 0;
    prm.max_cycle_error = params.max_cycle_error;
    prm.min_fraction = params.min_fraction;
    std::vector<uint8_t> keep(std::max<size_t>(np, 1));
    std::vector<ps_cycle_stats> cs(std::max<size_t>(np, 1));
    ps_view_graph_report r;
    check(ps_view_graph_filter(0, n_sets, (int)np, flat.data(), static_cast<const ps_two_view*>(d.p), &prm, keep.data(), cs.data(), nullptr,
                               &r),
          who, "ps_view_graph_filter");
    ViewGraph out;
    out.keep.resize(np);
    out.stats.resize(np);
    for (size_t p = 0; p < np; ++p) {
        out.keep[p] = keep[p] != 0;
        out.stats[p].n_triangles = cs[p].n_triangles;
        out.stats[p].n_consistent = cs[p].n_consistent;
        out.stats[p].min_error = cs[p].min_error;
    }
    ViewGraphReport& o = out.report;
    o.n_triangles = r.n_triangles;
    o.n_consistent_triangles = r.n_consistent_triangles;
    o.n_used = r.n_used;
    o.n_kept = r.n_kept;
    o.n_untested = r.n_untested;
    return out;
}

Positions globalPositioning(const std::vector<FeaturesDev*>& sets, const Tracks& tracks, const std::vector<Camera>& cameras,
                            const std::vector<Rigid>& rotations, const std::vector<bool>& registered, const PositionParams& params)
{
    const Batch b("globalPositioning", sets, {});
    if (cameras.size() != sets.size()) throw std::runtime_error(b.who + ": one camera per set expected");
    if (rotations.size() != sets.size() || registered.size() != sets.size())
        throw std::runtime_error(b.who + ": one rotation and one registered flag per set expected");
    if (tracks.start.empty() || tracks.set.size() != tracks.feature.size() || (size_t)tracks.start.back() != tracks.set.size())
        throw std::runtime_error(b.who + ": malformed tracks");
    std::vector<int32_t> n_feat(sets.size());
    std::vector<int64_t> off(sets.size() + 1, 0);
    for (size_t i = 0; i < sets.size(); ++i) {
        n_feat[i] = sets[i]->getFeatureCount();
        off[i + 1] = off[i] + std::max(n_feat[i], 0);
    }
    const size_t nt = tracks.start.size() - 1, nm = tracks.set.size();
    std::vector<int32_t> mem(nm);
    for (size_t k = 0; k < nm; ++k) {
        const int s = tracks.set[k], f = tracks.feature[k];
        if (s < 0 || (size_t)s >= sets.size() || f < 0 || f >= n_feat[s]) throw std::runtime_error(b.who + ": track member out of range");
        mem[k] = (int32_t)(off[s] + f);
    }
    std::vector<ps_camera> cams(sets.size());
    std::vector<double> R(9 * std::max<size_t>(sets.size(), 1));
    std::vector<uint8_t> reg(std::max<size_t>(sets.size(), 1)), pos(std::max<size_t>(sets.size(), 1));
    std::vector<ps_rigid> rig(std::max<size_t>(sets.size(), 1));
    for (size_t i = 0; i < sets.size(); ++i) {
        cams[i] = ps_camera{cameras[i].fx, cameras[i].fy, cameras[i].cx, cameras[i].cy};
        std::copy(rotations[i].R, rotations[i].R + 9, &R[9 * i]);
        reg[i] = registered[i] ? 1 : 0;
    }
    ps_position_params prm{};
    prm.loss = params.loss;
    prm.max_iters = params.max_iters;
    prm.cg_max_iters = params.cg_max_iters;
    prm.loss_scale = params.loss_scale;
    prm.function_tol = params.function_tol;
    prm.cg_tol = params.cg_tol;
    DevBuf start(tracks.start.size() * sizeof(int32_t), b.who), members(nm * sizeof(int32_t), b.who), X(nt * 3 * sizeof(double), b.who);
    check(ps_host_to_dev(start.p, tracks.start.data(), tracks.start.size() * sizeof(int32_t)), b.who);
    check(ps_host_to_dev(members.p, mem.data(), nm * sizeof(int32_t)), b.who);
    ps_position_report r;
    check(ps_global_positioning(b.dev, (int)sets.size(), n_feat.data(), b.feat.data(), cams.data(), R.data(), reg.data(), (int)nt,
                                static_cast<const int32_t*>(start.p), static_cast<const int32_t*>(members.p), (int)nm, &prm, rig.data(),
                                pos.data(), static_cast<double*>(X.p), &r),
          b.who, "ps_global_positioning");
    Positions out;
    out.X.resize(3 * nt);
    check(ps_dev_to_host(out.X.data(), X.p, 3 * nt * sizeof(double)), b.who);
    out.poses.resize(sets.size());
    out.positioned.resize(sets.size());
    for (size_t i = 0; i < sets.size(); ++i) {
        std::copy(rig[i].R, rig[i].R + 9, out.poses[i].R);
        std::copy(rig[i].t, rig[i].t + 3, out.poses[i].t);
        out.positioned[i] = pos[i] != 0;
    }
    PositionReport& o = out.report;
    o.initial_cost = r.initial_cost;
    o.final_cost = r.final_cost;
    o.iterations = r.iterations;
    o.cg_iterations = r.cg_iterations;
    o.n_obs = r.n_obs;
    o.n_points = r.n_points;
    o.n_cams = r.n_cams;
    o.termination = r.termination;
    return out;
}

} // namespace popsift
