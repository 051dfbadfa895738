// PopSift / SiftJob -- the reference's job pipeline (reference src/popsift/popsift.cpp:25-503)
// re-designed for many images in flight:
//
//   caller thread --enqueue--> job queue --> ONE worker thread per PopSift:
//        slot = next in round robin; if that slot still holds a job: finish it
//        (ps_counts + ps_download -> promise); ps_submit_* the new job (asynchronous: H2D + all
//        kernels on the slot's stream); when the queue runs dry, finish the remaining slots in order.
//
// Jobs therefore complete in FIFO order like the reference's, but `slots` images overlap on the
// GPU (upload of n+1 and kernels of n+1 run while the results of n are downloaded), where the
// reference has one image on the device at a time and >= 8 host synchronisations per image.
// The device context is created on the first image (or re-created when a larger image arrives),
// and the octave count is fixed by the first image exactly like the reference
// (popsift.cpp:118-122 writes it back into the stored Config).
#include "popsift/popsift.h"
#include "popsift_b200.h"
#include "pinned_pool.h"
#include "log_dump.h"

#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <iostream>
#include <mutex>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

using popsift::Config;

// ---------------------------------------------------------------- SiftJob

SiftJob::SiftJob(int w, int h, const unsigned char* imageData) : _w(w), _h(h), _isFloat(false)
{
    _f = _p.get_future();
    const size_t n = (size_t)w * h;
    // page-locked copy: ps_submit_* then DMA-copies straight from it (one host copy instead of the
    // reference's two, popsift.cpp:392-395 + s_image.cu:75)
    _imageData = static_cast<unsigned char*>(popsift::detail::pinned_pool().get(n ? n : 1));
    if (!_imageData) throw std::runtime_error("Memory limitation\nE    Failed to allocate memory for SiftJob");
    popsift::detail::parallel_copy(_imageData, imageData, n);
}

SiftJob::SiftJob(int w, int h, const float* imageData) : _w(w), _h(h), _isFloat(true)
{
    _f = _p.get_future();
    const size_t n = (size_t)w * h * sizeof(float);
    // page-locked copy: ps_submit_* then DMA-copies straight from it (one host copy instead of the
    // reference's two, popsift.cpp:392-395 + s_image.cu:75)
    _imageData = static_cast<unsigned char*>(popsift::detail::pinned_pool().get(n ? n : 1));
    if (!_imageData) throw std::runtime_error("Memory limitation\nE    Failed to allocate memory for SiftJob");
    popsift::detail::parallel_copy(_imageData, imageData, n);
}

static_assert(sizeof(popsift::Keypoint) == sizeof(ps_keypoint) && sizeof(popsift::Keypoint) == 24, "popsift::Keypoint is ps_keypoint");

SiftJob::SiftJob(int w, int h, const unsigned char* imageData, const std::vector<popsift::Keypoint>& kps, bool computeOrientations)
    : SiftJob(w, h, imageData)
{
    _describe = computeOrientations ? PS_DESCRIBE_ORIENT : PS_DESCRIBE_GIVEN;
    _keypoints = kps;
}

SiftJob::SiftJob(int w, int h, const float* imageData, const std::vector<popsift::Keypoint>& kps, bool computeOrientations)
    : SiftJob(w, h, imageData)
{
    _describe = computeOrientations ? PS_DESCRIBE_ORIENT : PS_DESCRIBE_GIVEN;
    _keypoints = kps;
}

SiftJob::~SiftJob() { popsift::detail::pinned_pool().put(_imageData); }

void SiftJob::setFeatures(popsift::FeaturesBase* f) { _p.set_value(f); }
void SiftJob::setError(std::exception_ptr ptr) { _err = ptr; }

popsift::FeaturesBase* SiftJob::getBase()
{
    popsift::FeaturesBase* f = _f.get();
    if (_err) std::rethrow_exception(_err);
    return f;
}
popsift::FeaturesHost* SiftJob::getHost() { return dynamic_cast<popsift::FeaturesHost*>(getBase()); }
popsift::FeaturesHost* SiftJob::get() { return getHost(); }
popsift::FeaturesDev* SiftJob::getDev() { return dynamic_cast<popsift::FeaturesDev*>(getBase()); }

// ---------------------------------------------------------------- PopSift::Pipe

struct PopSift::Pipe
{
    std::mutex                mu;
    std::condition_variable   cv;
    std::deque<SiftJob*>      queue;
    bool                      stop = false;
    std::thread               worker;

    // ctx and in_slot belong to the worker thread alone; what configure()/setSlots() need to know about them
    // is published through `started` (set under `mu` before the first context is created)
    ps_ctx*                   ctx = nullptr;
    bool                      started = false;
    int                       ctx_w = 0, ctx_h = 0;
    int                       slots = 4;
    std::vector<SiftJob*>     in_slot;
    int                       next_slot = 0;
    bool                      octaves_fixed = false;
    bool                      log_all = false;      // Config::LogMode::All, fixed when the context is created
    int                       log_levels = 3;
    bool                      tables_printed = false; // --print-gauss-tables: once per PopSift
    float                     log_upscale = 1.0f;
};

namespace {

void fail_job(SiftJob* job, const std::string& msg)
{
    job->setError(std::make_exception_ptr(std::runtime_error(msg)));
    job->setFeatures(nullptr);
}

} // namespace

PopSift::PopSift(ImageMode imode, int device) : _pipe(new Pipe), _image_mode(imode), _device(device)
{
    Pipe* p = _pipe.get();
    p->worker = std::thread([this, p] {
        auto finish = [&](int s) {
            SiftJob* job = p->in_slot[s];
            if (!job) return;
            p->in_slot[s] = nullptr;
            int32_t nf = 0, nd = 0;
            int rc = ps_counts(p->ctx, s, &nf, &nd);
            if (rc != PS_OK && rc != PS_ERR_OVERFLOW) { fail_job(job, ps_last_error(p->ctx)); return; }
            if (rc == PS_ERR_OVERFLOW) std::cerr << "popsift_b200 warning: " << ps_last_error(p->ctx) << std::endl;
            if (_proc_mode == Config::MatchingMode) {
                // device-resident results (reference popsift.cpp:346-383, sift_pyramid.cu:324-362)
                popsift::FeaturesDev* fd = nullptr;
                try {
                    fd = new popsift::FeaturesDev(nf, nd);
                    rc = ps_download_dev(p->ctx, s, reinterpret_cast<ps_feature*>(fd->getFeatures()),
                                         reinterpret_cast<ps_descriptor*>(fd->getDescriptors()), fd->getReverseMap());
                    if (rc != PS_OK) { delete fd; fail_job(job, ps_last_error(p->ctx)); return; }
                } catch (const std::exception& e) { delete fd; fail_job(job, e.what()); return; }
                job->setFeatures(fd);
                return;
            }
            popsift::FeaturesHost* fh = nullptr;
            try {
                fh = new popsift::FeaturesHost(nf, nd);
                rc = ps_download(p->ctx, s, reinterpret_cast<ps_feature*>(fh->getFeatures()),
                                 reinterpret_cast<ps_descriptor*>(fh->getDescriptors()));
                if (rc != PS_OK) { delete fh; fail_job(job, ps_last_error(p->ctx)); return; }
                if (p->log_all) {
                    // --log (reference popsift.cpp:330-337): plane and descriptor dumps of this image
                    popsift::detail::dump_slot_planes(p->ctx, s, p->log_levels, "pyramid");
                    popsift::detail::dump_descriptors(*fh, p->log_upscale, "pyramid");
                }
            } catch (const std::exception& e) { delete fh; fail_job(job, e.what()); return; }
            job->setFeatures(fh);
        };
        auto finish_all = [&] {
            if (!p->ctx) return;
            for (int i = 0; i < (int)p->in_slot.size(); ++i) finish((p->next_slot + i) % (int)p->in_slot.size());
        };
        for (;;) {
            SiftJob* job = nullptr;
            {
                std::unique_lock<std::mutex> lk(p->mu);
                if (p->queue.empty() && !p->stop) {
                    // nothing to submit: drain what is in flight, then sleep
                    lk.unlock();
                    finish_all();
                    lk.lock();
                    p->cv.wait(lk, [&] { return !p->queue.empty() || p->stop; });
                }
                if (p->queue.empty() && p->stop) break;
                job = p->queue.front();
                p->queue.pop_front();
            }
            const int w = job->width(), h = job->height();
            if (!p->ctx || w > p->ctx_w || h > p->ctx_h) {
                finish_all();
                if (p->ctx) { ps_destroy(p->ctx); p->ctx = nullptr; }
                ps_config c;
                int slots;
                bool print_tables = false;
                {
                    // _config and slots are written by configure()/setSlots() on caller threads: read (and fix
                    // the octave count) under the same mutex; from here on configure() refuses changes
                    std::lock_guard<std::mutex> lk(p->mu);
                    p->started = true;
                    if (!p->octaves_fixed) {
                        // first image fixes the octave count (reference popsift.cpp:118-122)
                        _config.toC(c);
                        if (c.octaves < 0) { const int n = ps_geometry(&c, w, h, nullptr, nullptr); if (n > 0) _config.octaves = n; }
                        p->octaves_fixed = true;
                    }
                    _config.toC(c);
                    slots = p->slots;
                    p->log_all = _config.getLogMode() == Config::All;
                    p->log_levels = std::max(2, _config.levels);
                    p->log_upscale = _config.getUpscaleFactor();
                    print_tables = _config.ifPrintGaussTables() && !p->tables_printed;
                    p->tables_printed = p->tables_printed || print_tables;
                }
                p->ctx_w = std::max(w, p->ctx_w); p->ctx_h = std::max(h, p->ctx_h);
                if (print_tables) {
                    // Config::setPrintGaussTables() (reference gauss_filter.cu:24-121,146-161,247-256): once, when the tables are built
                    const int n = ps_format_gauss_tables(&c, nullptr, 0);
                    if (n > 0) {
                        std::string txt((size_t)n + 1, '\0');
                        ps_format_gauss_tables(&c, &txt[0], txt.size());
                        std::fputs(txt.c_str(), stdout);
                        std::fflush(stdout);
                    }
                }
                p->ctx = ps_create(_device, &c, p->ctx_w, p->ctx_h, slots);
                p->in_slot.assign(slots, nullptr);
                p->next_slot = 0;
                if (!p->ctx) { fail_job(job, ps_last_error(nullptr)); p->ctx_w = p->ctx_h = 0; continue; }
            }
            const int s = p->next_slot;
            finish(s);
            int rc;
            if (job->describeFlags() >= 0) {
                const ps_keypoint* kps = reinterpret_cast<const ps_keypoint*>(job->keypoints().data());
                const int n = (int)job->keypoints().size();
                rc = job->isFloat() ? ps_describe_f32(p->ctx, s, reinterpret_cast<const float*>(job->pixels()), w, h, kps, n, job->describeFlags())
                                    : ps_describe_u8(p->ctx, s, job->pixels(), w, h, kps, n, job->describeFlags());
            } else {
                rc = job->isFloat() ? ps_submit_f32(p->ctx, s, reinterpret_cast<const float*>(job->pixels()), w, h)
                                    : ps_submit_u8(p->ctx, s, job->pixels(), w, h);
            }
            if (rc != PS_OK) {
                // the copy out of the job's page-locked image may already be queued: let it finish before
                // the caller can delete the job (and hand its block back to the pool)
                const std::string msg = ps_last_error(p->ctx);
                ps_sync(p->ctx, s);
                fail_job(job, msg);
                continue;
            }
            p->in_slot[s] = job;
            p->next_slot = (s + 1) % (int)p->in_slot.size();
        }
        finish_all();
        if (p->ctx) { ps_destroy(p->ctx); p->ctx = nullptr; }
    });
}

PopSift::PopSift(const Config& config, Config::ProcessingMode mode, ImageMode imode, int device)
    : PopSift(imode, device)
{
    _proc_mode = mode;
    configure(config);
}

PopSift::~PopSift()
{
    if (_isInit) uninit();
}

bool PopSift::configure(const Config& config, bool /*force*/)
{
    Pipe* p = _pipe.get();
    std::lock_guard<std::mutex> lk(p->mu);
    if (p->started) return false;            // like the reference: not after the pyramid exists
    _config = config;
    _config.levels = std::max(2, config.levels);
    return true;
}

void PopSift::setSlots(int n)
{
    Pipe* p = _pipe.get();
    std::lock_guard<std::mutex> lk(p->mu);
    if (!p->started && n >= 1 && n <= 64) p->slots = n;
}

void PopSift::uninit()
{
    if (!_isInit) {
        std::cerr << "[warning] Attempt to release resources from an uninitialized instance" << std::endl;
        return;
    }
    Pipe* p = _pipe.get();
    {
        std::lock_guard<std::mutex> lk(p->mu);
        p->stop = true;
    }
    p->cv.notify_all();
    if (p->worker.joinable()) p->worker.join();
    _isInit = false;
}

PopSift::AllocTest PopSift::testTextureFit(int width, int height)
{
    // linear HBM planes: no texture or surface limits; only absurd sizes are refused
    if (width < 1 || height < 1 || (long long)width * height > (1LL << 30)) return ImageExceedsLinearTextureLimit;
    return Ok;
}

std::string PopSift::testTextureFitErrorString(AllocTest err, int width, int height)
{
    std::ostringstream o;
    switch (err) {
        case Ok: o << "?    No error." << std::endl; break;
        case ImageExceedsLinearTextureLimit:
            o << "E    Cannot load unscaled image. " << std::endl
              << "E    Size (" << width << "," << height << ") is not supported." << std::endl; break;
        default: o << "E    Programming error, please report." << std::endl; break;
    }
    return o.str();
}

SiftJob* PopSift::enqueue(int w, int h, const unsigned char* imageData)
{
    if (_image_mode != ByteImages)
        throw std::runtime_error("Image mode error\nE    Cannot load byte images into a PopSift pipeline configured for float images");
    const AllocTest a = testTextureFit(w, h);
    if (a != Ok) {
        std::cerr << __FILE__ << ":" << __LINE__ << " Image too large" << std::endl << testTextureFitErrorString(a, w, h);
        return nullptr;
    }
    SiftJob* job = new SiftJob(w, h, imageData);
    Pipe* p = _pipe.get();
    { std::lock_guard<std::mutex> lk(p->mu); p->queue.push_back(job); }
    p->cv.notify_all();
    return job;
}

SiftJob* PopSift::enqueue(int w, int h, const float* imageData)
{
    if (_image_mode != FloatImages)
        throw std::runtime_error("Image mode error\nE    Cannot load float images into a PopSift pipeline configured for byte images");
    const AllocTest a = testTextureFit(w, h);
    if (a != Ok) {
        std::cerr << __FILE__ << ":" << __LINE__ << " Image too large" << std::endl << testTextureFitErrorString(a, w, h);
        return nullptr;
    }
    SiftJob* job = new SiftJob(w, h, imageData);
    Pipe* p = _pipe.get();
    { std::lock_guard<std::mutex> lk(p->mu); p->queue.push_back(job); }
    p->cv.notify_all();
    return job;
}

SiftJob* PopSift::describe(int w, int h, const unsigned char* imageData, const std::vector<popsift::Keypoint>& kps, bool computeOrientations)
{
    if (_image_mode != ByteImages)
        throw std::runtime_error("Image mode error\nE    Cannot load byte images into a PopSift pipeline configured for float images");
    const AllocTest a = testTextureFit(w, h);
    if (a != Ok) {
        std::cerr << __FILE__ << ":" << __LINE__ << " Image too large" << std::endl << testTextureFitErrorString(a, w, h);
        return nullptr;
    }
    if (kps.size() > (size_t)INT32_MAX) throw std::runtime_error("PopSift::describe: more than 2^31 - 1 keypoints");
    SiftJob* job = new SiftJob(w, h, imageData, kps, computeOrientations);
    Pipe* p = _pipe.get();
    { std::lock_guard<std::mutex> lk(p->mu); p->queue.push_back(job); }
    p->cv.notify_all();
    return job;
}

SiftJob* PopSift::describe(int w, int h, const float* imageData, const std::vector<popsift::Keypoint>& kps, bool computeOrientations)
{
    if (_image_mode != FloatImages)
        throw std::runtime_error("Image mode error\nE    Cannot load float images into a PopSift pipeline configured for byte images");
    const AllocTest a = testTextureFit(w, h);
    if (a != Ok) {
        std::cerr << __FILE__ << ":" << __LINE__ << " Image too large" << std::endl << testTextureFitErrorString(a, w, h);
        return nullptr;
    }
    if (kps.size() > (size_t)INT32_MAX) throw std::runtime_error("PopSift::describe: more than 2^31 - 1 keypoints");
    SiftJob* job = new SiftJob(w, h, imageData, kps, computeOrientations);
    Pipe* p = _pipe.get();
    { std::lock_guard<std::mutex> lk(p->mu); p->queue.push_back(job); }
    p->cv.notify_all();
    return job;
}
