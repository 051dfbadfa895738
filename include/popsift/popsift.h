// PopSift / SiftJob for the H100 (sm_90a) drop-in.
//
// Same public surface as the reference (reference src/popsift/popsift.h:44-317): construct with a
// Config, enqueue(w, h, pixels) copies the image and returns a SiftJob the caller owns,
// SiftJob::get() blocks and returns a FeaturesHost the caller owns, uninit() drains and frees.
// Underneath it is a thin C++ layer over the C ABI in <popsift_b200.h>: one worker thread per
// PopSift keeps `slots` images in flight on independent CUDA streams (the reference keeps one).
// Errors raised on the worker are delivered by get() as std::runtime_error (the reference's
// extracting mode would std::terminate, src/popsift/popsift.cpp:306-344).
#pragma once

#include "common/device_prop.h"
#include "features.h"
#include "sift_conf.h"
#include "sift_config.h"

#include <exception>
#include <future>
#include <memory>
#include <string>
#include <vector>

struct ps_ctx;

class SiftJob
{
    std::promise<popsift::FeaturesBase*> _p;
    std::future<popsift::FeaturesBase*>  _f;
    int            _w;
    int            _h;
    unsigned char* _imageData;
    bool           _isFloat;
    std::exception_ptr _err;
    int            _describe = -1;                // -1: detection; else the ps_describe_* flags
    std::vector<popsift::Keypoint> _keypoints;    // describe jobs: the caller's keypoints

public:
    SiftJob(int w, int h, const unsigned char* imageData);
    SiftJob(int w, int h, const float* imageData);
    /// a describe job (PopSift::describe): copies the image and the keypoints
    SiftJob(int w, int h, const unsigned char* imageData, const std::vector<popsift::Keypoint>& kps, bool computeOrientations);
    SiftJob(int w, int h, const float* imageData, const std::vector<popsift::Keypoint>& kps, bool computeOrientations);
    ~SiftJob();

    popsift::FeaturesHost* get();
    popsift::FeaturesBase* getBase();
    popsift::FeaturesHost* getHost();
    popsift::FeaturesDev*  getDev();

    void setFeatures(popsift::FeaturesBase* f);
    void setError(std::exception_ptr ptr);

    // used by the pipeline
    int                  width() const { return _w; }
    int                  height() const { return _h; }
    const unsigned char* pixels() const { return _imageData; }
    bool                 isFloat() const { return _isFloat; }
    int                  describeFlags() const { return _describe; }
    const std::vector<popsift::Keypoint>& keypoints() const { return _keypoints; }
};

class PopSift
{
public:
    enum ImageMode { ByteImages, FloatImages };
    enum AllocTest { Ok, ImageExceedsLinearTextureLimit, ImageExceedsLayeredSurfaceLimit };

    PopSift() = delete;
    PopSift(const PopSift&) = delete;

    explicit PopSift(ImageMode imode = ByteImages, int device = 0);
    explicit PopSift(const popsift::Config&          config,
                     popsift::Config::ProcessingMode mode = popsift::Config::ExtractingMode,
                     ImageMode imode = ByteImages, int device = 0);
    ~PopSift();

    bool configure(const popsift::Config& config, bool force = false);
    void uninit();

    AllocTest   testTextureFit(int width, int height);
    std::string testTextureFitErrorString(AllocTest err, int w, int h);

    SiftJob* enqueue(int w, int h, const unsigned char* imageData);
    SiftJob* enqueue(int w, int h, const float* imageData);

    /// Orientations (computeOrientations) and descriptors at the caller's keypoints instead of detected ones (extension;
    /// C ABI ps_describe_u8 / ps_describe_f32).  The job's features hold one Feature per keypoint, in input order, with
    /// num_ori = 0 for a rejected keypoint.  Describe and enqueue jobs share one FIFO; get() / getDev() as for enqueue.
    SiftJob* describe(int w, int h, const unsigned char* imageData, const std::vector<popsift::Keypoint>& kps,
                      bool computeOrientations = false);
    SiftJob* describe(int w, int h, const float* imageData, const std::vector<popsift::Keypoint>& kps,
                      bool computeOrientations = false);

    /// number of images in flight on the device (extension; the reference has 1)
    void setSlots(int n);

    // deprecated interface of the reference, kept
    inline void uninit(int /*pipe*/) { uninit(); }
    inline bool init(int /*pipe*/, int w, int h) { _last_init_w = w; _last_init_h = h; return true; }
    inline popsift::FeaturesBase* execute(int /*pipe*/, const unsigned char* imageData)
    {
        SiftJob* j = enqueue(_last_init_w, _last_init_h, imageData);
        if (!j) return nullptr;
        popsift::FeaturesBase* f = j->getBase();
        delete j;
        return f;
    }

private:
    struct Pipe;
    std::unique_ptr<Pipe> _pipe;
    popsift::Config _config;
    int       _last_init_w{};
    int       _last_init_h{};
    ImageMode _image_mode;
    int       _device;
    popsift::Config::ProcessingMode _proc_mode{popsift::Config::ExtractingMode};
    bool      _isInit{true};
};
