// popsift::Config for the H100 (sm_90a) drop-in.
//
// Same public surface as the reference's popsift::Config (reference src/popsift/sift_conf.h:29-419):
// public fields octaves / levels / sigma / _edge_limit / verbose, every setter, getter and enum, and
// operator== / != with the reference's notion of equality.  Unlike the reference
// (src/popsift/sift_conf.cu:42-50) constructing a Config does NOT need a CUDA device.
// `namespace popart` is an alias, because the reference README still uses that spelling.
#pragma once

#include <string>

#define MAX_OCTAVES 20
#define MAX_LEVELS  10

struct ps_config;

namespace popsift {

struct Config
{
    Config();

    enum GaussMode { VLFeat_Compute, VLFeat_Relative, VLFeat_Relative_All, OpenCV_Compute, Fixed9, Fixed15 };
    enum SiftMode { PopSift, OpenCV, VLFeat, Default = PopSift };
    enum LogMode { None, All };
    enum ScalingMode { ScaleDirect, ScaleDefault };
    enum DescMode { Loop, ILoop, Grid, IGrid, NoTile };
    enum NormMode { RootSift, Classic };
    enum GridFilterMode { RandomScale, LargestScaleFirst, SmallestScaleFirst };
    enum ProcessingMode { ExtractingMode, MatchingMode };

    void setGaussMode(const std::string& m);
    void setGaussMode(GaussMode m);
    void setMode(SiftMode m);
    void setLogMode(LogMode mode = All);
    void setScalingMode(ScalingMode mode = ScaleDefault);
    void setVerbose(bool on = true);
    void setDescMode(const std::string& byname);
    void setDescMode(DescMode mode = Loop);
    void setDownsampling(float v);
    void setOctaves(int v);
    void setLevels(int v);
    void setSigma(float v);
    void setEdgeLimit(float v);
    void setThreshold(float v);
    void setInitialBlur(float blur);
    void setPrintGaussTables();
    void setFilterMaxExtrema(int extrema);
    void setFilterGridSize(int sz);
    void setFilterSorting(const std::string& direction);
    void setFilterSorting(GridFilterMode m);
    void setNormMode(NormMode m);
    void setNormMode(const std::string& m);
    void setUseRootSift(bool on);
    void setNormalizationMultiplier(int mul);

    bool           hasInitialBlur() const;
    float          getInitialBlur() const;
    float          getPeakThreshold() const;
    bool           ifPrintGaussTables() const;
    GaussMode      getGaussMode() const;
    SiftMode       getSiftMode() const;
    LogMode        getLogMode() const;
    bool           getUseRootSift() const;
    NormMode       getNormMode(NormMode m = RootSift) const;
    int            getNormalizationMultiplier() const;
    float          getUpscaleFactor() const { return _upscale_factor; }
    int            getMaxExtrema() const { return _max_extrema; }
    bool           getCanFilterExtrema() const;
    int            getFilterMaxExtrema() const { return _filter_max_extrema; }
    int            getFilterGridSize() const { return _filter_grid_size; }
    GridFilterMode getFilterSorting() const { return _grid_filter_mode; }
    ScalingMode    getScalingMode() const { return _scaling_mode; }
    DescMode       getDescMode() const { return _desc_mode; }

    static GaussMode   getGaussModeDefault();
    static const char* getGaussModeUsage();
    static NormMode    getNormModeDefault();
    static const char* getNormModeUsage();

    bool equal(const Config& other) const;

    /// the plain-C view of this configuration handed to the C ABI (include/popsift_b200.h)
    void toC(ps_config& out) const;

    int   octaves;
    int   levels;
    float sigma;
    float _edge_limit;
    bool  verbose;

private:
    float          _threshold;
    float          _upscale_factor;
    LogMode        _log_mode;
    ScalingMode    _scaling_mode;
    DescMode       _desc_mode;
    GridFilterMode _grid_filter_mode;
    int            _max_extrema;
    int            _filter_max_extrema;
    int            _filter_grid_size;
    GaussMode      _gauss_mode;
    SiftMode       _sift_mode;
    bool           _assume_initial_blur;
    float          _initial_blur;
    NormMode       _normalization_mode;
    int            _normalization_multiplier;
    bool           _print_gauss_tables;
};

inline bool operator==(const Config& l, const Config& r) { return l.equal(r); }
inline bool operator!=(const Config& l, const Config& r) { return !l.equal(r); }

} // namespace popsift

namespace popart = popsift;
