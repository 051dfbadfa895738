// Result containers of the drop-in (reference src/popsift/features.h:23-122,
// src/popsift/sift_extremum.h:69-72).  Byte layouts are the reference's: Descriptor = 128 floats,
// Feature = 72 bytes with host pointers into the owning FeaturesHost's descriptor array.
#pragma once

#include <cstdint>
#include <iostream>
#include <utility>
#include <vector>

#define ORIENTATION_MAX_COUNT 4

namespace popsift {

struct Descriptor
{
    float features[128];   // index (iy*4+ix)*8 + bin
};

struct Feature
{
    int         debug_octave;
    float       xpos;
    float       ypos;
    float       sigma;
    int         num_ori;
    float       orientation[ORIENTATION_MAX_COUNT];
    Descriptor* desc[ORIENTATION_MAX_COUNT];

    void print(std::ostream& ostr, bool write_as_uchar) const;
};

std::ostream& operator<<(std::ostream& ostr, const Feature& feature);

/// A keypoint for PopSift::describe, in input-image units like Feature (same bytes as ps_keypoint, 24).
struct Keypoint
{
    float xpos;
    float ypos;
    float sigma;
    float orientation = 0.0f;   // radians; used unless describe() computes the orientations
    int   octave = -1;          // -1: derived from sigma; else the octave, as Feature::debug_octave
    int   level = -1;           // -1: derived from sigma; else the Gaussian level of the octave, 0 .. levels+2
};

class FeaturesBase
{
    int _num_ext;
    int _num_ori;

public:
    FeaturesBase();
    virtual ~FeaturesBase();

    int  size() const { return _num_ext; }
    int  getFeatureCount() const { return _num_ext; }
    int  getDescriptorCount() const { return _num_ori; }
    void setFeatureCount(int n) { _num_ext = n; }
    void setDescriptorCount(int n) { _num_ori = n; }
};

class FeaturesHost : public FeaturesBase
{
    Feature*    _ext;
    Descriptor* _ori;

public:
    FeaturesHost();
    FeaturesHost(int num_ext, int num_ori);
    ~FeaturesHost() override;

    typedef Feature*       F_iterator;
    typedef const Feature* F_const_iterator;

    F_iterator       begin() { return _ext; }
    F_const_iterator begin() const { return _ext; }
    F_iterator       end() { return _ext + size(); }
    F_const_iterator end() const { return _ext + size(); }

    void reset(int num_ext, int num_ori);
    void pin();     // no-op here: results arrive through the library's own pinned staging
    void unpin();

    Feature*    getFeatures() { return _ext; }
    Descriptor* getDescriptors() { return _ori; }

    void print(std::ostream& ostr, bool write_as_uchar) const;
};

using Features = FeaturesHost;

std::ostream& operator<<(std::ostream& ostr, const FeaturesHost& feature);

/// Device-resident results (Config::MatchingMode; reference features.h:104-122): Feature records,
/// descriptors and the descriptor -> feature reverse map live in device memory owned by this object;
/// Feature::desc[] are device pointers into getDescriptors().  match() is the reference's brute-force
/// 2-nearest-neighbour matcher (features.cu:282-304), computed on the tensor cores (C ABI ps_match).
class FeaturesDev : public FeaturesBase
{
    Feature*    _ext;
    Descriptor* _ori;
    int*        _rev;   // the reverse map from descriptors to extrema

public:
    FeaturesDev();
    FeaturesDev(int num_ext, int num_ori);
    ~FeaturesDev() override;

    void reset(int num_ext, int num_ori);

    /// reference behaviour: prints one "accept/reject feat ..." line per descriptor of *this to stdout
    void match(FeaturesDev* other);
    /// the same search without the printing: 3 ints (best index, second index, accept) per descriptor of *this
    /// (an addition to the reference's interface; flags as for ps_match)
    std::vector<int> matchIndices(FeaturesDev* other, int flags = 0);

    Feature*    getFeatures() { return _ext; }
    Descriptor* getDescriptors() { return _ori; }
    int*        getReverseMap() { return _rev; }
};

/// 2-nearest-neighbour matching of many pairs in one call (an addition to the reference's interface; C ABI
/// ps_match_batch): entry p equals sets[pairs[p].first]->matchIndices(sets[pairs[p].second], flags).  Every set is
/// prepared once per group of pairs and all pairs share one tensor-core launch; flags as for ps_match.
std::vector<std::vector<int>> matchPairs(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                         int flags = 0);

/// matchPairs on 8-bit descriptors (an addition to the reference's interface; C ABI ps_descriptors_to_u8 +
/// ps_match_u8_batch): entry p equals matchPairs(...) on the descriptors rounded as --write-as-uchar prints them
/// (saturated to [0, 255]; scale them with Config::setNormalizationMultiplier, e.g. 9).  Each set is quantised on the
/// device and matched with exact integer distances; flags as for ps_match.
std::vector<std::vector<int>> matchPairsU8(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                           int flags = 0);

/// RANSAC settings of verifyPairs (same fields and rules as ps_verify_params in popsift_b200.h).
struct VerifyParams
{
    enum Model { Homography = 0, Fundamental = 1 };
    int                model = Homography;
    int                n_samples = 1024;    // minimal samples per pair, 1 .. 65536 (fixed; no early exit)
    float              threshold = 4.0f;    // pixels: transfer error (H) or Sampson distance (F)
    bool               refine = true;       // one least-squares refit on the winner's inliers
    unsigned long long seed = 0;
};

/// The two-view model of one pair: model maps left to right in pixels (row-major; zero when none was found),
/// inlier_rows are the left descriptor indices of the inlier correspondences, ascending.
struct PairGeometry
{
    float            model[9];
    int              n_inliers;
    std::vector<int> inlier_rows;
};

/// Geometric verification of matched pairs on the device (an addition to the reference's interface; C ABI
/// ps_match_correspondences + ps_verify_batch): `matches` is the output of matchPairs / matchPairsU8 on the same sets and
/// pairs.  Correspondences are gathered from the sets' Features and reverse maps, then every pair gets one RANSAC
/// homography or fundamental matrix.  Throws like matchPairs.
std::vector<PairGeometry> verifyPairs(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                      const std::vector<std::vector<int>>& matches, const VerifyParams& params = VerifyParams());

/// Pinhole intrinsics of one image in pixels (ps_camera in popsift_b200_pose.h); points must be undistorted.
struct Camera
{
    float fx = 0.0f, fy = 0.0f, cx = 0.0f, cy = 0.0f;
};

/// RANSAC settings of relativePoses (same fields and rules as ps_pose_params in popsift_b200_pose.h).
struct PoseParams
{
    int                n_samples = 1024;    // minimal samples per pair, 1 .. 65536 (fixed; no early exit)
    float              threshold = 4.0f;    // pixels (Sampson distance, tested in calibrated coordinates)
    bool               refine = true;       // one least-squares refit on the winner's inliers
    unsigned long long seed = 0;
};

/// The calibrated two-view geometry of one pair (ps_two_view): E in calibrated coordinates, F in pixels (a model for
/// matchPairsGuided with VerifyParams::Fundamental), R and unit t with X_r = R X_l + t, all row-major and zero when none
/// was found.  inlier_rows / front_rows are the left descriptor indices of the inlier correspondences and of those also
/// in front of both cameras, ascending.
struct TwoViewPose
{
    float            E[9], F[9], R[9], t[3];
    int              n_inliers, n_front;
    std::vector<int> inlier_rows, front_rows;
};

/// Relative poses of matched calibrated pairs on the device (an addition to the reference's interface; C ABI
/// ps_match_correspondences + ps_relative_pose_batch): `matches` is the output of matchPairs / matchPairsU8 on the same
/// sets and pairs, `cameras` one per set.  Throws like verifyPairs, and when cameras.size() != sets.size().
std::vector<TwoViewPose> relativePoses(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                       const std::vector<std::vector<int>>& matches, const std::vector<Camera>& cameras,
                                       const PoseParams& params = PoseParams());

/// Guided matching (an addition to the reference's interface; C ABI ps_match_guided_batch in popsift_b200_guided.h): matchPairs
/// again with only the right descriptors whose keypoints pass the pair's model as candidates.  `geometry` is what
/// verifyPairs gave for the same sets and pairs; params.model and params.threshold select the test (the other fields are
/// unused).  Returns what matchPairs returns and throws like it (also when geometry.size() != pairs.size()).
std::vector<std::vector<int>> matchPairsGuided(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                               const std::vector<PairGeometry>& geometry, const VerifyParams& params, int flags = 0);
/// matchPairsGuided on 8-bit descriptors (quantised on the device as matchPairsU8 does; C ABI ps_match_u8_guided_batch)
std::vector<std::vector<int>> matchPairsGuidedU8(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                                 const std::vector<PairGeometry>& geometry, const VerifyParams& params, int flags = 0);

/// Codebook settings of vladCodebook (same rules as ps_vlad_train in popsift_b200_retrieval.h).
struct VladParams
{
    int                k = 64;       // centroids, 1 .. 1024 (at most the pooled descriptor count)
    int                iters = 10;   // k-means iterations, 0 .. 1000 (fixed; no convergence test)
    unsigned long long seed = 0;     // initial draw
};

/// k-means codebook of the pooled descriptors of `sets` (an addition to the reference's interface; C ABI ps_vlad_train):
/// k x 128 floats, row-major.  flags as for matchPairs (the assignment is its nearest-neighbour search).  Throws like
/// matchPairs, and for parameters ps_vlad_train refuses.
std::vector<float> vladCodebook(const std::vector<FeaturesDev*>& sets, const VladParams& params = VladParams(), int flags = 0);

/// VLAD vectors of `sets` under `codebook` (k x 128 floats; C ABI ps_vlad_encode): sets.size() rows of k * 128 floats.
std::vector<float> vladEncode(const std::vector<FeaturesDev*>& sets, const std::vector<float>& codebook, int flags = 0);

/// The pair list of image retrieval (C ABI ps_retrieve_pairs): `vectors` holds n rows of vectors.size() / n floats (a
/// multiple of 4, e.g. vladEncode's output); every row's m best neighbours under the inner product are taken, and the
/// result is the union of the unordered pairs (i, j), i < j, sorted.
std::vector<std::pair<int, int>> retrievePairs(const std::vector<float>& vectors, int n, int m);

/// Feature tracks (C ABI ps_tracks_from_matches in popsift_b200_tracks.h): the connected components of the matches over
/// all features of all sets, without those holding two features of one set and those shorter than min_length (>= 2).
/// Track t's members are set[k] / feature[k] for k in [start[t], start[t + 1]), ascending by set; tracks are sorted by
/// their smallest member; track_of[i][f] is feature f of set i's track, or -1.
struct Tracks
{
    std::vector<int>              start, set, feature;
    std::vector<std::vector<int>> track_of;
    int                           n_components = 0, n_conflicting = 0, n_short = 0;
};

/// Tracks of the verified inliers: `matches` and `geometry` are what matchPairs(U8) and verifyPairs gave for the same sets
/// and pairs, and the edges are geometry[p].inlier_rows.  Throws like verifyPairs.
Tracks buildTracks(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                   const std::vector<std::vector<int>>& matches, const std::vector<PairGeometry>& geometry, int min_length = 2);
/// Tracks of every correspondence of `matches`: the rows of matchPairsGuided(U8), which already passed the model.
Tracks buildTracks(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                   const std::vector<std::vector<int>>& matches, int min_length = 2);

/// A camera pose, world to camera: X_cam = R X_world + t, R row-major (ps_rigid in popsift_b200_triangulate.h).
struct Rigid
{
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double t[3] = {0, 0, 0};
};

/// Settings of triangulateTracks (same fields and rules as ps_triangulate_params).
struct TriangulateParams
{
    float              max_error = 4.0f;     // pixels
    float              min_angle = 1.5f;     // degrees, [0, 90)
    int                min_views = 2;        // >= 2
    int                n_samples = 256;      // hypotheses per track when not every pair is tried, 1 .. 65536
    int                refine_iters = 10;    // Gauss-Newton steps, 0 .. 32
    unsigned long long seed = 0;
};

/// One point per track (ps_track_point) and one entry per member of Tracks::set / Tracks::feature: the inlier mask and
/// the pixel reprojection error (+inf behind the camera or without a point).  n_status[s] counts the tracks of status s
/// (PS_TRI_OK .. PS_TRI_SMALL_ANGLE).
struct TrackPoint
{
    double X[3];
    float  error, angle;
    int    n_inliers, status;
};
struct TrackPoints
{
    std::vector<TrackPoint>   points;
    std::vector<std::uint8_t> mask;
    std::vector<float>        obs_error;
    int                       n_status[5] = {0, 0, 0, 0, 0};
    int                       n_inlier_obs = 0;
};

/// Multi-view triangulation of `tracks` (what buildTracks gave for `sets`) from known poses on the device (an addition to
/// the reference's interface; C ABI ps_triangulate_tracks): `cameras` and `poses` one per set.  Throws like
/// relativePoses, and when poses.size() != sets.size().
TrackPoints triangulateTracks(const std::vector<FeaturesDev*>& sets, const Tracks& tracks, const std::vector<Camera>& cameras,
                              const std::vector<Rigid>& poses, const TriangulateParams& params = TriangulateParams());

/// Settings of bundleAdjust (same fields and rules as ps_bundle_params in popsift_b200_bundle.h).
struct BundleParams
{
    enum Loss { Squared = 0, Huber = 1, Cauchy = 2 };
    int    loss = Squared;
    double loss_scale = 1.0;         // pixels
    int    max_iters = 50;           // LM iterations, 0 .. 10000
    double function_tol = 1e-6;      // relative cost decrease of an accepted step that stops
    int    cg_max_iters = 100;       // CG iterations per LM iteration, 1 .. 10000
    double cg_tol = 1e-6;            // relative residual that stops CG, [0, 1)
    double initial_lambda = 1e-4;
    int    scale_set = -1;           // -1, or the set one of whose translation components is held
    int    scale_axis = 0;           // that component, 0 .. 2
};

/// What bundleAdjust did (ps_bundle_report); termination is PS_BA_MAX_ITERS .. PS_BA_NONFINITE_START.
struct BundleReport
{
    double initial_cost = 0, final_cost = 0;
    int    iterations = 0, accepted = 0, cg_iterations = 0, termination = 0;
    int    n_obs = 0, n_points = 0, n_free_cams = 0;
};

/// Bundle adjustment on the device (an addition to the reference's interface; C ABI ps_bundle_adjust): the poses of the
/// sets with fixed[i] == false and the points of the OK tracks of `points` (what triangulateTracks gave for `tracks`;
/// its mask selects the observations) refined by Levenberg-Marquardt.  Returns the refined poses and the report, and
/// updates points (X, error, angle of the OK tracks, obs_error of every member).  Throws like triangulateTracks, and for
/// the arguments ps_bundle_adjust refuses.
std::pair<std::vector<Rigid>, BundleReport> bundleAdjust(const std::vector<FeaturesDev*>& sets, const Tracks& tracks,
                                                         const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
                                                         const std::vector<bool>& fixed, TrackPoints& points,
                                                         const BundleParams& params = BundleParams());

/// Settings of rotationAveraging (same fields and rules as ps_rotation_params in popsift_b200_global.h).
struct RotationParams
{
    int    loss = BundleParams::Cauchy;
    double loss_scale = 5.0;         // degrees
    int    max_iters = 100;          // IRLS iterations, 0 .. 10000
    double step_tol = 1e-4;          // degrees: the largest update that stops
    int    cg_max_iters = 100;       // 1 .. 10000
    double cg_tol = 1e-8;            // [0, 1)
    int    min_inliers = 15;         // a pair is used when its n_front reaches this
};

/// What rotationAveraging did (ps_rotation_report); termination is PS_RA_MAX_ITERS .. PS_RA_NO_PAIRS.
struct RotationReport
{
    double initial_cost = 0, final_cost = 0;
    int    iterations = 0, cg_iterations = 0, n_pairs = 0, n_registered = 0, termination = 0;
};

/// One world-to-camera rotation per set, registered flags and per-pair errors (degrees, +inf for pairs not used).
struct Rotations
{
    std::vector<Rigid>  R;               // t is zero
    std::vector<bool>   registered;
    std::vector<float>  pair_error;
    RotationReport      report;
};

/// Rotation averaging on device 0 (an addition to the reference's interface; C ABI ps_rotation_averaging): `poses` is
/// what relativePoses gave for `pairs` (its R and n_front are uploaded).  Throws when poses.size() != pairs.size(), and
/// for the arguments ps_rotation_averaging refuses.
Rotations rotationAveraging(int n_sets, const std::vector<std::pair<int, int>>& pairs, const std::vector<TwoViewPose>& poses,
                            const RotationParams& params = RotationParams());

/// Settings of filterViewGraph (same fields and rules as ps_view_graph_params in popsift_b200_viewgraph.h).
struct ViewGraphParams
{
    double max_cycle_error = 3.0;    // degrees: a triangle whose cycle error is at most this is consistent
    int    min_consistent = 1;       // a pair in some triangle is kept with at least this many consistent ones ...
    double min_fraction = 0.0;       // ... and at least this fraction of its triangles consistent, [0, 1]
    bool   keep_untested = false;    // the fate of a used pair that lies in no triangle
    int    min_inliers = 15;         // a pair is used when its n_front reaches this (as in RotationParams)
};

/// One pair's triangles (ps_cycle_stats): how many, how many consistent, the smallest cycle error in degrees (+inf: none).
struct CycleStats
{
    int   n_triangles = 0, n_consistent = 0;
    float min_error = 0;
};

/// What filterViewGraph did (ps_view_graph_report).
struct ViewGraphReport
{
    long long n_triangles = 0, n_consistent_triangles = 0;
    int       n_used = 0, n_kept = 0, n_untested = 0;
};

/// The pairs kept, one CycleStats per pair and the totals.
struct ViewGraph
{
    std::vector<bool>       keep;
    std::vector<CycleStats> stats;
    ViewGraphReport         report;
};

/// View-graph cleaning on device 0 (an addition to the reference's interface; C ABI ps_view_graph_filter): drops the pairs
/// whose relative rotations fail loop consistency over the triangles of the view graph.  `poses` is what relativePoses
/// gave for `pairs` (its R and n_front are uploaded); the kept pairs and their poses go to rotationAveraging.  Throws when
/// poses.size() != pairs.size(), and for the arguments ps_view_graph_filter refuses (a duplicate pair among them).
ViewGraph filterViewGraph(int n_sets, const std::vector<std::pair<int, int>>& pairs, const std::vector<TwoViewPose>& poses,
                          const ViewGraphParams& params = ViewGraphParams());

/// A grey image on the device: row-major 8-bit values, `pitch` bytes between rows (ps_image in popsift_b200_depth.h).
struct DeviceImage
{
    const std::uint8_t* data = nullptr;
    long long           pitch = 0;
    int                 width = 0, height = 0;
};

/// Settings of depthMaps (same fields and rules as ps_depth_params in popsift_b200_depth.h).
struct DepthParams
{
    int   n_depths = 128;                // planes, 2 .. 1024
    int   radius = 3;                    // NCC window half-size, 1 .. 7
    int   top_k = 3;                     // source costs averaged per plane, 1 .. 32
    int   min_sources = 1;               // valid sources a plane needs, 1 .. 32
    float max_cost = 0.5f;               // a depth is kept when its cost is at most this, (0, 2]
    float min_var = 1.0f;                // window variance floor, grey levels^2
};

/// One reference's maps, row-major width x height: depth (0 where there is none), cost (+inf without a winner) and the
/// valid sources at the winning plane.
struct DepthMap
{
    int                       width = 0, height = 0;
    std::vector<float>        depth, cost;
    std::vector<std::uint8_t> n_src;
};

/// depthMaps' maps, one per reference, and the totals of ps_depth_report.
struct DepthMaps
{
    std::vector<DepthMap> maps;
    long long             n_candidates = 0, n_depths = 0;
};

/// Dense depth maps by plane sweep on `device` (an addition to the reference's interface; C ABI ps_depth_maps):
/// `images`, `cameras` and `poses` one per set; for reference j the set refs[j], its source sets sources[j] and its depth
/// range ranges[j] = (d_min, d_max).  Throws for the arguments ps_depth_maps refuses.
DepthMaps depthMaps(const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
                    const std::vector<int>& refs, const std::vector<std::vector<int>>& sources,
                    const std::vector<std::pair<float, float>>& ranges, const DepthParams& params = DepthParams(), int device = 0);

/// Settings of filterDepthMaps (same fields and rules as ps_depth_filter_params).
struct DepthFilterParams
{
    float max_reproj_error = 1.0f;       // pixels
    float max_depth_diff = 0.01f;        // relative
    int   min_consistent = 2;            // 1 .. 255
};

/// One consistent pixel as a world point (ps_dense_point).
struct DensePoint
{
    float         X[3];
    int           ref;
    std::uint16_t x, y;
    std::uint8_t  n_consistent, grey;
};

/// filterDepthMaps' result: the consistent sources per pixel of each reference, the points in (ref, y, x) order and the
/// pixels with a depth.
struct DensePoints
{
    std::vector<std::vector<std::uint8_t>> n_consistent;
    std::vector<DensePoint>                points;
    long long                              n_tested = 0;
};

/// Geometric consistency between the maps of one depthMaps call and the consistent pixels as points (C ABI
/// ps_depth_filter): the same images, cameras, poses, refs and sources; `maps` is uploaded.  Throws for the arguments
/// ps_depth_filter refuses.
DensePoints filterDepthMaps(const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
                            const std::vector<int>& refs, const std::vector<std::vector<int>>& sources, const DepthMaps& maps,
                            const DepthFilterParams& params = DepthFilterParams(), int device = 0);

/// A dense truncated signed distance volume on `device` (ps_volume in popsift_b200_mesh.h): nx x ny x nz grid points from
/// `origin` at spacing `voxel`, grid point (i, j, k) at index i + nx (j + ny k) of the three device arrays it owns.
/// Constructed cleared; throws for the volumes ps_volume_clear refuses or when the allocation fails.
class DeviceVolume
{
public:
    DeviceVolume(const double origin[3], double voxel, int nx, int ny, int nz, int device = 0);
    ~DeviceVolume();
    DeviceVolume(const DeviceVolume&) = delete;
    DeviceVolume& operator=(const DeviceVolume&) = delete;

    const double* origin() const { return _origin; }
    double voxel() const { return _voxel; }
    int nx() const { return _n[0]; }
    int ny() const { return _n[1]; }
    int nz() const { return _n[2]; }
    int device() const { return _device; }
    float* tsdf() const { return _tsdf; }       // DEVICE
    float* weight() const { return _weight; }   // DEVICE
    float* grey() const { return _grey; }       // DEVICE

private:
    double _origin[3];
    double _voxel;
    int    _n[3];
    int    _device;
    float* _tsdf = nullptr;
    float* _weight = nullptr;
    float* _grey = nullptr;
};

/// Sets every grid point's tsdf, weight and grey to 0 (C ABI ps_volume_clear).
void clearVolume(DeviceVolume& volume);

/// Settings of integrateDepthMaps (same fields and rules as ps_tsdf_params in popsift_b200_mesh.h).
struct TsdfParams
{
    float trunc = 0.0f;                  // truncation distance in world units, > 0 (no default: it depends on the scene)
    int   min_consistent = 0;            // 0 .. 255; > 0: only pixels whose mask value is at least this
};

/// integrateDepthMaps' totals (ps_tsdf_report).
struct TsdfReport
{
    long long n_updates = 0, n_voxels_touched = 0;
};

/// Folds depth maps into `volume` (C ABI ps_tsdf_integrate): view v is images[v], cameras[v], poses[v] and the host map
/// maps[v] (its size that of images[v]), uploaded; masks[v] are the n_consistent values of filterDepthMaps, read when
/// params.min_consistent > 0 (masks may be empty otherwise).  Throws when the sizes disagree, and for the arguments
/// ps_tsdf_integrate refuses.
TsdfReport integrateDepthMaps(DeviceVolume& volume, const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras,
                              const std::vector<Rigid>& poses, const std::vector<DepthMap>& maps,
                              const std::vector<std::vector<std::uint8_t>>& masks, const TsdfParams& params);

/// Settings of extractMesh (ps_mesh_params).
struct MeshParams
{
    float min_weight = 1.0f;             // a cell is meshed when its 8 corners have at least this weight
};

/// One mesh vertex (ps_mesh_vertex): world position and interpolated grey level.
struct MeshVertex
{
    float X[3];
    float grey;
};

/// extractMesh's result: the vertices in edge-key order, the triangles as 3 vertex indices each (normals towards the
/// cameras) and the totals of ps_mesh_report.
struct Mesh
{
    std::vector<MeshVertex> vertices;
    std::vector<int>        triangles;   // 3 per triangle
    long long               n_cells = 0;
};

/// The surface of `volume` by marching tetrahedra (C ABI ps_tsdf_mesh: a count call, then the call that fills outputs of
/// that size).  Throws for the arguments ps_tsdf_mesh refuses.
Mesh extractMesh(const DeviceVolume& volume, const MeshParams& params = MeshParams());

/// Settings of renderMesh (ps_render_params in popsift_b200_render.h).
struct RenderParams
{
    float z_near = 1e-3f;                // triangles with a vertex closer than this are not drawn (no clipping)
};

/// One view's rendered maps, row-major width x height: camera-frame depth (0 where no triangle covers the pixel) and the
/// nearest triangle (-1 where none).
struct RenderMap
{
    int                width = 0, height = 0;
    std::vector<float> depth;
    std::vector<int>   triangle;
};

/// renderMesh's maps, one per view, and the totals of ps_render_report.
struct RenderedMesh
{
    std::vector<RenderMap> maps;
    long long              n_drawn = 0, n_big = 0, n_covered = 0;
};

/// Renders `mesh` into posed views with a z-buffer on `device` (an addition to the reference's interface; C ABI
/// ps_mesh_render): view v is cameras[v], poses[v] and sizes[v] = (width, height).  The maps are in depthMaps' layout.
/// Throws when the sizes disagree, and for the arguments ps_mesh_render refuses.
RenderedMesh renderMesh(const Mesh& mesh, const std::vector<Camera>& cameras, const std::vector<Rigid>& poses,
                        const std::vector<std::pair<int, int>>& sizes, const RenderParams& params = RenderParams(), int device = 0);

/// Settings of textureMesh (same fields and rules as ps_texture_params; cells_per_row 0 keeps the atlas close to square).
struct TextureParams
{
    int   cell = 8;                      // texels per cell side, 3 .. 64
    int   cells_per_row = 0;             // 0: ceil(sqrt(triangles)), at most 65535 / cell
    float depth_tol = 0.01f;             // relative occlusion tolerance
    float min_cos = 0.1f;                // facing test, [0, 1)
    float z_near = 1e-3f;
};

/// textureMesh's result: the atlas (width x height, row-major grey), the view per triangle (-1: the vertex-grey fallback)
/// and the totals of ps_texture_report.  Triangle m's corners sit at texel positions (b, b), (cell - b, b), (b, cell - b)
/// of cell (m mod cells_per_row, m div cells_per_row), b = 1.
struct TexturedMesh
{
    int                       width = 0, height = 0, cell = 0, cells_per_row = 0;
    std::vector<std::uint8_t> atlas;
    std::vector<int>          view;
    long long                 n_viewed = 0, n_fallback = 0;
};

/// A texture atlas of `mesh` from the images on `device` (C ABI ps_mesh_render, then ps_mesh_texture on the device maps,
/// with no host copy between them).  Throws when the sizes disagree, and for the arguments either call refuses.
TexturedMesh textureMesh(const Mesh& mesh, const std::vector<DeviceImage>& images, const std::vector<Camera>& cameras,
                         const std::vector<Rigid>& poses, const TextureParams& params = TextureParams(), int device = 0);

/// Settings of twoViewGeometries' classification (same fields and rules as ps_two_view_config_params in
/// popsift_b200_twoview.h; the pure-rotation test uses PoseParams::threshold).
struct TwoViewConfigParams
{
    int    min_inliers = 15;
    double min_ef_ratio = 0.95;
    double max_h_ratio = 0.8;
    double min_rotation_ratio = 0.9;
};

/// One pair's two-view configuration (ps_two_view_info and the record that replaces ps_relative_pose_batch's): config is
/// Degenerate, General, Planar, Panoramic or Uncalibrated (PS_TV_*); pose the essential pose (General), the homography's
/// (Planar), the rotation with t = 0 (Panoramic) or zero; normal the unit plane normal in the left frame (Planar);
/// tri_angle the median triangulation angle of the rows in front, degrees; the inlier counts of E, F and H and the H
/// inliers the pure rotation explains.
struct TwoViewGeometry
{
    enum { Degenerate = 0, General = 1, Planar = 2, Panoramic = 3, Uncalibrated = 4 };
    int         config = Degenerate;
    TwoViewPose pose;
    float       normal[3] = {0.0f, 0.0f, 0.0f};
    float       tri_angle = 0.0f;
    int         n_e = 0, n_f = 0, n_h = 0, n_rotation = 0;
};

/// Two-view configuration of matched calibrated pairs on the device (an addition to the reference's interface; C ABI
/// ps_match_correspondences, ps_verify_batch with the homography and the fundamental matrix, ps_relative_pose_batch, then
/// ps_two_view_config_batch in popsift_b200_twoview.h): the three RANSACs use `params`.  The poses feed
/// rotationAveraging and filterViewGraph unchanged.  Throws like relativePoses.
std::vector<TwoViewGeometry> twoViewGeometries(const std::vector<FeaturesDev*>& sets, const std::vector<std::pair<int, int>>& pairs,
                                               const std::vector<std::vector<int>>& matches, const std::vector<Camera>& cameras,
                                               const PoseParams& params = PoseParams(),
                                               const TwoViewConfigParams& config = TwoViewConfigParams());

/// Settings of globalPositioning (same fields and rules as ps_position_params).
struct PositionParams
{
    int    loss = BundleParams::Huber;
    double loss_scale = 0.1;
    int    max_iters = 100;
    double function_tol = 1e-8;
    int    cg_max_iters = 300;
    double cg_tol = 1e-8;
};

/// What globalPositioning did (ps_position_report); termination is PS_GP_MAX_ITERS .. PS_GP_NO_OBSERVATIONS.
struct PositionReport
{
    double initial_cost = 0, final_cost = 0;
    int    iterations = 0, cg_iterations = 0, n_obs = 0, n_points = 0, n_cams = 0, termination = 0;
};

/// Camera poses (world to camera) and one point per track (0 for tracks that took no part).
struct Positions
{
    std::vector<Rigid>   poses;
    std::vector<bool>    positioned;
    std::vector<double>  X;              // 3 per track
    PositionReport       report;
};

/// Global positioning of camera centres and track points with rotations held (an addition to the reference's interface;
/// C ABI ps_global_positioning): `tracks` as for triangulateTracks, `rotations` and `registered` what rotationAveraging
/// gave (only R of each Rigid is read).  Throws like triangulateTracks, and for the arguments ps_global_positioning refuses.
Positions globalPositioning(const std::vector<FeaturesDev*>& sets, const Tracks& tracks, const std::vector<Camera>& cameras,
                            const std::vector<Rigid>& rotations, const std::vector<bool>& registered,
                            const PositionParams& params = PositionParams());

} // namespace popsift
