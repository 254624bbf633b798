#pragma once
// kfusion::KinFuParams / kfusion::KinFu -- same interface as the reference's kfusion/kinfu.hpp:15-97, so apps/demo.cpp's use of
// it (default_params_dynamicfusion, KinFu::Ptr, operator()(depth), renderImage, getCameraPose, getWarp().getNodesAsMat())
// compiles unchanged.  The per-frame loop runs device-resident behind df_kinfu_* (include/dfusion.h).
#include <kfusion/types.hpp>
#include <vector>
#include <string>
#include <dual_quaternion.hpp>
#include <quaternion.hpp>
#include <kfusion/cuda/projective_icp.hpp>
#include <kfusion/cuda/tsdf_volume.hpp>
#include <kfusion/warp_field.hpp>
#include "warp_field_optimiser.hpp"

namespace kfusion
{
    struct KF_EXPORTS KinFuParams
    {
        static KinFuParams default_params();
        static KinFuParams default_params_dynamicfusion();

        int cols;  //pixels
        int rows;  //pixels
        Intr intr;  //Camera parameters
        Vec3i volume_dims; //number of voxels
        Vec3f volume_size; //meters
        Affine3f volume_pose; //meters, inital pose
        float bilateral_sigma_depth;   //meters
        float bilateral_sigma_spatial;   //pixels
        int   bilateral_kernel_size;   //pixels
        float icp_truncate_depth_dist; //meters
        float icp_dist_thres;          //meters
        float icp_angle_thres;         //radians
        std::vector<int> icp_iter_num; //iterations for level index 0,1,..,3
        float tsdf_min_camera_movement; //meters, integrate only if exceedes
        float tsdf_trunc_dist;             //meters;
        int tsdf_max_weight;               //frames
        float raycast_step_factor;   // in voxel sizes
        float gradient_delta_factor; // in voxel sizes
        Vec3f light_pose; //meters

        // not in the reference: opt-in extensions of the fusion step (SURVEY 8f), forwarded to df_kinfu_params; the defaults keep the
        // reference's behaviour.  (The same switches exist as environment variables for an unchanged apps/demo.cpp, dfusion.h.)
        int dfusion_flags = 0;             // DF_KINFU_WARPED_INTEGRATE (8) | DF_KINFU_EXTEND_FIELD (16) | DF_KINFU_COLOR (256) | DF_KINFU_COLOR_TRACKING (512)
                                           // | DF_KINFU_WARPED_COLOR (1024: with COLOR and WARPED_INTEGRATE, colour fused through the warp field)
                                           // | DF_KINFU_RELOCALISE (2048: keep the model through tracking loss, isLost())
        float fusion_weight_scale = 0.f;   // df_integrate_warped's weight quantisation (0: every sample weighs 1)
        float extend_radius = 0.f;         // df_extend_field's support radius in metres (0: 0.03)
    };

    class KF_EXPORTS KinFu
    {
    public:
        typedef cv::Ptr<KinFu> Ptr;

        KinFu(const KinFuParams& params);
        ~KinFu();

        const KinFuParams& params() const;
        KinFuParams& params();
        const cuda::TsdfVolume& tsdf() const;
        cuda::TsdfVolume& tsdf();
        const cuda::ProjectiveICP& icp() const;
        cuda::ProjectiveICP& icp();
        const WarpField& getWarp() const;
        WarpField& getWarp();

        void reset();
        bool operator()(const cuda::Depth& depth, const cuda::Image& image = cuda::Image());
        void renderImage(cuda::Image& image, int flags = 0);
        void dynamicfusion(cuda::Depth& depth, cuda::Cloud live_frame, cuda::Normals current_normals);
        void renderImage(cuda::Image& image, const Affine3f& pose, int flags = 0);
        Affine3f getCameraPose (int time = -1) const;

        // not in the reference: snapshots of the whole reconstruction (df_kinfu_save / df_kinfu_load, include/dfusion.h).  load() needs an
        // object made with the same parameters and resumes the sequence exactly where save() left it; both return false on failure
        // (I/O error, malformed file, other parameters, another colour camera), and a failed load leaves the object unchanged.
        // not in the reference: tracking loss (dfusion_flags DF_KINFU_RELOCALISE, 2048): true while the last frame failed the relocaliser's gate;
        // operator() then returned false and left the reconstruction as it was, and the camera is relocalised from keyframes by later frames
        bool isLost() const;
        bool save(const std::string& path) const;
        bool load(const std::string& path);
        // not in the reference: the triangle mesh of the canonical model (live = true: carried into the current frame by the warp field),
        // df_kinfu_mesh.  vertices / normals: 1 x N CV_32FC3, every extracted cloud point; faces: 1 x T CV_32SC3 of vertex indices.  Returns
        // false (outputs untouched) when the cloud does not match the volume or, for live, when there is no warp field.  io/ply.hpp writes it.
        bool getMesh(cv::Mat& vertices, cv::Mat& normals, cv::Mat& faces, bool live = false) const;
        // not in the reference: colour.  An object made with DF_KINFU_COLOR in dfusion_flags (or DF_KINFU_COLOR=1 in the environment) fuses
        // the image passed to operator()(depth, image) -- registered to the depth, b g r + pad per pixel, the frame's size -- into a colour
        // volume; an empty image fuses geometry only.  getMeshColors: 1 x N CV_8UC4 (r, g, b, a; a = 255 where coloured) for the vertices
        // of getMesh, live or not; false on an object without colour.  renderMeshImage flag 4 draws them.
        bool getMeshColors(cv::Mat& colors) const;
        // not in the reference: a colour camera with its own calibration (df_kinfu_set_color_camera): intrinsics, image size and the pose
        // taking a point from the depth camera's frame to the colour camera's.  From then on operator()(depth, image) fuses an image of that
        // size, taken by that camera, with an occlusion test against the frame's depth.  Only on a colour object before its first frame (or
        // after reset(), which keeps the camera); returns false and changes nothing otherwise or on invalid values.  A snapshot made with a
        // camera loads only into an object with the same camera set first (and one made without, only into an object without).
        bool setColorCamera(const Intr& intr, cv::Size size, const Affine3f& depth_to_color);
        // not in the reference: the same with the colour camera's lens distortion (df_kinfu_set_color_lens), and the depth camera's lens
        // (df_kinfu_set_depth_lens): from the next frame on, each depth frame (and an image registered to it) is undistorted on the GPU
        // before anything reads it.  The same rules as setColorCamera; a Lens with every coefficient 0 removes the lens.  Meshes, renders
        // and dynamicfusion() stay ideal pinhole images.
        bool setColorCamera(const Intr& intr, cv::Size size, const Affine3f& depth_to_color, const Lens& lens);
        bool setDepthLens(const Lens& lens);
        // not in the reference: that mesh rendered from a virtual camera (df_kinfu_render).  pose: camera-to-model; for the live model the
        // model frame is the current camera's, so Affine3f() is the current view.  renderMeshMaps fills cols x rows point and normal maps in
        // the camera frame (NaN where nothing is drawn) and returns false, leaving the maps as they were, where getMesh fails;
        // renderMeshImage shades them (flags 2 tangent colours, 3 shaded and tangent colours side by side, 4 the fused colours of a colour
        // object, any other value the shaded image)
        // and reports such a failure through the error handler.  renderImage itself still ray-casts the volume.
        bool renderMeshMaps(cuda::Cloud& points, cuda::Normals& normals, const Affine3f& pose, bool live = false);
        void renderMeshImage(cuda::Image& image, const Affine3f& pose, int flags = 0, bool live = false);
    private:
        void allocate_buffers();

        int frame_counter_;
        KinFuParams params_;
        std::vector<Affine3f> poses_;
        cuda::Dists dists_;
        cuda::Frame curr_, prev_, first_;
        cuda::Cloud points_;
        cuda::Normals normals_;
        cuda::Depth depths_;
        cv::Ptr<cuda::TsdfVolume> volume_;
        cv::Ptr<cuda::ProjectiveICP> icp_;
        cv::Ptr<WarpField> warp_;
        std::vector<std::pair<utils::DualQuaternion<float>, utils::DualQuaternion<float>>> edges_;
        cv::Ptr<WarpFieldOptimiser> optimiser_;
        void *handle_;          // df_kinfu_* pipeline object (not in the reference)
        long long resets_seen_ = 0;   // tracking-loss resets already mirrored into poses_
        cv::Size color_size_;         // setColorCamera's image size (0 x 0: images registered to the depth)
    };
}
