// reloc_export.cpp -- tracking loss through the C++ mirror: runs raw depth frames (u16) through a KinFu made with dfusion_flags =
// DF_KINFU_RELOCALISE (2048) and writes, per frame, operator()'s return value, isLost() and the 12 floats of getCameraPose(), then the live
// mesh as a PLY, so that tests/test_reloc_gpu.py can compare them with a Python run of the same frames.  Needs a GPU to RUN.
// argv: depth file, frame count, per-frame output, output PLY.
#include <kfusion/kinfu.hpp>
#include <kfusion/io/ply.hpp>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <vector>

using namespace kfusion;

int main(int argc, char **argv)
{
    if (argc < 5) { std::printf("usage: reloc_export depth.u16 frames frames.out out.ply\n"); return 2; }
    const int frames = std::atoi(argv[2]);
    KinFuParams params = KinFuParams::default_params_dynamicfusion();
    params.dfusion_flags = 2048;                                       // DF_KINFU_RELOCALISE
    const size_t npix = (size_t)params.cols * params.rows;
    std::vector<unsigned short> depth_all(npix * frames);
    std::ifstream in(argv[1], std::ios::binary);
    in.read((char *)depth_all.data(), (std::streamsize)(depth_all.size() * 2));
    if (!in) { std::printf("reloc_export: cannot read %s\n", argv[1]); return 1; }
    KinFu kf(params);
    std::ofstream out(argv[3], std::ios::binary);
    for (int t = 0; t < frames; ++t) {
        cuda::Depth depth;
        depth.upload(&depth_all[npix * t], params.cols * sizeof(unsigned short), params.rows, params.cols);
        const unsigned char flags[2] = {(unsigned char)kf(depth), (unsigned char)kf.isLost()};
        const Affine3f pose = kf.getCameraPose();
        float p[12];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) p[3 * r + c] = pose.matrix(r, c);
        for (int r = 0; r < 3; ++r) p[9 + r] = pose.matrix(r, 3);
        out.write((const char *)flags, 2);
        out.write((const char *)p, sizeof p);
    }
    cv::Mat v, n, f;
    if (!kf.getMesh(v, n, f, true) || writePly(argv[4], v, n, f) != (long)v.cols * v.rows) { std::printf("reloc_export: mesh failed\n"); return 1; }
    std::printf("reloc_export: done\n");
    return 0;
}
