// warped_color_export.cpp -- colour under per-voxel warped fusion through the C++ mirror: fuses raw depth (u16) and BGRA (u8) frames into a
// KinFu made with dfusion_flags = DF_KINFU_WARPED_INTEGRATE | DF_KINFU_COLOR | DF_KINFU_WARPED_COLOR (8 | 256 | 1024) through
// operator()(depth, image), then writes the live mesh with KinFu::getMeshColors as a coloured PLY (kfusion::writePly), so that
// tests/test_warped_color_gpu.py can produce the same file from Python and compare bytes.  Needs a GPU to RUN (exit code 0 = all checks
// passed).  argv: depth file, bgra file, frame count, output PLY.
#include <kfusion/kinfu.hpp>
#include <kfusion/io/ply.hpp>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <vector>

using namespace kfusion;

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK failed: %s (line %d)\n", #c, __LINE__); ++fails; } } while (0)

template <class T> static std::vector<T> read_all(const char *path, size_t count)
{
    std::vector<T> v(count);
    std::ifstream f(path, std::ios::binary);
    f.read((char *)v.data(), (std::streamsize)(count * sizeof(T)));
    if (!f) v.clear();
    return v;
}

int main(int argc, char **argv)
{
    if (argc < 5) { std::printf("usage: warped_color_export depth.u16 bgra.u8 frames out.ply\n"); return 2; }
    const int frames = std::atoi(argv[3]);
    KinFuParams params = KinFuParams::default_params_dynamicfusion();
    params.dfusion_flags = 8 | 256 | 1024;                              // WARPED_INTEGRATE | COLOR | WARPED_COLOR
    const size_t npix = (size_t)params.cols * params.rows;
    const std::vector<unsigned short> depth_all = read_all<unsigned short>(argv[1], npix * frames);
    const std::vector<unsigned char> bgra_all = read_all<unsigned char>(argv[2], npix * 4 * frames);
    CHECK(!depth_all.empty() && !bgra_all.empty());
    if (fails) return 1;

    KinFu kf(params);
    for (int t = 0; t < frames; ++t) {
        cuda::Depth depth;
        cuda::Image image;
        depth.upload(&depth_all[npix * t], params.cols * sizeof(unsigned short), params.rows, params.cols);
        image.upload(&bgra_all[npix * 4 * t], params.cols * 4, params.rows, params.cols);
        kf(depth, image);
    }
    cv::Mat v, n, f, c;
    CHECK(kf.getMesh(v, n, f, true));
    CHECK(kf.getMeshColors(c));
    CHECK(c.cols * c.rows == v.cols * v.rows && c.cols * c.rows > 1000);
    CHECK(writePly(argv[4], v, n, f, c) == (long)v.cols * v.rows);
    std::printf(fails ? "warped_color_export: %d check(s) FAILED\n" : "warped_color_export: all checks passed\n", fails);
    return fails ? 1 : 0;
}
