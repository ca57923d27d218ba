// The Monte-Carlo variance through the C++ shim class: segmentImage, then computeVariance on the classes it returned and
// generateVarianceImage on the result (bayesian_segnet.cpp:205-260, 330-344).
//
//   test_shim_variance <prototxt> <caffemodel> <bgr.bin> <out_dir>
//
// bgr.bin = int32 rows, int32 cols, int32 channels, then the pixels.  Dumps classes, variance and the normalised variance
// image for tests/test_shim_variance.py to compare with the Python mirror of the same C-ABI and with cv2.normalize.
#include <cstdio>
#include <fstream>
#include <stdexcept>
#include <string>

#include "bayesian_segnet/bayesian_segnet.hpp"

using namespace SIVO;

static int failures = 0;
#define EXPECT(cond) do { if (!(cond)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } } while (0)

static cv::Mat read_bin(const std::string &path) {
    std::ifstream f(path, std::ios::binary);
    int hdr[3] = {0, 0, 0};
    f.read(reinterpret_cast<char *>(hdr), sizeof hdr);
    cv::Mat m(hdr[0], hdr[1], hdr[2] == 3 ? CV_8UC3 : CV_8UC1);
    f.read(reinterpret_cast<char *>(m.data), static_cast<std::streamsize>(m.total() * m.elemSize()));
    if (!f) throw std::runtime_error("cannot read " + path);
    return m;
}
static void dump(const std::string &path, const void *p, size_t bytes) {
    std::ofstream f(path, std::ios::binary);
    f.write(static_cast<const char *>(p), static_cast<std::streamsize>(bytes));
}

int main(int argc, char **argv) {
    if (argc < 5) { std::printf("usage: test_shim_variance <prototxt> <caffemodel> <bgr.bin> <out_dir>\n"); return 2; }
    const std::string out = argv[4];
    cv::Mat image = read_bin(argv[3]);
    BayesianSegNet net{BayesianSegNetParams{argv[1], argv[2]}};
    cv::Size g = net.getInputGeometry();
    MatXu classes;
    MatXd confidence, entropy;
    net.segmentImage(image, classes, confidence, entropy);
    MatXd variance = net.computeVariance(classes);
    EXPECT(variance.rows() == g.height && variance.cols() == g.width);
    cv::Mat var_img = net.generateVarianceImage(variance);
    EXPECT(var_img.rows == g.height && var_img.cols == g.width);
    MatXu wrong(g.height + 1, g.width);
    bool threw = false;
    try { net.computeVariance(wrong); } catch (const std::invalid_argument &) { threw = true; }
    EXPECT(threw);
    dump(out + "/classes.bin", classes.data(), classes.size());
    dump(out + "/variance.bin", variance.data(), variance.size() * sizeof(double));
    cv::Mat vc = var_img.clone();
    dump(out + "/variance_image.bin", vc.data, vc.total() * sizeof(double));
    std::printf(failures ? "SHIM VARIANCE FAILED\n" : "SHIM VARIANCE OK\n");
    return failures ? 1 : 0;
}
