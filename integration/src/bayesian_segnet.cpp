/* Shim translation unit: SIVO::BayesianSegNet over the C-ABI.  Replaces src/bayesian_segnet/bayesian_segnet.cpp in
 * the `bayesian_segnet` target (CMakeLists.txt:74-81), which then links libsivo_b200.so instead of ${Caffe_LIBRARIES}. */
#include "bayesian_segnet/bayesian_segnet.hpp"

#include <cstdlib>
#include <iostream>
#include <stdexcept>

namespace SIVO {

double computeEntropy(const double probability) {
    return probability == 0 ? 0 : -1.0 * probability * std::log2(probability);
}

BayesianSegNet::BayesianSegNet(const BayesianSegNetParams &params) : params(params) {
    // extra knobs come from the environment so the host signatures stay untouched
    const char *dev = std::getenv("SIVO_B200_DEVICE");
    const char *seed = std::getenv("SIVO_B200_SEED");
    int rc = sivo_segnet_create(params.model_file.c_str(), params.weights_file.c_str(), dev ? std::atoi(dev) : 0,
                                seed ? std::strtoull(seed, nullptr, 10) : 1234ull, &this->handle);
    if (rc == SIVO_EINVAL) throw std::invalid_argument(sivo_last_error());  // bayesian_segnet.cpp:66,68,82,86
    if (rc != SIVO_OK) throw std::runtime_error(sivo_last_error());        // the reference LOG(FATAL)s here
    int w = 0, h = 0;
    sivo_segnet_geometry(this->handle, &w, &h, nullptr, nullptr);
    this->input_geometry = cv::Size{w, h};
    const cv::Vec3b colours[14] = {{128, 64, 128}, {232, 35, 244}, {69, 69, 69}, {156, 102, 102}, {153, 153, 153},
                                   {30, 170, 250}, {0, 220, 220}, {35, 142, 107}, {152, 251, 152}, {180, 130, 70},
                                   {60, 20, 220}, {142, 0, 0}, {70, 0, 0}, {32, 11, 119}};
    for (int i = 0; i < 14; ++i) this->class_colours.at<cv::Vec3b>(i) = colours[i];
    std::cout << "Class colours loaded!" << std::endl;
}

BayesianSegNet::~BayesianSegNet() { sivo_segnet_destroy(this->handle); }

void BayesianSegNet::segmentImage(const cv::Mat &image, MatXu &classes, MatXd &confidence, MatXd &entropy) {
    CV_Assert(image.type() == CV_8UC3);
    classes.resize(input_geometry.height, input_geometry.width);
    confidence.resize(input_geometry.height, input_geometry.width);
    entropy.resize(input_geometry.height, input_geometry.width);
    int rc = sivo_segnet_run(this->handle, image.data, image.rows, image.cols, image.step, classes.data(),
                             confidence.data(), entropy.data());
    if (rc != SIVO_OK) throw std::runtime_error(sivo_last_error());
}

MatXd BayesianSegNet::computeVariance(const MatXu &classes) {
    if (classes.rows() != input_geometry.height || classes.cols() != input_geometry.width)
        throw std::invalid_argument("computeVariance: the class map must have the network's input geometry");
    MatXd variance(input_geometry.height, input_geometry.width);
    int rc = sivo_segnet_variance(this->handle, classes.data(), variance.data());
    if (rc != SIVO_OK) throw std::runtime_error(sivo_last_error());
    return variance;
}

cv::Mat BayesianSegNet::resizeImage(const cv::Mat &image) {
    if (image.size() == this->input_geometry) return image;
    cv::Mat out;
    if (image.rows >= input_geometry.height && image.cols >= input_geometry.width) {
        cv::Rect roi{image.cols / 2 - input_geometry.width / 2, image.rows / 2 - input_geometry.height / 2,
                     input_geometry.width, input_geometry.height};
        out = image(roi).clone();
    }
    return out;
}

cv::Mat BayesianSegNet::generateConfidenceImage(const MatXd &confidence) {
    cv::Mat img(static_cast<int>(confidence.rows()), static_cast<int>(confidence.cols()), CV_64FC1);
    cv::eigen2cv(confidence, img);
    return img;
}

static cv::Mat normalised(const MatXd &m) {
    cv::Mat img(static_cast<int>(m.rows()), static_cast<int>(m.cols()), CV_64FC1), out;
    cv::eigen2cv(m, img);
    cv::normalize(img, out, 0.0, 1.0, cv::NORM_MINMAX, CV_64FC1);
    return out;
}
cv::Mat BayesianSegNet::generateVarianceImage(MatXd &variance) { return normalised(variance); }
cv::Mat BayesianSegNet::generateEntropyImage(MatXd &entropy) { return normalised(entropy); }

cv::Mat BayesianSegNet::generateSegmentedImage(const MatXu &classes, const cv::Mat &test_image) {
    cv::Mat cls(static_cast<int>(classes.rows()), static_cast<int>(classes.cols()), CV_8UC1), cls3, seg;
    cv::eigen2cv(classes, cls);
    cv::cvtColor(cls, cls3, cv::COLOR_GRAY2BGR);
    cv::LUT(cls3, this->class_colours, seg);
    cv::addWeighted(seg, 0.5, this->resizeImage(test_image), 0.5, 0, seg);
    return seg;
}
}  // namespace SIVO
