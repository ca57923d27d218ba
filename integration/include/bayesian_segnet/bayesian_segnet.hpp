/* Drop-in replacement for SIVO's include/bayesian_segnet/bayesian_segnet.hpp (public API :46-50,67-105,108-170):
 * same namespace, typedefs, enum, params struct and member signatures; the Caffe members (:254-257) become an
 * opaque handle into libsivo_b200.so.  System.cc:94-95,127,158 and Frame.cc:232-245 compile unchanged. */
#ifndef SIVO_BAYESIAN_SEGNET_HPP
#define SIVO_BAYESIAN_SEGNET_HPP

#include <Eigen/Core>
#include <opencv2/core/core.hpp>
#include <opencv2/core/eigen.hpp>
#include <opencv2/imgproc/imgproc.hpp>

#include <cstdint>
#include <string>

#include "sivo_b200.h"

namespace SIVO {

using MatXd = Eigen::Matrix<double, Eigen::Dynamic, Eigen::Dynamic, Eigen::RowMajor>;
using MatXu = Eigen::Matrix<uint8_t, Eigen::Dynamic, Eigen::Dynamic, Eigen::RowMajor>;

double computeEntropy(const double probability);

enum Classes {
    ROAD, SIDEWALK, BUILDING, WALL, POLE, TRAFFIC_LIGHT, TRAFFIC_SIGN, VEGETATION, TERRAIN, SKY, PERSON, CAR,
    COMMERCIAL_VEHICLE, BIKE, VOID = 255
};

struct BayesianSegNetParams {
    BayesianSegNetParams(const std::string model_filepath, const std::string weights_filepath)
        : model_file(model_filepath), weights_file(weights_filepath) {}
    bool use_gpu = true;  // kept for source compatibility; this backend always runs on the GPU
    std::string model_file;
    std::string weights_file;
};

class BayesianSegNet {
 public:
    EIGEN_MAKE_ALIGNED_OPERATOR_NEW
    explicit BayesianSegNet(const BayesianSegNetParams &params);
    ~BayesianSegNet();
    BayesianSegNet(const BayesianSegNet &) = delete;
    BayesianSegNet &operator=(const BayesianSegNet &) = delete;

    void segmentImage(const cv::Mat &image, MatXu &classes, MatXd &confidence, MatXd &entropy);
    cv::Size getInputGeometry() { return this->input_geometry; }
    // Private and never called in the reference (bayesian_segnet.hpp, bayesian_segnet.cpp:205-260); public here because the
    // Monte-Carlo samples stay on the device and only the library can compute it.  Per pixel, the sample variance over the
    // last segmentImage's T samples of the softmax probability of classes(row, col); 0 where that class does not exist.
    MatXd computeVariance(const MatXu &classes);
    cv::Mat generateConfidenceImage(const MatXd &confidence);
    cv::Mat generateVarianceImage(MatXd &variance);
    cv::Mat generateEntropyImage(MatXd &entropy);
    cv::Mat generateSegmentedImage(const MatXu &classes, const cv::Mat &test_image);

 private:
    cv::Mat resizeImage(const cv::Mat &image);
    BayesianSegNetParams params;
    sivo_segnet_t *handle = nullptr;
    cv::Size input_geometry;
    cv::Mat class_colours = cv::Mat(256, 1, CV_8UC3, cv::Scalar(0, 0, 0));
};
}  // namespace SIVO
#endif
