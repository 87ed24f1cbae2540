// exporter_ref facade — TEST INFRASTRUCTURE ONLY.  imgproc slice (see core.hpp); each function is forwarded to the
// OpenCV kernel of the same name in cv2 (facade.cpp).
#pragma once
#include <string>

#include "opencv2/core.hpp"

namespace cv {

enum ColorConversionCodes { COLOR_GRAY2BGR = 8 };
enum InterpolationFlags { INTER_LINEAR = 1 };
enum HersheyFonts { FONT_HERSHEY_SIMPLEX = 0 };
enum LineTypes { LINE_8 = 8, LINE_AA = 16 };

void cvtColor(const Mat& src, Mat& dst, int code);
void resize(const Mat& src, Mat& dst, Size dsize, double fx = 0, double fy = 0, int interpolation = INTER_LINEAR);
void addWeighted(const Mat& a, double alpha, const Mat& b, double beta, double gamma, Mat& dst);
Size getTextSize(const std::string& text, int fontFace, double fontScale, int thickness, int* baseLine);
void putText(Mat& img, const std::string& text, Point org, int fontFace, double fontScale, Scalar color, int thickness = 1,
             int lineType = LINE_8, bool bottomLeftOrigin = false);

}  // namespace cv
