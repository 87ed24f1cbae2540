// exporter_ref facade — TEST INFRASTRUCTURE ONLY.  An inert VideoWriter, so that Exporter.cpp, which also encodes files,
// compiles for its canvas functions: it opens nothing and writes nothing.
#pragma once
#include <string>

#include "opencv2/core.hpp"

namespace cv {

class VideoWriter {
public:
    static int fourcc(char c1, char c2, char c3, char c4) {
        return (c1 & 255) | ((c2 & 255) << 8) | ((c3 & 255) << 16) | ((c4 & 255) << 24);
    }
    bool open(const std::string&, int, double, Size, bool = true) { return false; }
    bool isOpened() const { return false; }
    void write(const Mat&) {}
    void release() {}
};

}  // namespace cv
