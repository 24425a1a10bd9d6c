// se2lam::ORBextractor(1000, 1.2f, 8, HARRIS_SCORE) through the drop-in header, called like Frame::Frame (src/Frame.cpp:25).
// usage: orb_harris_demo <in.bin> <out.bin>   in: int w, int h, w*h bytes; out: int N, N cv::KeyPoint, N x 32 descriptor bytes
#include <cstdio>
#include <vector>

#include "se2lam/ORBextractor.h"

using namespace se2lam;

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb"); FILE* fo = fopen(argv[2], "wb");
    if (!fi || !fo) return 2;
    int w, h;
    if (fread(&w, 4, 1, fi) != 1 || fread(&h, 4, 1, fi) != 1) return 2;
    std::vector<unsigned char> pix((size_t)w * h);
    if (fread(pix.data(), 1, pix.size(), fi) != pix.size()) return 2;
    cv::Mat img(h, w, CV_8UC1, pix.data());
    ORBextractor ext(1000, 1.2f, 8, ORBextractor::HARRIS_SCORE);
    std::vector<cv::KeyPoint> keyPoints;
    cv::Mat descriptors;
    ext(img, cv::Mat(), keyPoints, descriptors);
    const int N = (int)keyPoints.size();
    fwrite(&N, 4, 1, fo);
    fwrite(keyPoints.data(), sizeof(cv::KeyPoint), keyPoints.size(), fo);
    for (int i = 0; i < N; ++i) fwrite(descriptors.ptr<unsigned char>(i), 1, 32, fo);
    fclose(fi); fclose(fo);
    return 0;
}
