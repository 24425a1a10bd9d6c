// Drop-in replacement of se2lam's include/se2lam/ORBextractor.h (reference lines 36-84): same class, same
// public signatures, so Frame.cpp:25 `(*mpORBExtractor)(img, cv::Mat(), keyPoints, descriptors)`,
// Track.cpp:34 / Localizer.cpp:21 `new ORBextractor(Config::MaxFtrNumber, Config::ScaleFactor, Config::MaxLevel)`
// and Frame.cpp:47-48 GetLevels()/GetScaleFactor() compile unchanged. The implementation forwards to the
// C ABI (se2gpu_orb_*) of libse2gpu.so; there is no CPU path. Header-only: link with -lse2gpu.
#ifndef ORBEXTRACTOR_H
#define ORBEXTRACTOR_H

#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <vector>

#if defined(__has_include)
#if __has_include(<opencv2/core/core.hpp>)
#include <opencv2/core/core.hpp>
#include <opencv2/features2d/features2d.hpp>
#include <opencv2/imgproc/imgproc.hpp>
#define SE2LAM_HAVE_OPENCV 1
#endif
#endif
#ifndef SE2LAM_HAVE_OPENCV
#include "cv_compat.h"
#endif

#include "../se2gpu.h"

namespace se2lam
{

class ORBextractor
{
public:

    enum {HARRIS_SCORE=0, FAST_SCORE=1 };

    ORBextractor(int nfeatures = 1000, float scaleFactor = 1.2f, int nlevels = 8, int scoreType=FAST_SCORE, int fastTh = 20)
        : nfeatures(nfeatures), scaleFactor(scaleFactor), nlevels(nlevels), scoreType(scoreType), fastTh(fastTh),
          mHandle(nullptr), mMaxW(0), mMaxH(0)
    {
    }

    ~ORBextractor(){ if (mHandle) se2gpu_orb_destroy(mHandle); }

    // Compute the ORB features and descriptors on an image
    void operator()( cv::InputArray image, cv::InputArray mask,
      std::vector<cv::KeyPoint>& keypoints,
      cv::OutputArray descriptors)
    {
        if (image.empty())
            return;                                    // reference: silent return (ORBextractor.cpp:730-731)
        cv::Mat img = image.getMat();
        assert(img.type() == CV_8UC1);                 // :734
        (void)mask;                                    // always empty at the only call site (Frame.cpp:25)
        ensure(img.cols, img.rows);
        mKps.resize(nfeatures);
        mDesc.resize((size_t)nfeatures * 32);
        int count = 0;
        const int rc = se2gpu_orb_extract(mHandle, img.data, 1, img.cols, img.rows, (int)img.step, 0,
                                          reinterpret_cast<se2gpu_keypoint*>(mKps.data()), mDesc.data(), &count);
        if (rc != SE2GPU_OK) {
            std::fprintf(stderr, "se2lam::ORBextractor (GPU): %s\n", se2gpu_last_error());
            std::abort();                              // no CPU fallback by design
        }
        keypoints.assign(mKps.begin(), mKps.begin() + count);
        if (count == 0) { descriptors.release(); return; }          // :747-748
        descriptors.create(count, 32, CV_8U);                        // :751
        cv::Mat d = descriptors.getMat();
        for (int i = 0; i < count; ++i) std::memcpy(d.ptr<unsigned char>(i), &mDesc[(size_t)i * 32], 32);
    }

    // Extension (not in the reference class): fold Frame::Frame's cv::undistort(im, img, Kcam, Dcam) (Frame.cpp:22) into
    // the pyramid's level 0, so the frame stays on the device. K: Config::Kcam.ptr<float>() (3x3 row-major), dist:
    // Config::Dcam.ptr<float>() with n = 4, 5, 8 or 12 coefficients. After this call operator() takes the RAW frame.
    void SetUndistort(const float* K, const float* dist, int n)
    {
        for (int i = 0; i < 9; ++i) mUndK[i] = K[i];
        mUndN = n;
        for (int i = 0; i < n && i < 14; ++i) mUndD[i] = dist[i];
        mUndOn = true;
        if (mHandle) applyUndistort();
    }

    int inline GetLevels(){
        return nlevels;}

    float inline GetScaleFactor(){
        return scaleFactor;}

protected:
    void ensure(int w, int h)
    {
        if (mHandle && w <= mMaxW && h <= mMaxH) return;
        if (mHandle) se2gpu_orb_destroy(mHandle);
        mMaxW = w > mMaxW ? w : mMaxW; mMaxH = h > mMaxH ? h : mMaxH;
        mHandle = se2gpu_orb_create_scored(nfeatures, (float)scaleFactor, nlevels, scoreType, fastTh, mMaxW, mMaxH, 1, 0);
        if (!mHandle) {
            std::fprintf(stderr, "se2lam::ORBextractor (GPU): %s\n", se2gpu_last_error());
            std::abort();
        }
        if (mUndOn) applyUndistort();
    }

    void applyUndistort()
    {
        if (se2gpu_orb_set_undistort(mHandle, mUndK, mUndN ? mUndD : 0, mUndN) != SE2GPU_OK) {
            std::fprintf(stderr, "se2lam::ORBextractor (GPU): %s\n", se2gpu_last_error());
            std::abort();
        }
    }

    int nfeatures;
    double scaleFactor;
    int nlevels;
    int scoreType;
    int fastTh;

    se2gpu_orb* mHandle;
    int mMaxW, mMaxH;
    bool mUndOn = false;
    float mUndK[9], mUndD[14];
    int mUndN = 0;
    std::vector<cv::KeyPoint> mKps;
    std::vector<unsigned char> mDesc;

private:
    ORBextractor(const ORBextractor&);
    ORBextractor& operator=(const ORBextractor&);
};

} //namespace se2lam

#endif
