// ORB front-end ORACLE, HARRIS_SCORE branch — TEST INFRASTRUCTURE ONLY.
//
// se2lam::ORBextractor with scoreType == HARRIS_SCORE: after the FAST(fastTh) / FAST(7) fallback of every grid cell,
// HarrisResponses(cellImage, cellKeyPoints, 7, HARRIS_K) (reference src/ORBextractor.cpp:85-126, called at :625-629)
// overwrites each keypoint's response, and everything downstream (retainBest per cell and per level, the output
// KeyPoint.response) uses that float instead of the FAST score.
//
// Built as a library of its own (oracle/liborb_harris_oracle.so, oracle/pyharris.py) with liboracle.so's flags (no
// -march, -ffp-contract=off). It compiles oracle/orb_oracle.cpp into the same translation unit to reuse the pinned
// primitives and the Extractor (pyramid, FAST, retainBest, IC_Angle, blur, rBRIEF) and restates only the keypoint
// orchestration (:531-716) with the Harris step; -fvisibility=hidden keeps orb_oracle.cpp's own exports out of this
// library. Pinned against cv2 4.13.0 by oracle/pin_orb_harris_against_cv2.py (tests/golden/orb_harris_golden.npz).
#include "orb_oracle.cpp"

#define HARRIS_EXPORT extern "C" __attribute__((visibility("default")))

namespace {

const float HARRIS_K = 0.04f;   // ORBextractor.cpp:84

// HarrisResponses(img, pts, blockSize, harris_k), ORBextractor.cpp:85-126: pixel (x, y) of the cell ROI is img[y*step + x] and
// pts are in cell coordinates; the 3x3 gradients of the block reach one pixel beyond it on every side.
// The float expression in C++ evaluation order; this file is compiled without contraction.
void harris_responses(const uint8_t* img, int step, std::vector<KeyPoint>& pts, int blockSize, float harris_k) {
    const int r = blockSize / 2;
    float scale = (1 << 2) * blockSize * 255.0f;
    scale = 1.0f / scale;
    const float scale_sq_sq = scale * scale * scale * scale;
    for (KeyPoint& kp : pts) {
        const int x0 = cv_round_f(kp.x - r), y0 = cv_round_f(kp.y - r);
        const uint8_t* ptr0 = img + (ptrdiff_t)y0 * step + x0;
        int a = 0, b = 0, c = 0;
        for (int i = 0; i < blockSize; ++i)
            for (int j = 0; j < blockSize; ++j) {
                const uint8_t* ptr = ptr0 + (ptrdiff_t)i * step + j;
                const int Ix = (ptr[1] - ptr[-1]) * 2 + (ptr[-step + 1] - ptr[-step - 1]) + (ptr[step + 1] - ptr[step - 1]);
                const int Iy = (ptr[step] - ptr[-step]) * 2 + (ptr[step - 1] - ptr[-step - 1]) + (ptr[step + 1] - ptr[-step + 1]);
                a += Ix * Ix;
                b += Iy * Iy;
                c += Ix * Iy;
            }
        kp.response = ((float)a * b - (float)c * c - harris_k * ((float)a + b) * ((float)a + b)) * scale_sq_sq;
    }
}

struct HarrisExtractor : Extractor {
    HarrisExtractor(int nf, float sf, int nl, int ft) : Extractor(nf, sf, nl, ft) {}

    // ORBextractor.cpp:531-716 with scoreType == HARRIS_SCORE
    void computeKeyPoints(std::vector<std::vector<KeyPoint>>& all) {
        all.assign(nlevels, {});
        float imageRatio = (float)pyr[0].w / pyr[0].h;
        for (int level = 0; level < nlevels; ++level) {
            const int nDesiredFeatures = mnFeaturesPerLevel[level];
            const int levelCols = (int)sqrtf((float)nDesiredFeatures / (5 * imageRatio));
            const int levelRows = (int)(imageRatio * levelCols);
            const int minBorderX = EDGE_THRESHOLD, minBorderY = minBorderX;
            const int maxBorderX = pyr[level].w - EDGE_THRESHOLD;
            const int maxBorderY = pyr[level].h - EDGE_THRESHOLD;
            const int W = maxBorderX - minBorderX, H = maxBorderY - minBorderY;
            const int cellW = (int)ceilf((float)W / levelCols);
            const int cellH = (int)ceilf((float)H / levelRows);
            const int nCells = levelRows * levelCols;
            const int nfeaturesCell = (int)ceilf((float)nDesiredFeatures / nCells);
            std::vector<std::vector<std::vector<KeyPoint>>> cellKeyPoints(levelRows, std::vector<std::vector<KeyPoint>>(levelCols));
            std::vector<std::vector<int>> nToRetain(levelRows, std::vector<int>(levelCols, 0));
            std::vector<std::vector<int>> nTotal(levelRows, std::vector<int>(levelCols, 0));
            std::vector<std::vector<bool>> bNoMore(levelRows, std::vector<bool>(levelCols, false));
            std::vector<int> iniXCol(levelCols), iniYRow(levelRows);
            int nNoMore = 0, nToDistribute = 0;
            float hY = cellH + 6;
            const Plane& P = pyr[level];
            for (int i = 0; i < levelRows; i++) {
                const float iniY = minBorderY + i * cellH - 3;
                iniYRow[i] = iniY;
                if (i == levelRows - 1) {
                    hY = maxBorderY + 3 - iniY;
                    if (hY <= 0) continue;
                }
                float hX = cellW + 6;
                for (int j = 0; j < levelCols; j++) {
                    float iniX;
                    if (i == 0) { iniX = minBorderX + j * cellW - 3; iniXCol[j] = iniX; }
                    else iniX = iniXCol[j];
                    if (j == levelCols - 1) {
                        hX = maxBorderX + 3 - iniX;
                        if (hX <= 0) continue;
                    }
                    int r0 = (int)iniY, r1 = (int)(iniY + hY), c0 = (int)iniX, c1 = (int)(iniX + hX);
                    const uint8_t* cell = P.roi() + (ptrdiff_t)r0 * P.pitch + c0;
                    std::vector<KeyPoint>& kc = cellKeyPoints[i][j];
                    fast9_16_nms(cell, c1 - c0, r1 - r0, P.pitch, fastTh, kc);
                    if (kc.size() <= 3) {
                        kc.clear();
                        fast9_16_nms(cell, c1 - c0, r1 - r0, P.pitch, 7, kc);
                    }
                    harris_responses(cell, P.pitch, kc, 7, HARRIS_K);   // :625-629
                    const int nKeys = (int)kc.size();
                    nTotal[i][j] = nKeys;
                    if (nKeys > nfeaturesCell) { nToRetain[i][j] = nfeaturesCell; bNoMore[i][j] = false; }
                    else { nToRetain[i][j] = nKeys; nToDistribute += nfeaturesCell - nKeys; bNoMore[i][j] = true; nNoMore++; }
                }
            }
            while (nToDistribute > 0 && nNoMore < nCells) {
                int nNewFeaturesCell = (int)(nfeaturesCell + ceilf((float)nToDistribute / (nCells - nNoMore)));
                nToDistribute = 0;
                for (int i = 0; i < levelRows; i++)
                    for (int j = 0; j < levelCols; j++)
                        if (!bNoMore[i][j]) {
                            if (nTotal[i][j] > nNewFeaturesCell) { nToRetain[i][j] = nNewFeaturesCell; bNoMore[i][j] = false; }
                            else { nToRetain[i][j] = nTotal[i][j]; nToDistribute += nNewFeaturesCell - nTotal[i][j]; bNoMore[i][j] = true; nNoMore++; }
                        }
            }
            std::vector<KeyPoint>& keypoints = all[level];
            const int scaledPatchSize = (int)(PATCH_SIZE * mvScaleFactor[level]);
            for (int i = 0; i < levelRows; i++)
                for (int j = 0; j < levelCols; j++) {
                    std::vector<KeyPoint>& keysCell = cellKeyPoints[i][j];
                    retain_best(keysCell, nToRetain[i][j]);
                    if ((int)keysCell.size() > nToRetain[i][j]) keysCell.resize(nToRetain[i][j]);
                    for (size_t k = 0; k < keysCell.size(); k++) {
                        keysCell[k].x += iniXCol[j];
                        keysCell[k].y += iniYRow[i];
                        keysCell[k].octave = level;
                        keysCell[k].size = (float)scaledPatchSize;
                        keypoints.push_back(keysCell[k]);
                    }
                }
            if ((int)keypoints.size() > nDesiredFeatures) {
                retain_best(keypoints, nDesiredFeatures);
                keypoints.resize(nDesiredFeatures);
            }
        }
        for (int level = 0; level < nlevels; ++level)
            for (auto& kp : all[level]) kp.angle = icAngle(pyr[level], kp.x, kp.y);
    }

    // ORBextractor.cpp:727-788 (Extractor::extract with this computeKeyPoints)
    int extract(const uint8_t* img, int w, int h, int stride, KeyPoint* kps_out, uint8_t* desc_out) {
        if (!img || w <= 0 || h <= 0) return 0;
        computePyramid(img, w, h, stride);
        std::vector<std::vector<KeyPoint>> all;
        computeKeyPoints(all);
        blurred.assign(nlevels, Plane());
        int offset = 0;
        for (int level = 0; level < nlevels; ++level) {
            std::vector<KeyPoint>& kps = all[level];
            if (kps.empty()) continue;
            blurLevel(level);
            for (size_t i = 0; i < kps.size(); ++i) descriptor(blurred[level], kps[i], desc_out + (size_t)(offset + i) * 32);
            if (level != 0) {
                float scale = mvScaleFactor[level];
                for (auto& kp : kps) { kp.x *= scale; kp.y *= scale; }
            }
            memcpy(kps_out + offset, kps.data(), kps.size() * sizeof(KeyPoint));
            offset += (int)kps.size();
        }
        return offset;
    }
};

}  // namespace

// ORBextractor(nfeatures, scaleFactor, nlevels, HARRIS_SCORE, fastTh)
HARRIS_EXPORT void* orb_harris_oracle_create(int nfeatures, float scaleFactor, int nlevels, int fastTh) {
    return new HarrisExtractor(nfeatures, scaleFactor, nlevels, fastTh);
}
HARRIS_EXPORT void orb_harris_oracle_destroy(void* h) { delete (HarrisExtractor*)h; }
// kps: n x 28 bytes (cv::KeyPoint layout), desc: n x 32 bytes; both sized for >= nfeatures entries
HARRIS_EXPORT int orb_harris_oracle_extract(void* h, const uint8_t* img, int w, int h_, int stride, void* kps, uint8_t* desc) {
    return ((HarrisExtractor*)h)->extract(img, w, h_, stride, (KeyPoint*)kps, desc);
}
// HarrisResponses(img, pts, 7, 0.04f) at n points (xs[i], ys[i]) of an 8-bit image with row pitch `pitch`: out[i] = response
HARRIS_EXPORT void orb_harris_oracle_responses(const uint8_t* img, int pitch, const float* xs, const float* ys, int n, float* out) {
    std::vector<KeyPoint> k(n);
    for (int i = 0; i < n; ++i) k[i] = KeyPoint{xs[i], ys[i], 7.f, -1.f, 0.f, 0, -1};
    harris_responses(img, pitch, k, 7, HARRIS_K);
    for (int i = 0; i < n; ++i) out[i] = k[i].response;
}
