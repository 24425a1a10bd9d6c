// SE(2)-XYZ subset of the g2o graph API that se2lam's local BA drives, implemented as a thin recorder that
// hands the graph to the C ABI (se2gpu_ba_*). It exists so that Map::loadLocalGraph (reference
// src/Map.cpp:891-1053), LocalMapper::localBA (src/LocalMapper.cpp:232-302) and Map::optimizeLocalGraph
// (src/Map.cpp:754-783) keep their source shape when real g2o is NOT installed (this build container has
// neither g2o nor Eigen). Covered: VertexSE2, VertexSBAPointXYZ, CameraParameters, EdgeSE2XYZ, PreEdgeSE2,
// SparseOptimizer::{setAlgorithm,setVerbose,setForceStopFlag,vertex,addVertex,addEdge,addParameter,
// initializeOptimization,optimize,clear,clearParameters}. SE(3) vertex/edge types (GlobalMapper, Localizer)
// are out of scope (SURVEY.md section 8b option ii). With real g2o installed use the GPU-backed
// OptimizationAlgorithm described in INTEGRATION.md instead of this file.
#pragma once
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <vector>

#include "../se2gpu.h"

namespace g2o {

template <int R, int C>
struct Mat {
    double d[R * C];
    Mat() { for (int i = 0; i < R * C; ++i) d[i] = 0; }
    double& operator()(int r, int c) { return d[r * C + c]; }
    double operator()(int r, int c) const { return d[r * C + c]; }
    double& operator()(int i) { return d[i]; }
    double operator()(int i) const { return d[i]; }
    double& operator[](int i) { return d[i]; }
    double operator[](int i) const { return d[i]; }
    static Mat Identity() { Mat m; for (int i = 0; i < (R < C ? R : C); ++i) m(i, i) = 1; return m; }
};
typedef Mat<2, 1> Vector2D; typedef Mat<3, 1> Vector3D; typedef Mat<2, 2> Matrix2D; typedef Mat<3, 3> Matrix3D;
inline Vector2D makeVector2D(double a, double b) { Vector2D v; v[0] = a; v[1] = b; return v; }
inline Vector3D makeVector3D(double a, double b, double c) { Vector3D v; v[0] = a; v[1] = b; v[2] = c; return v; }

class SE2 {
public:
    SE2() : x_(0), y_(0), th_(0) {}
    SE2(double x, double y, double theta) : x_(x), y_(y), th_(theta) {}
    Vector3D toVector() const { return makeVector3D(x_, y_, th_); }
    double x_, y_, th_;
};

struct SE3Quat {   // rotation matrix + translation is all the SE(2)-XYZ edge needs from it
    Matrix3D R; Vector3D t;
    SE3Quat() { R = Matrix3D::Identity(); }
    SE3Quat(const Matrix3D& R_, const Vector3D& t_) : R(R_), t(t_) {}
    SE3Quat inverse() const {
        SE3Quat o;
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) o.R(i, j) = R(j, i);
        for (int i = 0; i < 3; ++i) o.t[i] = -(o.R(i, 0) * t[0] + o.R(i, 1) * t[1] + o.R(i, 2) * t[2]);
        return o;
    }
};

struct Vertex { int id = -1; bool fixed = false; virtual ~Vertex() {} void setId(int i) { id = i; } void setFixed(bool f) { fixed = f; } };
struct VertexSE2 : Vertex { SE2 est; void setEstimate(const SE2& e) { est = e; } const SE2& estimate() const { return est; } };
struct VertexSBAPointXYZ : Vertex {
    Vector3D est; bool marginalized = true;
    void setEstimate(const Vector3D& e) { est = e; } const Vector3D& estimate() const { return est; } void setMarginalized(bool m) { marginalized = m; }
};
struct CameraParameters {
    double focal_length; Vector2D principle_point; double baseline; int id = 0;
    CameraParameters(double f, const Vector2D& pp, double b) : focal_length(f), principle_point(pp), baseline(b) {}
    void setId(int i) { id = i; }
};
struct RobustKernelHuber { double delta = 1.0; void setDelta(double d) { delta = d; } };

struct Edge {
    Vertex* v[2] = {nullptr, nullptr};
    virtual ~Edge() {}
    Vertex** vertices() { return v; }
    int level() const { return level_; }
    void setLevel(int l) { level_ = l; }
    virtual void computeError() = 0;
    virtual double chi2() const = 0;
protected:
    int level_ = 0;
};
inline double normalize_theta(double theta) {                // g2o/stuff/misc.h
    if (theta >= -M_PI && theta < M_PI) return theta;
    const double multiplier = std::floor(theta / (2 * M_PI));
    theta = theta - multiplier * 2 * M_PI;
    if (theta >= M_PI) theta -= 2 * M_PI;
    if (theta < -M_PI) theta += 2 * M_PI;
    return theta;
}
// g2o::SE2ToSE3 (reference src/EdgeSE2XYZ.cpp:27-33): planar pose -> rotation about z + translation in the plane
inline SE3Quat SE2ToSE3(const SE2& se2) {
    SE3Quat T;
    const double c = std::cos(se2.th_), s = std::sin(se2.th_);
    T.R(0, 0) = c; T.R(0, 1) = -s; T.R(1, 0) = s; T.R(1, 1) = c; T.R(2, 2) = 1;
    T.t[0] = se2.x_; T.t[1] = se2.y_; T.t[2] = 0;
    return T;
}
struct EdgeSE2XYZ : Edge {
    Vector2D meas; Matrix2D info; CameraParameters* cam = nullptr; SE3Quat Tbc, Tcb; RobustKernelHuber* rk = nullptr;
    ~EdgeSE2XYZ() { delete rk; }
    void setMeasurement(const Vector2D& m) { meas = m; }
    void setInformation(const Matrix2D& i) { info = i; }
    const Matrix2D& information() const { return info; }
    void setCameraParameter(CameraParameters* c) { cam = c; }
    void setExtParameter(const SE3Quat& Tbc_) { Tbc = Tbc_; Tcb = Tbc.inverse(); }      // EdgeSE2XYZ.h:52
    void setRobustKernel(RobustKernelHuber* k) { rk = k; }
    // one edge, on the host, for the per-edge outlier test after a BA (EdgeSE2XYZ.cpp:61-72): e = cam_map(Tcb Tbw lw) - uv
    void computeError() override {
        const SE2& p = static_cast<VertexSE2*>(v[0])->estimate();
        const Vector3D& lw = static_cast<VertexSBAPointXYZ*>(v[1])->estimate();
        const SE3Quat Tbw = SE2ToSE3(p).inverse();
        double lb[3], lc[3];
        for (int r = 0; r < 3; ++r) lb[r] = Tbw.R(r, 0) * lw[0] + Tbw.R(r, 1) * lw[1] + Tbw.R(r, 2) * lw[2] + Tbw.t[r];
        for (int r = 0; r < 3; ++r) lc[r] = Tcb.R(r, 0) * lb[0] + Tcb.R(r, 1) * lb[1] + Tcb.R(r, 2) * lb[2] + Tcb.t[r];
        const double f = cam ? cam->focal_length : 1.0, cx = cam ? cam->principle_point[0] : 0.0, cy = cam ? cam->principle_point[1] : 0.0;
        err[0] = f * lc[0] / lc[2] + cx - meas[0];
        err[1] = f * lc[1] / lc[2] + cy - meas[1];
    }
    const Vector2D& error() const { return err; }
    double chi2() const override { return err[0] * (info(0, 0) * err[0] + info(0, 1) * err[1]) + err[1] * (info(1, 0) * err[0] + info(1, 1) * err[1]); }
private:
    Vector2D err;
};
struct PreEdgeSE2 : Edge {
    Vector3D meas; Matrix3D info;
    void setMeasurement(const Vector3D& m) { meas = m; }
    void setInformation(const Matrix3D& i) { info = i; }
    const Matrix3D& information() const { return info; }
    void computeError() override {                                                     // EdgeSE2XYZ.h:68-82
        const SE2& a = static_cast<VertexSE2*>(v[0])->estimate();
        const SE2& b = static_cast<VertexSE2*>(v[1])->estimate();
        const double c = std::cos(a.th_), s = std::sin(a.th_), dx = b.x_ - a.x_, dy = b.y_ - a.y_;
        err[0] = c * dx + s * dy - meas[0]; err[1] = -s * dx + c * dy - meas[1]; err[2] = b.th_ - a.th_ - meas[2];
    }
    const Vector3D& error() const { return err; }
    double chi2() const override {
        double s = 0;
        for (int r = 0; r < 3; ++r) for (int c2 = 0; c2 < 3; ++c2) s += err[r] * info(r, c2) * err[c2];
        return s;
    }
private:
    Vector3D err;
};

// the solver stack is fixed on the GPU (LM + Schur + Cholesky); these exist so that
// `new SlamLinearSolver(); new SlamBlockSolver(ls); new SlamAlgorithm(bs); optimizer.setAlgorithm(solver)` compiles
struct LinearSolverGpu {};
struct BlockSolverGpu { explicit BlockSolverGpu(LinearSolverGpu* l) : ls(l) {} ~BlockSolverGpu() { delete ls; } LinearSolverGpu* ls; };
struct OptimizationAlgorithmGpuLM { explicit OptimizationAlgorithmGpuLM(BlockSolverGpu* b) : bs(b) {} ~OptimizationAlgorithmGpuLM() { delete bs; } BlockSolverGpu* bs; };

class SparseOptimizer {
public:
    SparseOptimizer() {}
    ~SparseOptimizer() { clear(); clearParameters(); delete alg_; if (ba_) se2gpu_ba_destroy(ba_); }
    void setAlgorithm(OptimizationAlgorithmGpuLM* a) { delete alg_; alg_ = a; }
    void setVerbose(bool v) { verbose_ = v; }
    void setForceStopFlag(bool* f) { stop_ = f; }
    Vertex* vertex(int id) { auto it = vertices_.find(id); return it == vertices_.end() ? nullptr : it->second; }
    bool addVertex(Vertex* v) { if (vertices_.count(v->id)) return false; vertices_[v->id] = v; return true; }
    bool addEdge(Edge* e) { if (!e->v[0] || !e->v[1]) return false; edges_.push_back(e); return true; }
    bool addParameter(CameraParameters* p) { params_.push_back(p); return true; }
    void clear() { for (auto& kv : vertices_) delete kv.second; vertices_.clear(); for (Edge* e : edges_) delete e; edges_.clear(); ready_ = false; }
    void clearParameters() { for (auto* p : params_) delete p; params_.clear(); }
    const std::vector<Edge*>& edges() const { return edges_; }

    // builds the SoA problem (poses in id order first, then points: g2o's index mapping) and uploads it
    bool initializeOptimization(int level = 0) {
        ready_ = false;          // a rejected graph must not leave the previous window to optimize() (its vertices are gone)
        poses_.clear(); points_.clear();
        std::vector<double> xp, xl, uv, info, om, oinf;
        std::vector<uint8_t> fixed;
        std::vector<int> ep, el, oi, oj;
        std::map<int, int> pidx, lidx;
        for (auto& kv : vertices_) {
            if (auto* v = dynamic_cast<VertexSE2*>(kv.second)) {
                pidx[v->id] = (int)poses_.size(); poses_.push_back(v);
                xp.push_back(v->est.x_); xp.push_back(v->est.y_); xp.push_back(v->est.th_); fixed.push_back(v->fixed ? 1 : 0);
            } else if (auto* p = dynamic_cast<VertexSBAPointXYZ*>(kv.second)) {
                if (!p->marginalized || p->fixed) { std::fprintf(stderr, "se2gpu: only free, marginalised VertexSBAPointXYZ are supported\n"); return false; }
                lidx[p->id] = (int)points_.size(); points_.push_back(p);
                for (int k = 0; k < 3; ++k) xl.push_back(p->est[k]);
            } else { std::fprintf(stderr, "se2gpu: unsupported vertex type in an SE(2)-XYZ graph\n"); return false; }
        }
        const EdgeSE2XYZ* first = nullptr;
        for (Edge* e : edges_) {
            if (e->level() != level) continue;                // only the edges of this level are active (removeOutlierChi2 moves outliers to level 1)
            if (auto* x = dynamic_cast<EdgeSE2XYZ*>(e)) {
                if (!first) first = x;
                else if (x->cam != first->cam || std::memcmp(x->Tcb.R.d, first->Tcb.R.d, sizeof first->Tcb.R.d) || std::memcmp(x->Tcb.t.d, first->Tcb.t.d, sizeof first->Tcb.t.d) ||
                         (x->rk ? x->rk->delta : -1.0) != (first->rk ? first->rk->delta : -1.0)) {
                    std::fprintf(stderr, "se2gpu: EdgeSE2XYZ edges with different camera / extrinsic / Huber delta are not supported (Map::loadLocalGraph uses one of each)\n");
                    return false;
                }
                ep.push_back(pidx.at(x->v[0]->id)); el.push_back(lidx.at(x->v[1]->id));
                uv.push_back(x->meas[0]); uv.push_back(x->meas[1]);
                info.push_back(x->info(0, 0)); info.push_back(0.5 * (x->info(0, 1) + x->info(1, 0))); info.push_back(x->info(1, 1));
            } else if (auto* o = dynamic_cast<PreEdgeSE2*>(e)) {
                oi.push_back(pidx.at(o->v[0]->id)); oj.push_back(pidx.at(o->v[1]->id));
                for (int k = 0; k < 3; ++k) om.push_back(o->meas[k]);
                oinf.push_back(o->info(0, 0)); oinf.push_back(o->info(0, 1)); oinf.push_back(o->info(0, 2));
                oinf.push_back(o->info(1, 1)); oinf.push_back(o->info(1, 2)); oinf.push_back(o->info(2, 2));
            } else { std::fprintf(stderr, "se2gpu: unsupported edge type in an SE(2)-XYZ graph\n"); return false; }
        }
        if (poses_.empty()) return false;
        double Tcb[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0}, fx = 1, cx = 0, cy = 0, delta = 1;
        if (first) {
            for (int i = 0; i < 9; ++i) Tcb[i] = first->Tcb.R.d[i];
            for (int i = 0; i < 3; ++i) Tcb[9 + i] = first->Tcb.t[i];
            if (first->cam) { fx = first->cam->focal_length; cx = first->cam->principle_point[0]; cy = first->cam->principle_point[1]; }
            if (first->rk) delta = first->rk->delta;
        }
        const int P = (int)poses_.size(), L = (int)points_.size(), E = (int)ep.size(), O = (int)oi.size();
        // the device context (all buffers, the occupancy query, pinned staging) is kept across BAs while its capacity suffices
        if (ba_ && (P > capP_ || L > capL_ || E > capE_ || O > capO_)) { se2gpu_ba_destroy(ba_); ba_ = nullptr; }
        if (!ba_) {
            capP_ = P + P / 2 + 8; capL_ = L + L / 2 + 64; capE_ = E + E / 2 + 256; capO_ = O + O / 2 + 8;
            ba_ = se2gpu_ba_create(capP_, capL_, capE_, capO_, 0);
        }
        if (!ba_) { std::fprintf(stderr, "se2gpu: %s\n", se2gpu_last_error()); return false; }
        static const double zero3[3] = {0, 0, 0};
        int rc = se2gpu_ba_set_problem(ba_, P, L, E, O, xp.data(), fixed.data(), L ? xl.data() : zero3, ep.data(), el.data(), uv.data(),
                                       info.data(), oi.data(), oj.data(), om.data(), oinf.data(), fx, cx, cy, Tcb, delta);
        if (rc != SE2GPU_OK) { std::fprintf(stderr, "se2gpu: %s\n", se2gpu_last_error()); return false; }
        ready_ = true;
        return true;
    }

    // SparseOptimizer::optimize: returns the number of iterations performed; estimates are written back to the vertices
    int optimize(int iterations) {
        if (!ready_) { std::fprintf(stderr, "optimize: 0 vertices to optimize, maybe forgot to call initializeOptimization()\n"); return -1; }
        stats_.assign(iterations > 0 ? iterations : 1, se2gpu_ba_iter_stats());
        int n = se2gpu_ba_optimize(ba_, iterations, (const volatile unsigned char*)stop_, stats_.data(), nullptr, nullptr);
        if (n < 0) { std::fprintf(stderr, "se2gpu: %s\n", se2gpu_last_error()); return 0; }
        if (verbose_) for (int k = 0; k < n; ++k)
            std::fprintf(stderr, "iteration= %d\t chi2= %f\t lambda= %f\t levenbergIter= %d\n", k, stats_[k].chi2_after, stats_[k].lambda, stats_[k].trials);
        std::vector<double> xp(3 * poses_.size()), xl(3 * points_.size() + 3);
        if (se2gpu_ba_get(ba_, xp.data(), xl.data()) != SE2GPU_OK) { std::fprintf(stderr, "se2gpu: %s\n", se2gpu_last_error()); return 0; }
        for (size_t i = 0; i < poses_.size(); ++i) poses_[i]->est = SE2(xp[3 * i], xp[3 * i + 1], xp[3 * i + 2]);
        for (size_t j = 0; j < points_.size(); ++j) for (int k = 0; k < 3; ++k) points_[j]->est[k] = xl[3 * j + k];
        return n;
    }
    const std::vector<se2gpu_ba_iter_stats>& stats() const { return stats_; }

private:
    std::map<int, Vertex*> vertices_;
    std::vector<Edge*> edges_;
    std::vector<CameraParameters*> params_;
    std::vector<VertexSE2*> poses_;
    std::vector<VertexSBAPointXYZ*> points_;
    std::vector<se2gpu_ba_iter_stats> stats_;
    OptimizationAlgorithmGpuLM* alg_ = nullptr;
    se2gpu_ba* ba_ = nullptr;
    int capP_ = 0, capL_ = 0, capE_ = 0, capO_ = 0;
    bool* stop_ = nullptr;
    bool verbose_ = false, ready_ = false;
};

}  // namespace g2o
