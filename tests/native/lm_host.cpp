// Host test of the Levenberg-Marquardt control every LM solver of the library runs (se2lam_b200/csrc/lm.h): lambda_0, the
// gain-ratio test, the lambda schedule, the retry and terminate rules, the iteration statistics and the NOT_PD rule, against
// g2o's OptimizationAlgorithmLevenberg::solve. Prints "OK <checks>" and exits 0, or names the first failed check.
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "../../se2lam_b200/csrc/lm.h"

using namespace se2gpu;

static int checks = 0;

#define CHECK(cond)                                                       \
    do {                                                                  \
        ++checks;                                                         \
        if (!(cond)) {                                                    \
            std::printf("FAIL line %d: %s\n", __LINE__, #cond);           \
            std::exit(1);                                                 \
        }                                                                 \
    } while (0)

// one LM trial as the kernels run it: the solve's outcome, chi2 at the trial point and the computeScale() sum
struct Lm {
    double chi, lambda, ni;
    int trials = 0, accepted = 0, failed = 0;
    double rho = 0;
    bool trial(bool solve_ok, double temp, double scale) {
        if (!solve_ok) ++failed;
        const bool acc = lm_gain_step(temp, scale, solve_ok, chi, lambda, ni, rho);
        if (acc) accepted = 1;
        ++trials;
        return acc;
    }
};

int main() {
    // lambda_0 = 1e-5 max |diag H|, nu = 2
    {
        double lambda = -1, ni = -1;
        lm_lambda_init(4.0, lambda, ni);
        CHECK(lambda == 1e-5 * 4.0 && ni == 2.0);
        lm_lambda_init(0.0, lambda, ni);
        CHECK(lambda == 0.0 && ni == 2.0);
    }
    // accept with rho = 1: alpha = 1 - 1 = 0, clamped to 1/3; nu back to 2, chi2 takes the trial's
    {
        Lm m{10.0, 3.0, 8.0};
        // scale + 1e-3 = 2, chi - temp = 2: rho = 1 exactly
        CHECK(m.trial(true, 8.0, 2.0 - 1e-3));
        CHECK(m.rho == (10.0 - 8.0) / ((2.0 - 1e-3) + 1e-3));
        CHECK(m.lambda == 3.0 * (1. / 3.) && m.ni == 2.0 && m.chi == 8.0 && m.accepted == 1);
        CHECK(!lm_retry(m.rho, m.trials) && !lm_terminate(m.rho, m.trials));
    }
    // accept with rho = 0.5: alpha = 1 - 0 = 1, clamped to 2/3
    {
        Lm m{10.0, 3.0, 2.0};
        CHECK(m.trial(true, 9.0, 2.0 - 1e-3));
        CHECK(std::fabs(m.rho - 0.5) < 1e-12);
        CHECK(m.lambda == 3.0 * (2. / 3.) && m.ni == 2.0 && m.chi == 9.0);
    }
    // accept between the clamps: alpha = 1 - (2 rho - 1)^3
    {
        Lm m{10.0, 3.0, 2.0};
        CHECK(m.trial(true, 10.0 - 0.9 * 2.0, 2.0 - 1e-3));
        const double rho = (10.0 - (10.0 - 0.9 * 2.0)) / ((2.0 - 1e-3) + 1e-3);
        CHECK(m.rho == rho && m.lambda == 3.0 * (1. - pow(2 * rho - 1, 3)));
        CHECK(m.lambda > 1.0 && m.lambda < 2.0);
    }
    // consecutive rejections: lambda *= nu, nu doubles each time; chi2 unchanged; retry while rho < 0
    {
        Lm m{10.0, 1.0, 2.0};
        double lambda = 1.0, ni = 2.0;
        for (int k = 0; k < 4; ++k) {
            CHECK(!m.trial(true, 11.0, 1.0));
            lambda *= ni; ni *= 2;
            CHECK(m.lambda == lambda && m.ni == ni && m.chi == 10.0 && m.rho < 0);
            CHECK(lm_retry(m.rho, m.trials) && !lm_terminate(m.rho, m.trials));
        }
        CHECK(m.ni == 32.0 && m.lambda == 1024.0);
        // an accepted trial resets nu
        CHECK(m.trial(true, 9.0, 1.0));
        CHECK(m.ni == 2.0 && m.accepted == 1);
    }
    // a failed solve: chi2 = DBL_MAX, scale = 0 (+ 1e-3) whatever was passed in; rejected
    {
        double temp = 5.0, scale = 7.0, rho = 0;
        double chi = 10.0, lambda = 1.0, ni = 2.0;
        CHECK(!lm_gain_step(temp, scale, false, chi, lambda, ni, rho));
        CHECK(temp == DBL_MAX && scale == 1e-3 && rho == (10.0 - DBL_MAX) / 1e-3 && rho < 0);
        CHECK(chi == 10.0 && lambda == 2.0 && ni == 4.0);
    }
    // ten failed solves: the iteration terminates with every trial failed, which is NOT_PD
    {
        Lm m{10.0, 1.0, 2.0};
        for (int k = 0; k < kLmMaxTrials; ++k) {
            CHECK(!m.trial(false, 0.0, 0.0));
            if (k + 1 < kLmMaxTrials) CHECK(lm_retry(m.rho, m.trials));
        }
        CHECK(kLmMaxTrials == 10);
        CHECK(!lm_retry(m.rho, m.trials) && lm_terminate(m.rho, m.trials));
        const se2gpu_ba_iter_stats st = lm_iter_stats(10.0, m.chi, m.lambda, m.rho, m.trials, m.accepted);
        CHECK(st.chi2_before == 10.0 && st.chi2_after == 10.0 && st.lambda == std::ldexp(1.0, 55) && st.rho == m.rho);
        CHECK(st.trials == 10 && st.accepted == 0 && st.terminate == 1 && st.pad == 0);
        CHECK(lm_not_pd(st, m.failed));
    }
    // ten rejected trials that solved: terminate, but not NOT_PD; nor when one of them failed to solve
    {
        Lm m{10.0, 1.0, 2.0};
        for (int k = 0; k < kLmMaxTrials; ++k) m.trial(k != 3, 11.0, 1.0);
        const se2gpu_ba_iter_stats st = lm_iter_stats(10.0, m.chi, m.lambda, m.rho, m.trials, m.accepted);
        CHECK(st.terminate == 1 && m.failed == 1 && !lm_not_pd(st, m.failed));
    }
    // a failed solve, then an accepted trial: no terminate, no NOT_PD
    {
        Lm m{10.0, 1.0, 2.0};
        CHECK(!m.trial(false, 0.0, 0.0));
        CHECK(lm_retry(m.rho, m.trials));
        CHECK(m.trial(true, 9.0, 1.0));
        const se2gpu_ba_iter_stats st = lm_iter_stats(10.0, m.chi, m.lambda, m.rho, m.trials, m.accepted);
        CHECK(st.trials == 2 && st.accepted == 1 && st.terminate == 0 && st.chi2_after == 9.0 && !lm_not_pd(st, m.failed));
    }
    // rho == 0 (the trial's chi2 equals the current one): rejected, no retry, terminate
    {
        Lm m{10.0, 1.0, 2.0};
        CHECK(!m.trial(true, 10.0, 1.0));
        CHECK(m.rho == 0 && m.lambda == 2.0 && m.ni == 4.0);
        CHECK(!lm_retry(m.rho, m.trials) && lm_terminate(m.rho, m.trials));
        const se2gpu_ba_iter_stats st = lm_iter_stats(10.0, m.chi, m.lambda, m.rho, m.trials, m.accepted);
        CHECK(st.terminate == 1 && st.trials == 1 && !lm_not_pd(st, m.failed));
    }
    // a NaN trial chi2: rejected; rho is NaN, so do ... while (rho < 0 && ...) stops without terminating
    {
        Lm m{10.0, 1.0, 2.0};
        CHECK(!m.trial(true, std::nan(""), 1.0));
        CHECK(std::isnan(m.rho) && m.chi == 10.0 && m.lambda == 2.0 && m.ni == 4.0);
        CHECK(!lm_retry(m.rho, m.trials) && !lm_terminate(m.rho, m.trials));
        const se2gpu_ba_iter_stats st = lm_iter_stats(10.0, m.chi, m.lambda, m.rho, m.trials, m.accepted);
        CHECK(st.terminate == 0 && st.accepted == 0 && !lm_not_pd(st, m.failed));
    }
    // every trial failed to solve, but the iteration did not terminate (a NaN current chi2 gives a NaN rho): not NOT_PD
    {
        Lm m{std::nan(""), 1.0, 2.0};
        CHECK(!m.trial(false, 0.0, 0.0));
        CHECK(std::isnan(m.rho) && !lm_retry(m.rho, m.trials) && !lm_terminate(m.rho, m.trials));
        const se2gpu_ba_iter_stats st = lm_iter_stats(m.chi, m.chi, m.lambda, m.rho, m.trials, m.accepted);
        CHECK(st.terminate == 0 && m.failed == st.trials && !lm_not_pd(st, m.failed));
    }
    // a positive rho from a non-finite trial chi2 is rejected
    {
        double temp = -INFINITY, scale = 1.0, rho = 0, chi = 10.0, lambda = 1.0, ni = 2.0;
        CHECK(!lm_gain_step(temp, scale, true, chi, lambda, ni, rho));
        CHECK(rho > 0 && chi == 10.0 && lambda == 2.0 && ni == 4.0);
    }
    std::printf("OK %d checks\n", checks);
    return 0;
}
