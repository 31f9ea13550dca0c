// The reference's two self-checking examples (examples/example-rosenbrock-comparison.cpp and example-rosenbrock-bracketing.cpp)
// at their own size, with the small-batch solver: for n = 2, 4, .., 24, `trials` (default 1024, as there) seeded random starts in
// [-1,1]^n minimised with each of the four line searches (max_linesearch = 256) -- ONE launch per (n, line search) for all starts --
// and |x - 1|_inf <= 1e-4 checked for every start like validate_solution() there.  Prints the average evaluation / iteration counts.
#include <cmath>
#include <cstdlib>
#include <iostream>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include <LBFGSSmallBatch.h>

using namespace LBFGSpp;
typedef DeviceVector<double> Vector;

static void validate_solutions(const Vector& X, long trials, int n)
{
    const std::vector<double> x = X.to_std_vector();
    for (long b = 0; b < trials; b++)
        for (int i = 0; i < n; i++)
            if (std::abs(x[size_t(b) * n + i] - 1.0) > 1e-4)
                throw std::runtime_error("start " + std::to_string(b) + ": error is larger than 1e-4");
}

template <template <class> class LS>
static void run(const char* name, const LBFGSParam<double>& param, const std::vector<double>& starts, long trials, int n)
{
    LBFGSSmallBatchSolver<double, LS> solver(param);
    BuiltinObjective<double> fun(LBFGS_B200_OBJ_ROSENBROCK_PAIRED);
    Vector X = Vector::from_host(starts);
    const std::vector<BatchOutcome<double> > out = solver.minimize(fun, X, trials);
    long niter = 0;
    for (const BatchOutcome<double>& o : out)
    {
        if (o.status != 0) ls_throw(o.status);
        niter += o.niter;
    }
    validate_solutions(X, trials, n);
    std::cout << "  " << name << ": " << fun.ncalls() / trials << " calls, " << niter / trials << " iterations" << std::endl;
}

int main(int argc, char** argv)
{
    const long trials = argc > 1 ? std::atol(argv[1]) : 1024;
    LBFGSParam<double> param;
    param.linesearch = LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE;
    param.max_linesearch = 256;
    std::mt19937_64 rng(12345);
    std::uniform_real_distribution<double> unif(-1.0, 1.0);
    try
    {
        for (int n = 2; n <= 24; n += 2)
        {
            std::vector<double> starts(size_t(trials) * n);
            for (double& v : starts) v = unif(rng);
            std::cout << "n = " << n << std::endl;
            run<LineSearchBacktracking>("LineSearchBacktracking ", param, starts, trials, n);
            run<LineSearchBracketing>("LineSearchBracketing   ", param, starts, trials, n);
            run<LineSearchNocedalWright>("LineSearchNocedalWright", param, starts, trials, n);
            run<LineSearchMoreThuente>("LineSearchMoreThuente  ", param, starts, trials, n);
        }
    }
    catch (const std::exception& e)
    {
        std::cout << "FAILED: " << e.what() << std::endl;
        return 1;
    }
    return 0;
}
