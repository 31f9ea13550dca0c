// The reference's two self-checking examples (examples/example-rosenbrock-comparison.cpp and
// example-rosenbrock-bracketing.cpp) on the GPU front: for n = 2, 4, .., 24 and `trials` seeded random starts in
// [-1,1]^n, minimise the paired Rosenbrock function with all four line searches (max_linesearch = 256), check
// |x - 1|_inf <= 1e-4 like validate_solution() there, and report the average evaluation / iteration counts.
#include <cmath>
#include <cstdlib>
#include <iostream>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include <LBFGS.h>
#include <LBFGSpp/DeviceObjectives.h>

using namespace LBFGSpp;
typedef DeviceVector<double> Vector;

static void validate_solution(const Vector& x)
{
    for (double v : x.to_std_vector())
        if (std::abs(v - 1.0) > 1e-4) throw std::runtime_error("Error is larger than 1e-4");
}

static int g_solver_loop = -1;   // -1: automatic (device-resident for built-in objectives up to n = 4e6), 0: host-driven, 1: resident

template <template <class> class LS>
static void run(const char* name, const LBFGSParam<double>& param, const std::vector<std::vector<double> >& starts)
{
    LBFGSSolver<double, LS> solver(param);
    if (g_solver_loop >= 0) solver.set_device_resident(g_solver_loop == 1);
    BuiltinObjective<double> fun(LBFGS_B200_OBJ_ROSENBROCK_PAIRED);
    long niter = 0;
    for (const std::vector<double>& x0 : starts)
    {
        Vector x = Vector::from_host(x0);
        double fx;
        niter += solver.minimize(fun, x, fx);
        validate_solution(x);
    }
    std::cout << "  " << name << ": " << fun.ncalls() / long(starts.size()) << " calls, " << niter / long(starts.size()) << " iterations" << std::endl;
}

int main(int argc, char** argv)
{
    const int trials = argc > 1 ? std::atoi(argv[1]) : 32;
    if (argc > 2) g_solver_loop = (std::string(argv[2]) == "resident") ? 1 : 0;   // usage: line_search_comparison [trials [host|resident]]
    LBFGSParam<double> param;
    param.linesearch = LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE;
    param.max_linesearch = 256;
    std::mt19937_64 rng(12345);
    std::uniform_real_distribution<double> unif(-1.0, 1.0);
    try
    {
        for (int n = 2; n <= 24; n += 2)
        {
            std::vector<std::vector<double> > starts(trials, std::vector<double>(n));
            for (auto& s : starts)
                for (double& v : s) v = unif(rng);
            std::cout << "n = " << n << std::endl;
            run<LineSearchBacktracking>("LineSearchBacktracking ", param, starts);
            run<LineSearchBracketing>("LineSearchBracketing   ", param, starts);
            run<LineSearchNocedalWright>("LineSearchNocedalWright", param, starts);
            run<LineSearchMoreThuente>("LineSearchMoreThuente  ", param, starts);
        }
    }
    catch (const std::exception& e)
    {
        std::cout << "FAILED: " << e.what() << std::endl;
        return 1;
    }
    return 0;
}
