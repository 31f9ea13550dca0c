// examples/example-rosenbrock-box.cpp of the reference on the GPU front: chained Rosenbrock, n = 25, bounds [2, 4] with the
// third variable unbounded and some start values on the bounds, LBFGSBSolver with default LBFGSBParam.  Vectors live on the
// device; the objective is the built-in device kernel for this function.
#include <cmath>
#include <iostream>
#include <limits>
#include <vector>

#include <LBFGSB.h>
#include <LBFGSpp/DeviceObjectives.h>

using namespace LBFGSpp;
typedef DeviceVector<double> Vector;

int main()
{
    const int n = 25;
    LBFGSBParam<double> param;
    LBFGSBSolver<double> solver(param);
    BuiltinObjective<double> fun(LBFGS_B200_OBJ_ROSENBROCK_CHAINED);

    std::vector<double> lb(n, 2.0), ub(n, 4.0), x0(n, 3.0);
    lb[2] = -std::numeric_limits<double>::infinity();
    ub[2] = std::numeric_limits<double>::infinity();
    x0[0] = x0[1] = 2.0;
    x0[5] = x0[7] = 4.0;
    Vector x = Vector::from_host(x0), l = Vector::from_host(lb), u = Vector::from_host(ub);

    double fx;
    const int niter = solver.minimize(fun, x, fx, l, u);
    const std::vector<double> xs = x.to_std_vector();
    std::cout << niter << " iterations\nx =";
    for (double v : xs) std::cout << ' ' << v;
    std::cout.precision(16);
    std::cout << "\nf(x) = " << fx << "\nprojected grad norm = " << solver.final_grad_norm() << std::endl;
    // the reference headers give 13 iterations and f = 360.2835855511515 (tests/golden/lbfgs_ref.json)
    return (niter == 13 && std::abs(fx - 360.2835855511515) < 1e-8) ? 0 : 1;
}
