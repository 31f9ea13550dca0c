// examples/example-quadratic.cpp of the reference on the GPU front: a free function over host vectors,
// f(x) = |x - (0,1,...,n-1)|^2, double precision, default parameters.
#include <cmath>
#include <iostream>

#include <LBFGS.h>

using namespace LBFGSpp;
typedef HostVector<double> Vec;

double foo(const Vec& x, Vec& grad)
{
    double f = 0.0;
    for (std::ptrdiff_t i = 0; i < x.size(); i++)
    {
        const double r = x[i] - double(i);
        f += r * r;
        grad[i] = 2.0 * r;
    }
    return f;
}

int main()
{
    const int n = 10;
    LBFGSParam<double> param;
    LBFGSSolver<double> solver(param);
    Vec x = Vec::Zero(n);
    double fx;
    const int niter = solver.minimize(foo, x, fx);
    std::cout << niter << " iterations\nf(x) = " << fx << "\nx =";
    for (int i = 0; i < n; i++) std::cout << ' ' << x[i];
    std::cout << std::endl;
    for (int i = 0; i < n; i++)
        if (std::abs(x[i] - i) > 1e-8) return 1;
    return niter == 2 ? 0 : 2;
}
