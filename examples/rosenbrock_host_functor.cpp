// The reference's first example (examples/example-rosenbrock.cpp) on the GPU front, host-vector compatibility mode:
// the objective is an ordinary host functor, exactly as an LBFGSpp user writes it; only the vector type changed
// (Eigen::VectorXf -> LBFGSpp::HostVector<float>; with Eigen installed, Eigen::VectorXf works unchanged).
#include <iostream>

#include <LBFGS.h>

using namespace LBFGSpp;
typedef HostVector<float> Vec;

class Rosenbrock
{
    int n;

public:
    explicit Rosenbrock(int n_) : n(n_) {}
    float operator()(const Vec& x, Vec& grad)
    {
        float fx = 0.0f;
        for (int i = 0; i < n; i += 2)
        {
            const float a = 1.0f - x[i];
            const float b = 10.0f * (x[i + 1] - x[i] * x[i]);
            grad[i + 1] = 20.0f * b;
            grad[i] = -2.0f * (x[i] * grad[i + 1] + a);
            fx += a * a + b * b;
        }
        return fx;
    }
};

int main()
{
    const int n = 10;
    LBFGSParam<float> param;
    LBFGSSolver<float> solver(param);   // default line search: LineSearchNocedalWright, as in the reference
    Rosenbrock fun(n);
    Vec x = Vec::Zero(n);
    float fx;
    const int niter = solver.minimize(fun, x, fx);

    std::cout << niter << " iterations\nx =";
    for (int i = 0; i < n; i++) std::cout << ' ' << x[i];
    std::cout << "\nf(x) = " << fx << "\n||grad|| = " << solver.final_grad_norm() << std::endl;
    const SmallMatrix<float> B = solver.final_approx_hessian(), H = solver.final_approx_inverse_hessian();
    std::cout << "approx_hess[0][0..2] = " << B(0, 0) << ' ' << B(0, 1) << ' ' << B(0, 2) << "\n";
    std::cout << "approx_inv_hess[0][0..2] = " << H(0, 0) << ' ' << H(0, 1) << ' ' << H(0, 2) << std::endl;
    // B * H must be the identity
    float worst = 0;
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++)
        {
            float acc = 0;
            for (int k = 0; k < n; k++) acc += B(i, k) * H(k, j);
            worst = std::max(worst, std::abs(acc - (i == j ? 1.0f : 0.0f)));
        }
    std::cout << "max |B*H - I| = " << worst << std::endl;
    for (int i = 0; i < n; i++)
        if (std::abs(x[i] - 1.0f) > 1e-2f) return 1;
    return worst < 1e-2f ? 0 : 2;
}
