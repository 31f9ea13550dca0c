// owlqn_weights_front_check.cpp -- OWLQNSolver(param, lambda, w) refusing weights of the wrong size or device, linked with the driver
// units and a test double of the C ABI.  TEST INFRASTRUCTURE ONLY.
#include <stdexcept>

#include "../../include/OWLQN.h"
#include "../../include/LBFGSpp/DeviceObjectives.h"
#include "../../lbfgspp_b200/csrc/driver_common.h"

extern "C" __attribute__((visibility("default")))
// minimize() with n_w weights for n coordinates (other_device: the weights live on another Device object): 1 when it throws
// std::invalid_argument before any evaluation, 0 otherwise
int owlqn_weights_front_check(long n, long n_w, int other_device)
{
    using namespace LBFGSpp;
    Device& dev = lbfgsb200_drv::device(0);
    Device& dev2 = lbfgsb200_drv::device(1);
    DeviceVector<double> x(dev, n), w(other_device ? dev2 : dev, n_w);
    x.setZero();
    w.setZero();
    LBFGSParam<double> prm;
    OWLQNSolver<double> solver(prm, 1.0, w);
    BuiltinObjective<double> f(0, nullptr, nullptr);
    double fx = 0;
    try { solver.minimize(f, x, fx); }
    catch (const std::invalid_argument&) { return solver.num_evaluations() == 0 && f.ncalls() == 0 ? 1 : 0; }
    return 0;
}
