// CPU harness around the activations of zuko_b200/csrc/activations.cuh (what the CNF backward kernel runs on the
// GPU), compiled by g++ from tests/test_cnf_grad_host.py.
#include <stdint.h>

#include "../../zuko_b200/csrc/activations.cuh"

extern "C" {

// d1[i] = act'(v[i]), d2[i] = act''(v[i]) for the internal activation code `act` (1 = ReLU, ZK_ACT_* otherwise)
void act_derivs(const float* v, int64_t n, int act, float* d1, float* d2) {
    for (int64_t i = 0; i < n; ++i) {
        d1[i] = zk::act_deriv(v[i], act);
        d2[i] = zk::act_deriv2(v[i], act);
    }
}
}
