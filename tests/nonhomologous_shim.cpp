// Host build of the product's nonhomologous line-distance header (tardis_b200/csrc/nonhomologous.cuh) for
// tests/test_nonhomologous.py: the same source the transport kernel compiles, here with g++ -ffp-contract=off.
#include "../tardis_b200/csrc/nonhomologous.cuh"

extern "C" {
void shim_depressed_quartic(double A, double B, double C, double D, double E, double *roots) {
    const nh::Roots r = nh::depressed_quartic(A, B, C, D, E);
    for (int i = 0; i < 4; i++) roots[i] = r.x[i];
}
double shim_distance_line(double r, double mu, double nu, double nu_line, double r_inner, double r_outer, double v_inner,
                          double v_outer) {
    const double dvdr = nh::velocity_gradient(r_inner, r_outer, v_inner, v_outer);
    return nh::distance_line(r, mu, nu, nu_line, r_inner, r_outer, v_inner, v_outer, dvdr, nh::velocity(r, r_inner, v_inner, dvdr));
}
double shim_velocity_gradient(double r_inner, double r_outer, double v_inner, double v_outer) {
    return nh::velocity_gradient(r_inner, r_outer, v_inner, v_outer);
}
double shim_cbrt(double x) { return nh::cbrt_pos(x); }
double shim_atan2(double y, double x) { return nh::atan2_(y, x); }
double shim_sin(double x) { return nh::sin_(x); }
double shim_cos(double x) { return nh::cos_(x); }
double shim_hypot(double x, double y) { return nh::hypot_(x, y); }
}
