/* TEST INFRASTRUCTURE ONLY (oracle shim) - stands in for <boost/math/distributions/chi_squared.hpp>: the chi-squared
 * distribution, complement() and the upper-tail quantile, the one use pulse_blanking_cc.cc:57-58 makes of it.  With k
 * degrees of freedom, quantile(complement(chi2(k), q)) = 2 gamma_p_inv(k / 2, 1 - q), computed in double (as Boost
 * promotes float) and rounded once to the distribution's type. */
#pragma once
#include <boost/math/special_functions/gamma.hpp>
namespace boost
{
namespace math
{
template <class RealType = double, class Policy = void>
class chi_squared_distribution
{
public:
    explicit chi_squared_distribution(RealType df) : df_(df) {}
    RealType degrees_of_freedom() const { return df_; }

private:
    RealType df_;
};
template <class Dist, class RealType>
struct complemented2_type
{
    const Dist& dist;
    RealType param;
};
template <class Dist, class RealType>
inline complemented2_type<Dist, RealType> complement(const Dist& d, const RealType& p)
{
    return complemented2_type<Dist, RealType>{d, p};
}
template <class RealType, class Policy, class T>
inline RealType quantile(const complemented2_type<chi_squared_distribution<RealType, Policy>, T>& c)
{
    const double k = static_cast<double>(c.dist.degrees_of_freedom());
    const double q = static_cast<double>(c.param);
    return static_cast<RealType>(2.0 * gamma_p_inv(0.5 * k, 1.0 - q));
}
}  // namespace math
}  // namespace boost
