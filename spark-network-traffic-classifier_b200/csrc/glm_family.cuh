// glm_family.cuh — GeneralizedLinearRegression's families and links, DESIGN.md §5o.
//
// Every mode of glm.cu evaluates a row through these functions, so the working response, the training summary and
// transform's prediction see the same bits for the same (y, mu, weight).  tests/glm_oracle.py restates them.
// Formulas are Spark 3's as recalled in b200flow/glm.py; log / exp / pow / lgamma / normcdf / normcdfinv are CUDA's.
#pragma once
#include <cfloat>
#include <math.h>

#include "../../include/b200flow.h"

namespace b200flow {

struct GlmSpec {
    int family, link;
    double variance_power, link_power;            // tweedie's V(mu) = mu^variance_power; the power link's mu^link_power
};

constexpr double kGlmEpsilon = 1e-16;             // project's floor (and 1 - epsilon binomial ceiling)
constexpr double kTweedieDelta = 0.1;             // initialize / deviance stand-in for y = 0

__device__ __forceinline__ double glm_link(const GlmSpec& s, double mu) {
    switch (s.link) {
        case B200FLOW_GLM_IDENTITY: return mu;
        case B200FLOW_GLM_LOG: return log(mu);
        case B200FLOW_GLM_INVERSE: return 1.0 / mu;
        case B200FLOW_GLM_LOGIT: return log(mu / (1.0 - mu));
        case B200FLOW_GLM_PROBIT: return normcdfinv(mu);
        case B200FLOW_GLM_CLOGLOG: return log(-log1p(-mu));
        case B200FLOW_GLM_SQRT: return sqrt(mu);
        default: return s.link_power == 0.0 ? log(mu) : pow(mu, s.link_power);
    }
}

__device__ __forceinline__ double glm_unlink(const GlmSpec& s, double eta) {
    switch (s.link) {
        case B200FLOW_GLM_IDENTITY: return eta;
        case B200FLOW_GLM_LOG: return exp(eta);
        case B200FLOW_GLM_INVERSE: return 1.0 / eta;
        case B200FLOW_GLM_LOGIT: return 1.0 / (1.0 + exp(-eta));
        case B200FLOW_GLM_PROBIT: return normcdf(eta);
        case B200FLOW_GLM_CLOGLOG: return 1.0 - exp(-exp(eta));
        case B200FLOW_GLM_SQRT: return eta * eta;
        default: return s.link_power == 0.0 ? exp(eta) : pow(eta, 1.0 / s.link_power);
    }
}

// g'(mu)
__device__ __forceinline__ double glm_deriv(const GlmSpec& s, double mu) {
    switch (s.link) {
        case B200FLOW_GLM_IDENTITY: return 1.0;
        case B200FLOW_GLM_LOG: return 1.0 / mu;
        case B200FLOW_GLM_INVERSE: return -1.0 / (mu * mu);
        case B200FLOW_GLM_LOGIT: return 1.0 / (mu * (1.0 - mu));
        case B200FLOW_GLM_PROBIT: {
            const double q = normcdfinv(mu);
            return 1.0 / (exp(-0.5 * (q * q)) * 0.3989422804014327);     // 1 / phi(Phi^-1(mu)), 1/sqrt(2 pi) rounded
        }
        case B200FLOW_GLM_CLOGLOG: return 1.0 / ((mu - 1.0) * log1p(-mu));
        case B200FLOW_GLM_SQRT: return 1.0 / (2.0 * sqrt(mu));
        default: return s.link_power == 0.0 ? 1.0 / mu : s.link_power * pow(mu, s.link_power - 1.0);
    }
}

__device__ __forceinline__ double glm_variance(const GlmSpec& s, double mu) {
    switch (s.family) {
        case B200FLOW_GLM_GAUSSIAN: return 1.0;
        case B200FLOW_GLM_BINOMIAL: return mu * (1.0 - mu);
        case B200FLOW_GLM_POISSON: return mu;
        case B200FLOW_GLM_GAMMA: return mu * mu;
        default: return pow(mu, s.variance_power);
    }
}

// clip mu into the family's domain; NaN passes through
__device__ __forceinline__ double glm_project(const GlmSpec& s, double mu) {
    if (s.family == B200FLOW_GLM_GAUSSIAN) return isinf(mu) ? (mu > 0.0 ? DBL_MAX : -DBL_MAX) : mu;
    if (s.family == B200FLOW_GLM_BINOMIAL) return mu < kGlmEpsilon ? kGlmEpsilon : (mu > 1.0 - kGlmEpsilon ? 1.0 - kGlmEpsilon : mu);
    return mu < kGlmEpsilon ? kGlmEpsilon : (isinf(mu) ? DBL_MAX : mu);
}

// the family's starting mean
__device__ __forceinline__ double glm_initialize(const GlmSpec& s, double y, double w) {
    if (s.family == B200FLOW_GLM_BINOMIAL) return (w * y + 0.5) / (w + 1.0);
    if (s.family == B200FLOW_GLM_POISSON || s.family == B200FLOW_GLM_TWEEDIE) return y == 0.0 ? kTweedieDelta : y;
    return y;
}

__device__ __forceinline__ double glm_ylogy(double y, double mu) { return y == 0.0 ? 0.0 : y * log(y / mu); }

// the row's deviance term
__device__ __forceinline__ double glm_deviance(const GlmSpec& s, double y, double mu, double w) {
    switch (s.family) {
        case B200FLOW_GLM_GAUSSIAN: return w * (y - mu) * (y - mu);
        case B200FLOW_GLM_BINOMIAL: return 2.0 * w * (glm_ylogy(y, mu) + glm_ylogy(1.0 - y, 1.0 - mu));
        case B200FLOW_GLM_POISSON: return 2.0 * w * (glm_ylogy(y, mu) - (y - mu));
        case B200FLOW_GLM_GAMMA: return -2.0 * w * (log(y / mu) - (y - mu) / mu);
        default: {
            const double p = s.variance_power;
            const double y1 = p >= 1.0 && p < 2.0 && y < kTweedieDelta ? kTweedieDelta : y;
            return 2.0 * w * (y * (pow(y1, 1.0 - p) - pow(mu, 1.0 - p)) / (1.0 - p) -
                              (pow(y, 2.0 - p) - pow(mu, 2.0 - p)) / (2.0 - p));
        }
    }
}

// the row's share of the AIC's log-likelihood sum: gaussian log w; binomial the log pmf of Binomial(round(w), mu) at
// round(y w) (0 when round(w) = 0); poisson w times the log pmf of Poisson(mu) at trunc(y); 0 for gamma (glm.py
// combines its separate sums) and tweedie
__device__ __forceinline__ double glm_aic_term(const GlmSpec& s, double y, double mu, double w) {
    switch (s.family) {
        case B200FLOW_GLM_GAUSSIAN: return log(w);
        case B200FLOW_GLM_BINOMIAL: {
            const double n = floor(w + 0.5), k = floor(y * w + 0.5);
            if (n == 0.0) return 0.0;
            return lgamma(n + 1.0) - lgamma(k + 1.0) - lgamma(n - k + 1.0) + k * log(mu) + (n - k) * log(1.0 - mu);
        }
        case B200FLOW_GLM_POISSON: {
            const double k = trunc(y);
            return w * (-mu + k * log(mu) - lgamma(k + 1.0));
        }
        default: return 0.0;
    }
}

}  // namespace b200flow
