// resample.cpp -- the filter design of the rate conversion (resample.h).
#include "resample.h"

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <numeric>

namespace namb200
{

namespace
{

std::string hz(double r)
{
  char b[48];
  std::snprintf(b, sizeof b, "%.10g Hz", r);
  return b;
}

bool integer_rate(double r)
{
  return std::isfinite(r) && r > 0.0 && r <= 2147483647.0 && std::floor(r) == r;
}

// modified Bessel function of the first kind, order 0 (power series; converges fast for the Kaiser beta used here)
double bessel_i0(double x)
{
  double sum = 1.0, term = 1.0;
  const double q = 0.25 * x * x;
  for (int k = 1; k < 200; k++)
  {
    term *= q / ((double)k * (double)k);
    sum += term;
    if (term < sum * 1e-17)
      break;
  }
  return sum;
}

} // namespace

bool design_resampler(double host_rate, double model_rate, ResamplerDesign* out, std::string* why)
{
  const std::string pair = "host rate " + hz(host_rate) + ", model rate " + (model_rate == -1.0 ? std::string("unknown (-1)") : hz(model_rate));
  if (model_rate == -1.0)
  {
    *why = "resample: " + pair + ": the model's expected sample rate is unknown, so there is nothing to convert to";
    return false;
  }
  if (!integer_rate(host_rate) || !integer_rate(model_rate))
  {
    *why = "resample: " + pair + ": both rates must be positive integers in Hz";
    return false;
  }
  const int64_t h = (int64_t)host_rate, mo = (int64_t)model_rate, g = std::gcd(h, mo);
  const int64_t L = mo / g, M = h / g;
  if (L > kResampleMaxFactor || M > kResampleMaxFactor)
  {
    *why = "resample: " + pair + ": model / host = " + std::to_string(L) + "/" + std::to_string(M) + " in lowest terms, beyond "
           + std::to_string(kResampleMaxFactor) + "/" + std::to_string(kResampleMaxFactor);
    return false;
  }
  // Kaiser-windowed sinc at the common rate fs = host * L: cutoff 0.45 * min(rates), transition 0.1 * min(rates)
  // (passband to 0.4, stopband from 0.5), attenuation A; N from Kaiser's estimate
  const double fs = (double)h * (double)L, fmin = (double)std::min(h, mo);
  const double A = kResampleStopbandDb, beta = 0.1102 * (A - 8.7);
  const double fc = 0.45 * fmin / fs, df = 0.1 * fmin / fs; // cycles per sample at fs
  const int N = (int)std::ceil((A - 7.95) / (2.285 * 2.0 * M_PI * df)) + 1;
  const int taps_up = (N + (int)L - 1) / (int)L, taps_dn = (N + (int)M - 1) / (int)M;
  if (std::max(taps_up, taps_dn) > kResampleMaxTaps)
  {
    *why = "resample: " + pair + ": the filter needs " + std::to_string(std::max(taps_up, taps_dn))
           + " taps per output sample, more than " + std::to_string(kResampleMaxTaps) + " (rates too far apart)";
    return false;
  }
  ResamplerDesign d;
  d.host_rate = host_rate;
  d.model_rate = model_rate;
  d.L = (int)L;
  d.M = (int)M;
  d.n_taps = N;
  d.taps_up = taps_up;
  d.taps_dn = taps_dn;
  d.latency_frames = (double)(N - 1) / (double)L;
  d.g_up.resize((size_t)N);
  d.g_dn.resize((size_t)N);
  const double c = 0.5 * (N - 1), i0b = bessel_i0(beta);
  for (int n = 0; n < N; n++)
  {
    const double t = n - c, r = t / c;
    const double x = 2.0 * fc * t;
    const double sinc = (x == 0.0) ? 1.0 : std::sin(M_PI * x) / (M_PI * x);
    const double w = bessel_i0(beta * std::sqrt(std::max(0.0, 1.0 - r * r))) / i0b;
    const double gn = 2.0 * fc * sinc * w;
    d.g_up[(size_t)n] = (float)((double)L * gn);
    d.g_dn[(size_t)n] = (float)((double)M * gn);
  }
  *out = std::move(d);
  return true;
}

std::vector<float> resampler_phase_table(const std::vector<float>& g, int B, int T)
{
  std::vector<float> t((size_t)B * T, 0.0f);
  for (int u = 0; u < T; u++)
    for (int p = 0; p < B; p++)
    {
      const size_t k = (size_t)p + (size_t)u * B;
      if (k < g.size())
        t[(size_t)u * B + p] = g[k];
    }
  return t;
}

std::string resampler_json(const ResamplerDesign& d)
{
  std::string s = "{\"host_rate\": " + std::to_string((int64_t)d.host_rate) + ", \"model_rate\": " + std::to_string((int64_t)d.model_rate)
                  + ", \"L\": " + std::to_string(d.L) + ", \"M\": " + std::to_string(d.M) + ", \"n_taps\": " + std::to_string(d.n_taps)
                  + ", \"taps_per_output_up\": " + std::to_string(d.taps_up) + ", \"taps_per_output_down\": " + std::to_string(d.taps_dn);
  char b[64];
  std::snprintf(b, sizeof b, "%.9g", d.latency_frames);
  s += std::string(", \"latency_frames\": ") + b;
  auto arr = [&](const char* name, const std::vector<float>& v) {
    s += std::string(", \"") + name + "\": [";
    for (size_t i = 0; i < v.size(); i++)
    {
      std::snprintf(b, sizeof b, i ? ", %.9g" : "%.9g", (double)v[i]);
      s += b;
    }
    s += "]";
  };
  arr("g_up", d.g_up);
  arr("g_dn", d.g_dn);
  return s + "}";
}

} // namespace namb200
