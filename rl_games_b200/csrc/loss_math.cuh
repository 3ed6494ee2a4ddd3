// Per-sample PPO loss forward + analytic backward to the heads, shared by the fp32 (loss.cu) and the wgmma
// (mlp_tc.cu) kernels.  Follows a2c_continuous.py:97-134 (calc_losses), :241-257 (bound/reg loss),
// common_losses.py:16-82 (actor / smoothed actor / critic loss), torch_ext.py:27-36 (policy_kl),
// models.py:335-364 (sigma = exp(logstd), neglogp, entropy) and torch_ext.py:217-227 (clip fraction).
#pragma once
#include "common.cuh"

struct LossCfgDev {
    float e_clip, critic_coef, bounds_coef;
    int has_bounds, bound_type, clip_value, smooth, ppo;
    float log_lo, log_hi;    // log(1 - e_clip), log(1 + e_clip) for the clip-fraction diagnostic (filled on the host)
};

// fill sSig[0..4A): sigma, logstd, 1/sigma, log(sigma)  (one thread per action); returns nothing
__device__ __forceinline__ void loss_fill_sigma(float* sSig, const float* __restrict__ logstd, int A, int j) {
    const float ls = __ldg(logstd + j);
    const float sg = expf(ls);
    sSig[j] = sg; sSig[A + j] = ls; sSig[2 * A + j] = 1.0f / sg; sSig[3 * A + j] = logf(sg);
}

// sigma parametrisations (models.py apply_sigma_parametrization); the codes of b200rl_sigma_cfg.parametrization
constexpr int SIGMA_EXP = 0, SIGMA_SOFTPLUS = 1, SIGMA_LINEAR = 2;

struct SigmaCfgDev {
    int param, has_bounds;
    float min_sigma, lo, hi;    // lo / hi: logstd_bounds of 'exp'
};

inline SigmaCfgDev sigma_cfg_dev(const b200rl_sigma_cfg& h) {
    SigmaCfgDev c;
    c.param = h.parametrization; c.has_bounds = h.has_logstd_bounds;
    c.min_sigma = h.min_sigma; c.lo = h.logstd_lo; c.hi = h.logstd_hi;
    return c;
}

// torch.nn.functional.softplus (beta 1, threshold 20) and its derivative
__host__ __device__ __forceinline__ float softplus_t20(float x, float& dx) {
    if (x > 20.0f) { dx = 1.0f; return x; }
    const float z = expf(x);
    dx = z / (z + 1.0f);
    return log1pf(z);
}

// raw sigma-head output r -> sigma, logstd, and d logstd / d r (the factor that turns dL/dlogstd into dL/dr):
//   exp:      r clamped to the bounds (gradient 1 on the closed interval, 0 outside), sigma = e^r, logstd = r;
//             with a floor sigma = e^r + min_sigma, logstd = log(sigma)
//   softplus: sigma = softplus(r) + min_sigma, logstd = log(sigma)
//   linear:   floor = max(min_sigma, 1e-3), sigma = floor + softplus(r - floor), logstd = log(sigma)
__host__ __device__ __forceinline__ void sigma_param(float r, const SigmaCfgDev& c, float& sg, float& ls, float& dls_dr) {
    if (c.param == SIGMA_SOFTPLUS || c.param == SIGMA_LINEAR) {
        const float floor_ = c.param == SIGMA_LINEAR ? fmaxf(c.min_sigma, 1e-3f) : c.min_sigma;
        float dsp;
        const float sp = softplus_t20(c.param == SIGMA_LINEAR ? r - floor_ : r, dsp);
        sg = sp + floor_;
        ls = logf(sg);
        dls_dr = dsp / sg;
        return;
    }
    float g = 1.0f;
    if (c.has_bounds) {
        g = (r >= c.lo && r <= c.hi) ? 1.0f : 0.0f;
        r = fminf(fmaxf(r, c.lo), c.hi);
    }
    const float e = expf(r);
    if (c.min_sigma > 0.0f) {
        sg = e + c.min_sigma;
        ls = logf(sg);
        dls_dr = e * g / sg;
    } else {
        sg = e;
        ls = r;
        dls_dr = g;
    }
}

// per-row sigma of a state-dependent head (one entry per action): sigma, logstd and d logstd / d raw from sigma_param
template <int MAXA>
struct RowSigma {
    float sg[MAXA], ls[MAXA], dr[MAXA];
};

constexpr int LOSS_NSC = 8;   // scalar partial slots: w*a_loss, w*c_loss, w*entropy, w*b_loss, w*kl, mask, mask*clipped, w

struct LossArena {
    const float* actions; float* old_mu; float* old_sigma;
    const float* old_values_n; const float* returns_n; const float* old_neglogp; const float* advs_n; const float* mask;
};

// All arena inputs of one sample, fetched up front (vector loads when A % 4 == 0) so that their latency overlaps with the
// GEMM that produces the heads instead of serialising inside the loss arithmetic.
template <int MAXA>
struct LossRow {
    float act[MAXA], omu[MAXA], osg[MAXA];
    float old_v, ret, old_nlp, adv, mk;
};

template <int MAXA>
__device__ __forceinline__ void loss_row_load(const LossArena& a, int64_t ar, int A, LossRow<MAXA>& r) {
    r.old_v = __ldg(a.old_values_n + ar); r.ret = __ldg(a.returns_n + ar);
    r.old_nlp = __ldg(a.old_neglogp + ar); r.adv = __ldg(a.advs_n + ar);
    r.mk = a.mask ? __ldg(a.mask + ar) : 1.f;
    if ((A & 3) == 0) {
        const float4* pa = reinterpret_cast<const float4*>(a.actions + ar * A);
        const float4* pm = reinterpret_cast<const float4*>(a.old_mu + ar * A);
        const float4* ps = reinterpret_cast<const float4*>(a.old_sigma + ar * A);
#pragma unroll
        for (int q = 0; q < (MAXA - 1 + 3) / 4; ++q) {
            if (q * 4 < A) {
                const float4 x = __ldg(pa + q), y = pm[q], z = ps[q];
                if (q * 4 + 0 < MAXA) { r.act[q * 4 + 0] = x.x; r.omu[q * 4 + 0] = y.x; r.osg[q * 4 + 0] = z.x; }
                if (q * 4 + 1 < MAXA) { r.act[q * 4 + 1] = x.y; r.omu[q * 4 + 1] = y.y; r.osg[q * 4 + 1] = z.y; }
                if (q * 4 + 2 < MAXA) { r.act[q * 4 + 2] = x.z; r.omu[q * 4 + 2] = y.z; r.osg[q * 4 + 2] = z.z; }
                if (q * 4 + 3 < MAXA) { r.act[q * 4 + 3] = x.w; r.omu[q * 4 + 3] = y.w; r.osg[q * 4 + 3] = z.w; }
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < MAXA - 1; ++j) {
            if (j < A) { r.act[j] = __ldg(a.actions + ar * A + j); r.omu[j] = a.old_mu[ar * A + j]; r.osg[j] = a.old_sigma[ar * A + j]; }
        }
    }
}

// head[0] = value, head[1..A] = mu.  sSig (shared memory): sigma[A], logstd[A], 1/sigma[A], log(sigma)[A].
// FAST (bf16 tensor-core path): divisions -> reciprocal multiplies, exp/log -> ex2/lg2 approximations (the operands were
// already rounded to bf16 upstream); !FAST (fp32 path): IEEE divisions and full-precision expf/logf for tight parity.
// ar = arena row.  Outputs: dh[0] = dL/dvalue, dh[1+j] = dL/dmu_j, dls[j] = per-sample dL/dlogstd_j (without the
// entropy term), sc[] = weighted scalar contributions; writes the new mu / sigma over the old ones
// (datasets.py:33-43) and returns the sample's neglogp.
// SD (state-dependent sigma, fp32 only): sigma / logstd come per row from `rs` instead of sSig, and dls[j] is the row's dL/draw_j of
// the sigma head, the entropy bonus -ent_coef * w included (the fixed-sigma form leaves that term to the finalisation).
template <int MAXA, bool FAST, bool SD = false>
__device__ __forceinline__ float ppo_sample_loss(const float (&head)[MAXA], int A, const float* __restrict__ sSig,
                                                 const LossArena& ar_, int64_t ar, const LossRow<MAXA>& row, float inv_cnt,
                                                 const LossCfgDev& cfg, float (&dh)[MAXA], float (&dls)[MAXA], float (&sc)[LOSS_NSC],
                                                 const RowSigma<MAXA>* rs = nullptr, float ent_coef = 0.f) {
    static_assert(!(SD && FAST), "state-dependent sigma has no FAST form");
    const float val = head[0];
    const float old_v = row.old_v, ret = row.ret, old_nlp = row.old_nlp, adv = row.adv, mk = row.mk;
    const float w = mk * inv_cnt;
    float sumz2 = 0.f, sumls = 0.f, ent = 0.f, kl = 0.f, bl = 0.f;
    float z[MAXA];
#pragma unroll
    for (int j = 0; j < MAXA - 1; ++j) {
        if (j < A) {
            const float mu = head[1 + j], sg = SD ? rs->sg[j] : sSig[j], ls = SD ? rs->ls[j] : sSig[A + j];
            const float act = row.act[j];
            const float omu = row.omu[j], osg = row.osg[j];
            z[j] = FAST ? (act - mu) * sSig[2 * A + j] : (act - mu) / sg;
            sumz2 += z[j] * z[j];
            sumls += ls;
            ent += 0.5f + 0.9189385332046727f + (SD ? logf(sg) : sSig[3 * A + j]);     // 0.5 + 0.5*log(2*pi) + log(sigma)
            const float c1 = FAST ? __logf(osg * sSig[2 * A + j] + 1e-5f) : logf(osg / sg + 1e-5f);
            const float dm = omu - mu;
            const float c2 = FAST ? (sg * sg + dm * dm) * __frcp_rn(2.0f * (osg * osg + 1e-5f))
                                  : (sg * sg + dm * dm) / (2.0f * (osg * osg + 1e-5f));
            kl += c1 + c2 - 0.5f;
            if (cfg.has_bounds) {
                if (cfg.bound_type == 1) {
                    const float hi = fmaxf(mu - 1.1f, 0.f), lo = fminf(mu + 1.1f, 0.f);
                    bl += lo * lo + hi * hi;
                } else if (cfg.bound_type == 2) {
                    bl += mu * mu;
                }
            }
        } else {
            z[j] = 0.f;
        }
    }
    z[MAXA - 1] = 0.f;
    const float nlp = 0.5f * sumz2 + 0.9189385332046727f * (float)A + sumls;
    // ---- actor loss + d/dnlp ----
    float a_loss, g_a;
    if (cfg.ppo) {
        const float ratio = FAST ? __expf(old_nlp - nlp) : expf(old_nlp - nlp);
        const float mi = 1.0f - cfg.e_clip, mx = 1.0f + cfg.e_clip;
        float clamped, dcl;
        if (cfg.smooth) {
            const float s = FAST ? __frcp_rn(1.0f + __expf((-(ratio - mi) * __frcp_rn(mx - mi) + 0.5f) * 4.0f))
                                 : 1.0f / (1.0f + expf((-(ratio - mi) / (mx - mi) + 0.5f) * 4.0f));
            clamped = s * (mx - mi) + mi;
            dcl = 4.0f * s * (1.0f - s);
        } else {
            clamped = fminf(fmaxf(ratio, mi), mx);
            dcl = (ratio >= mi && ratio <= mx) ? 1.0f : 0.0f;
        }
        const float t1 = -(adv * ratio), t2 = -(adv * clamped);
        a_loss = fmaxf(t1, t2);
        const float d1 = adv * ratio, d2 = adv * dcl * ratio;
        g_a = (t1 > t2) ? d1 : ((t1 < t2) ? d2 : 0.5f * (d1 + d2));
    } else {
        a_loss = nlp * adv;
        g_a = adv;
    }
    // ---- critic loss + d/dvalue ----
    float c_loss, dc;
    if (cfg.clip_value) {
        const float delta = val - old_v;
        const float vpc = old_v + fminf(fmaxf(delta, -cfg.e_clip), cfg.e_clip);
        const float e1 = val - ret, e2 = vpc - ret;
        const float l1 = e1 * e1, l2 = e2 * e2;
        c_loss = fmaxf(l1, l2);
        const float g1 = 2.0f * e1;
        const float g2 = (delta >= -cfg.e_clip && delta <= cfg.e_clip) ? 2.0f * e2 : 0.0f;
        dc = (l1 > l2) ? g1 : ((l1 < l2) ? g2 : 0.5f * (g1 + g2));
    } else {
        const float e1 = ret - val;
        c_loss = e1 * e1;
        dc = -2.0f * e1;
    }
    const float lr_ = old_nlp - nlp;
    const float clipped = (lr_ < cfg.log_lo || lr_ > cfg.log_hi) ? 1.f : 0.f;
    // ---- gradients at the heads ----
    dh[0] = w * 0.5f * cfg.critic_coef * dc;
#pragma unroll
    for (int j = 0; j < MAXA - 1; ++j) {
        if (j < A) {
            const float mu = head[1 + j], sg = SD ? rs->sg[j] : sSig[j];
            float db = 0.f;
            if (cfg.has_bounds) {
                if (cfg.bound_type == 1) db = 2.0f * fmaxf(mu - 1.1f, 0.f) + 2.0f * fminf(mu + 1.1f, 0.f);
                else if (cfg.bound_type == 2) db = 2.0f * mu;
            }
            dh[1 + j] = w * (g_a * (FAST ? -(z[j] * sSig[2 * A + j]) : -(z[j] / sg)) + cfg.bounds_coef * db);
            dls[j] = w * g_a * (1.0f - z[j] * z[j]);
            if (SD) dls[j] = (dls[j] - ent_coef * w) * rs->dr[j];
            ar_.old_mu[ar * A + j] = mu;          // new mu/sigma overwrite the old ones (datasets.py:33-43)
            ar_.old_sigma[ar * A + j] = sg;
        } else {
            dh[1 + j] = 0.f;
            dls[j] = 0.f;
        }
    }
    dls[MAXA - 1] = 0.f;
    sc[0] = w * a_loss; sc[1] = w * c_loss; sc[2] = w * ent; sc[3] = w * bl; sc[4] = w * kl;
    sc[5] = mk; sc[6] = mk * clipped; sc[7] = w;
    return nlp;
}
