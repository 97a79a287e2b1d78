// C ABI of the engine, part 4 of 5: EC-FFT and batch normalisation (ecfft.cuh), hash_to_curve and Params::new (h2c.cuh),
// point (de)compression (codec.cuh).
#include "util_kernels.cuh"
#include "msm.cuh"
#include "ecfft.cuh"
#include "codec.cuh"
#include "h2c.cuh"

// ------------------------------------------------------------------------------------------------
// EC-FFT (best_fft with G = curve point) and batch normalisation (ecfft.cuh)
// ------------------------------------------------------------------------------------------------
// the log n butterfly stages (+ the optional `*g *= scale` pass) on an XYZZ work array already in network order
template <class P, class PS>
static int ecfft_stages(xyzz *work, uint32_t log_n, const fe &omega_mont, const fe *scale_canon, cudaStream_t s) {
    const fe *tw = nullptr;
    if (get_twiddles_any(PS::ID, omega_mont, log_n, s, &tw)) return 1;
    const uint64_t n = 1ull << log_n;
    // one QUAD of lanes per butterfly (ecfft.cuh) unless the test hook asks for the one-thread form
    // A quad level costs ~3 multiply latencies (selects, call, 32 shuffles, limb carries), so the quad form only
    // wins while a stage has too few butterflies to give every SM a warp.  ecfft_quad: 1 = by size (default), 0 / 2 = force
    // the thread / quad form (test hook).
    const bool use_quad = g_ctx.ecfft_quad == 2 || (g_ctx.ecfft_quad == 1 && log_n <= 12);
    const uint32_t q = use_quad ? 4u : 1u;
    auto stage = use_quad ? ecfft_stage_quad_kernel<P, PS> : ecfft_stage_kernel<P, PS>;
    for (uint32_t st = 1; st <= log_n; st++) LAUNCH(stage, blocks_for(n / 2 * q, 64), 64, 0, s, work, tw, log_n, st);
    if (scale_canon) {
        auto sc = use_quad ? ecfft_scale_quad_kernel<P, PS> : ecfft_scale_kernel<P, PS>;
        LAUNCH(sc, blocks_for(n * q, 64), 64, 0, s, work, *scale_canon, n);
    }
    return 0;
}
// mode 0: Jacobian in -> Jacobian out (h2_ec_fft); mode 1: affine in -> scaled, normalised affine out (h2_params_lagrange)
// `in` == nullptr: the input is already in X.ec_io on the device (h2_params_new)
template <class P, class PS>
static int ecfft_host(int mode, const void *in, uint32_t log_n, const void *omega, const void *scale, const HostArgs &h, void *out) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint64_t n = 1ull << log_n;
    const int canon = h.canon();
    const size_t in_sz = mode == 0 ? sizeof(jacobian) : sizeof(affine);
    if (in) {
        if (X.ec_io.ensure(n * sizeof(jacobian))) return 1;
        if (upload_async(X.ec_io.p, in, n * in_sz, s)) return 1;
    }
    if (X.ec_work.ensure(n * sizeof(xyzz)) || X.ec_out.ensure(n * sizeof(affine))) return 1;
    xyzz *work = X.ec_work.as<xyzz>();
    if (mode == 0) {
        auto k = ecfft_load_jac_kernel<P, PS>;
        LAUNCH(k, blocks_for(n, 128), 128, 0, s, X.ec_io.as<jacobian>(), canon, work, log_n);
    } else {
        auto k = ecfft_load_affine_kernel<P, PS>;
        LAUNCH(k, blocks_for(n, 128), 128, 0, s, X.ec_io.as<affine>(), canon, work, log_n);
    }
    fe sc, *scp = nullptr;
    if (scale) {
        memcpy(sc.v, scale, 32);
        if (!canon) sc = fe_from_mont<PS>(sc);
        scp = &sc;
    }
    if (ecfft_stages<P, PS>(work, log_n, h.elem<PS>(omega), scp, s)) return 1;
    if (mode == 0) {
        auto k = ecfft_store_jac_kernel<P, PS>;
        LAUNCH(k, blocks_for(n, 128), 128, 0, s, work, X.ec_io.as<jacobian>(), canon, n);
        CU(cudaMemcpyAsync(out, X.ec_io.p, n * sizeof(jacobian), cudaMemcpyDeviceToHost, s));
    } else {
        LAUNCH(normalize_kernel<P>, blocks_for((n + H2_NORM_CHUNK - 1) / H2_NORM_CHUNK, 64), 64, 0, s, work, (const jacobian *)nullptr, 0,
               X.ec_out.as<affine>(), canon, n);
        CU(cudaMemcpyAsync(out, X.ec_out.p, n * sizeof(affine), cudaMemcpyDeviceToHost, s));
    }
    CU(cudaStreamSynchronize(s));
    return 0;
}
static int ecfft_host_dispatch(int curve, int mode, const void *in, uint32_t log_n, const void *omega, const void *scale, const HostArgs &h,
                               std::initializer_list<HostArgs::Need> needs, void *out) {
    CtxLock lk;
    if (require_ready() || h.check(needs)) return 1;
    if (log_n > 26) return fail("ec_fft: log_n > 26 not supported");
    return by_curve(curve, [&](auto p, auto ps) { return ecfft_host<decltype(p), decltype(ps)>(mode, in, log_n, omega, scale, h, out); });
}
extern "C" int h2_ec_fft(int curve, void *points_xyz, const void *omega, uint32_t log_n, const void *scale, int repr) {
    return ecfft_host_dispatch(curve, 0, points_xyz, log_n, omega, scale, {"h2_ec_fft", repr}, {{points_xyz, "points_xyz"}, {omega, "omega"}}, points_xyz);
}
// minv is required here (poly/commitment.rs:83)
extern "C" int h2_params_lagrange(int curve, const void *g_xy, uint32_t k, const void *omega_inv, const void *minv, int repr, void *out_xy) {
    return ecfft_host_dispatch(curve, 1, g_xy, k, omega_inv, minv, {"h2_params_lagrange", repr},
                               {{g_xy, "g_xy"}, {omega_inv, "omega_inv"}, {minv, "minv"}, {out_xy, "out_g_lagrange_xy"}}, out_xy);
}

// ------------------------------------------------------------------------------------------------
// hash_to_curve (h2c.cuh) and Params::new (poly/commitment.rs:38-114)
// ------------------------------------------------------------------------------------------------
// n messages -> n affine points in X.ec_io (device, `repr`).  msgs == nullptr: generator
// messages 0 || (first + i) as u32 LE
template <class P>
static int h2c_issue(const H2cConst &K, const void *msgs, size_t msg_len, uint64_t first, size_t n, const HostArgs &h, affine *d_out, cudaStream_t s) {
    Context &X = g_ctx;
    const uint8_t *d_msgs = nullptr;
    if (msgs && n * msg_len) {
        if (X.misc.ensure(n * msg_len)) return 1;
        CU(cudaMemcpyAsync(X.misc.p, msgs, n * msg_len, cudaMemcpyHostToDevice, s));
        d_msgs = X.misc.as<uint8_t>();
    }
    LAUNCH(h2c_kernel<P>, blocks_for(n, 64), 64, 0, s, d_msgs, (uint32_t)msg_len, msgs ? 0 : 1, first, K, d_out, h.mont() ? 1 : 0,
           (uint64_t)n);
    return 0;
}
template <class P>
static int hash_to_curve_host(const char *domain_prefix, const void *msgs, size_t msg_len, size_t n, const HostArgs &h, void *out_xy) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const H2cConst K = make_h2c_const<P>(domain_prefix);
    if (!K.ok) return fail("h2_hash_to_curve: domain prefix too long (DST must be < 256 bytes)");
    if (X.ec_io.ensure(n * sizeof(affine))) return 1;
    if (h2c_issue<P>(K, msgs, msg_len, 0, n, h, X.ec_io.as<affine>(), s)) return 1;
    CU(cudaMemcpyAsync(out_xy, X.ec_io.p, n * sizeof(affine), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return 0;
}
extern "C" int h2_hash_to_curve(int curve, const char *domain_prefix, const void *messages, size_t msg_len, size_t n, int repr, void *out_xy) {
    CtxLock lk;
    const HostArgs h("h2_hash_to_curve", repr);
    if (require_ready() || check_curve(curve) || h.check({{out_xy, "out_xy", n != 0}})) return 1;
    if (!domain_prefix) return fail("h2_hash_to_curve: domain_prefix is NULL");
    if (msg_len && !messages && n) return fail("h2_hash_to_curve: messages is NULL");
    if (msg_len >= (1ull << 31) || n >= (1ull << 32)) return fail("h2_hash_to_curve: message or batch too large");
    if (n == 0) return 0;
    static const uint8_t empty = 0;
    const void *m = messages ? messages : &empty;      // msg_len == 0: n hashes of the empty message
    return by_curve(curve, [&](auto p, auto) { return hash_to_curve_host<decltype(p)>(domain_prefix, m, msg_len, n, h, out_xy); });
}
// Params::new: g[i] = H(0 || i), w = H(1), u = H(2) with H = hash_to_curve("Halo2-Parameters"), then g_lagrange from g
template <class P, class PS>
static int params_new_host(uint32_t k, const HostArgs &h, void *g_xy, void *gl_xy, void *w_xy, void *u_xy) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint64_t n = 1ull << k;
    static const H2cConst K = make_h2c_const<P>("Halo2-Parameters");
    if (!K.ok) return fail("h2_params_new: internal constant check failed");
    // alpha_inv = ROOT_OF_UNITY_INV^(2^(S-k)) (commitment.rs:77-80), minv = TWO_INV^k (:83)
    static const SqrtConst KS = make_sqrt_const<PS>();
    fe alpha_inv = fe_inv<PS>(KS.root);
    for (uint32_t i = k; i < 32; i++) alpha_inv = fe_sqr<PS>(alpha_inv);
    const fe two_inv = fe_inv<PS>(fe_dbl<PS>(fe_one<PS>()));
    fe minv = fe_one<PS>();
    for (uint32_t i = 0; i < k; i++) minv = fe_mul<PS>(minv, two_inv);
    if (h.canon()) { alpha_inv = fe_from_mont<PS>(alpha_inv); minv = fe_from_mont<PS>(minv); }   // ecfft_host reads them in repr
    if (X.ec_io.ensure((n + 2) * sizeof(jacobian))) return 1;
    affine *d_g = X.ec_io.as<affine>();
    static const uint8_t wu[2] = {1, 2};
    if (h2c_issue<P>(K, wu, 1, 0, 2, h, d_g + n, s)) return 1;       // w, u behind g
    if (h2c_issue<P>(K, nullptr, 0, 0, n, h, d_g, s)) return 1;
    CU(cudaMemcpyAsync(g_xy, d_g, n * sizeof(affine), cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(w_xy, d_g + n, sizeof(affine), cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(u_xy, d_g + n + 1, sizeof(affine), cudaMemcpyDeviceToHost, s));
    return ecfft_host<P, PS>(1, nullptr, k, alpha_inv.v, minv.v, h, gl_xy);   // synchronises
}
extern "C" int h2_params_new(int curve, uint32_t k, int repr, void *out_g_xy, void *out_g_lagrange_xy, void *out_w_xy, void *out_u_xy) {
    CtxLock lk;
    const HostArgs h("h2_params_new", repr);
    if (require_ready() || h.check({{out_g_xy, "out_g_xy"}, {out_g_lagrange_xy, "out_g_lagrange_xy"}, {out_w_xy, "out_w_xy"}, {out_u_xy, "out_u_xy"}})) return 1;
    if (k > 26) return fail("h2_params_new: k > 26 not supported");
    return by_curve(curve, [&](auto p, auto ps) {
        return params_new_host<decltype(p), decltype(ps)>(k, h, out_g_xy, out_g_lagrange_xy, out_w_xy, out_u_xy);
    });
}
extern "C" int h2_batch_normalize(int curve, const void *points_xyz, size_t n, int repr, void *out_xy) {
    CtxLock lk;
    const HostArgs h("h2_batch_normalize", repr);
    if (require_ready() || check_curve(curve) || h.check({{points_xyz, "points_xyz", n != 0}, {out_xy, "out_xy", n != 0}})) return 1;
    if (n == 0) return 0;
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const int canon = h.canon();
    if (X.ec_io.ensure(n * sizeof(jacobian)) || X.ec_out.ensure(n * sizeof(affine))) return 1;
    CU(cudaMemcpyAsync(X.ec_io.p, points_xyz, n * sizeof(jacobian), cudaMemcpyHostToDevice, s));
    const uint32_t nb = blocks_for((n + H2_NORM_CHUNK - 1) / H2_NORM_CHUNK, 64);
    if (by_curve(curve, [&](auto p, auto) {
            LAUNCH(normalize_kernel<decltype(p)>, nb, 64, 0, s, (const xyzz *)nullptr, X.ec_io.as<jacobian>(), canon, X.ec_out.as<affine>(), canon, (uint64_t)n);
            return 0;
        }))
        return 1;
    CU(cudaMemcpyAsync(out_xy, X.ec_out.p, n * sizeof(affine), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// point (de)compression (codec.cuh): C::to_bytes / C::from_bytes, the encoding of Params::{write, read} and of every
// point in a proof transcript
// ------------------------------------------------------------------------------------------------
template <class P> static int points_codec(int decompress, const void *in, size_t n, const HostArgs &h, void *out) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const int mont = h.mont();
    if (X.ec_io.ensure(n * sizeof(affine)) || X.ec_out.ensure(n * sizeof(affine)) || X.misc.ensure(64)) return 1;
    uint32_t bad = 0xffffffffu;
    if (!decompress) {
        CU(cudaMemcpyAsync(X.ec_io.p, in, n * sizeof(affine), cudaMemcpyHostToDevice, s));
        LAUNCH(compress_kernel<P>, blocks_for(n, 128), 128, 0, s, X.ec_io.as<affine>(), mont, X.ec_out.as<fe>(), (uint64_t)n);
        CU(cudaMemcpyAsync(out, X.ec_out.p, n * sizeof(fe), cudaMemcpyDeviceToHost, s));
    } else {
        static const SqrtConst K = make_sqrt_const<P>();
        CU(cudaMemcpyAsync(X.ec_io.p, in, n * sizeof(fe), cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(X.misc.p, &bad, 4, cudaMemcpyHostToDevice, s));
        LAUNCH(decompress_kernel<P>, blocks_for(n, 128), 128, 0, s, X.ec_io.as<fe>(), X.ec_out.as<affine>(), mont, K, X.misc.as<uint32_t>(), (uint64_t)n);
        CU(cudaMemcpyAsync(out, X.ec_out.p, n * sizeof(affine), cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(&bad, X.misc.p, 4, cudaMemcpyDeviceToHost, s));
    }
    CU(cudaStreamSynchronize(s));
    if (bad != 0xffffffffu) return fail("h2_points_decompress: invalid point encoding at index " + std::to_string(bad));
    return 0;
}
static int points_codec_dispatch(int curve, int decompress, const void *in, size_t n, const HostArgs &h, std::initializer_list<HostArgs::Need> needs,
                                 void *out) {
    CtxLock lk;
    if (require_ready() || check_curve(curve) || h.check(needs)) return 1;
    if (n >= (1ull << 32)) return fail("points codec: n >= 2^32");
    if (n == 0) return 0;
    return by_curve(curve, [&](auto p, auto) { return points_codec<decltype(p)>(decompress, in, n, h, out); });
}
extern "C" int h2_points_compress(int curve, const void *points_xy, size_t n, int repr, void *out_bytes) {
    return points_codec_dispatch(curve, 0, points_xy, n, {"h2_points_compress", repr}, {{points_xy, "points_xy", n != 0}, {out_bytes, "out_bytes", n != 0}},
                                 out_bytes);
}
extern "C" int h2_points_decompress(int curve, const void *bytes, size_t n, int repr, void *out_xy) {
    return points_codec_dispatch(curve, 1, bytes, n, {"h2_points_decompress", repr}, {{bytes, "bytes", n != 0}, {out_xy, "out_xy", n != 0}}, out_xy);
}

