// nyxb_api.cu — C-ABI implementation (include/nyxb.h): engine lifetime, table packing and
// upload, launches.  Host side of `Propagator::new` + `MonteCarlo::run_until_epoch`'s fan-out.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include <map>

#include "nyxb_coop.h"
#include "nyxb_tx.h"
#include "nyxb_device.cuh"
#include "nyxb_od.cuh"
#include "nyxb_tableaux.h"
#include "nyxb_target_dev.h"

// kernels (nyxb_kernels.cu built twice, nyxb_coop.cu)
extern "C" cudaError_t nyxb_launch_thread_strict(const DevSetup*, size_t, const double*, const double*, const long long*,
                                                 long long, long long*, double*, long long*, nyxb_details*, int*, int,
                                                 const DevSink*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_thread_fast(const DevSetup*, size_t, const double*, const double*, const long long*,
                                               long long, long long*, double*, long long*, nyxb_details*, int*, int,
                                               const DevSink*, cudaStream_t);
extern "C" double nyxb_fp64_probe(int device, int iters);
extern "C" cudaError_t nyxb_launch_frame_shift(const DevBody*, double, size_t, double*, const long long*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_traj_resample(long long, const long long*, const double*, const long long*, size_t, size_t,
                                                 const long long*, double*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_event_locate(long long, const long long*, const double*, const long long*, size_t, int, double, long long,
                                                const int*, long long*, double*, int*, cudaStream_t);
extern "C" cudaError_t nyxb_launch_mvn(unsigned long long, unsigned long long, size_t, const double*, const double*, const double*,
                                       double*, double*, cudaStream_t);

// layout of the PODs the host mirrors rely on (nyx_b200/abi.py, tests/test_abi.py)
static_assert(sizeof(nyxb_integ_opts) == 56 && sizeof(nyxb_gravity_field) == 104 && sizeof(nyxb_dynamics) == 96 && sizeof(nyxb_rotation) == 56 && sizeof(nyxb_srp) == 40 && sizeof(nyxb_details) == 48, "ABI layout");
static_assert(sizeof(nyxb_ground_station) == 176 && sizeof(nyxb_od_config) == 72 && sizeof(nyxb_tracking_arc) == 32 && sizeof(nyxb_od_outputs) == 96, "ABI layout");
static_assert(sizeof(nyxb_bls_config) == 80 && sizeof(nyxb_bls_outputs) == 72, "ABI layout");
static_assert(sizeof(nyxb_od_records) == 64 && sizeof(nyxb_smooth_outputs) == 48, "ABI layout");
static_assert(sizeof(nyxb_position_device) == 64 && sizeof(nyxb_position_arc) == 32 && sizeof(nyxb_aer_station) == 256, "ABI layout");
static_assert(sizeof(nyxb_interlink_tx) == 56, "ABI layout");
static_assert(sizeof(nyxb_tgt_variable) == 48 && sizeof(nyxb_tgt_objective) == 40 && sizeof(nyxb_target_config) == 544, "ABI layout");

static thread_local std::string g_err;
static void set_err(const std::string& s) { g_err = s; }
#define CUDA_TRY(x)                                                                                   \
    do {                                                                                              \
        cudaError_t _e = (x);                                                                         \
        if (_e != cudaSuccess) {                                                                      \
            set_err(std::string(#x) + ": " + cudaGetErrorString(_e));                                 \
            return NYXB_RC_CUDA;                                                                      \
        }                                                                                             \
    } while (0)

struct nyxb_engine {
    int device = 0;
    int mode = NYXB_MODE_STRICT;
    int lanes = 0;  // 0 = auto
    DevSetup S;
    std::vector<void*> dev_allocs;
    long long launches = 0;
    double last_ms = 0.0;
    // grow-only device staging slab of the host-pointer entry point (no cudaMalloc/cudaFree per call)
    size_t cap = 0;
    double* d_f64 = nullptr;
    long long* d_i64 = nullptr;
    nyxb_details* d_det = nullptr;
    int* d_status = nullptr;
    cudaStream_t stream = nullptr;
    // grow-only device buffers of the trajectory sink (host-pointer entry point)
    size_t sink_bytes = 0;
    unsigned char* d_sink = nullptr;
    size_t rec_n = 0;        // the recording resident in d_sink: trajectories and capacity (nyxb_traj_resample with sink == NULL)
    long long rec_cap = 0;
    std::vector<double> h_cnm, h_snm;      // host copies for building cooperative tables lazily
    std::map<int, DevCoop> coop;           // lanes -> device tables
    std::map<int, DevCoopStrict> scoop;    // lanes -> STRICT cooperative schedules
    int kernel = NYXB_KERNEL_AUTO;         // nyxb_engine_set_kernel
    int last_kernel = NYXB_KERNEL_AUTO;    // family the last launch used
    std::map<int, DevTx> tx;               // positions -> tables of the transposed kernel
    int tx_slice = 64;                     // step attempts per time slice of the persistent transposed kernel
    int tx_positions = 0;                  // walker warps per set (0: by degree)
    int tx_max_ctas = 0;                   // 0: every resident slot (SMs x occupancy); tests shrink it to force time slicing
    size_t txq_bytes = 0;                  // grow-only queue + parking workspace of the transposed kernel
    unsigned char* d_txq = nullptr;
    int sms = 0;
    size_t frame_n = 0;                    // grow-only copy of the input states translated into the integration frame
    double* d_frame = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    ~nyxb_engine() {
        for (void* p : dev_allocs) cudaFree(p);
        cudaFree(d_f64); cudaFree(d_i64); cudaFree(d_det); cudaFree(d_status); cudaFree(d_sink); cudaFree(d_txq); cudaFree(d_frame);
        if (stream) cudaStreamDestroy(stream);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
    }
};

static bool tableau_for(int method, int& order, int& stages, const NyxbCoef*& a, const NyxbCoef*& b) {
    switch (method) {  // rk_methods/mod.rs:81-133
    case NYXB_RK89: order = 9; stages = 16; a = NYXB_RK89_A; b = NYXB_RK89_B; return true;
    case NYXB_DP78: order = 8; stages = 13; a = NYXB_DP78_A; b = NYXB_DP78_B; return true;
    case NYXB_DP45: order = 5; stages = 7; a = NYXB_DP45_A; b = NYXB_DP45_B; return true;
    case NYXB_RK4: order = 4; stages = 4; a = NYXB_RK4_A; b = NYXB_RK4_B; return true;
    case NYXB_CK45: order = 5; stages = 6; a = NYXB_CK45_A; b = NYXB_CK45_B; return true;
    case NYXB_V56: order = 6; stages = 8; a = NYXB_V56_A; b = NYXB_V56_B; return true;
    default: return false;
    }
}

static double host_dur_to_seconds(long long total_ns) {
    const long long NPC = 3155760000000000000LL, NPS = 1000000000LL;
    long long cent = total_ns / NPC;
    if (total_ns % NPC < 0) cent -= 1;
    long long nanos = total_ns - cent * NPC;
    volatile double s = (double)(nanos / NPS);
    volatile double f = (double)(nanos % NPS) * 1e-9;
    if (cent == 0) return s + f;
    volatile double c = (double)cent * 3155760000.0;
    volatile double cs = c + s;
    return cs + f;
}

static DevRotation pack_rot(const nyxb_rotation& r) {
    DevRotation d;
    d.kind = r.kind;
    d.ra0 = r.ra0_deg; d.ra1 = r.ra1_deg_cy; d.dec0 = r.dec0_deg; d.dec1 = r.dec1_deg_cy; d.w0 = r.w0_deg; d.w1 = r.w1_deg_day;
    volatile double w = r.w1_deg_day * 1.7453292519943295e-2;
    d.wdot = (r.kind == 0) ? 0.0 : w / 86400.0;
    d.ra_dot = r.ra1_deg_cy * 1.7453292519943295e-2 / (36525.0 * 86400.0);
    d.dec_dot = r.dec1_deg_cy * 1.7453292519943295e-2 / (36525.0 * 86400.0);
    return d;
}

template <typename T>
static T* upload(nyxb_engine* e, const T* host, size_t count) {
    T* d = nullptr;
    if (cudaMalloc(&d, sizeof(T) * (count ? count : 1)) != cudaSuccess) return nullptr;
    e->dev_allocs.push_back(d);
    if (count && cudaMemcpy(d, host, sizeof(T) * count, cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
    return d;
}

// GravityField::new (gravity_field.rs:52-92) for one field: recursion factors, diagonal, per-thread column-walk records
static bool build_grav(nyxb_engine* e, const nyxb_gravity_field& g, DevGrav& G, bool primary) {
        if (g.degree < 1 || g.degree > NYXB_MAX_DEGREE || g.order < 0 || g.order > g.degree) {
            set_err("gravity field degree/order out of range (1..96)"); return false;
        }
        const int N = g.degree, np2 = N + 2;
        G.N = N; G.M = g.order; G.mu = g.mu_km3_s2; G.r_eq = g.r_eq_km; G.inv_r_eq = 1.0 / g.r_eq_km;
        G.rot = pack_rot(g.rot);
        // GravityField::new gravity_field.rs:52-92 (same formulas; sqrt and / are correctly rounded)
        std::vector<double> adiag(N + 3), offd(N + 2);
        adiag[0] = 1.0;
        for (int n = 1; n <= np2; ++n) {
            double nf = (double)n;
            volatile double t = 1.0 + 1.0 / (2.0 * nf);
            volatile double s = std::sqrt(t);
            volatile double v = s * adiag[n - 1];
            adiag[n] = v;
        }
        for (int n = 0; n <= N + 1; ++n) offd[n] = std::sqrt(2.0 * (double)n + 3.0);
        std::vector<DevHarm> tab((size_t)(N + 2) * (N + 3) / 2);
        const double sqrt2 = std::sqrt(2.0);
        for (int n = 0; n <= N + 1; ++n) {
            for (int m = 0; m <= n; ++m) {
                double nf = (double)n, mf = (double)m;
                DevHarm h;
                volatile double cnum = (2.0 * nf + 1.0) * (nf + mf - 1.0) * (nf - mf - 1.0);
                volatile double cden = (nf - mf) * (nf + mf) * (2.0 * nf - 3.0);
                volatile double cq = cnum / cden;
                h.c = std::sqrt(cq);
                volatile double bnum = (2.0 * nf + 1.0) * (2.0 * nf - 1.0);
                volatile double bden = (nf + mf) * (nf - mf);
                volatile double bq = bnum / bden;
                h.b = std::sqrt(bq);
                volatile double v01 = (nf - mf) * (nf + mf + 1.0);
                h.vr01 = std::sqrt(v01);
                volatile double v11n = (2.0 * nf + 1.0) * (nf + mf + 2.0) * (nf + mf + 1.0);
                volatile double v11 = v11n / (2.0 * nf + 3.0);
                h.vr11 = std::sqrt(v11);
                if (m == 0) { h.vr01 = h.vr01 / sqrt2; h.vr11 = h.vr11 / sqrt2; }
                if (n <= N) { h.cbar = g.c_nm[(size_t)n * (N + 1) + m]; h.sbar = g.s_nm[(size_t)n * (N + 1) + m]; }
                else { h.cbar = 0.0; h.sbar = 0.0; }
                if (!(n >= m + 2)) { h.b = 0.0; h.c = 0.0; }  // never read; avoid NaN/inf noise
                tab[(size_t)n * (n + 1) / 2 + m] = h;
            }
        }
        if (primary) {
            e->h_cnm.assign(g.c_nm, g.c_nm + (size_t)(N + 1) * (N + 1));
            e->h_snm.assign(g.s_nm, g.s_nm + (size_t)(N + 1) * (N + 1));
        }
        G.tab = upload(e, tab.data(), tab.size());
        G.a_diag = upload(e, adiag.data(), adiag.size());
        G.offdiag = upload(e, offd.data(), offd.size());
        {   // records of the FAST per-thread column walk (grav_accel_cols, nyxb_device.cuh), in walk order
            const int ncols = std::min(N, g.order) + 1;
            auto T = [&](int n, int m) -> const DevHarm& { return tab[(size_t)n * (n + 1) / 2 + m]; };
            std::vector<double> cr;
            cr.reserve((size_t)ncols * (N + 2) * 8);
            const double inv_req = 1.0 / g.r_eq_km;
            auto push = [&](int k, int j) {
                double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                if (j <= N && k <= g.order) { v[0] = (double)k * sqrt2 * T(j, k).cbar * inv_req; v[1] = (double)k * sqrt2 * T(j, k).sbar * inv_req; }
                if (j <= N) { v[2] = sqrt2 * T(j, k - 1).vr01 * T(j, k - 1).cbar * inv_req; v[3] = sqrt2 * T(j, k - 1).vr01 * T(j, k - 1).sbar * inv_req; }
                if (j >= 2) { v[4] = sqrt2 * T(j - 1, k - 1).vr11 * T(j - 1, k - 1).cbar * inv_req; v[5] = sqrt2 * T(j - 1, k - 1).vr11 * T(j - 1, k - 1).sbar * inv_req; }
                if (j <= N) {
                    if (j == k) { v[6] = offd[k]; v[7] = 0.0; }
                    else { v[6] = T(j + 1, k).b; v[7] = T(j + 1, k).c; }
                }
                cr.insert(cr.end(), v, v + 8);
            };
            for (int k = 1; k <= ncols; k += 2) {   // walk order of grav_accel_cols: columns in pairs, rows interleaved
                const bool two = k + 1 <= ncols;
                push(k, k);
                for (int j = k + 1; j <= N + 1; ++j) { push(k, j); if (two) push(k + 1, j); }
            }
            cr.insert(cr.end(), 16, 0.0);           // two null records: targets of the last prefetches
            G.colrec = upload(e, cr.data(), cr.size());
            G.ncols = ncols;
            if (!G.colrec) { set_err("gravity table upload failed"); return false; }
        }
        if (!G.tab || !G.a_diag || !G.offdiag) { set_err("gravity table upload failed"); return false; }
    return true;
}

extern "C" nyxb_engine* nyxb_engine_create(const nyxb_dynamics* dyn, const nyxb_integ_opts* opts, int32_t mode,
                                            int32_t device) {
    if (!dyn || !opts) { set_err("null dynamics/options"); return nullptr; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_err("no CUDA device available: nyxb has no CPU fallback");
        return nullptr;
    }
    if (device < 0 || device >= ndev) { set_err("bad device ordinal"); return nullptr; }
    if (cudaSetDevice(device) != cudaSuccess) { set_err("cudaSetDevice failed"); return nullptr; }
    if (mode != NYXB_MODE_STRICT && mode != NYXB_MODE_FAST) { set_err("bad mode"); return nullptr; }
    if (dyn->n_bodies < 0 || dyn->n_bodies > NYXB_MAX_BODIES) { set_err("n_bodies out of range"); return nullptr; }

    nyxb_engine* e = new nyxb_engine();
    e->device = device;
    e->mode = mode;
    DevSetup& S = e->S;
    memset(&S, 0, sizeof(S));

    // ---- tableau (dense rows, c accumulated left to right as instance.rs:379-386 does)
    int order, stages;
    const NyxbCoef *a, *b;
    if (!tableau_for(opts->method, order, stages, a, b)) { set_err("unknown integration method"); delete e; return nullptr; }
    S.tb.stages = stages;
    S.tb.order = order;
    int idx = 0;
    for (int i = 0; i < stages - 1; ++i) {
        volatile double ci = 0.0;
        for (int j = 0; j <= i; ++j) {
            double aij = nyxb_tableau_value(a[idx++]);
            ci = ci + aij;
            S.tb.a[i * NYXB_MAX_STAGES + j] = aij;
        }
        S.tb.c[i] = ci;
    }
    for (int i = 0; i < stages; ++i) {
        S.tb.b[i] = nyxb_tableau_value(b[i]);
        volatile double d = S.tb.b[i] - nyxb_tableau_value(b[i + stages]);
        S.tb.e[i] = d;
    }
    S.error_ctrl = opts->error_ctrl;
    S.attempts = opts->attempts;
    S.fixed_step = opts->fixed_step;
    S.init_step_ns = opts->init_step_ns;
    S.min_step_ns = opts->min_step_ns;
    S.max_step_ns = opts->max_step_ns;
    S.tolerance = opts->tolerance;
    S.min_step_s = host_dur_to_seconds(opts->min_step_ns);
    S.max_step_s = host_dur_to_seconds(opts->max_step_ns);
    S.inv_order = 1.0 / (double)order;
    S.inv_order_m1 = 1.0 / (double)(order - 1);

    // ---- dynamics
    S.mu_central = dyn->mu_central_km3_s2;
    S.central_radius = dyn->central_radius_km;
    S.n_bodies = dyn->n_bodies;
    S.point_mass_mask = dyn->point_mass_mask;
    S.n_pm = 0;
    if (dyn->n_point_masses > 0) {   // `celestial_objects` order (orbital.rs:217)
        if (dyn->n_point_masses > dyn->n_bodies) { set_err("n_point_masses out of range"); delete e; return nullptr; }
        for (int q = 0; q < dyn->n_point_masses; ++q) {
            const int j = dyn->point_mass_order[q];
            if (j < 0 || j >= dyn->n_bodies) { set_err("point_mass_order: bad body index"); delete e; return nullptr; }
            S.pm_order[S.n_pm++] = (signed char)j;
        }
    } else {
        for (int j = 0; j < dyn->n_bodies; ++j)
            if ((dyn->point_mass_mask >> j) & 1u) S.pm_order[S.n_pm++] = (signed char)j;
    }
    S.state_center = -1;
    if (opts->state_center != 0) {
        if (opts->state_center < 0 || opts->state_center > dyn->n_bodies) { set_err("state_center: bad body index"); delete e; return nullptr; }
        S.state_center = opts->state_center - 1;
    }
    for (int j = 0; j < dyn->n_bodies; ++j) {
        const nyxb_body& hb = dyn->bodies[j];
        DevBody& db = S.bodies[j];
        db.mu = hb.mu_km3_s2; db.radius = hb.radius_km; db.t0_ns = hb.t0_ns; db.interval_ns = hb.interval_ns;
        db.n_intervals = hb.n_intervals; db.n_coeffs = hb.n_coeffs;
        db.inv_interval = 1.0 / (double)hb.interval_ns;
        db.coeffs = upload(e, hb.coeffs, (size_t)hb.n_intervals * 3 * hb.n_coeffs);
        if (!db.coeffs) { set_err("ephemeris upload failed"); delete e; return nullptr; }
    }
    const int n_grav = dyn->gravity ? std::max(1, dyn->n_gravity) : 0;
    if (n_grav > NYXB_MAX_FIELDS) { set_err("too many gravity fields"); delete e; return nullptr; }
    S.grav_body = NYXB_CENTRAL_BODY;
    for (int f = 0; f < n_grav; ++f) {
        const nyxb_gravity_field& g = dyn->gravity[f];
        if (g.body != NYXB_CENTRAL_BODY && (g.body < 0 || g.body >= dyn->n_bodies)) { set_err("gravity field: bad body index"); delete e; return nullptr; }
        if (f == 0) {
            if (!build_grav(e, g, S.grav, true)) { delete e; return nullptr; }
            S.has_grav = 1;
            S.grav_body = g.body;
        } else {
            if (!build_grav(e, g, S.xgrav[f - 1], false)) { delete e; return nullptr; }
            S.xgrav_body[f - 1] = g.body;
            S.n_xgrav = f;
        }
    }
    if (dyn->srp) {
        const nyxb_srp& s = *dyn->srp;
        if (s.sun_body < 0 || s.sun_body >= dyn->n_bodies || s.n_shadow < 0 || s.n_shadow > 4) {
            set_err("bad SRP descriptor"); delete e; return nullptr;
        }
        S.has_srp = 1;
        S.srp.phi = s.phi_w_m2; S.srp.sun_body = s.sun_body; S.srp.n_shadow = s.n_shadow; S.srp.estimate = s.estimate;
        for (int q = 0; q < 4; ++q) {
            S.srp.shadow_body[q] = s.shadow_body[q];
            if (q < s.n_shadow && s.shadow_body[q] != NYXB_CENTRAL_BODY && (s.shadow_body[q] < 0 || s.shadow_body[q] >= dyn->n_bodies)) {
                set_err("bad shadow body index"); delete e; return nullptr;
            }
        }
    }
    if (dyn->drag) {
        const nyxb_drag& d = *dyn->drag;
        S.has_drag = 1;
        S.drag.density = d.density; S.drag.rho0 = d.rho0; S.drag.r0 = d.r0; S.drag.ref_alt_m = d.ref_alt_m; S.drag.r_eq = d.r_eq_km;
        S.drag.rot = pack_rot(d.rot);
    }
    cudaEventCreate(&e->ev0);
    cudaEventCreate(&e->ev1);
    return e;
}

extern "C" void nyxb_engine_destroy(nyxb_engine* eng) {
    if (!eng) return;
    cudaSetDevice(eng->device);
    delete eng;
}

static bool coop_supported(const nyxb_engine* e, int lanes) {
    if (!e->S.has_grav) return false;
    return lanes == 8 || lanes == 16 || lanes == 32;
}

static int pick_lanes(const nyxb_engine* e, size_t n) {
    if (e->lanes > 0) return e->lanes;
    // auto: cooperative lanes only pay off when the harmonic sum dominates
    if (!e->S.has_grav || e->S.grav.N < 6) return 1;
    // FAST, moderate degree, very large ensembles: one thread per trajectory (column walk, grav_accel_cols) has enough warps to
    // hide its latencies and issues ~3x fewer instructions per trajectory than the cooperative kernel.  Only degrees 6-7 reach this
    // rule (the transposed kernel takes degree 8-70 from 1 024 trajectories); H100, degree 7: 3.7e8 against 1.4e8 steps/s for 8
    // lanes at 32 768 trajectories and above (scripts/dispatch_sweep.py)
    if (e->mode == NYXB_MODE_FAST && e->S.grav.N < 30 && n >= 32768) return 1;
    return (e->S.grav.N >= 48) ? 32 : ((e->S.grav.N >= 30) ? 16 : 8);
}

static const DevCoopStrict* get_scoop(nyxb_engine* e, int lanes) {
    auto it = e->scoop.find(lanes);
    if (it != e->scoop.end()) return &it->second;
    CoopStrictHost h;
    nyxb_coop_strict_build_host(e->S.grav.N, e->S.grav.M, lanes, h);
    DevCoopStrict d;
    d.G = h.G; d.kc = h.kc; d.kr = h.kr;
    d.cols = upload(e, h.cols.data(), h.cols.size());
    d.rows = upload(e, h.rows.data(), h.rows.size());
    if (!d.cols || !d.rows) return nullptr;
    return &(e->scoop[lanes] = d);
}

static const DevCoop* get_coop(nyxb_engine* e, int lanes) {
    auto it = e->coop.find(lanes);
    if (it != e->coop.end()) return &it->second;
    CoopHost h;
    nyxb_coop_build_host(e->S.grav.N, e->S.grav.M, e->h_cnm.data(), e->h_snm.data(), lanes, h);
    DevCoop d;
    d.G = h.G; d.L = h.L; d.kmax = h.kmax;
    d.recs = upload(e, h.recs.data(), h.recs.size());
    d.colseed = upload(e, h.colseed.data(), h.colseed.size());
    d.col_start = upload(e, h.col_start.data(), h.col_start.size());
    d.col_m = upload(e, h.col_m.data(), h.col_m.size());
    if (!d.recs || !d.col_start || !d.col_m || !d.colseed) return nullptr;
    return &(e->coop[lanes] = d);
}

static const DevTx* get_tx(nyxb_engine* e, int P) {
    auto it = e->tx.find(P);
    if (it != e->tx.end()) return &it->second;
    TxHost h;
    nyxb_tx_build_host(e->S.grav.N, e->S.grav.M, e->h_cnm.data(), e->h_snm.data(), P, h);
    std::vector<unsigned char> blob(nyxb_tx_pack_blob(&h, e->S.grav.N, nullptr));
    nyxb_tx_pack_blob(&h, e->S.grav.N, blob.data());
    DevTx d;
    d.P = h.P; d.n_rec = h.n_rec; d.kmax = h.kmax;
    d.recA = reinterpret_cast<const double*>(upload(e, blob.data(), blob.size()));
    if (!d.recA) return nullptr;
    return &(e->tx[P] = d);
}

// positions of the transposed kernel for this field: 8 warps per set up to degree 40, 16 beyond (shared-memory footprint of the table)
static int tx_positions(const nyxb_engine* e) {
    if (e->tx_positions) return e->tx_positions;
    return e->S.grav.N <= 40 ? 8 : 16;
}

static bool tx_supported(const nyxb_engine* e) {
    return e->mode == NYXB_MODE_FAST && e->S.has_grav && e->S.grav.N >= 8 && e->S.grav.N <= 70;
}

// Transposed kernel (nyxb_tx.cu): persistent CTAs, one set of 32 trajectories per CTA, (set, time-slice) tickets.
static int32_t launch_tx(nyxb_engine* e, size_t n, const double* state, const double* consts, const int64_t* epoch0, int64_t end_epoch,
                         int64_t* step_io, double* out_state, int64_t* out_epoch, nyxb_details* out_details, int32_t* out_status,
                         const DevSink& sink, cudaStream_t stream) {
    const DevTx* tx = get_tx(e, tx_positions(e));
    if (!tx) { set_err("transposed-kernel table upload failed"); return NYXB_RC_CUDA; }
    size_t smem = 0;
    // sets of 32 trajectories.  Sets of 64 (a walker lane carrying two trajectories through every record load: half the shared-
    // memory wavefronts per FP64 instruction, but only one set context fits a CTA, so nothing covers the serial stretch between two
    // attempts) were built and measured slower; not dispatched.
    const int set_len = 32;
    const int occ = nyxb_tx_occupancy(&e->S, tx, &smem);
    if (occ < 1) { set_err("transposed kernel: tables do not fit in shared memory"); return NYXB_RC_UNSUPPORTED; }
    if (!e->sms) CUDA_TRY(cudaDeviceGetAttribute(&e->sms, cudaDevAttrMultiProcessorCount, e->device));
    const size_t n_sets = (n + set_len - 1) / set_len;
    // one persistent CTA per SM, `occ` set contexts each; tx_max_ctas (tests) shrinks the grid to force time slicing
    size_t ctas = (size_t)e->sms;
    if (e->tx_max_ctas > 0 && (size_t)e->tx_max_ctas < ctas) ctas = (size_t)e->tx_max_ctas;
    // fewer sets than SMs x contexts: spread them over all SMs (one set per CTA runs its stages at the helpers' pace instead of
    // alternating with a second set, and twice as many SMs work)
    ctas = std::min(ctas, n_sets);
    const size_t slots = ctas * occ;
    const int grid = (int)ctas;
    // workspace: [ctl 4 x i32 | ring n_sets x i32 | ws_step n i64 | ws_f64 2n | ws_flags n | details n]
    const size_t ctl_bytes = (16 + 4 * n_sets + 15) & ~(size_t)15;
    const size_t need = ctl_bytes + n * (8 + 16 + 8) + n * sizeof(nyxb_details);
    if (need > e->txq_bytes) {
        cudaFree(e->d_txq); e->d_txq = nullptr; e->txq_bytes = 0;
        CUDA_TRY(cudaMalloc(&e->d_txq, need));
        e->txq_bytes = need;
    }
    CUDA_TRY(cudaMemsetAsync(e->d_txq, 0, ctl_bytes, stream));
    DevTxQueue q;
    q.ctl = reinterpret_cast<int*>(e->d_txq);
    q.ring = q.ctl + 4;
    unsigned char* ws = e->d_txq + ctl_bytes;
    q.ws_step = reinterpret_cast<long long*>(ws);
    q.ws_f64 = reinterpret_cast<double*>(ws + 8 * n);
    q.ws_flags = reinterpret_cast<int*>(ws + 24 * n);
    q.details = out_details ? out_details : reinterpret_cast<nyxb_details*>(ws + 32 * n);
    q.n_sets = (int)n_sets;
    q.slice = (n_sets > slots) ? e->tx_slice : 0;   // every set resident: no parking
    q.trace = nullptr;
#ifdef NYXB_TX_TRACE
    // diagnostic build: timeline of CTA 0, dumped to $NYXB_TX_TRACE_FILE after the launch (synchronises the stream)
    const size_t trace_bytes = (size_t)32 * NYXB_TX_TRACE_CAP * sizeof(unsigned long long);
    const char* trace_file = getenv("NYXB_TX_TRACE_FILE");
    if (trace_file) {
        CUDA_TRY(cudaMalloc(&q.trace, trace_bytes));
        CUDA_TRY(cudaMemsetAsync(q.trace, 0, trace_bytes, stream));
    }
#endif
    cudaError_t err = nyxb_launch_tx(&e->S, tx, &q, n, state, consts, (const long long*)epoch0, end_epoch, (long long*)step_io, out_state,
                                     (long long*)out_epoch, out_status, &sink, grid, stream);
    if (err != cudaSuccess) { set_err(std::string("kernel launch: ") + cudaGetErrorString(err)); return NYXB_RC_CUDA; }
#ifdef NYXB_TX_TRACE
    if (q.trace) {
        std::vector<unsigned long long> host((size_t)32 * NYXB_TX_TRACE_CAP);
        CUDA_TRY(cudaStreamSynchronize(stream));
        CUDA_TRY(cudaMemcpy(host.data(), q.trace, trace_bytes, cudaMemcpyDeviceToHost));
        cudaFree(q.trace);
        if (FILE* f = fopen(trace_file, "wb")) { fwrite(host.data(), 1, trace_bytes, f); fclose(f); }
    }
#endif
    e->launches += 1;
    e->last_kernel = NYXB_KERNEL_TRANSPOSED;
    return NYXB_RC_OK;
}

// kernel family for this call (nyxb_engine_set_kernel overrides the automatic choice)
static int pick_kernel(const nyxb_engine* e, size_t n) {
    if (e->kernel == NYXB_KERNEL_TRANSPOSED) return tx_supported(e) ? NYXB_KERNEL_TRANSPOSED : NYXB_KERNEL_COOP;
    if (e->kernel != NYXB_KERNEL_AUTO) return e->kernel;
    if (e->lanes > 0) return e->lanes == 1 ? NYXB_KERNEL_THREAD : NYXB_KERNEL_COOP;
    // auto: transposed kernel from 32 sets up, for every degree it serves (8..70; 16 walker positions and one set context per CTA
    // above degree 40); below that the lane-cooperative kernel.  H100 (scripts/dispatch_sweep.py, FAST; 3 days up to 5 000 trajectories, 1 day
    // above, 6 hours at 70x70): 21x21 from 1 024 to 100 000 trajectories it is ahead of every lane count of the cooperative kernel and of the per-thread kernel (1 024: 2.6e7 against
    // 2.5e7 for 16 lanes; 5 000: 7.5e7 / 6.5e7; 100 000: 1.11e8 against 9.4e7 per-thread); 70x70 at 1 024 and 2 000: 4.5e6 / 3.6e6 and
    // 8.8e6 / 5.4e6 for 32 lanes
    if (tx_supported(e) && n >= (size_t)1024) return NYXB_KERNEL_TRANSPOSED;
    return NYXB_KERNEL_AUTO;
}

static int32_t launch_inner(nyxb_engine* e, size_t n, const double* state, const double* consts, const int64_t* epoch0,
                            int64_t end_epoch, int64_t* step_io, double* out_state, int64_t* out_epoch,
                            nyxb_details* out_details, int32_t* out_status, const DevSink& sink, cudaStream_t stream);

// propagation launch with the integration_frame translations around it (instance.rs:117-142, 167-176, 211-220)
static int32_t launch(nyxb_engine* e, size_t n, const double* state, const double* consts, const int64_t* epoch0,
                      int64_t end_epoch, int64_t* step_io, double* out_state, int64_t* out_epoch,
                      nyxb_details* out_details, int32_t* out_status, const DevSink& sink, cudaStream_t stream) {
    if (e->S.state_center < 0 || n == 0)
        return launch_inner(e, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    if (n > e->frame_n) {
        cudaFree(e->d_frame); e->d_frame = nullptr; e->frame_n = 0;
        CUDA_TRY(cudaMalloc(&e->d_frame, sizeof(double) * 9 * n));
        e->frame_n = n;
    }
    const DevBody* body = &e->S.bodies[e->S.state_center];
    CUDA_TRY(cudaMemcpyAsync(e->d_frame, state, sizeof(double) * 9 * n, cudaMemcpyDeviceToDevice, stream));
    CUDA_TRY(nyxb_launch_frame_shift(body, 1.0, n, e->d_frame, (const long long*)epoch0, nullptr, stream));
    const int32_t rc = launch_inner(e, n, e->d_frame, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    if (rc != NYXB_RC_OK) return rc;
    CUDA_TRY(nyxb_launch_frame_shift(body, -1.0, n, out_state, (const long long*)out_epoch, out_status, stream));
    e->launches += 2;
    return NYXB_RC_OK;
}

// The family a launch of n trajectories runs: TRANSPOSED, or COOP / THREAD with `lanes` lanes per trajectory (1 for THREAD)
static int launch_family(const nyxb_engine* e, size_t n, int& lanes) {
    lanes = 1;
    if (pick_kernel(e, n) == NYXB_KERNEL_TRANSPOSED) return NYXB_KERNEL_TRANSPOSED;
    lanes = pick_lanes(e, n);
    if (e->kernel == NYXB_KERNEL_THREAD) lanes = 1;
    if (e->kernel == NYXB_KERNEL_COOP && lanes == 1 && e->S.has_grav) lanes = (e->S.grav.N >= 48) ? 32 : ((e->S.grav.N >= 30) ? 16 : 8);
    return lanes > 1 ? NYXB_KERNEL_COOP : NYXB_KERNEL_THREAD;
}

static int32_t launch_inner(nyxb_engine* e, size_t n, const double* state, const double* consts, const int64_t* epoch0,
                            int64_t end_epoch, int64_t* step_io, double* out_state, int64_t* out_epoch,
                            nyxb_details* out_details, int32_t* out_status, const DevSink& sink, cudaStream_t stream) {
    int lanes;
    if (launch_family(e, n, lanes) == NYXB_KERNEL_TRANSPOSED)
        return launch_tx(e, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details, out_status, sink, stream);
    e->last_kernel = lanes > 1 ? NYXB_KERNEL_COOP : NYXB_KERNEL_THREAD;
    cudaError_t err;
    if (lanes > 1 && e->mode == NYXB_MODE_STRICT) {
        const DevCoopStrict* cs = get_scoop(e, lanes);
        if (!cs) { set_err("cooperative schedule upload failed"); return NYXB_RC_CUDA; }
        err = nyxb_launch_coop_strict(&e->S, cs, n, state, consts, (const long long*)epoch0, end_epoch, (long long*)step_io,
                                      out_state, (long long*)out_epoch, out_details, out_status, &sink, stream);
    } else if (lanes > 1) {
        const DevCoop* cp = get_coop(e, lanes);
        if (!cp) { set_err("cooperative table upload failed"); return NYXB_RC_CUDA; }
        err = nyxb_launch_coop(&e->S, cp, n, state, consts, (const long long*)epoch0, end_epoch, (long long*)step_io,
                               out_state, (long long*)out_epoch, out_details, out_status, &sink, stream);
    } else if (e->mode == NYXB_MODE_STRICT) {
        err = nyxb_launch_thread_strict(&e->S, n, state, consts, (const long long*)epoch0, end_epoch, (long long*)step_io,
                                        out_state, (long long*)out_epoch, out_details, out_status, 64, &sink, stream);
    } else {
        const int blk = 64;   // 32 / 128 threads per CTA measured no better
        err = nyxb_launch_thread_fast(&e->S, n, state, consts, (const long long*)epoch0, end_epoch, (long long*)step_io,
                                      out_state, (long long*)out_epoch, out_details, out_status, blk, &sink, stream);
    }
    if (err != cudaSuccess) { set_err(std::string("kernel launch: ") + cudaGetErrorString(err)); return NYXB_RC_CUDA; }
    e->launches += 1;
    return NYXB_RC_OK;
}

static DevSink make_sink(const nyxb_traj_sink* sink) {
    DevSink d{};
    if (sink && sink->capacity > 0 && sink->epoch_ns && sink->state && sink->count) {
        d.cap = sink->capacity; d.epoch = (long long*)sink->epoch_ns; d.state = sink->state; d.count = (long long*)sink->count;
    }
    return d;
}

extern "C" int32_t nyxb_propagate_batch_traj_dev(nyxb_engine* eng, size_t n, const double* state_soa, const double* consts_soa,
                                                 const int64_t* epoch0_ns, int64_t end_epoch_ns, int64_t* step_ns,
                                                 double* out_state_soa, int64_t* out_epoch_ns, nyxb_details* out_details,
                                                 int32_t* out_status, const nyxb_traj_sink* sink, void* cuda_stream) {
    if (!eng || !state_soa || !consts_soa || !epoch0_ns || !out_state_soa || !out_epoch_ns || !out_status) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    CUDA_TRY(cudaSetDevice(eng->device));
    return launch(eng, n, state_soa, consts_soa, epoch0_ns, end_epoch_ns, step_ns, out_state_soa, out_epoch_ns, out_details,
                  out_status, make_sink(sink), (cudaStream_t)cuda_stream);
}

extern "C" int32_t nyxb_propagate_batch_dev(nyxb_engine* eng, size_t n, const double* state_soa, const double* consts_soa,
                                            const int64_t* epoch0_ns, int64_t end_epoch_ns, int64_t* step_ns,
                                            double* out_state_soa, int64_t* out_epoch_ns, nyxb_details* out_details,
                                            int32_t* out_status, void* cuda_stream) {
    return nyxb_propagate_batch_traj_dev(eng, n, state_soa, consts_soa, epoch0_ns, end_epoch_ns, step_ns, out_state_soa,
                                         out_epoch_ns, out_details, out_status, nullptr, cuda_stream);
}

extern "C" int32_t nyxb_propagate_batch_event(nyxb_engine* eng, size_t n, const double* state_soa, const double* consts_soa,
                                              const int64_t* epoch0_ns, int64_t end_epoch_ns, int64_t* step_ns,
                                              double* out_state_soa, int64_t* out_epoch_ns, nyxb_details* out_details,
                                              int32_t* out_status, const nyxb_traj_sink* sink, const nyxb_event* event) {
    if (event && event->kind != NYXB_EVENT_NONE &&
        (event->kind < NYXB_EVENT_RMAG || event->kind > NYXB_EVENT_VMAG || event->trigger < 1 || !event->crossings)) {
        set_err("bad event descriptor");
        return NYXB_RC_BAD_ARG;
    }
    const bool has_ev = event && event->kind != NYXB_EVENT_NONE;
    if (!eng || !state_soa || !consts_soa || !epoch0_ns || !out_state_soa || !out_epoch_ns || !out_status) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (n == 0) return NYXB_RC_OK;
    CUDA_TRY(cudaSetDevice(eng->device));
    // device slab: [state 9n | consts 4n | out_state 9n] doubles, [epoch0 n | out_epoch n | step n] i64, details, status
    int32_t rc = NYXB_RC_OK;
    cudaError_t ce;
#define TRY2(x) do { ce = (x); if (ce != cudaSuccess) { set_err(std::string(#x) + ": " + cudaGetErrorString(ce)); return NYXB_RC_CUDA; } } while (0)
    if (!eng->stream) TRY2(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
    if (n > eng->cap) {
        cudaFree(eng->d_f64); cudaFree(eng->d_i64); cudaFree(eng->d_det); cudaFree(eng->d_status);
        eng->d_f64 = nullptr; eng->d_i64 = nullptr; eng->d_det = nullptr; eng->d_status = nullptr; eng->cap = 0;
        TRY2(cudaMalloc(&eng->d_f64, sizeof(double) * 22 * n));
        TRY2(cudaMalloc(&eng->d_i64, sizeof(long long) * 3 * n));
        TRY2(cudaMalloc(&eng->d_det, sizeof(nyxb_details) * n));
        TRY2(cudaMalloc(&eng->d_status, sizeof(int) * 2 * n));  // status | event crossings
        eng->cap = n;
    }
    double* d_f64 = eng->d_f64;
    long long* d_i64 = eng->d_i64;
    nyxb_details* d_det = eng->d_det;
    int* d_status = eng->d_status;
    cudaStream_t st = eng->stream;
    TRY2(cudaMemcpyAsync(d_f64, state_soa, sizeof(double) * 9 * n, cudaMemcpyHostToDevice, st));
    TRY2(cudaMemcpyAsync(d_f64 + 9 * n, consts_soa, sizeof(double) * 4 * n, cudaMemcpyHostToDevice, st));
    TRY2(cudaMemcpyAsync(d_i64, epoch0_ns, sizeof(long long) * n, cudaMemcpyHostToDevice, st));
    if (step_ns) TRY2(cudaMemcpyAsync(d_i64 + 2 * n, step_ns, sizeof(long long) * n, cudaMemcpyHostToDevice, st));
    // trajectory sink on the device: [epoch cap*n i64 | state 6*cap*n f64 | count n i64]
    DevSink dsink{};
    if (has_ev) { dsink.ev_kind = event->kind; dsink.ev_trigger = event->trigger; dsink.ev_value = event->value; dsink.ev_crossings = d_status + n; }
    const bool rec = sink && sink->capacity > 0 && sink->epoch_ns && sink->state && sink->count;
    eng->rec_n = 0; eng->rec_cap = 0;   // a propagation that does not record invalidates the resident recording (sink == NULL calls)
    if (rec) {
        const size_t cap = (size_t)sink->capacity;
        const size_t need = (cap * n * 7 + n) * 8;
        if (need > eng->sink_bytes) {
            cudaFree(eng->d_sink); eng->d_sink = nullptr; eng->sink_bytes = 0;
            TRY2(cudaMalloc(&eng->d_sink, need));
            eng->sink_bytes = need;
        }
        dsink.cap = sink->capacity;
        dsink.epoch = (long long*)eng->d_sink;
        dsink.state = (double*)(eng->d_sink + cap * n * 8);
        dsink.count = (long long*)(eng->d_sink + cap * n * 56);
        eng->rec_n = n; eng->rec_cap = sink->capacity;
        // slots past count[i] come back as zeros, not as whatever the allocation held (the whole sink is copied to the caller)
        TRY2(cudaMemsetAsync(eng->d_sink, 0, cap * n * 56, st));
    }
    TRY2(cudaEventRecord(eng->ev0, st));
    rc = launch(eng, n, d_f64, d_f64 + 9 * n, (const int64_t*)d_i64, end_epoch_ns, step_ns ? (int64_t*)(d_i64 + 2 * n) : nullptr,
                d_f64 + 13 * n, (int64_t*)(d_i64 + n), d_det, d_status, dsink, st);
    if (rc != NYXB_RC_OK) return rc;
    TRY2(cudaEventRecord(eng->ev1, st));
    TRY2(cudaMemcpyAsync(out_state_soa, d_f64 + 13 * n, sizeof(double) * 9 * n, cudaMemcpyDeviceToHost, st));
    TRY2(cudaMemcpyAsync(out_epoch_ns, d_i64 + n, sizeof(long long) * n, cudaMemcpyDeviceToHost, st));
    if (step_ns) TRY2(cudaMemcpyAsync(step_ns, d_i64 + 2 * n, sizeof(long long) * n, cudaMemcpyDeviceToHost, st));
    if (out_details) TRY2(cudaMemcpyAsync(out_details, d_det, sizeof(nyxb_details) * n, cudaMemcpyDeviceToHost, st));
    TRY2(cudaMemcpyAsync(out_status, d_status, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    if (has_ev) TRY2(cudaMemcpyAsync(event->crossings, d_status + n, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    if (rec) {
        const size_t cap = (size_t)sink->capacity;
        TRY2(cudaMemcpyAsync(sink->epoch_ns, dsink.epoch, cap * n * 8, cudaMemcpyDeviceToHost, st));
        TRY2(cudaMemcpyAsync(sink->state, dsink.state, cap * n * 48, cudaMemcpyDeviceToHost, st));
        TRY2(cudaMemcpyAsync(sink->count, dsink.count, n * 8, cudaMemcpyDeviceToHost, st));
    }
    TRY2(cudaStreamSynchronize(st));
    {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, eng->ev0, eng->ev1) == cudaSuccess) eng->last_ms = ms;
    }
    return rc;
#undef TRY2
}

extern "C" int32_t nyxb_propagate_batch_traj(nyxb_engine* eng, size_t n, const double* state_soa, const double* consts_soa,
                                             const int64_t* epoch0_ns, int64_t end_epoch_ns, int64_t* step_ns,
                                             double* out_state_soa, int64_t* out_epoch_ns, nyxb_details* out_details,
                                             int32_t* out_status, const nyxb_traj_sink* sink) {
    return nyxb_propagate_batch_event(eng, n, state_soa, consts_soa, epoch0_ns, end_epoch_ns, step_ns, out_state_soa, out_epoch_ns,
                                      out_details, out_status, sink, nullptr);
}

extern "C" int32_t nyxb_propagate_batch(nyxb_engine* eng, size_t n, const double* state_soa, const double* consts_soa,
                                        const int64_t* epoch0_ns, int64_t end_epoch_ns, int64_t* step_ns,
                                        double* out_state_soa, int64_t* out_epoch_ns, nyxb_details* out_details,
                                        int32_t* out_status) {
    return nyxb_propagate_batch_traj(eng, n, state_soa, consts_soa, epoch0_ns, end_epoch_ns, step_ns, out_state_soa, out_epoch_ns,
                                     out_details, out_status, nullptr);
}

// ---------------------------------------------------------------------------------------------------------------------
// Multi-GPU fan-out behind the boundary (SURVEY.md section 8e; mc/montecarlo.rs:233-253: contiguous run-index ranges, no exchange while
// integrating).  engines[g] must have been created from the same (dynamics, options) on DIFFERENT devices (or the same device, for
// tests); shard g = runs [g n / G, (g+1) n / G).  All uploads and launches are enqueued first, then the results of every shard are
// copied straight into the caller's [9][n] arrays — for a host caller that IS the gather of final states.
// ---------------------------------------------------------------------------------------------------------------------
static int32_t ensure_slab(nyxb_engine* eng, size_t n) {
    cudaError_t ce;
#define TRY3(x) do { ce = (x); if (ce != cudaSuccess) { set_err(std::string(#x) + ": " + cudaGetErrorString(ce)); return NYXB_RC_CUDA; } } while (0)
    if (!eng->stream) TRY3(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
    if (n > eng->cap) {
        cudaFree(eng->d_f64); cudaFree(eng->d_i64); cudaFree(eng->d_det); cudaFree(eng->d_status);
        eng->d_f64 = nullptr; eng->d_i64 = nullptr; eng->d_det = nullptr; eng->d_status = nullptr; eng->cap = 0;
        TRY3(cudaMalloc(&eng->d_f64, sizeof(double) * 22 * n));
        TRY3(cudaMalloc(&eng->d_i64, sizeof(long long) * 3 * n));
        TRY3(cudaMalloc(&eng->d_det, sizeof(nyxb_details) * n));
        TRY3(cudaMalloc(&eng->d_status, sizeof(int) * 2 * n));
        eng->cap = n;
    }
    return NYXB_RC_OK;
#undef TRY3
}

extern "C" int32_t nyxb_propagate_batch_multi(nyxb_engine* const* engines, int32_t n_engines, size_t n, const double* state_soa,
                                              const double* consts_soa, const int64_t* epoch0_ns, int64_t end_epoch_ns, int64_t* step_ns,
                                              double* out_state_soa, int64_t* out_epoch_ns, nyxb_details* out_details, int32_t* out_status) {
    if (!engines || n_engines < 1 || !state_soa || !consts_soa || !epoch0_ns || !out_state_soa || !out_epoch_ns || !out_status) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    for (int32_t g = 0; g < n_engines; ++g)
        if (!engines[g]) { set_err("null engine"); return NYXB_RC_BAD_ARG; }
    if (n == 0) return NYXB_RC_OK;
    const size_t G = (size_t)n_engines;
    auto lo_of = [&](size_t g) { return g * n / G; };
    cudaError_t ce;
#define TRY4(x) do { ce = (x); if (ce != cudaSuccess) { set_err(std::string(#x) + ": " + cudaGetErrorString(ce)); return NYXB_RC_CUDA; } } while (0)
    // ---- phase 1: uploads + launches on every device (asynchronous: the devices integrate concurrently)
    for (size_t g = 0; g < G; ++g) {
        nyxb_engine* eng = engines[g];
        const size_t lo = lo_of(g), m = lo_of(g + 1) - lo;
        if (m == 0) continue;
        TRY4(cudaSetDevice(eng->device));
        int32_t rc = ensure_slab(eng, m);
        if (rc != NYXB_RC_OK) return rc;
        cudaStream_t st = eng->stream;
        // strided rows of the caller's [rows][n] arrays -> dense [rows][m] shards
        TRY4(cudaMemcpy2DAsync(eng->d_f64, m * 8, state_soa + lo, n * 8, m * 8, 9, cudaMemcpyHostToDevice, st));
        TRY4(cudaMemcpy2DAsync(eng->d_f64 + 9 * m, m * 8, consts_soa + lo, n * 8, m * 8, 4, cudaMemcpyHostToDevice, st));
        TRY4(cudaMemcpyAsync(eng->d_i64, epoch0_ns + lo, m * 8, cudaMemcpyHostToDevice, st));
        if (step_ns) TRY4(cudaMemcpyAsync(eng->d_i64 + 2 * m, step_ns + lo, m * 8, cudaMemcpyHostToDevice, st));
        eng->rec_n = 0; eng->rec_cap = 0;
        TRY4(cudaEventRecord(eng->ev0, st));
        rc = launch(eng, m, eng->d_f64, eng->d_f64 + 9 * m, (const int64_t*)eng->d_i64, end_epoch_ns,
                    step_ns ? (int64_t*)(eng->d_i64 + 2 * m) : nullptr, eng->d_f64 + 13 * m, (int64_t*)(eng->d_i64 + m), eng->d_det,
                    eng->d_status, DevSink{}, st);
        if (rc != NYXB_RC_OK) return rc;
        TRY4(cudaEventRecord(eng->ev1, st));
    }
    // ---- phase 2: every shard's results straight into the caller's arrays (the gather), then one synchronisation per device
    for (size_t g = 0; g < G; ++g) {
        nyxb_engine* eng = engines[g];
        const size_t lo = lo_of(g), m = lo_of(g + 1) - lo;
        if (m == 0) continue;
        TRY4(cudaSetDevice(eng->device));
        cudaStream_t st = eng->stream;
        TRY4(cudaMemcpy2DAsync(out_state_soa + lo, n * 8, eng->d_f64 + 13 * m, m * 8, m * 8, 9, cudaMemcpyDeviceToHost, st));
        TRY4(cudaMemcpyAsync(out_epoch_ns + lo, eng->d_i64 + m, m * 8, cudaMemcpyDeviceToHost, st));
        if (step_ns) TRY4(cudaMemcpyAsync(step_ns + lo, eng->d_i64 + 2 * m, m * 8, cudaMemcpyDeviceToHost, st));
        if (out_details) TRY4(cudaMemcpyAsync(out_details + lo, eng->d_det, sizeof(nyxb_details) * m, cudaMemcpyDeviceToHost, st));
        TRY4(cudaMemcpyAsync(out_status + lo, eng->d_status, sizeof(int) * m, cudaMemcpyDeviceToHost, st));
    }
    for (size_t g = 0; g < G; ++g) {
        nyxb_engine* eng = engines[g];
        if (lo_of(g + 1) == lo_of(g)) continue;
        TRY4(cudaSetDevice(eng->device));
        TRY4(cudaStreamSynchronize(eng->stream));
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, eng->ev0, eng->ev1) == cudaSuccess) eng->last_ms = ms;
    }
    return NYXB_RC_OK;
#undef TRY4
}

// ---------------------------------------------------------------------------------------------------------------------
// (f)-2: STM propagation and the batched sequential filter (kernels in nyxb_od.cu).  Host-pointer entry points with
// per-call device buffers (these calls run for seconds; allocation cost is irrelevant).
// ---------------------------------------------------------------------------------------------------------------------
namespace {
// The device buffers of one call.  A failed allocation or upload sets `failed`; the call checks it before its launch.
struct DevBufs {
    std::vector<void*> p;
    bool failed = false;
    ~DevBufs() { for (void* q : p) cudaFree(q); }
    template <typename T> T* alloc(size_t count) {
        T* d = nullptr;
        if (cudaMalloc(&d, sizeof(T) * (count ? count : 1)) != cudaSuccess) { failed = true; return nullptr; }
        p.push_back(d);
        return d;
    }
    template <typename T> T* put(const T* host, size_t count, cudaStream_t st) {
        T* d = alloc<T>(count);
        if (d && count && cudaMemcpyAsync(d, host, sizeof(T) * count, cudaMemcpyHostToDevice, st) != cudaSuccess) { failed = true; return nullptr; }
        return d;
    }
    int32_t check(const char* what = "device allocation / upload failed") const {
        if (!failed) return NYXB_RC_OK;
        set_err(what);
        return NYXB_RC_CUDA;
    }
};
// copies count entries of dev back to host, unless host is null
template <typename H, typename D>
cudaError_t get(H* host, const D* dev, size_t count, cudaStream_t st) {
    static_assert(sizeof(H) == sizeof(D), "host and device entries differ");
    return host ? cudaMemcpyAsync(host, dev, sizeof(D) * count, cudaMemcpyDeviceToHost, st) : cudaSuccess;
}

// uploads the per-filter inputs and allocates the per-filter outputs every OD kernel has
OdIo od_io(DevBufs& B, cudaStream_t st, size_t n, const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns) {
    return OdIo{B.put(state_soa, 9 * n, st), B.put(consts_soa, 4 * n, st), B.put((const long long*)epoch0_ns, n, st), B.alloc<double>(9 * n),
                B.alloc<long long>(n), B.alloc<nyxb_details>(n), B.alloc<int>(n)};
}
int32_t od_io_get(const OdIo& io, size_t n, cudaStream_t st, double* out_state, int64_t* out_epoch, nyxb_details* out_details, int32_t* out_status) {
    CUDA_TRY(get(out_state, io.out_state, 9 * n, st));
    CUDA_TRY(get(out_epoch, io.out_epoch, n, st));
    CUDA_TRY(get(out_details, io.out_details, n, st));
    CUDA_TRY(get(out_status, io.out_status, n, st));
    return NYXB_RC_OK;
}

// The start and finish of every call below: od_stream selects the engine's device and stream; timed_launch runs one launch between
// the events ev0 and ev1 and counts it; od_finish waits for the copies back and keeps the kernel time.
int32_t od_stream(nyxb_engine* eng, cudaStream_t& st) {
    CUDA_TRY(cudaSetDevice(eng->device));
    if (!eng->stream) CUDA_TRY(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
    st = eng->stream;
    return NYXB_RC_OK;
}
template <class F>
int32_t timed_launch(nyxb_engine* eng, int family, F launch) {
    CUDA_TRY(cudaEventRecord(eng->ev0, eng->stream));
    cudaError_t err = launch();
    if (err != cudaSuccess) { set_err(std::string("kernel launch: ") + cudaGetErrorString(err)); return NYXB_RC_CUDA; }
    eng->launches += 1;
    eng->last_kernel = family;
    CUDA_TRY(cudaEventRecord(eng->ev1, eng->stream));
    return NYXB_RC_OK;
}
int32_t od_finish(nyxb_engine* eng) {
    CUDA_TRY(cudaStreamSynchronize(eng->stream));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, eng->ev0, eng->ev1) == cudaSuccess) eng->last_ms = ms;
    return NYXB_RC_OK;
}

bool stm_supported(const nyxb_engine* e) {
    if (e->S.grav_body >= 0 || e->S.n_xgrav > 0 || e->S.state_center >= 0) {
        set_err("the STM / filter kernels take one harmonic field, of the integration centre, and states in the integration frame");
        return false;
    }
    if (e->S.has_drag) { set_err("PartialsUndefined: the drag model has no partials (drag.rs:109-118, 286-295)"); return false; }
    if (!e->S.fixed_step && e->S.error_ctrl != NYXB_RSS_CARTESIAN_STATE && e->S.error_ctrl != NYXB_RSS_CARTESIAN_STEP) {
        set_err("STM propagation accepts the Cartesian error controls or a fixed step");
        return false;
    }
    return true;
}

// The column deal of the warp kernels (nyxb_od_coop.cu), used in FAST mode with a gravity field of degree >= 8: one WARP per filter,
// the harmonic gradient split by columns over the lanes, columns -> lanes by longest-processing-time.  Empty for the per-thread kernel:
// nyxb_engine_set_kernel(NYXB_KERNEL_THREAD) forces it, and so does a deal that needs more than ODC_KMAX columns on one lane.
std::vector<int> coop_cols(const nyxb_engine* eng) {
    bool coop = eng->mode == NYXB_MODE_FAST && eng->S.has_grav && eng->S.grav.N >= 8 && eng->kernel != NYXB_KERNEL_THREAD;
    if (!coop) return {};
    const int N = eng->S.grav.N, mtop = eng->S.grav.M < N ? eng->S.grav.M : N;
    std::vector<int> cols(32 * (size_t)ODC_KMAX, -1), cnt(32, 0);
    std::vector<long long> load(32, 0);
    for (int m = 0; m <= mtop; ++m) {   // columns in decreasing length order: m = 0, 1 (same length), 2, ...
        int best = 0;
        for (int l = 1; l < 32; ++l)
            if (load[l] < load[best] || (load[l] == load[best] && cnt[l] < cnt[best])) best = l;
        if (cnt[best] >= ODC_KMAX) return {};
        cols[(size_t)best * ODC_KMAX + cnt[best]++] = m;
        load[best] += N - (m > 0 ? m : 1) + 1 + 6;   // entries + per-column overhead
    }
    return cols;
}

template <class Job>
cudaError_t thread_launch(const nyxb_engine* eng, const Job& job, size_t n, const OdIo& io) {
    return eng->mode == NYXB_MODE_STRICT ? nyxb_od_strict::launch(eng->S, job, n, io, eng->stream)
                                         : nyxb_od_fast::launch(eng->S, job, n, io, eng->stream);
}

// One timed launch of an OD job in the engine's kernel family: warp-cooperative when coop_cols deals the columns (uploaded into B),
// else per-thread STRICT or FAST.
template <class Job>
int32_t od_launch(nyxb_engine* eng, const Job& job, DevBufs& B, size_t n, const OdIo& io) {
    const std::vector<int> cols = coop_cols(eng);
    if (cols.empty()) return timed_launch(eng, NYXB_KERNEL_THREAD, [&] { return thread_launch(eng, job, n, io); });
    const int* d_cols = B.put(cols.data(), cols.size(), eng->stream);
    if (int32_t rc = B.check()) return rc;
    return timed_launch(eng, NYXB_KERNEL_COOP, [&] { return nyxb_od_coop_launch(eng->S, job, d_cols, n, io, eng->stream); });
}
}  // namespace

extern "C" int32_t nyxb_propagate_batch_stm(nyxb_engine* eng, size_t n, const double* state_soa, const double* consts_soa,
                                            const int64_t* epoch0_ns, int64_t end_epoch_ns, int64_t* step_ns,
                                            const double* stm_in_soa, double* out_state_soa, int64_t* out_epoch_ns,
                                            double* out_stm_soa, nyxb_details* out_details, int32_t* out_status) {
    if (!eng || !state_soa || !consts_soa || !epoch0_ns || !out_state_soa || !out_epoch_ns || !out_stm_soa || !out_status) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (!stm_supported(eng)) return NYXB_RC_UNSUPPORTED;
    if (n == 0) return NYXB_RC_OK;
    cudaStream_t st;
    if (int32_t rc = od_stream(eng, st)) return rc;
    DevBufs B;
    const OdIo io = od_io(B, st, n, state_soa, consts_soa, epoch0_ns);
    OdStmJob job{end_epoch_ns, step_ns ? B.put((const long long*)step_ns, n, st) : nullptr, stm_in_soa ? B.put(stm_in_soa, 81 * n, st) : nullptr,
                 B.alloc<double>(81 * n)};
    if (int32_t rc = B.check()) return rc;
    if (int32_t rc = timed_launch(eng, NYXB_KERNEL_THREAD, [&] { return thread_launch(eng, job, n, io); })) return rc;
    if (int32_t rc = od_io_get(io, n, st, out_state_soa, out_epoch_ns, out_details, out_status)) return rc;
    CUDA_TRY(get(out_stm_soa, job.out_stm, 81 * n, st));
    CUDA_TRY(get(step_ns, job.step_io, n, st));
    return od_finish(eng);
}

namespace {
bool station_ok(const nyxb_engine* eng, const nyxb_ground_station& g) {
    if (g.n_types < 1 || g.n_types > 2 || (g.body != NYXB_CENTRAL_BODY && (g.body < 0 || g.body >= eng->S.n_bodies))) {
        set_err("bad ground station descriptor");
        return false;
    }
    return true;
}
DevStation pack_station(const nyxb_ground_station& g) {
    DevStation d{};
    for (int q = 0; q < 3; ++q) { d.pos[q] = g.pos_fixed_km[q]; d.up[q] = g.up_fixed[q]; }
    d.mask_deg = g.elevation_mask_deg; d.rot = pack_rot(g.rot); d.body = g.body; d.n_types = g.n_types;
    for (int q = 0; q < 2; ++q) { d.types[q] = g.types[q]; d.noise_var[q] = g.noise_var[q]; d.bias[q] = g.bias[q]; }
    d.body_radius = g.body_radius_km;
    return d;
}
// the checks and packing of a list of stations with angles (nyxb_od_aer_batch / _smooth_batch)
int32_t pack_aer_stations(const nyxb_engine* eng, int32_t n_stations, const nyxb_aer_station* stations, std::vector<DevAerStation>& hs) {
    hs.assign((size_t)(n_stations > 0 ? n_stations : 0), DevAerStation{});
    for (int32_t s = 0; s < n_stations; ++s) {
        const nyxb_aer_station& g = stations[s];
        if (g.n_types < 1 || g.n_types > 4) { set_err("bad station: n_types must be 1 to 4"); return NYXB_RC_BAD_ARG; }
        if (g.body != NYXB_CENTRAL_BODY && (g.body < 0 || g.body >= eng->S.n_bodies)) { set_err("bad ground station descriptor"); return NYXB_RC_BAD_ARG; }
        for (int q = 0; q < g.n_types; ++q) {
            if (g.types[q] < NYXB_MSR_RANGE || g.types[q] > NYXB_MSR_ELEVATION) {
                set_err("bad station: measurement types must be Range, Doppler, Azimuth or Elevation");
                return NYXB_RC_BAD_ARG;
            }
            for (int p = 0; p < q; ++p)
                if (g.types[p] == g.types[q]) { set_err("bad station: duplicate measurement type"); return NYXB_RC_BAD_ARG; }
        }
        DevAerStation& d = hs[s];
        for (int q = 0; q < 3; ++q) { d.pos[q] = g.pos_fixed_km[q]; d.up[q] = g.up_fixed[q]; d.north[q] = g.north_fixed[q]; d.east[q] = g.east_fixed[q]; }
        d.mask_deg = g.elevation_mask_deg; d.rot = pack_rot(g.rot); d.body = g.body; d.n_types = g.n_types;
        for (int q = 0; q < 4; ++q) { d.types[q] = g.types[q]; d.noise_var[q] = g.noise_var[q]; d.bias[q] = g.bias[q]; }
        d.body_radius = g.body_radius_km;
    }
    return NYXB_RC_OK;
}
// the checks and packing of a position device list (nyxb_od_position_batch / _smooth_batch)
int32_t pack_position_devices(int32_t n_devices, const nyxb_position_device* devices, std::vector<DevPosDevice>& hs) {
    hs.assign((size_t)(n_devices > 0 ? n_devices : 0), DevPosDevice{});
    for (int32_t s = 0; s < n_devices; ++s) {
        const nyxb_position_device& g = devices[s];
        if (g.n_types < 1 || g.n_types > 3) { set_err("bad position device: n_types must be 1 to 3"); return NYXB_RC_BAD_ARG; }
        DevPosDevice& d = hs[s];
        d.n_types = g.n_types;
        for (int q = 0; q < 3; ++q) { d.types[q] = g.types[q]; d.noise_var[q] = g.noise_var[q]; d.bias[q] = g.bias[q]; }
        for (int q = 0; q < g.n_types; ++q) {
            if (g.types[q] != NYXB_MSR_X && g.types[q] != NYXB_MSR_Y && g.types[q] != NYXB_MSR_Z) {
                set_err("bad position device: measurement types must be X, Y or Z");
                return NYXB_RC_BAD_ARG;
            }
            for (int p = 0; p < q; ++p)
                if (g.types[p] == g.types[q]) { set_err("bad position device: duplicate measurement type"); return NYXB_RC_BAD_ARG; }
        }
    }
    return NYXB_RC_OK;
}
bool records_ok(const nyxb_od_records* rec) {
    if (rec->capacity < 0 || !rec->count ||
        (rec->capacity > 0 && (!rec->epoch_ns || !rec->tag || !rec->nominal || !rec->deviation || !rec->covar || !rec->stm))) {
        set_err("bad estimate records: count is required, and every record array when capacity > 0");
        return false;
    }
    return true;
}

// The argument checks the ground-station (Dev = DevStation or DevAerStation) and position-fix filter calls share, in this order.  The
// ground-station calls check the engine's setup after the records; nyxb_od_position_batch checks it after its devices.
template <class Dev, class Arc, class Trk>
int32_t filter_args(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_dev, const Trk* devs, const Arc* arc, const double* state_soa,
                    const double* consts_soa, const int64_t* epoch0_ns, const double* covar0_soa, const nyxb_od_outputs* out,
                    const nyxb_od_records* rec) {
    constexpr bool ground = !std::is_same<Dev, DevPosDevice>::value;
    if (!eng || !cfg || !arc || !state_soa || !consts_soa || !epoch0_ns || !covar0_soa || !out || !out->state_soa || !out->epoch_ns ||
        !out->covar_soa || !out->status || (n_dev > 0 && !devs) || n_dev < 0) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (rec && !records_ok(rec)) return NYXB_RC_BAD_ARG;
    if (ground && !stm_supported(eng)) return NYXB_RC_UNSUPPORTED;
    if (cfg->msr_size < 1 || cfg->msr_size > (ground ? 2 : 3)) { set_err(ground ? "msr_size must be 1 or 2" : "msr_size must be 1, 2 or 3"); return NYXB_RC_BAD_ARG; }
    if (cfg->variant != NYXB_KF_REFERENCE_UPDATE && cfg->variant != NYXB_KF_DEVIATION_TRACKING) { set_err("bad filter variant"); return NYXB_RC_BAD_ARG; }
    if (cfg->max_step_ns <= 0) { set_err("StepSize: max_step must be positive (process/mod.rs:147-150)"); return NYXB_RC_BAD_ARG; }
    if (arc->n_msr < 2) { set_err("TooFewMeasurements: need 2 (process/mod.rs:139-145)"); return NYXB_RC_BAD_ARG; }
    if (!arc->epoch_ns || !arc->tracker || !arc->obs) { set_err("null tracking arc arrays"); return NYXB_RC_BAD_ARG; }
    return NYXB_RC_OK;
}

// The common part of the ground-station and position-fix filter calls: upload, one launch, read-back.  hs: the packed devices;
// rec: null, or the estimate records.
template <class Dev>
int32_t od_filter_run(nyxb_engine* eng, const nyxb_od_config* cfg, const std::vector<Dev>& hs, int64_t n_msr, const int64_t* arc_epoch,
                      const int32_t* arc_tracker, const double* arc_obs, size_t n, const double* state_soa, const double* consts_soa,
                      const int64_t* epoch0_ns, const double* covar0_soa, const nyxb_od_outputs* out, const nyxb_od_records* rec) {
    constexpr int NS = Dev::NS;
    cudaStream_t st;
    if (int32_t rc = od_stream(eng, st)) return rc;
    const size_t m = (size_t)n_msr;
    DevBufs B;
    DevOdT<Dev> od{};
    od.variant = cfg->variant; od.msr_size = cfg->msr_size; od.reject = cfg->reject_num_sigmas;
    od.max_step_ns = cfg->max_step_ns; od.eps_ns = cfg->epoch_precision_ns;
    od.snc_enabled = cfg->snc_enabled; od.snc_frame = cfg->snc_frame;
    for (int q = 0; q < 3; ++q) od.snc_diag[q] = cfg->snc_diag[q];
    od.snc_disable_ns = cfg->snc_disable_time_ns;
    od.n_stations = (int32_t)hs.size();
    od.stations = B.put(hs.data(), hs.size(), st);
    od.n_msr = n_msr;
    od.msr_epoch = B.put((const long long*)arc_epoch, m, st);
    od.msr_tracker = B.put((const int*)arc_tracker, m, st);
    od.obs = B.put(arc_obs, m * NS * n, st);
    od.covar0 = B.put(covar0_soa, 81 * n, st);
    const OdIo io = od_io(B, st, n, state_soa, consts_soa, epoch0_ns);
    od.covar = B.alloc<double>(81 * n);
    od.state_dev = out->state_dev_soa ? B.alloc<double>(9 * n) : nullptr;
    od.ratio = out->resid_ratio ? B.alloc<double>(m * NS * n) : nullptr;
    od.prefit = out->prefit ? B.alloc<double>(m * NS * n) : nullptr;
    od.postfit = out->postfit ? B.alloc<double>(m * NS * n) : nullptr;
    od.flags = out->msr_flags ? B.alloc<int>(m * n) : nullptr;
    od.est_state = out->est_state ? B.alloc<double>(m * 9 * n) : nullptr;
    od.est_cov = out->est_covar_diag ? B.alloc<double>(m * 9 * n) : nullptr;
    if (int32_t rc = B.check()) return rc;
    OdEstRecords er{};
    const size_t rcap = rec ? (size_t)rec->capacity : 0;
    if (rec) {
        er.cap = (long long)rcap;
        er.count = B.alloc<long long>(n);
        if (rcap) {
            er.epoch = B.alloc<long long>(rcap * n);
            er.tag = B.alloc<long long>(rcap * n);
            er.nominal = B.alloc<double>(rcap * 9 * n);
            er.dev = B.alloc<double>(rcap * 9 * n);
            er.covar = B.alloc<double>(rcap * 81 * n);
            er.stm = B.alloc<double>(rcap * 81 * n);
        }
        if (int32_t rc = B.check("device allocation failed (estimate records)")) return rc;
    }
    // per-measurement records default to NaN (0xFF bytes) / 0 flags where nothing is written
    if (od.ratio) CUDA_TRY(cudaMemsetAsync(od.ratio, 0xFF, sizeof(double) * m * NS * n, st));
    if (od.prefit) CUDA_TRY(cudaMemsetAsync(od.prefit, 0xFF, sizeof(double) * m * NS * n, st));
    if (od.postfit) CUDA_TRY(cudaMemsetAsync(od.postfit, 0xFF, sizeof(double) * m * NS * n, st));
    if (od.flags) CUDA_TRY(cudaMemsetAsync(od.flags, 0, sizeof(int) * m * n, st));
    if (od.est_state) CUDA_TRY(cudaMemsetAsync(od.est_state, 0xFF, sizeof(double) * m * 9 * n, st));
    if (od.est_cov) CUDA_TRY(cudaMemsetAsync(od.est_cov, 0xFF, sizeof(double) * m * 9 * n, st));
    if (rec) CUDA_TRY(cudaMemsetAsync(er.count, 0, sizeof(long long) * n, st));
    if (rcap) {                                  // records a filter does not reach: -1 / NaN
        CUDA_TRY(cudaMemsetAsync(er.epoch, 0xFF, sizeof(long long) * rcap * n, st));
        CUDA_TRY(cudaMemsetAsync(er.tag, 0xFF, sizeof(long long) * rcap * n, st));
        CUDA_TRY(cudaMemsetAsync(er.nominal, 0xFF, sizeof(double) * rcap * 9 * n, st));
        CUDA_TRY(cudaMemsetAsync(er.dev, 0xFF, sizeof(double) * rcap * 9 * n, st));
        CUDA_TRY(cudaMemsetAsync(er.covar, 0xFF, sizeof(double) * rcap * 81 * n, st));
        CUDA_TRY(cudaMemsetAsync(er.stm, 0xFF, sizeof(double) * rcap * 81 * n, st));
    }
    if (int32_t rc = rec ? od_launch(eng, OdFilterJob<Dev, true>{od, er}, B, n, io) : od_launch(eng, OdFilterJob<Dev, false>{od}, B, n, io))
        return rc;
    if (int32_t rc = od_io_get(io, n, st, out->state_soa, out->epoch_ns, out->details, out->status)) return rc;
    CUDA_TRY(get(out->covar_soa, od.covar, 81 * n, st));
    CUDA_TRY(get(out->state_dev_soa, od.state_dev, 9 * n, st));
    CUDA_TRY(get(out->resid_ratio, od.ratio, m * NS * n, st));
    CUDA_TRY(get(out->prefit, od.prefit, m * NS * n, st));
    CUDA_TRY(get(out->postfit, od.postfit, m * NS * n, st));
    CUDA_TRY(get(out->msr_flags, od.flags, m * n, st));
    CUDA_TRY(get(out->est_state, od.est_state, m * 9 * n, st));
    CUDA_TRY(get(out->est_covar_diag, od.est_cov, m * 9 * n, st));
    if (rec) CUDA_TRY(get(rec->count, er.count, n, st));
    if (rcap) {
        CUDA_TRY(get(rec->epoch_ns, er.epoch, rcap * n, st));
        CUDA_TRY(get(rec->tag, er.tag, rcap * n, st));
        CUDA_TRY(get(rec->nominal, er.nominal, rcap * 9 * n, st));
        CUDA_TRY(get(rec->deviation, er.dev, rcap * 9 * n, st));
        CUDA_TRY(get(rec->covar, er.covar, rcap * 81 * n, st));
        CUDA_TRY(get(rec->stm, er.stm, rcap * 81 * n, st));
    }
    return od_finish(eng);
}

// nyxb_od_ekf_batch and nyxb_od_ekf_record_batch: argument checks, packing, one launch, read-back.  rec: null, or the estimate records.
int32_t od_ekf_run(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations, const nyxb_ground_station* stations,
                   const nyxb_tracking_arc* arc, size_t n, const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                   const double* covar0_soa, const nyxb_od_outputs* out, const nyxb_od_records* rec) {
    if (int32_t rc = filter_args<DevStation>(eng, cfg, n_stations, stations, arc, state_soa, consts_soa, epoch0_ns, covar0_soa, out, rec))
        return rc;
    std::vector<DevStation> hs;
    for (int32_t s = 0; s < n_stations; ++s) {
        const nyxb_ground_station& g = stations[s];
        if (!station_ok(eng, g)) return NYXB_RC_BAD_ARG;
        for (int q = 0; q < g.n_types; ++q)
            if (g.types[q] != NYXB_MSR_RANGE && g.types[q] != NYXB_MSR_DOPPLER) { set_err("unsupported measurement type"); return NYXB_RC_UNSUPPORTED; }
        if (g.n_types % cfg->msr_size != 0) { set_err("filter misconfigured: measurement types per device must be a multiple of msr_size"); return NYXB_RC_UNSUPPORTED; }
        hs.push_back(pack_station(g));
    }
    if (n == 0) return NYXB_RC_OK;
    return od_filter_run(eng, cfg, hs, arc->n_msr, arc->epoch_ns, arc->tracker, arc->obs, n, state_soa, consts_soa, epoch0_ns, covar0_soa,
                         out, rec);
}
}  // namespace

extern "C" int32_t nyxb_od_ekf_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations,
                                     const nyxb_ground_station* stations, const nyxb_tracking_arc* arc, size_t n,
                                     const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                                     const double* covar0_soa, const nyxb_od_outputs* out) {
    return od_ekf_run(eng, cfg, n_stations, stations, arc, n, state_soa, consts_soa, epoch0_ns, covar0_soa, out, nullptr);
}

extern "C" int32_t nyxb_od_ekf_record_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations,
                                            const nyxb_ground_station* stations, const nyxb_tracking_arc* arc, size_t n,
                                            const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                                            const double* covar0_soa, const nyxb_od_outputs* out, const nyxb_od_records* rec) {
    if (!rec) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    return od_ekf_run(eng, cfg, n_stations, stations, arc, n, state_soa, consts_soa, epoch0_ns, covar0_soa, out, rec);
}

namespace {
// The record tags and windows of each tracker kind (NYXB_OD_TAG_*, NYXB_OD_POS_TAG_*, include/nyxb.h).  A ground station's window must
// lie within its types; the window of a position device or of a station with angles need only start within them.
struct GroundTags {
    static int64_t msr(int64_t tg) { return NYXB_OD_TAG_MSR(tg); }
    static int window(int64_t tg) { return (int)NYXB_OD_TAG_WINDOW(tg); }
    static int64_t msr_size(int64_t tg) { return NYXB_OD_TAG_MSR_SIZE(tg); }
    static bool outside(int w, int M, int n_types) { return (w + 1) * M > n_types; }
};
struct PosTags {
    static int64_t msr(int64_t tg) { return NYXB_OD_POS_TAG_MSR(tg); }
    static int window(int64_t tg) { return (int)NYXB_OD_POS_TAG_WINDOW(tg); }
    static int64_t msr_size(int64_t tg) { return NYXB_OD_POS_TAG_MSR_SIZE(tg); }
    static bool outside(int w, int M, int n_types) { return w * M >= n_types; }
};
// interlink records: the ground station's tags, with a short last window as a station with angles
struct LinkTags : GroundTags {
    static bool outside(int w, int M, int n_types) { return PosTags::outside(w, M, n_types); }
};

// The common part of the two smoothing calls: the per-filter statuses decided on the host, then upload, the smoothing launch and
// read-back.  The records of the filters left to smooth must belong to this arc and msr_size.  hs: the packed devices.
// win_err: the status of a window that cannot be formed (the even err_key of nyxb_k_smooth).
template <class Tags, class Dev>
int32_t od_smooth_run(nyxb_engine* eng, int M, const std::vector<Dev>& hs, int64_t n_msr, const int32_t* arc_tracker, const double* arc_obs,
                      size_t n, const nyxb_od_records* rec, const int32_t* filter_status, nyxb_smooth_outputs* out,
                      int32_t win_err = NYXB_ERR_EPHEMERIS) {
    constexpr int NS = Dev::NS;
    const size_t m = (size_t)n_msr, cap = (size_t)rec->capacity;
    const int32_t n_stations = (int32_t)hs.size();
    std::vector<int> pre(n);
    for (size_t i = 0; i < n; ++i) {
        const long long cnt = rec->count[i];
        pre[i] = filter_status[i] ? filter_status[i]
               : (cnt > (long long)cap) ? NYXB_ERR_RECORDS_TRUNCATED
               : (cnt < 2) ? NYXB_ERR_TOO_FEW_MEASUREMENTS : 0;
        if (pre[i]) continue;
        for (long long k = 0; k < cnt; ++k) {
            const int64_t tg = rec->tag[(size_t)k * n + i];
            if (tg == NYXB_OD_TAG_TIME_UPDATE) continue;
            const int64_t mk = Tags::msr(tg);
            const int w = Tags::window(tg);
            if (tg < 0 || Tags::msr_size(tg) != M) { set_err("estimate records written with another msr_size"); return NYXB_RC_BAD_ARG; }
            if (mk >= n_msr || arc_tracker[mk] < 0 || arc_tracker[mk] >= n_stations || Tags::outside(w, M, hs[arc_tracker[mk]].n_types)) {
                set_err("estimate records do not match this tracking arc");
                return NYXB_RC_BAD_ARG;
            }
        }
    }
    for (size_t i = 0; i < n; ++i) out->status[i] = pre[i];
    if (n == 0 || cap == 0) return NYXB_RC_OK;
    cudaStream_t st;
    if (int32_t rc = od_stream(eng, st)) return rc;
    DevBufs B;
    DevSmoothT<Dev> sm{};
    sm.msr_size = M;
    sm.n_stations = n_stations;
    sm.stations = n_stations ? B.put(hs.data(), hs.size(), st) : nullptr;
    sm.msr_tracker = m ? B.put((const int*)arc_tracker, m, st) : nullptr;
    sm.obs = m ? B.put(arc_obs, m * NS * n, st) : nullptr;
    sm.cap = (long long)cap;
    sm.epoch = B.put((const long long*)rec->epoch_ns, cap * n, st);
    sm.tag = B.put((const long long*)rec->tag, cap * n, st);
    sm.nominal = B.put(rec->nominal, cap * 9 * n, st);
    sm.dev = B.put(rec->deviation, cap * 9 * n, st);
    sm.covar = B.put(rec->covar, cap * 81 * n, st);
    sm.stm = B.put(rec->stm, cap * 81 * n, st);
    sm.count = B.put((const long long*)rec->count, n, st);
    sm.pre_status = B.put(pre.data(), n, st);
    sm.state = out->state ? B.alloc<double>(cap * 9 * n) : nullptr;
    sm.sdev = out->deviation ? B.alloc<double>(cap * 9 * n) : nullptr;
    sm.scov = out->covar ? B.alloc<double>(cap * 81 * n) : nullptr;
    sm.ratio = out->fs_ratio ? B.alloc<double>(cap * 9 * n) : nullptr;
    sm.postfit = out->postfit ? B.alloc<double>(cap * NS * n) : nullptr;
    sm.err_key = B.alloc<long long>(n);
    if (int32_t rc = B.check()) return rc;
    if (sm.state) CUDA_TRY(cudaMemsetAsync(sm.state, 0xFF, sizeof(double) * cap * 9 * n, st));
    if (sm.sdev) CUDA_TRY(cudaMemsetAsync(sm.sdev, 0xFF, sizeof(double) * cap * 9 * n, st));
    if (sm.scov) CUDA_TRY(cudaMemsetAsync(sm.scov, 0xFF, sizeof(double) * cap * 81 * n, st));
    if (sm.ratio) CUDA_TRY(cudaMemsetAsync(sm.ratio, 0xFF, sizeof(double) * cap * 9 * n, st));
    if (sm.postfit) CUDA_TRY(cudaMemsetAsync(sm.postfit, 0xFF, sizeof(double) * cap * NS * n, st));
    CUDA_TRY(cudaMemsetAsync(sm.err_key, 0xFF, sizeof(long long) * n, st));
    if (int32_t rc = timed_launch(eng, NYXB_KERNEL_THREAD, [&] { return nyxb_smooth_launch(eng->S, sm, n, st); })) return rc;
    std::vector<long long> key(n);
    CUDA_TRY(get(key.data(), sm.err_key, n, st));
    CUDA_TRY(get(out->state, sm.state, cap * 9 * n, st));
    CUDA_TRY(get(out->deviation, sm.sdev, cap * 9 * n, st));
    CUDA_TRY(get(out->covar, sm.scov, cap * 81 * n, st));
    CUDA_TRY(get(out->fs_ratio, sm.ratio, cap * 9 * n, st));
    CUDA_TRY(get(out->postfit, sm.postfit, cap * NS * n, st));
    if (int32_t rc = od_finish(eng)) return rc;
    // the reference's error is the first one met going backwards from the last estimate: the largest k (singular before measure);
    // the outputs of such a filter were set to NaN on the device
    for (size_t i = 0; i < n; ++i)
        if (key[i] >= 0) out->status[i] = (key[i] & 1) ? NYXB_ERR_SINGULAR_STM : win_err;
    return NYXB_RC_OK;
}
}  // namespace

extern "C" int32_t nyxb_od_smooth_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations, const nyxb_ground_station* stations,
                                        const nyxb_tracking_arc* arc, size_t n, const nyxb_od_records* rec, const int32_t* filter_status,
                                        nyxb_smooth_outputs* out) {
    if (!eng || !cfg || !arc || !rec || !filter_status || !out || !out->status || (n_stations > 0 && !stations) || n_stations < 0) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (cfg->msr_size != 1 && cfg->msr_size != 2) { set_err("msr_size must be 1 or 2"); return NYXB_RC_BAD_ARG; }
    if (!records_ok(rec)) return NYXB_RC_BAD_ARG;
    if (arc->n_msr < 0 || (arc->n_msr > 0 && (!arc->tracker || !arc->obs))) { set_err("null tracking arc arrays"); return NYXB_RC_BAD_ARG; }
    std::vector<DevStation> hs;
    for (int32_t s = 0; s < n_stations; ++s) {
        if (!station_ok(eng, stations[s])) return NYXB_RC_BAD_ARG;
        hs.push_back(pack_station(stations[s]));
    }
    return od_smooth_run<GroundTags>(eng, cfg->msr_size, hs, arc->n_msr, arc->tracker, arc->obs, n, rec, filter_status, out);
}

extern "C" int32_t nyxb_od_position_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_devices, const nyxb_position_device* devices,
                                          const nyxb_position_arc* arc, size_t n, const double* state_soa, const double* consts_soa,
                                          const int64_t* epoch0_ns, const double* covar0_soa, const nyxb_od_outputs* out,
                                          const nyxb_od_records* rec) {
    if (int32_t rc = filter_args<DevPosDevice>(eng, cfg, n_devices, devices, arc, state_soa, consts_soa, epoch0_ns, covar0_soa, out, rec))
        return rc;
    std::vector<DevPosDevice> hs;
    if (int32_t rc = pack_position_devices(n_devices, devices, hs)) return rc;
    if (!stm_supported(eng)) return NYXB_RC_UNSUPPORTED;
    if (n == 0) return NYXB_RC_OK;
    return od_filter_run(eng, cfg, hs, arc->n_msr, arc->epoch_ns, arc->tracker, arc->obs, n, state_soa, consts_soa, epoch0_ns, covar0_soa,
                         out, rec);
}

extern "C" int32_t nyxb_od_position_smooth_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_devices,
                                                 const nyxb_position_device* devices, const nyxb_position_arc* arc, size_t n,
                                                 const nyxb_od_records* rec, const int32_t* filter_status, nyxb_smooth_outputs* out) {
    if (!eng || !cfg || !arc || !rec || !filter_status || !out || !out->status || (n_devices > 0 && !devices) || n_devices < 0) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (cfg->msr_size < 1 || cfg->msr_size > 3) { set_err("msr_size must be 1, 2 or 3"); return NYXB_RC_BAD_ARG; }
    if (!records_ok(rec)) return NYXB_RC_BAD_ARG;
    if (arc->n_msr < 0 || (arc->n_msr > 0 && (!arc->tracker || !arc->obs))) { set_err("null tracking arc arrays"); return NYXB_RC_BAD_ARG; }
    std::vector<DevPosDevice> hs;
    if (int32_t rc = pack_position_devices(n_devices, devices, hs)) return rc;
    return od_smooth_run<PosTags>(eng, cfg->msr_size, hs, arc->n_msr, arc->tracker, arc->obs, n, rec, filter_status, out);
}

extern "C" int32_t nyxb_od_aer_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations, const nyxb_aer_station* stations,
                                     const nyxb_tracking_arc* arc, size_t n, const double* state_soa, const double* consts_soa,
                                     const int64_t* epoch0_ns, const double* covar0_soa, const nyxb_od_outputs* out, const nyxb_od_records* rec) {
    if (int32_t rc = filter_args<DevAerStation>(eng, cfg, n_stations, stations, arc, state_soa, consts_soa, epoch0_ns, covar0_soa, out, rec))
        return rc;
    std::vector<DevAerStation> hs;
    if (int32_t rc = pack_aer_stations(eng, n_stations, stations, hs)) return rc;
    if (n == 0) return NYXB_RC_OK;
    return od_filter_run(eng, cfg, hs, arc->n_msr, arc->epoch_ns, arc->tracker, arc->obs, n, state_soa, consts_soa, epoch0_ns, covar0_soa,
                         out, rec);
}

extern "C" int32_t nyxb_od_aer_smooth_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_stations, const nyxb_aer_station* stations,
                                            const nyxb_tracking_arc* arc, size_t n, const nyxb_od_records* rec, const int32_t* filter_status,
                                            nyxb_smooth_outputs* out) {
    if (!eng || !cfg || !arc || !rec || !filter_status || !out || !out->status || (n_stations > 0 && !stations) || n_stations < 0) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (cfg->msr_size != 1 && cfg->msr_size != 2) { set_err("msr_size must be 1 or 2"); return NYXB_RC_BAD_ARG; }
    if (!records_ok(rec)) return NYXB_RC_BAD_ARG;
    if (arc->n_msr < 0 || (arc->n_msr > 0 && (!arc->tracker || !arc->obs))) { set_err("null tracking arc arrays"); return NYXB_RC_BAD_ARG; }
    std::vector<DevAerStation> hs;
    if (int32_t rc = pack_aer_stations(eng, n_stations, stations, hs)) return rc;
    return od_smooth_run<PosTags>(eng, cfg->msr_size, hs, arc->n_msr, arc->tracker, arc->obs, n, rec, filter_status, out);
}

namespace {
// The checks and packing of interlink transmitters and of their recordings (nyxb_od_interlink_batch / _smooth_batch): every column of
// the sink holds 1 to capacity records, every device names a column and one or two distinct types of Range and Doppler.
int32_t pack_links(int32_t n_devices, const nyxb_interlink_tx* devices, size_t n_tx, const nyxb_traj_sink* sink, std::vector<DevLink>& hs) {
    if (!sink || sink->capacity < 0 || (n_tx > 0 && (!sink->epoch_ns || !sink->state || !sink->count))) {
        set_err("null argument: the transmitter recordings");
        return NYXB_RC_BAD_ARG;
    }
    for (size_t j = 0; j < n_tx; ++j)
        if (sink->count[j] < 1 || sink->count[j] > sink->capacity) {
            set_err("bad transmitter recording: count must be 1 to capacity (a recording that dropped records is incomplete)");
            return NYXB_RC_BAD_ARG;
        }
    hs.assign((size_t)(n_devices > 0 ? n_devices : 0), DevLink{});
    for (int32_t s = 0; s < n_devices; ++s) {
        const nyxb_interlink_tx& g = devices[s];
        if (g.n_types < 1 || g.n_types > 2) { set_err("bad interlink device: n_types must be 1 or 2"); return NYXB_RC_BAD_ARG; }
        if (g.tx < 0 || (size_t)g.tx >= n_tx) { set_err("bad interlink device: transmitter column outside the recordings"); return NYXB_RC_BAD_ARG; }
        for (int q = 0; q < g.n_types; ++q) {
            if (g.types[q] != NYXB_MSR_RANGE && g.types[q] != NYXB_MSR_DOPPLER) {
                set_err("bad interlink device: measurement types must be Range or Doppler");
                return NYXB_RC_BAD_ARG;
            }
            if (q == 1 && g.types[0] == g.types[1]) { set_err("bad interlink device: duplicate measurement type"); return NYXB_RC_BAD_ARG; }
        }
        DevLink& d = hs[s];
        d.tx_n = (long long)n_tx;
        d.col = g.tx; d.n_types = g.n_types;
        for (int q = 0; q < 2; ++q) { d.types[q] = g.types[q]; d.noise_var[q] = g.noise_var[q]; d.bias[q] = g.bias[q]; }
        d.body_radius = g.body_radius_km;
    }
    return NYXB_RC_OK;
}
// uploads the recordings into B and points every device at them
int32_t put_links(DevBufs& B, size_t n_tx, const nyxb_traj_sink* sink, cudaStream_t st, std::vector<DevLink>& hs) {
    const size_t cap = (size_t)sink->capacity;
    const NyxbTrajView tv{(long long)cap, B.put((const long long*)sink->epoch_ns, cap * n_tx, st), B.put(sink->state, 6 * cap * n_tx, st),
                          B.put((const long long*)sink->count, n_tx, st)};
    if (int32_t rc = B.check("device allocation / upload failed (transmitter recordings)")) return rc;
    for (DevLink& d : hs) d.tx = tv;
    return NYXB_RC_OK;
}
}  // namespace

extern "C" int32_t nyxb_od_interlink_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_devices, const nyxb_interlink_tx* devices,
                                           size_t n_tx, const nyxb_traj_sink* tx_sink, const nyxb_tracking_arc* arc, size_t n,
                                           const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                                           const double* covar0_soa, const nyxb_od_outputs* out, const nyxb_od_records* rec) {
    if (int32_t rc = filter_args<DevLink>(eng, cfg, n_devices, devices, arc, state_soa, consts_soa, epoch0_ns, covar0_soa, out, rec))
        return rc;
    std::vector<DevLink> hs;
    if (int32_t rc = pack_links(n_devices, devices, n_tx, tx_sink, hs)) return rc;
    if (n == 0) return NYXB_RC_OK;
    cudaStream_t st;
    if (int32_t rc = od_stream(eng, st)) return rc;
    DevBufs B;
    if (int32_t rc = put_links(B, n_tx, tx_sink, st, hs)) return rc;
    return od_filter_run(eng, cfg, hs, arc->n_msr, arc->epoch_ns, arc->tracker, arc->obs, n, state_soa, consts_soa, epoch0_ns, covar0_soa,
                         out, rec);
}

extern "C" int32_t nyxb_od_interlink_smooth_batch(nyxb_engine* eng, const nyxb_od_config* cfg, int32_t n_devices,
                                                  const nyxb_interlink_tx* devices, size_t n_tx, const nyxb_traj_sink* tx_sink,
                                                  const nyxb_tracking_arc* arc, size_t n, const nyxb_od_records* rec,
                                                  const int32_t* filter_status, nyxb_smooth_outputs* out) {
    if (!eng || !cfg || !arc || !rec || !filter_status || !out || !out->status || (n_devices > 0 && !devices) || n_devices < 0) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (cfg->msr_size != 1 && cfg->msr_size != 2) { set_err("msr_size must be 1 or 2"); return NYXB_RC_BAD_ARG; }
    if (!records_ok(rec)) return NYXB_RC_BAD_ARG;
    if (arc->n_msr < 0 || (arc->n_msr > 0 && (!arc->tracker || !arc->obs))) { set_err("null tracking arc arrays"); return NYXB_RC_BAD_ARG; }
    std::vector<DevLink> hs;
    if (int32_t rc = pack_links(n_devices, devices, n_tx, tx_sink, hs)) return rc;
    cudaStream_t st;
    if (int32_t rc = od_stream(eng, st)) return rc;
    DevBufs B;
    if (int32_t rc = put_links(B, n_tx, tx_sink, st, hs)) return rc;
    return od_smooth_run<LinkTags>(eng, cfg->msr_size, hs, arc->n_msr, arc->tracker, arc->obs, n, rec, filter_status, out, NYXB_ERR_TX_NO_DATA);
}

extern "C" int32_t nyxb_od_predict_batch(nyxb_engine* eng, const nyxb_od_config* cfg, size_t n, const double* state_soa,
                                         const double* consts_soa, const int64_t* epoch0_ns, const int64_t* end_epoch_ns,
                                         const double* covar0_soa, const double* state_dev0_soa, const nyxb_predict_outputs* out) {
    if (!cfg) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    if (cfg->variant != NYXB_KF_REFERENCE_UPDATE && cfg->variant != NYXB_KF_DEVIATION_TRACKING) { set_err("bad filter variant"); return NYXB_RC_BAD_ARG; }
    // the reference does not check max_step here: a value <= 0 would never reach the end epoch
    if (cfg->max_step_ns <= 0) { set_err("StepSize: max_step must be positive"); return NYXB_RC_BAD_ARG; }
    if (!eng || !state_soa || !consts_soa || !epoch0_ns || !end_epoch_ns || !covar0_soa || !out || !out->state_soa || !out->epoch_ns ||
        !out->covar_soa || !out->status) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (out->capacity < 0) { set_err("negative record capacity"); return NYXB_RC_BAD_ARG; }
    if (!stm_supported(eng)) return NYXB_RC_UNSUPPORTED;
    if (n == 0) return NYXB_RC_OK;
    cudaStream_t st;
    if (int32_t rc = od_stream(eng, st)) return rc;
    const size_t cap = (size_t)out->capacity;
    DevBufs B;
    OdPredictJob job{};
    DevOd& od = job.od;
    od.variant = cfg->variant;
    od.max_step_ns = cfg->max_step_ns;
    od.snc_enabled = cfg->snc_enabled; od.snc_frame = cfg->snc_frame;
    for (int q = 0; q < 3; ++q) od.snc_diag[q] = cfg->snc_diag[q];
    od.snc_disable_ns = cfg->snc_disable_time_ns;
    od.covar0 = B.put(covar0_soa, 81 * n, st);
    od.covar = B.alloc<double>(81 * n);
    od.state_dev = out->state_dev_soa ? B.alloc<double>(9 * n) : nullptr;
    const OdIo io = od_io(B, st, n, state_soa, consts_soa, epoch0_ns);
    job.end_epoch = B.put((const long long*)end_epoch_ns, n, st);
    job.dev0 = state_dev0_soa ? B.put(state_dev0_soa, 9 * n, st) : nullptr;
    job.rec_count = out->rec_count ? B.alloc<long long>(n) : nullptr;
    job.rec.cap = (long long)cap;
    if (cap && out->rec_state) job.rec.state = B.alloc<double>(cap * 9 * n);
    if (cap && out->rec_covar) job.rec.covar = B.alloc<double>(cap * 81 * n);
    if (int32_t rc = B.check()) return rc;
    // records a run does not reach read back as NaN (0xFF bytes)
    if (job.rec.state) CUDA_TRY(cudaMemsetAsync(job.rec.state, 0xFF, sizeof(double) * cap * 9 * n, st));
    if (job.rec.covar) CUDA_TRY(cudaMemsetAsync(job.rec.covar, 0xFF, sizeof(double) * cap * 81 * n, st));
    if (int32_t rc = od_launch(eng, job, B, n, io)) return rc;
    if (int32_t rc = od_io_get(io, n, st, out->state_soa, out->epoch_ns, out->details, out->status)) return rc;
    CUDA_TRY(get(out->covar_soa, od.covar, 81 * n, st));
    CUDA_TRY(get(out->state_dev_soa, od.state_dev, 9 * n, st));
    CUDA_TRY(get(out->rec_count, job.rec_count, n, st));
    if (job.rec.state) CUDA_TRY(get(out->rec_state, job.rec.state, cap * 9 * n, st));
    if (job.rec.covar) CUDA_TRY(get(out->rec_covar, job.rec.covar, cap * 81 * n, st));
    return od_finish(eng);
}

namespace {
// nyxb_od_bls_batch / nyxb_od_bls_evaluate_batch: argument checks, packing, one launch, read-back.  `bl` carries the solver settings;
// its output pointers are filled here.  out_* host pointers may be null except status.
int32_t od_bls_run(nyxb_engine* eng, const nyxb_bls_config* cfg, int32_t n_stations, const nyxb_ground_station* stations,
                   const nyxb_tracking_arc* arc, size_t n, const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns,
                   DevBls bl, double* out_state, int64_t* out_epoch, double* out_covar, int32_t* out_iters, double* out_rms,
                   double* out_corr, int32_t* out_conv, nyxb_details* out_details, int32_t* out_status) {
    if (!eng || !cfg || !arc || !state_soa || !consts_soa || !epoch0_ns || !out_status || (n_stations > 0 && !stations) || n_stations < 0) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    // stricter than the reference, which would loop forever (max_step <= 0) or take a usize (max_iterations)
    if (cfg->max_step_ns <= 0) { set_err("StepSize: max_step must be positive"); return NYXB_RC_BAD_ARG; }
    if (!bl.evaluate) {
        if (cfg->solver != NYXB_BLS_NORMAL_EQUATIONS && cfg->solver != NYXB_BLS_LEVENBERG_MARQUARDT) { set_err("bad BLS solver"); return NYXB_RC_BAD_ARG; }
        if (cfg->max_iterations < 0) { set_err("max_iterations must not be negative"); return NYXB_RC_BAD_ARG; }
        if (cfg->solver == NYXB_BLS_LEVENBERG_MARQUARDT &&
            !(cfg->lm_lambda_init > 0.0 && cfg->lm_lambda_decrease > 0.0 && cfg->lm_lambda_increase > 0.0 && cfg->lm_lambda_min > 0.0 &&
              cfg->lm_lambda_max > 0.0)) {
            set_err("Levenberg-Marquardt lambda settings must be positive");
            return NYXB_RC_BAD_ARG;
        }
    }
    if (arc->n_msr < 0 || (arc->n_msr > 0 && (!arc->epoch_ns || !arc->tracker || !arc->obs))) { set_err("null tracking arc arrays"); return NYXB_RC_BAD_ARG; }
    if (!stm_supported(eng)) return NYXB_RC_UNSUPPORTED;
    std::vector<DevStation> hs;
    for (int32_t s = 0; s < n_stations; ++s) {
        const nyxb_ground_station& g = stations[s];
        if (!station_ok(eng, g)) return NYXB_RC_BAD_ARG;
        for (int q = 0; q < g.n_types; ++q) {
            if (g.types[q] != NYXB_MSR_RANGE && g.types[q] != NYXB_MSR_DOPPLER) { set_err("unsupported measurement type"); return NYXB_RC_UNSUPPORTED; }
            // earlier than the reference, which fails with SingularNoiseRk at the first measurement of this station
            if (!(g.noise_var[q] > 0.0)) { set_err("SingularNoiseRk: a station's noise variance must be positive"); return NYXB_RC_BAD_ARG; }
        }
        hs.push_back(pack_station(g));
    }
    if (n == 0) return NYXB_RC_OK;
    cudaStream_t st;
    if (int32_t rc = od_stream(eng, st)) return rc;
    const size_t m = (size_t)arc->n_msr;
    DevBufs B;
    OdBlsJob job{};
    DevOd& od = job.od;
    od.msr_size = 1;
    od.max_step_ns = cfg->max_step_ns; od.eps_ns = cfg->epoch_precision_ns;
    od.n_stations = n_stations;
    od.stations = n_stations ? B.put(hs.data(), hs.size(), st) : nullptr;
    od.n_msr = arc->n_msr;
    od.msr_epoch = m ? B.put((const long long*)arc->epoch_ns, m, st) : nullptr;
    od.msr_tracker = m ? B.put((const int*)arc->tracker, m, st) : nullptr;
    od.obs = m ? B.put(arc->obs, m * 2 * n, st) : nullptr;
    const OdIo io = od_io(B, st, n, state_soa, consts_soa, epoch0_ns);
    job.bl = bl;
    job.bl.covar = out_covar ? B.alloc<double>(81 * n) : nullptr;
    job.bl.iters = out_iters ? B.alloc<int>(n) : nullptr;
    job.bl.rms = out_rms ? B.alloc<double>(n) : nullptr;
    job.bl.corr_pos_km = out_corr ? B.alloc<double>(n) : nullptr;
    job.bl.converged = out_conv ? B.alloc<int>(n) : nullptr;
    if (int32_t rc = B.check()) return rc;
    if (int32_t rc = od_launch(eng, job, B, n, io)) return rc;
    if (int32_t rc = od_io_get(io, n, st, out_state, out_epoch, out_details, out_status)) return rc;
    CUDA_TRY(get(out_covar, job.bl.covar, 81 * n, st));
    CUDA_TRY(get(out_iters, job.bl.iters, n, st));
    CUDA_TRY(get(out_rms, job.bl.rms, n, st));
    CUDA_TRY(get(out_corr, job.bl.corr_pos_km, n, st));
    CUDA_TRY(get(out_conv, job.bl.converged, n, st));
    return od_finish(eng);
}
}  // namespace

extern "C" int32_t nyxb_od_bls_batch(nyxb_engine* eng, const nyxb_bls_config* cfg, int32_t n_stations, const nyxb_ground_station* stations,
                                     const nyxb_tracking_arc* arc, size_t n, const double* state_soa, const double* consts_soa,
                                     const int64_t* epoch0_ns, const nyxb_bls_outputs* out) {
    if (!cfg || !out) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    DevBls bl{};
    bl.evaluate = 0;
    bl.solver = cfg->solver; bl.max_iter = cfg->max_iterations; bl.lm_diag = cfg->lm_use_diag_scaling;
    bl.tol_pos_km = cfg->tolerance_pos_km;
    bl.lm_init = cfg->lm_lambda_init; bl.lm_dec = cfg->lm_lambda_decrease; bl.lm_inc = cfg->lm_lambda_increase;
    bl.lm_min = cfg->lm_lambda_min; bl.lm_max = cfg->lm_lambda_max;
    return od_bls_run(eng, cfg, n_stations, stations, arc, n, state_soa, consts_soa, epoch0_ns, bl, out->state_soa, out->epoch_ns,
                      out->covar_soa, out->iterations, out->final_rms, out->final_corr_pos_km, out->converged, out->details, out->status);
}

extern "C" int32_t nyxb_od_bls_evaluate_batch(nyxb_engine* eng, const nyxb_bls_config* cfg, int32_t n_stations,
                                              const nyxb_ground_station* stations, const nyxb_tracking_arc* arc, size_t n,
                                              const double* state_soa, const double* consts_soa, const int64_t* epoch0_ns, double* rms,
                                              int32_t* status) {
    DevBls bl{};
    bl.evaluate = 1;
    return od_bls_run(eng, cfg, n_stations, stations, arc, n, state_soa, consts_soa, epoch0_ns, bl, nullptr, nullptr, nullptr, nullptr,
                      rms, nullptr, nullptr, nullptr, status);
}

// ---------------------------------------------------------------------------------------------------------------------
// Impulsive targeting (Targeter::try_achieve_fd, md/opti/raphson_finite_diff.rs:41-747): update kernels in nyxb_target.cu.
// ---------------------------------------------------------------------------------------------------------------------
namespace {
bool target_config_ok(const nyxb_target_config& c) {
    if (c.n_vars < 1 || c.n_vars > 6 || c.n_objs < 1 || c.n_objs > 6) { set_err("n_vars and n_objs must be 1..6"); return false; }
    if (c.correction_frame < NYXB_TGT_FRAME_NONE || c.correction_frame > NYXB_TGT_FRAME_RIC) { set_err("unknown correction frame"); return false; }
    if (c.iterations < 0) { set_err("iterations must not be negative"); return false; }
    for (int j = 0; j < c.n_vars; ++j) {
        const nyxb_tgt_variable& v = c.vars[j];
        if (v.component < NYXB_VARY_POSITION_X || v.component > NYXB_VARY_VELOCITY_Z) { set_err("unknown variable component"); return false; }
        if (c.correction_frame != NYXB_TGT_FRAME_NONE && v.component < NYXB_VARY_VELOCITY_X) {
            set_err("FrameError: a position variable cannot be corrected in a local frame");
            return false;
        }
        // Variable::valid (target_variable.rs:143-168)
        if (v.max_step < 0.0 || v.max_value < 0.0 || v.min_value > v.max_value) { set_err("VariableError: bad max step or bounds"); return false; }
        if (!(std::isfinite(v.perturbation) && v.perturbation != 0.0)) { set_err("a perturbation must be finite and nonzero"); return false; }
    }
    for (int i = 0; i < c.n_objs; ++i)
        if (c.objs[i].parameter < 0 || c.objs[i].parameter >= NYXB_TGT_N_PARAMS) { set_err("unknown objective parameter"); return false; }
    return true;
}

// Fix the kernel family and lane count that launch_inner would pick for n trajectories, so that every launch of a call uses it.
struct FamilyPin {
    nyxb_engine* e;
    int kernel, lanes;
    FamilyPin(nyxb_engine* eng, size_t n) : e(eng), kernel(eng->kernel), lanes(eng->lanes) {
        int l;
        e->kernel = launch_family(e, n, l);
        if (e->kernel != NYXB_KERNEL_TRANSPOSED) e->lanes = l;
    }
    ~FamilyPin() { e->kernel = kernel; e->lanes = lanes; }
};
}  // namespace

extern "C" int32_t nyxb_target_batch(nyxb_engine* eng, const nyxb_target_config* cfg, size_t n, const double* state_soa,
                                     const double* consts_soa, const int64_t* epoch0_ns, int64_t correction_epoch_ns,
                                     int64_t achievement_epoch_ns, double* out_corrected_soa, double* out_achieved_soa,
                                     double* out_correction, double* out_errors, int32_t* out_iterations, int32_t* out_status) {
    if (!eng || !cfg || !state_soa || !consts_soa || !epoch0_ns || !out_corrected_soa || !out_achieved_soa || !out_correction ||
        !out_errors || !out_iterations || !out_status) {
        set_err("null argument");
        return NYXB_RC_BAD_ARG;
    }
    if (!target_config_ok(*cfg)) return NYXB_RC_BAD_ARG;
    // problem and slab indices are int on the device: n (n_vars + 1) must fit
    if (n > (size_t)INT32_MAX / 7) { set_err("too many problems"); return NYXB_RC_BAD_ARG; }
    if (eng->S.state_center >= 0) { set_err("targeting takes states in the integration frame"); return NYXB_RC_UNSUPPORTED; }
    if (n == 0) return NYXB_RC_OK;
    cudaStream_t st;
    if (int32_t rc = od_stream(eng, st)) return rc;
    const nyxb_target_config& c = *cfg;
    const size_t V = (size_t)c.n_vars, O = (size_t)c.n_objs, W = V + 1, M = n * W;
    const double mu = eng->S.mu_central;
    DevBufs B;
    TgtDev t{};
    t.n = n;
    const double* d_state = B.put(state_soa, 9 * n, st);
    t.consts = B.put(consts_soa, 4 * n, st);
    const long long* d_epoch0 = B.put((const long long*)epoch0_ns, n, st);
    t.start = B.alloc<double>(9 * n); t.epoch_c = B.alloc<long long>(n); t.xi = B.alloc<double>(6 * n); t.total = B.alloc<double>(V * n);
    t.err = B.alloc<double>(O * n); t.prev_norm = B.alloc<double>(n); t.achieved = B.alloc<double>(9 * n); t.corrected = B.alloc<double>(9 * n);
    t.iters = B.alloc<int>(n); t.status = B.alloc<int>(n); t.flag = B.alloc<int>(n);
    int* idx[2] = {B.alloc<int>(n), B.alloc<int>(n)};
    int* d_count = B.alloc<int>(1);
    t.idx = idx[0];
    t.l_state = B.alloc<double>(9 * M); t.l_consts = B.alloc<double>(4 * M); t.l_epoch = B.alloc<long long>(M);
    t.o_state = B.alloc<double>(9 * M); t.o_status = B.alloc<int>(M);
    long long* o_epoch = B.alloc<long long>(M);
    nyxb_details* o_det = B.alloc<nyxb_details>(M);
    size_t temp_bytes = 0;
    CUDA_TRY(nyxb_tgt_compact(nullptr, &temp_bytes, idx[0], t.flag, idx[1], d_count, (int)n, st));
    void* temp = B.alloc<unsigned char>(temp_bytes);
    if (int32_t rc = B.check()) return rc;

    FamilyPin pin(eng, M);
    int cur = 0;
    int A = 0;
    auto compact = [&](int count) -> int32_t {
        CUDA_TRY(nyxb_tgt_compact(temp, &temp_bytes, idx[cur], t.flag, idx[cur ^ 1], d_count, count, st));
        CUDA_TRY(cudaMemcpyAsync(&A, d_count, sizeof(int), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        cur ^= 1;
        eng->launches += 1;
        return NYXB_RC_OK;
    };
    CUDA_TRY(cudaEventRecord(eng->ev0, st));
    // xi_start: the states at the correction epoch, from opts.init_step (the slab's first n slots serve as the outputs)
    if (int32_t rc = launch(eng, n, d_state, t.consts, (const int64_t*)d_epoch0, correction_epoch_ns, nullptr, t.o_state,
                            (int64_t*)o_epoch, o_det, t.o_status, DevSink{}, st))
        return rc;
    CUDA_TRY(nyxb_tgt_launch_init(t, c, t.o_state, o_epoch, t.o_status, st));
    eng->launches += 1;
    if (int32_t rc = compact((int)n)) return rc;
    while (A > 0) {
        const size_t m = (size_t)A * W;
        CUDA_TRY(nyxb_tgt_launch_stage(t, c, A, idx[cur], st));
        eng->launches += 1;
        if (int32_t rc = launch(eng, m, t.l_state, t.l_consts, (const int64_t*)t.l_epoch, achievement_epoch_ns, nullptr, t.o_state,
                                (int64_t*)o_epoch, o_det, t.o_status, DevSink{}, st))
            return rc;
        CUDA_TRY(nyxb_tgt_launch_update(t, c, mu, A, idx[cur], st));
        eng->launches += 1;
        if (int32_t rc = compact(A)) return rc;
    }
    CUDA_TRY(nyxb_tgt_launch_finish(t, c, st));
    eng->launches += 1;
    CUDA_TRY(cudaEventRecord(eng->ev1, st));
    CUDA_TRY(get(out_corrected_soa, t.corrected, 9 * n, st));
    CUDA_TRY(get(out_achieved_soa, t.achieved, 9 * n, st));
    CUDA_TRY(get(out_correction, t.total, V * n, st));
    CUDA_TRY(get(out_errors, t.err, O * n, st));
    CUDA_TRY(get(out_iterations, t.iters, n, st));
    CUDA_TRY(get(out_status, t.status, n, st));
    return od_finish(eng);
}

extern "C" int32_t nyxb_mvn_sample_dev(int32_t device, uint64_t seed, uint64_t first_index, size_t n, const double* template_state,
                                       const double* mean, const double* sqrt_s_v, double* out_state_soa, double* out_dispersion_soa,
                                       void* cuda_stream) {
    if (!template_state || !sqrt_s_v || !out_state_soa) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_err("no CUDA device available: nyxb has no CPU fallback"); return NYXB_RC_NO_DEVICE; }
    if (device < 0 || device >= ndev) { set_err("bad device ordinal"); return NYXB_RC_BAD_ARG; }
    CUDA_TRY(cudaSetDevice(device));
    cudaError_t err = nyxb_launch_mvn(seed, first_index, n, template_state, mean, sqrt_s_v, out_state_soa, out_dispersion_soa,
                                      (cudaStream_t)cuda_stream);
    if (err != cudaSuccess) { set_err(std::string("kernel launch: ") + cudaGetErrorString(err)); return NYXB_RC_CUDA; }
    return NYXB_RC_OK;
}

extern "C" int32_t nyxb_mvn_sample(int32_t device, uint64_t seed, uint64_t first_index, size_t n, const double* template_state,
                                   const double* mean, const double* sqrt_s_v, double* out_state_soa, double* out_dispersion_soa) {
    if (!template_state || !sqrt_s_v || !out_state_soa) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    if (n == 0) return NYXB_RC_OK;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_err("no CUDA device available: nyxb has no CPU fallback"); return NYXB_RC_NO_DEVICE; }
    if (device < 0 || device >= ndev) { set_err("bad device ordinal"); return NYXB_RC_BAD_ARG; }
    CUDA_TRY(cudaSetDevice(device));
    DevBufs B;
    double* d_out = B.alloc<double>(9 * n);
    double* d_disp = out_dispersion_soa ? B.alloc<double>(9 * n) : nullptr;
    if (!d_out || (out_dispersion_soa && !d_disp)) { set_err("device allocation failed"); return NYXB_RC_CUDA; }
    int32_t rc = nyxb_mvn_sample_dev(device, seed, first_index, n, template_state, mean, sqrt_s_v, d_out, d_disp, nullptr);
    if (rc != NYXB_RC_OK) return rc;
    CUDA_TRY(cudaMemcpy(out_state_soa, d_out, sizeof(double) * 9 * n, cudaMemcpyDeviceToHost));
    if (d_disp) CUDA_TRY(cudaMemcpy(out_dispersion_soa, d_disp, sizeof(double) * 9 * n, cudaMemcpyDeviceToHost));
    return NYXB_RC_OK;
}

// ---- batched Hermite resampling of recorded trajectories (nyxb_traj.cu)
extern "C" int32_t nyxb_traj_resample_dev(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink, size_t m, const int64_t* query_epoch_ns,
                                          double* out_state, int32_t* out_status, void* cuda_stream) {
    if (!eng || !sink || !query_epoch_ns || !out_state || !out_status) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    if (sink->capacity <= 0 || !sink->epoch_ns || !sink->state || !sink->count) { set_err("empty trajectory sink"); return NYXB_RC_BAD_ARG; }
    CUDA_TRY(cudaSetDevice(eng->device));
    cudaError_t err = nyxb_launch_traj_resample(sink->capacity, (const long long*)sink->epoch_ns, sink->state, (const long long*)sink->count,
                                                n, m, (const long long*)query_epoch_ns, out_state, out_status, (cudaStream_t)cuda_stream);
    if (err != cudaSuccess) { set_err(std::string("kernel launch: ") + cudaGetErrorString(err)); return NYXB_RC_CUDA; }
    if (n && m) eng->launches += 1;
    return NYXB_RC_OK;
}

// upload `sink` into the engine's slab (or check the resident recording when sink == NULL) and describe it with device pointers
static int32_t resident_sink(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink, cudaStream_t st, nyxb_traj_sink* dsink) {
    if (sink && (sink->capacity <= 0 || !sink->epoch_ns || !sink->state || !sink->count)) { set_err("empty trajectory sink"); return NYXB_RC_BAD_ARG; }
    if (!sink && (eng->rec_cap <= 0 || eng->rec_n != n || !eng->d_sink)) {
        set_err("no resident recording of this many trajectories: pass the sink of nyxb_propagate_batch_traj");
        return NYXB_RC_BAD_ARG;
    }
    if (sink) {   // [epoch cap*n i64 | state 6*cap*n f64 | count n i64]
        const size_t cap = (size_t)sink->capacity;
        const size_t need = (cap * n * 7 + n) * 8;
        if (need > eng->sink_bytes) {
            cudaFree(eng->d_sink); eng->d_sink = nullptr; eng->sink_bytes = 0; eng->rec_n = 0; eng->rec_cap = 0;
            CUDA_TRY(cudaMalloc(&eng->d_sink, need));
            eng->sink_bytes = need;
        }
        CUDA_TRY(cudaMemcpyAsync(eng->d_sink, sink->epoch_ns, cap * n * 8, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(eng->d_sink + cap * n * 8, sink->state, cap * n * 48, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(eng->d_sink + cap * n * 56, sink->count, n * 8, cudaMemcpyHostToDevice, st));
        eng->rec_n = n; eng->rec_cap = sink->capacity;
    }
    const size_t cap = (size_t)eng->rec_cap;
    dsink->capacity = eng->rec_cap;
    dsink->epoch_ns = (int64_t*)eng->d_sink;
    dsink->state = (double*)(eng->d_sink + cap * n * 8);
    dsink->count = (int64_t*)(eng->d_sink + cap * n * 56);
    return NYXB_RC_OK;
}

extern "C" int32_t nyxb_traj_resample(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink, size_t m, const int64_t* query_epoch_ns,
                                      double* out_state, int32_t* out_status) {
    if (!eng || !query_epoch_ns || !out_state || !out_status) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    if (sink && (sink->capacity <= 0 || !sink->epoch_ns || !sink->state || !sink->count)) { set_err("empty trajectory sink"); return NYXB_RC_BAD_ARG; }
    if (!sink && (eng->rec_cap <= 0 || eng->rec_n != n || !eng->d_sink)) {
        set_err("no resident recording of this many trajectories: pass the sink of nyxb_propagate_batch_traj");
        return NYXB_RC_BAD_ARG;
    }
    if (n == 0 || m == 0) return NYXB_RC_OK;
    CUDA_TRY(cudaSetDevice(eng->device));
    if (!eng->stream) CUDA_TRY(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
    cudaStream_t st = eng->stream;
    nyxb_traj_sink dsink;
    int32_t rc = resident_sink(eng, n, sink, st, &dsink);
    if (rc != NYXB_RC_OK) return rc;
    DevBufs B;
    long long* d_q = B.put((const long long*)query_epoch_ns, m, st);
    double* d_out = B.alloc<double>(6 * m * n);
    int* d_status = B.alloc<int>(m * n);
    if (!d_q || !d_out || !d_status) { set_err("device allocation / upload failed"); return NYXB_RC_CUDA; }
    CUDA_TRY(cudaEventRecord(eng->ev0, st));
    rc = nyxb_traj_resample_dev(eng, n, &dsink, m, (const int64_t*)d_q, d_out, d_status, st);
    if (rc != NYXB_RC_OK) return rc;
    CUDA_TRY(cudaEventRecord(eng->ev1, st));
    CUDA_TRY(cudaMemcpyAsync(out_state, d_out, sizeof(double) * 6 * m * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out_status, d_status, sizeof(int) * m * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, eng->ev0, eng->ev1) == cudaSuccess) eng->last_ms = ms;
    return NYXB_RC_OK;
}

// ---- event location on recorded trajectories (nyxb_traj.cu)
static bool event_kind_ok(int32_t kind) { return kind >= NYXB_EVENT_RMAG && kind <= NYXB_EVENT_VMAG; }

extern "C" int32_t nyxb_event_locate_dev(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink, int32_t kind, double value,
                                         int64_t epoch_precision_ns, const int32_t* run_status, int64_t* out_event_epoch_ns,
                                         double* out_event_state, int32_t* out_status, void* cuda_stream) {
    if (!eng || !sink || !out_event_epoch_ns || !out_event_state || !out_status) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    if (sink->capacity <= 0 || !sink->epoch_ns || !sink->state || !sink->count) { set_err("empty trajectory sink"); return NYXB_RC_BAD_ARG; }
    if (!event_kind_ok(kind) || epoch_precision_ns < 0) { set_err("bad event descriptor"); return NYXB_RC_BAD_ARG; }
    CUDA_TRY(cudaSetDevice(eng->device));
    cudaError_t err = nyxb_launch_event_locate(sink->capacity, (const long long*)sink->epoch_ns, sink->state, (const long long*)sink->count, n,
                                               kind, value, epoch_precision_ns, run_status, (long long*)out_event_epoch_ns, out_event_state,
                                               out_status, (cudaStream_t)cuda_stream);
    if (err != cudaSuccess) { set_err(std::string("kernel launch: ") + cudaGetErrorString(err)); return NYXB_RC_CUDA; }
    if (n) eng->launches += 1;
    return NYXB_RC_OK;
}

extern "C" int32_t nyxb_event_locate(nyxb_engine* eng, size_t n, const nyxb_traj_sink* sink, int32_t kind, double value,
                                     int64_t epoch_precision_ns, const int32_t* run_status, int64_t* out_event_epoch_ns,
                                     double* out_event_state, int32_t* out_status) {
    if (!eng || !out_event_epoch_ns || !out_event_state || !out_status) { set_err("null argument"); return NYXB_RC_BAD_ARG; }
    if (!event_kind_ok(kind) || epoch_precision_ns < 0) { set_err("bad event descriptor"); return NYXB_RC_BAD_ARG; }
    if (n == 0) return NYXB_RC_OK;
    CUDA_TRY(cudaSetDevice(eng->device));
    if (!eng->stream) CUDA_TRY(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
    cudaStream_t st = eng->stream;
    nyxb_traj_sink dsink;
    int32_t rc = resident_sink(eng, n, sink, st, &dsink);
    if (rc != NYXB_RC_OK) return rc;
    DevBufs B;
    int* d_run = run_status ? B.put((const int*)run_status, n, st) : nullptr;
    long long* d_ep = B.alloc<long long>(n);
    double* d_out = B.alloc<double>(6 * n);
    int* d_status = B.alloc<int>(n);
    if ((run_status && !d_run) || !d_ep || !d_out || !d_status) { set_err("device allocation / upload failed"); return NYXB_RC_CUDA; }
    CUDA_TRY(cudaEventRecord(eng->ev0, st));
    rc = nyxb_event_locate_dev(eng, n, &dsink, kind, value, epoch_precision_ns, d_run, (int64_t*)d_ep, d_out, d_status, st);
    if (rc != NYXB_RC_OK) return rc;
    CUDA_TRY(cudaEventRecord(eng->ev1, st));
    CUDA_TRY(cudaMemcpyAsync(out_event_epoch_ns, d_ep, sizeof(long long) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out_event_state, d_out, sizeof(double) * 6 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out_status, d_status, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, eng->ev0, eng->ev1) == cudaSuccess) eng->last_ms = ms;
    return NYXB_RC_OK;
}

extern "C" int32_t nyxb_engine_set_lanes(nyxb_engine* eng, int32_t lanes) {
    if (!eng) return NYXB_RC_BAD_ARG;
    if (lanes != 0 && lanes != 1 && lanes != 8 && lanes != 16 && lanes != 32) { set_err("lanes must be 0,1,8,16,32"); return NYXB_RC_BAD_ARG; }
    if (lanes > 1 && !coop_supported(eng, lanes)) {
        set_err("cooperative lanes need a gravity field");
        return NYXB_RC_UNSUPPORTED;
    }
    if (lanes > 1 && eng->mode == NYXB_MODE_STRICT && nyxb_coop_strict_smem(eng->S.grav.N, lanes) > NYXB_COOP_STRICT_SMEM_MAX) {
        set_err("STRICT cooperative kernel: the shared-memory slabs of a degree-" + std::to_string(eng->S.grav.N) + " field at " +
                std::to_string(lanes) + " lanes per trajectory exceed the 227 KB of a block (8 lanes: degree <= 50, 16 lanes: <= 75)");
        return NYXB_RC_UNSUPPORTED;
    }
    eng->lanes = lanes;
    return NYXB_RC_OK;
}
extern "C" int32_t nyxb_engine_set_kernel(nyxb_engine* eng, int32_t kernel) {
    if (!eng) return NYXB_RC_BAD_ARG;
    if (kernel < NYXB_KERNEL_AUTO || kernel > NYXB_KERNEL_TRANSPOSED) { set_err("unknown kernel family"); return NYXB_RC_BAD_ARG; }
    if (kernel == NYXB_KERNEL_TRANSPOSED && !tx_supported(eng)) {
        set_err("the transposed kernel needs FAST mode and a gravity field of degree 8..70");
        return NYXB_RC_UNSUPPORTED;
    }
    if (kernel == NYXB_KERNEL_COOP && !eng->S.has_grav) { set_err("cooperative lanes need a gravity field"); return NYXB_RC_UNSUPPORTED; }
    eng->kernel = kernel;
    return NYXB_RC_OK;
}
extern "C" int32_t nyxb_engine_last_kernel(const nyxb_engine* eng) { return eng ? eng->last_kernel : 0; }
extern "C" int32_t nyxb_engine_set_tx_tuning(nyxb_engine* eng, int32_t slice_attempts, int32_t max_ctas) {
    if (!eng || slice_attempts < 1 || max_ctas < 0) { set_err("slice_attempts >= 1, max_ctas >= 0"); return NYXB_RC_BAD_ARG; }
    eng->tx_slice = slice_attempts;
    eng->tx_max_ctas = max_ctas;
    return NYXB_RC_OK;
}
extern "C" int32_t nyxb_engine_set_tx_positions(nyxb_engine* eng, int32_t positions) {
    if (!eng || (positions != 0 && positions != 8 && positions != 10 && positions != 16)) { set_err("positions: 0 (auto), 8, 10, 16"); return NYXB_RC_BAD_ARG; }
    eng->tx_positions = positions;
    return NYXB_RC_OK;
}
extern "C" int32_t nyxb_engine_get_lanes(const nyxb_engine* eng) { return eng ? pick_lanes(eng, 0) : 0; }
extern "C" int64_t nyxb_engine_launch_count(const nyxb_engine* eng) { return eng ? eng->launches : 0; }
extern "C" double nyxb_engine_last_kernel_ms(const nyxb_engine* eng) { return eng ? eng->last_ms : 0.0; }
extern "C" double nyxb_measure_fp64_tflops(int32_t device, int32_t iters) { return nyxb_fp64_probe(device, iters); }
extern "C" int32_t nyxb_coop_table_dump(const nyxb_gravity_field* f, int32_t lanes, int32_t* out_L, int32_t* out_kmax,
                                        double* recs, int32_t* col_start, int32_t* col_m, double* colseed) {
    if (!f || !f->c_nm || !f->s_nm || f->degree < 2 || (lanes != 8 && lanes != 16 && lanes != 32) || !out_L || !out_kmax) {
        set_err("bad argument");
        return NYXB_RC_BAD_ARG;
    }
    CoopHost h;
    nyxb_coop_build_host(f->degree, f->order, f->c_nm, f->s_nm, lanes, h);
    *out_L = h.L; *out_kmax = h.kmax;
    if (recs) std::copy(h.recs.begin(), h.recs.end(), recs);
    if (col_start) std::copy(h.col_start.begin(), h.col_start.end(), col_start);
    if (col_m) std::copy(h.col_m.begin(), h.col_m.end(), col_m);
    if (colseed) std::copy(h.colseed.begin(), h.colseed.end(), colseed);
    return NYXB_RC_OK;
}

extern "C" int32_t nyxb_tx_table_dump(const nyxb_gravity_field* f, int32_t positions, int32_t* out_n_rec, int32_t* out_kmax,
                                      double* recA, double* recK, double* colseed, int32_t* sched) {
    if (!f || !f->c_nm || !f->s_nm || f->degree < 2 || (positions != 8 && positions != 10 && positions != 16) || !out_n_rec || !out_kmax) {
        set_err("bad argument");
        return NYXB_RC_BAD_ARG;
    }
    TxHost h;
    nyxb_tx_build_host(f->degree, f->order, f->c_nm, f->s_nm, positions, h);
    *out_n_rec = h.n_rec; *out_kmax = h.kmax;
    if (recA) std::copy(h.recA.begin(), h.recA.end(), recA);
    if (recK) std::copy(h.recK.begin(), h.recK.end(), recK);
    if (colseed) std::copy(h.colseed.begin(), h.colseed.end(), colseed);
    if (sched) std::copy(h.sched.begin(), h.sched.end(), sched);
    return NYXB_RC_OK;
}

extern "C" int32_t nyxb_abi_version(void) { return NYXB_ABI_VERSION; }
extern "C" const char* nyxb_last_error(void) { return g_err.c_str(); }
