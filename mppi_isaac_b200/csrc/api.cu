// api.cu -- the C ABI of include/mppib.h (handle lifetime + thin launch wrappers).
#include <stdarg.h>
#include <stdlib.h>

#include "common.cuh"

static thread_local char g_err[1024] = "";

void mppib_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}


// Which planning modes cannot run together (make_params refuses the same pairs): validate checks the block with anneal = false; a schedule
// is checked with anneal = true at registration and at every launch, so that a later mppib_set_params cannot slip past it.
enum Feature { F_CEM, F_SMOOTH, F_UPDATE_COV, F_UPDATE_LAMBDA, F_COV_HORIZON, F_FILTER_U, F_WORLDS, F_MODES, F_KNOTS, F_CONSTRAINT, F_ANNEAL,
               F_ESS, F_COUNT };
static const char* const kFeatureNames[] = {"mode cem", "mode smooth", "update_cov", "update_lambda", "cov_horizon", "filter_u", "n_worlds > 1",
                                            "n_modes > 1", "control_knots > 0", "constraint_mode", "annealed MPPI", "lambda_mode: ess"};
#define FBIT(f) (1u << (f))
static const unsigned F_CEM_SMOOTH = FBIT(F_CEM) | FBIT(F_SMOOTH), F_ADAPTIVE = FBIT(F_UPDATE_COV) | FBIT(F_UPDATE_LAMBDA);
struct Exclusion { Feature feature; unsigned excludes; const char* why; };     // excludes: FBIT mask; why: "" or the reason
static const Exclusion kExclusions[] = {
    {F_SMOOTH, F_ADAPTIVE, ""},
    {F_SMOOTH, FBIT(F_FILTER_U), " (the derivative is integrated, not smoothed)"},
    {F_CEM, F_ADAPTIVE, ""},
    {F_WORLDS, F_CEM_SMOOTH | FBIT(F_COV_HORIZON), ""},
    {F_MODES, F_CEM_SMOOTH | FBIT(F_WORLDS), ""},
    {F_MODES, F_ADAPTIVE, " (the adapted distribution belongs to one mean)"},
    {F_KNOTS, F_CEM_SMOOTH | F_ADAPTIVE | FBIT(F_MODES) | FBIT(F_WORLDS), ""},
    {F_KNOTS, FBIT(F_FILTER_U), ": the spline is smooth already, switch filter_u off"},
    {F_CONSTRAINT, F_CEM_SMOOTH | F_ADAPTIVE | FBIT(F_MODES) | FBIT(F_WORLDS) | FBIT(F_KNOTS), ""},
    {F_ANNEAL, FBIT(F_CEM), " (it has its own sigma)"},
    {F_ANNEAL, FBIT(F_SMOOTH) | F_ADAPTIVE | FBIT(F_KNOTS) | FBIT(F_CONSTRAINT), ""},
    {F_ANNEAL, FBIT(F_MODES), " (the Stein coupling's Sigma^-1 metric would need the schedule)"},
    {F_ESS, FBIT(F_UPDATE_LAMBDA), " (two rules for one temperature)"},
    {F_ESS, FBIT(F_COV_HORIZON), " (the shift computes lambda Sigma_H^-1 U before the temperature is known)"},
    {F_ESS, F_CEM_SMOOTH, " (it does not weight the samples with the temperature)"},
    {F_ESS, FBIT(F_WORLDS) | FBIT(F_MODES) | FBIT(F_KNOTS) | FBIT(F_CONSTRAINT) | FBIT(F_ANNEAL), ""},
};

int check_exclusions(const MppibParams& p, bool anneal, const char* who) {
    const bool on[] = {p.mode == MPPIB_MODE_CEM, p.mode == MPPIB_MODE_SMOOTH, p.update_cov != 0, p.update_lambda != 0, p.cov_horizon != 0,
                       p.filter_u != 0, p.n_worlds > 1, p.n_modes > 1, p.control_knots > 0, p.constraint_mode != 0, anneal, p.lambda_ess != 0};
    for (const Exclusion& e : kExclusions)
        for (int f = 0; f < F_COUNT; ++f)
            MPPIB_REQUIRE(!(on[e.feature] && on[f] && (e.excludes & FBIT(f))), "%s%s%s excludes %s%s", who, *who ? ": " : "", kFeatureNames[e.feature],
                          kFeatureNames[f], e.why);
    return 0;
}

static int validate(const MppibModel* m, const MppibParams* p) {
    MPPIB_REQUIRE(m != nullptr && p != nullptr, "null model/params");
    MPPIB_REQUIRE(m->abi_version == MPPIB_ABI_VERSION, "model abi_version %d != library %d", m->abi_version, MPPIB_ABI_VERSION);
    MPPIB_REQUIRE(m->nb >= 1 && m->nb <= MPPIB_MAX_BODIES, "nb=%d out of range", m->nb);
    MPPIB_REQUIRE(m->nlinks >= 0 && m->nlinks <= MPPIB_MAX_LINKS, "nlinks=%d out of range", m->nlinks);
    MPPIB_REQUIRE(m->nu >= 1 && m->nu <= MPPIB_MAX_NU, "nu=%d out of range", m->nu);
    MPPIB_REQUIRE(m->nfree >= 0 && m->nfree <= MPPIB_MAX_FREE && m->nshapes >= 0 && m->nshapes <= MPPIB_MAX_SHAPES, "nfree / nshapes out of range");
    for (int s = 0; s < m->nshapes; ++s) {
        MPPIB_REQUIRE(m->shape_slot[s] >= -1 && m->shape_slot[s] < MPPIB_MAX_SLOTS, "shape %d: contact slot out of range", s);
        if (m->shape_owner_kind[s] != MPPIB_OWNER_LINK) MPPIB_REQUIRE(m->shape_actor[s] >= 0 && m->shape_actor[s] < m->nactors, "shape %d: actor index out of range", s);
        if (m->shape_owner_kind[s] == MPPIB_OWNER_LINK) MPPIB_REQUIRE(m->shape_owner[s] >= -1 && m->shape_owner[s] < m->nb, "shape %d: body index out of range", s);
        if (m->shape_owner_kind[s] == MPPIB_OWNER_FREE) MPPIB_REQUIRE(m->shape_owner[s] >= 0 && m->shape_owner[s] < m->nfree, "shape %d: free body index out of range", s);
    }
    MPPIB_REQUIRE((m->nshapes == 0 && m->nfree == 0) || (m->max_contacts >= 1 && m->max_contacts <= MPPIB_MAX_CONTACTS), "max_contacts %d out of range 1..%d", m->max_contacts, MPPIB_MAX_CONTACTS);
    for (int f = 0; f < m->nfree; ++f) MPPIB_REQUIRE(m->free_actor[f] >= 0 && m->free_actor[f] < m->nactors && m->free_mass[f] > 0.f, "free body %d invalid", f);
    for (int i = 0; i < m->nb; ++i) {
        MPPIB_REQUIRE(m->parent[i] >= -1 && m->parent[i] < i, "parent[%d]=%d is not topologically sorted", i, m->parent[i]);
        MPPIB_REQUIRE(m->cmd_i0[i] >= 0 && m->cmd_i0[i] < m->nu && m->cmd_i1[i] >= 0 && m->cmd_i1[i] < m->nu, "cmd map of dof %d out of range", i);
    }
    MPPIB_REQUIRE(!m->planar_base || (m->nb >= 3 && m->nu >= 2), "planar_base needs three virtual joints and a (v, omega) command");
    MPPIB_REQUIRE(p->K >= 1, "K=%d must be positive", p->K);     // K % 4 == 0 is a requirement of the reduction only (checked there)
    MPPIB_REQUIRE(p->T >= 1 && p->substeps >= 1 && p->dt > 0.f, "bad T/substeps/dt");
    MPPIB_REQUIRE(p->lambda_ > 0.f, "lambda must be positive");
    MPPIB_REQUIRE(isfinite(p->gamma) && p->gamma >= 0.f, "gamma = %g must be finite and >= 0 (rollout_var_discount)", p->gamma);
    MPPIB_REQUIRE(!(p->filter_u && p->T < 9), "filter_u needs T >= 9");
    MPPIB_REQUIRE(p->nobs >= 0 && p->nobs <= MPPIB_MAX_OBS, "nobs out of range");
    if (p->update_cov || p->update_lambda)
        MPPIB_REQUIRE(p->step_size_cov >= 0.f && p->step_size_cov <= 1.f && p->kappa >= 0.f && p->lambda_mult >= 0.f && p->lambda_mult < 1.f,
                      "adaptive MPPI: step_size_cov %g, kappa %g or lambda_mult %g out of range", p->step_size_cov, p->kappa, p->lambda_mult);
    MPPIB_REQUIRE(!p->cov_full || p->update_cov, "cov_full selects the update rule of update_cov and needs update_cov");
    MPPIB_REQUIRE(!p->cov_horizon || (p->update_cov && !p->cov_full), "cov_horizon selects the update rule of update_cov: it needs update_cov and excludes cov_full");
    MPPIB_REQUIRE(!p->cov_horizon || p->T * m->nu <= MPPIB_HZ_MAX_N, "cov_horizon: n = T*nu = %d exceeds %d", p->T * m->nu, MPPIB_HZ_MAX_N);
    MPPIB_REQUIRE(p->mode >= MPPIB_MODE_SIMPLE && p->mode <= MPPIB_MODE_SMOOTH, "mode %d unknown", p->mode);
    if (p->mode == MPPIB_MODE_SMOOTH) {
        MPPIB_REQUIRE(isfinite(p->smooth_weight) && p->smooth_weight >= 0.f, "mode smooth: smooth_weight = %g must be finite and >= 0", p->smooth_weight);
        MPPIB_REQUIRE(p->dt > 0.f, "mode smooth: the integration step dt = %g must be positive", p->dt);
        for (int j = 0; j < m->nu; ++j)
            MPPIB_REQUIRE(p->du_min[j] <= p->du_max[j], "mode smooth: du_min[%d] = %g > du_max[%d] = %g", j, p->du_min[j], j, p->du_max[j]);
        MPPIB_REQUIRE(p->T <= 256 && p->T * m->nu <= 512, "mode smooth needs T <= 256 and T*nu <= 512, got T = %d, T*nu = %d", p->T, p->T * m->nu);
    }
    if (p->mode == MPPIB_MODE_CEM) {
        MPPIB_REQUIRE(p->n_elites >= 1 && p->n_elites <= MPPIB_CEM_MAX_ELITES, "mode cem: n_elites = %d out of range [1, %d]", p->n_elites, MPPIB_CEM_MAX_ELITES);
        MPPIB_REQUIRE(p->n_keep >= 0 && p->n_keep <= p->n_elites, "mode cem: n_keep = %d out of range [0, n_elites = %d]", p->n_keep, p->n_elites);
        MPPIB_REQUIRE(p->elite_alpha >= 0.f && p->elite_alpha <= 1.f, "mode cem: elite_alpha = %g outside [0, 1]", p->elite_alpha);
        MPPIB_REQUIRE(p->T <= 256 && p->T * m->nu <= 512, "mode cem needs T <= 256 and T*nu <= 512, got T = %d, T*nu = %d", p->T, p->T * m->nu);
        for (int j = 0; j < m->nu; ++j)
            for (int i = 0; i < m->nu; ++i) MPPIB_REQUIRE(i == j || p->sigma_chol[j * m->nu + i] == 0.f, "mode cem needs a diagonal noise_sigma");
    }
    if (p->n_worlds > 1) {
        const int R = p->n_worlds;
        MPPIB_REQUIRE(R <= MPPIB_MAX_WORLDS && (R & (R - 1)) == 0, "n_worlds = %d must be a power of two in 1 .. %d", R, MPPIB_MAX_WORLDS);
        MPPIB_REQUIRE(p->risk_tail >= 1 && p->risk_tail <= R, "risk_tail = %d out of range [1, n_worlds = %d]", p->risk_tail, R);
        MPPIB_REQUIRE(p->K % R == 0 && p->k_offset % (uint32_t)R == 0, "n_worlds = %d: the shard K = %d, k_offset = %u must be multiples of it", R,
                      p->K, p->k_offset);
    }
    MPPIB_REQUIRE(p->n_modes >= 0 && p->n_modes <= MPPIB_MAX_MODES, "n_modes = %d out of range [1, %d]", p->n_modes, MPPIB_MAX_MODES);
    MPPIB_REQUIRE(isfinite(p->mode_margin) && p->mode_margin >= 0.f, "mode_margin = %g must be finite and >= 0", p->mode_margin);
    if (p->n_modes > 1) {
        const int M = p->n_modes;
        MPPIB_REQUIRE(p->mode_samples >= 32, "n_modes = %d: mode_samples = %d must be at least 32 (a 32-sample tile straddles at most two modes)", M,
                      p->mode_samples);
        MPPIB_REQUIRE((uint64_t)p->k_offset + (uint64_t)p->K <= (uint64_t)M * (uint64_t)p->mode_samples,
                      "n_modes = %d: the shard [%u, +%d) exceeds n_modes * mode_samples = %d", M, p->k_offset, p->K, M * p->mode_samples);
        MPPIB_REQUIRE(p->T * m->nu <= 512, "n_modes > 1 needs T*nu <= 512, got %d", p->T * m->nu);
    }
    MPPIB_REQUIRE(p->control_knots >= 0, "control_knots = %d must be >= 0", p->control_knots);
    if (p->control_knots > 0) {
        const int P = p->control_knots, d = p->spline_degree;
        MPPIB_REQUIRE(d >= 1 && d <= MPPIB_MAX_SPLINE_DEGREE, "spline_degree = %d out of range [1, %d]", d, MPPIB_MAX_SPLINE_DEGREE);
        MPPIB_REQUIRE(P >= d + 1 && P <= p->T, "control_knots = %d out of range [spline_degree + 1 = %d, T = %d]", P, d + 1, p->T);
        MPPIB_REQUIRE(P * m->nu <= 512 && p->T <= 256, "control_knots needs P*nu <= 512 and T <= 256, got P*nu = %d, T = %d", P * m->nu, p->T);
    }
    MPPIB_REQUIRE(p->constraint_mode == 0 || p->constraint_mode == 1, "constraint_mode = %d must be 0 or 1", p->constraint_mode);
    if (p->constraint_mode) {
        MPPIB_REQUIRE(isfinite(p->constraint_tol) && p->constraint_tol >= 0.f, "constraint_tol = %g must be finite and >= 0", p->constraint_tol);
        MPPIB_REQUIRE(isfinite(p->constraint_lambda) && p->constraint_lambda > 0.f, "constraint_lambda = %g must be finite and > 0", p->constraint_lambda);
        // a tile carries T violation rows beside the cost rows: (T*nu + 2T) * 32 floats per ring stage, and K3 needs two stages
        MPPIB_REQUIRE(reduce_ws_stages(*p, m->nu, RULE_FEASIBLE) >= 2, "constraint_mode needs two ring stages of (T*nu + 2T) * 32 floats in "
                      "K3's shared memory; T = %d, nu = %d leaves room for fewer", p->T, m->nu);
    }
    MPPIB_REQUIRE(p->lambda_ess == 0 || p->lambda_ess == 1, "lambda_ess = %d must be 0 or 1", p->lambda_ess);
    if (p->lambda_ess)
        MPPIB_REQUIRE(isfinite(p->ess_target) && p->ess_target > 0.f && p->ess_target <= 1.f, "ess_target = %g must be finite and in (0, 1]", p->ess_target);
    if (int rc = check_exclusions(*p, false, "")) return rc;
    for (int i = 0; i < p->nobs; ++i) {
        const int kd = p->obs[i].kind, ix = p->obs[i].index;
        MPPIB_REQUIRE(kd >= 0 && kd <= MPPIB_OBS_CONTACT, "obs[%d].kind invalid", i);
        if (kd == MPPIB_OBS_LINK_STATE) MPPIB_REQUIRE(ix >= 0 && ix < m->nlinks, "obs[%d] link index %d out of range", i, ix);
        if (kd == MPPIB_OBS_FREE_STATE) MPPIB_REQUIRE(ix >= 0 && ix < MPPIB_MAX_FREE, "obs[%d] free body index %d out of range", i, ix);
        if (kd == MPPIB_OBS_CONTACT) MPPIB_REQUIRE(ix >= 0 && ix < MPPIB_MAX_SLOTS, "obs[%d] contact slot %d out of range", i, ix);
    }
    return 0;
}

static void derive(MppibContext* c) {
    int r = 0;
    for (int i = 0; i < c->params.nobs; ++i) r += obs_item_width(c->model, c->params.obs[i].kind);
    c->obs_rows = r;
    c->state_rows = 2 * c->model.nb + 13 * c->model.nfree;
}

static int alloc_scratch(MppibContext* c) {
    if (c->reduce_scratch) { cudaFree(c->reduce_scratch); c->reduce_scratch = nullptr; }
    c->reduce_max_ctas = c->num_sms * 4;
    const size_t P = ((size_t)partial_row_capacity(c->params, c->model.nu) + 3) & ~(size_t)3;   // rows padded to 16 bytes
    MPPIB_CHECK_CUDA(cudaMalloc(&c->reduce_scratch, sizeof(float) * P * c->reduce_max_ctas));
    if (!c->reduce_ticket) {
        MPPIB_CHECK_CUDA(cudaMalloc(&c->reduce_ticket, sizeof(unsigned int)));
        MPPIB_CHECK_CUDA(cudaMemset(c->reduce_ticket, 0, sizeof(unsigned int)));
    }
    return 0;
}

int check_anneal(const MppibContext* c, const char* who) {
    if (!c->anneal) return 0;
    MPPIB_REQUIRE(c->params.T == c->anneal_T, "%s: the annealing schedule was registered for T = %d, the parameter block has T = %d; register a schedule "
                  "for the new horizon (mppib_set_anneal)", who, c->anneal_T, c->params.T);
    return check_exclusions(c->params, true, who);
}

int check_spline(const MppibContext* c, const char* who) {
    const MppibParams& p = c->params;
    if (p.control_knots == 0) return 0;
    MPPIB_REQUIRE(c->spline != nullptr, "%s: control_knots = %d needs its spline table registered (mppib_set_spline)", who, p.control_knots);
    MPPIB_REQUIRE(c->spline_T == p.T && c->spline_P == p.control_knots && c->spline_d == p.spline_degree && c->spline_nu == c->model.nu,
                  "%s: the spline table was registered for (T, P, d, nu) = (%d, %d, %d, %d), the handle has (%d, %d, %d, %d); register a table "
                  "for the new block (mppib_set_spline)", who, c->spline_T, c->spline_P, c->spline_d, c->spline_nu, p.T, p.control_knots,
                  p.spline_degree, c->model.nu);
    MPPIB_REQUIRE(update_rule(c) == RULE_PLAIN, "%s: control_knots > 0 runs plain MPPI; register no distribution", who);
    return 0;
}

int check_constraint(const MppibContext* c, const char* who) {
    const MppibParams& p = c->params;
    if (!p.constraint_mode) {
        MPPIB_REQUIRE(c->viol == nullptr, "%s: a constraint buffer is registered but constraint_mode is 0; register none (mppib_set_constraint(h, NULL, NULL))", who);
        return 0;
    }
    MPPIB_REQUIRE(c->viol != nullptr, "%s: constraint_mode needs its violation buffer registered (mppib_set_constraint)", who);
    MPPIB_REQUIRE(c->viol_T == p.T && c->viol_K == p.K, "%s: the violation buffer was registered for (T, K) = (%d, %d), the handle has (%d, %d); register a "
                  "buffer for the new block (mppib_set_constraint)", who, c->viol_T, c->viol_K, p.T, p.K);
    MPPIB_REQUIRE(c->dist == nullptr, "%s: constraint_mode runs plain MPPI; register no distribution", who);
    return 0;
}

int check_temperature(const MppibContext* c, const char* who) {
    if (!c->params.lambda_ess) return 0;
    MPPIB_REQUIRE(c->dist != nullptr && c->temp != nullptr, "%s: lambda_mode ess needs a distribution (mppib_set_distribution) and a temperature "
                  "state (mppib_set_temperature) registered; without them K3 would weight with the fixed lambda_", who);
    return 0;
}

extern "C" {

int32_t mppib_abi_version(void) { return MPPIB_ABI_VERSION; }
const char* mppib_last_error(void) { return g_err; }

// the K2 mapping switches of the environment: MPPIB_K2_LANES=0 / MPPIB_K2_TEAM=0 turn a mapping off (the thread-per-rollout
// kernel as the reference of the other two)
static void read_mapping_knobs(MppibContext* c) {
    c->k2_lanes = true;
    if (const char* e = getenv("MPPIB_K2_LANES")) c->k2_lanes = atoi(e) != 0;
    c->k2_team = true;
    if (const char* e = getenv("MPPIB_K2_TEAM")) c->k2_team = atoi(e) != 0;
}

int32_t mppib_create(const MppibModel* model_h, const MppibParams* params_h, int32_t device, MppibHandle* out) {
    MPPIB_REQUIRE(out != nullptr, "null out handle");
    if (int rc = validate(model_h, params_h)) return rc;
    int ndev = 0;
    MPPIB_CHECK_CUDA(cudaGetDeviceCount(&ndev));
    MPPIB_REQUIRE(device >= 0 && device < ndev, "device %d not present (%d CUDA devices)", device, ndev);
    DeviceGuard guard(device);                   // the caller's current device is restored on return
    MPPIB_CHECK_CUDA(guard.err);
    cudaDeviceProp prop;
    MPPIB_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
    MPPIB_REQUIRE(prop.major == 9 && prop.minor == 0, "this library is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
    MppibContext* c = new MppibContext();
    memset(c, 0, sizeof(*c));
    c->device = device;
    c->model = *model_h;
    c->params = *params_h;
    c->num_sms = prop.multiProcessorCount;
    read_mapping_knobs(c);                                                      // read once per handle, not per launch
    derive(c);
    if (int rc = alloc_scratch(c)) { delete c; return rc; }
    if (int rc = alloc_horizon(c)) { cudaFree(c->reduce_scratch); cudaFree(c->reduce_ticket); delete c; return rc; }
    *out = c;
    return 0;
}

int32_t mppib_peer_close(MppibHandle h) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    bool any = false;
    for (int g = 0; g < MPPIB_MAX_PEERS; ++g) any = any || h->peer_win[g] != nullptr;
    if (!any) { h->peer_world = 0; return 0; }
    MPPIB_ON_DEVICE(h);
    cudaDeviceSynchronize();
    for (int g = 0; g < MPPIB_MAX_PEERS; ++g) {
        if (!h->peer_win[g]) continue;
        if (g == h->peer_rank) cudaFree(h->peer_win[g]); else cudaIpcCloseMemHandle(h->peer_win[g]);
        h->peer_win[g] = nullptr;
    }
    h->peer_world = 0; h->peer_rank = 0; h->peer_pcap = 0;
    return 0;
}

int32_t mppib_peer_alloc(MppibHandle h, int32_t world, int32_t rank, unsigned char* ipc_handle_out_h) {
    MPPIB_REQUIRE(h && ipc_handle_out_h, "mppib_peer_alloc: null argument");
    MPPIB_REQUIRE(world >= 2 && world <= MPPIB_MAX_PEERS && rank >= 0 && rank < world, "mppib_peer_alloc: world %d / rank %d out of range (max %d ranks)", world, rank, MPPIB_MAX_PEERS);
    static_assert(sizeof(cudaIpcMemHandle_t) == MPPIB_IPC_HANDLE_BYTES, "IPC handle size");
    mppib_peer_close(h);
    MPPIB_ON_DEVICE(h);
    const int P = partial_row_capacity(h->params, h->model.nu);
    const int pcap = ((P + 3) >> 2) << 2;
    void* win = nullptr;
    MPPIB_CHECK_CUDA(cudaMalloc(&win, peer_window_bytes(world, pcap)));
    MPPIB_CHECK_CUDA(cudaMemset(win, 0, peer_window_bytes(world, pcap)));
    MPPIB_CHECK_CUDA(cudaDeviceSynchronize());     // zeroed before the handle leaves this process
    cudaIpcMemHandle_t hd;
    cudaError_t e = cudaIpcGetMemHandle(&hd, win);
    if (e != cudaSuccess) { cudaFree(win); MPPIB_REQUIRE(false, "cudaIpcGetMemHandle: %s", cudaGetErrorString(e)); }
    memcpy(ipc_handle_out_h, &hd, sizeof(hd));
    h->peer_world = world; h->peer_rank = rank; h->peer_pcap = pcap;
    h->peer_win[rank] = win;
    const char* to = getenv("MPPIB_PEER_TIMEOUT_S");
    const double sec = to ? atof(to) : 20.0;
    h->peer_timeout_ns = (unsigned long long)((sec > 0.0 ? sec : 20.0) * 1e9);
    return 0;
}

int32_t mppib_peer_open(MppibHandle h, int32_t peer, const unsigned char* ipc_handle_h) {
    MPPIB_REQUIRE(h && ipc_handle_h, "mppib_peer_open: null argument");
    MPPIB_REQUIRE(h->peer_world >= 2, "mppib_peer_open: call mppib_peer_alloc first");
    MPPIB_REQUIRE(peer >= 0 && peer < h->peer_world && peer != h->peer_rank, "mppib_peer_open: peer %d out of range", peer);
    MPPIB_REQUIRE(h->peer_win[peer] == nullptr, "mppib_peer_open: peer %d is already open", peer);
    MPPIB_ON_DEVICE(h);
    cudaIpcMemHandle_t hd;
    memcpy(&hd, ipc_handle_h, sizeof(hd));
    void* win = nullptr;
    MPPIB_CHECK_CUDA(cudaIpcOpenMemHandle(&win, hd, cudaIpcMemLazyEnablePeerAccess));
    h->peer_win[peer] = win;
    return 0;
}

int32_t mppib_destroy(MppibHandle h) {
    if (!h) return 0;
    MPPIB_ON_DEVICE(h);
    mppib_peer_close(h);
    if (h->reduce_scratch) cudaFree(h->reduce_scratch);
    if (h->reduce_ticket) cudaFree(h->reduce_ticket);
    h->params.cov_horizon = 0;
    alloc_horizon(h);                            // frees the cov_horizon buffers
    delete h;
    return 0;
}

int32_t mppib_set_params(MppibHandle h, const MppibParams* params_h) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    if (int rc = validate(&h->model, params_h)) return rc;
    const bool resize = partial_row_capacity(*params_h, h->model.nu) != partial_row_capacity(h->params, h->model.nu);
    MPPIB_REQUIRE(h->peer_world <= 1 || partial_row_capacity(*params_h, h->model.nu) <= h->peer_pcap, "mppib_set_params: T*nu outgrows the open peer window; close and re-open the peers");
    h->params = *params_h;
    derive(h);
    MPPIB_ON_DEVICE(h);
    if (resize) if (int rc = alloc_scratch(h)) return rc;
    return alloc_horizon(h);
}

int32_t mppib_set_model(MppibHandle h, const MppibModel* model_h) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    if (int rc = validate(model_h, &h->params)) return rc;
    const bool resize = model_h->nu != h->model.nu;
    MPPIB_REQUIRE(h->peer_world <= 1 || partial_row_capacity(h->params, model_h->nu) <= h->peer_pcap, "mppib_set_model: T*nu outgrows the open peer window; close and re-open the peers");
    h->model = *model_h;
    derive(h);
    MPPIB_ON_DEVICE(h);
    if (resize) if (int rc = alloc_scratch(h)) return rc;
    return alloc_horizon(h);
}

int32_t mppib_state_size(MppibHandle h) { return h ? h->state_rows : -1; }
int32_t mppib_obs_size(MppibHandle h) { return h ? h->obs_rows : -1; }

int32_t mppib_sample(MppibHandle h, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total, const float* U,
                     const float* prior_row, float* actions, float* noise, void* stream) {
    if (int rc = k1_admit(h, K1_SAMPLE, U && actions, k_offset, k_total)) return rc;
    MPPIB_ON_DEVICE(h);
    return launch_sample(h, seed, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, actions, noise, (cudaStream_t)stream);
}

int32_t mppib_sample_spline(MppibHandle h, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                            const float* U, float* actions, float* xk, void* stream) {
    if (int rc = k1_admit(h, K1_SPLINE, U && actions && xk, k_offset, k_total)) return rc;
    MPPIB_ON_DEVICE(h);
    return launch_sample_spline(h, seed, plan_idx, plan_ctr, k_offset, k_total, U, actions, xk, (cudaStream_t)stream);
}

int32_t mppib_sample_colored(MppibHandle h, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                             const float* U, const float* prior_row, const float* Lt, float* actions, float* noise, void* stream) {
    if (int rc = k1_admit(h, K1_COLORED, U && Lt && actions, k_offset, k_total)) return rc;
    MPPIB_ON_DEVICE(h);
    return launch_sample_colored(h, seed, plan_idx, plan_ctr, k_offset, k_total, U, prior_row, Lt, actions, noise, (cudaStream_t)stream);
}

int32_t mppib_sample_smooth(MppibHandle h, uint64_t seed, uint64_t plan_idx, const uint32_t* plan_ctr, uint32_t k_offset, uint32_t k_total,
                            const float* U, float* actions, float* noise, void* stream) {
    if (int rc = k1_admit(h, K1_SMOOTH, U && actions, k_offset, k_total)) return rc;
    MPPIB_ON_DEVICE(h);
    return launch_sample_smooth(h, seed, plan_idx, plan_ctr, k_offset, k_total, U, actions, noise, (cudaStream_t)stream);
}

int32_t mppib_noise_library(MppibHandle h, uint32_t k_offset, uint32_t k_total, const int32_t* halton_tab, const float* B, int32_t n_knots,
                            float* Z, void* stream) {
    if (int rc = k1_admit(h, K1_NOISE_LIBRARY, halton_tab && B && Z, k_offset, k_total, n_knots)) return rc;
    MPPIB_ON_DEVICE(h);
    return launch_noise_library(h, k_offset, k_total, halton_tab, B, n_knots, Z, (cudaStream_t)stream);
}

int32_t mppib_sample_library(MppibHandle h, uint32_t k_offset, uint32_t k_total, const float* U, const float* prior_row, const float* Z,
                             float* actions, float* noise, void* stream) {
    if (int rc = k1_admit(h, K1_SAMPLE_LIBRARY, U && Z && actions, k_offset, k_total)) return rc;
    MPPIB_ON_DEVICE(h);
    return launch_sample_library(h, k_offset, k_total, U, prior_row, Z, actions, noise, (cudaStream_t)stream);
}

int32_t mppib_rollout(MppibHandle h, const float* state0, const float* root0, float* state, const float* actions, int32_t t0, int32_t nsteps,
                      float* obs, void* stream) {
    MPPIB_REQUIRE(h && actions, "mppib_rollout: null argument");
    MPPIB_REQUIRE(state0 || state, "mppib_rollout: need state0 (broadcast) or state (continue)");
    MPPIB_REQUIRE(t0 >= 0 && nsteps >= 0 && t0 + (nsteps > 0 ? nsteps : 1) <= h->params.T, "mppib_rollout: steps [%d,%d) outside horizon %d", t0, t0 + nsteps, h->params.T);
    MPPIB_ON_DEVICE(h);
    return launch_rollout(h, state0, root0, state, actions, t0, nsteps, obs, (cudaStream_t)stream);
}

int32_t mppib_reduce(MppibHandle h, const float* cost, const float* x, const float* U, float* partial, void* stream) {
    MPPIB_REQUIRE(h && cost && x && U && partial, "mppib_reduce: null argument");
    if (int rc = check_anneal(h, "mppib_reduce")) return rc;
    if (int rc = check_spline(h, "mppib_reduce")) return rc;
    if (int rc = check_constraint(h, "mppib_reduce")) return rc;
    if (int rc = check_temperature(h, "mppib_reduce")) return rc;
    MPPIB_REQUIRE(((uintptr_t)cost & 15) == 0 && ((uintptr_t)x & 15) == 0, "mppib_reduce: cost/x must be 16-byte aligned");
    MPPIB_ON_DEVICE(h);
    return launch_reduce(h, cost, x, U, partial, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int32_t mppib_reduce_finalize(MppibHandle h, const float* cost, const float* x, float* U, float* partial, float* action_out, float* stats, void* stream) {
    MPPIB_REQUIRE(h && cost && x && U && partial && action_out, "mppib_reduce_finalize: null argument");
    if (int rc = check_anneal(h, "mppib_reduce_finalize")) return rc;
    if (int rc = check_spline(h, "mppib_reduce_finalize")) return rc;
    if (int rc = check_constraint(h, "mppib_reduce_finalize")) return rc;
    if (int rc = check_temperature(h, "mppib_reduce_finalize")) return rc;
    MPPIB_REQUIRE(h->peer_world <= 1, "mppib_reduce_finalize is the single-GPU plan tail; with an open peer window use mppib_reduce + mppib_finalize");
    MPPIB_ON_DEVICE(h);
    return launch_reduce(h, cost, x, U, partial, U, action_out, stats, (cudaStream_t)stream);
}

int32_t mppib_finalize(MppibHandle h, const float* partials, int32_t G, float* U, float* action_out, float* stats, void* stream) {
    MPPIB_REQUIRE(h && U && action_out && G >= 1, "mppib_finalize: bad argument");
    if (int rc = check_anneal(h, "mppib_finalize")) return rc;
    if (int rc = check_spline(h, "mppib_finalize")) return rc;
    if (int rc = check_constraint(h, "mppib_finalize")) return rc;
    if (int rc = check_temperature(h, "mppib_finalize")) return rc;
    if (!partials) {
        MPPIB_REQUIRE(h->peer_world >= 2 && G == h->peer_world, "mppib_finalize: partials == NULL needs an open peer window and G == world (G=%d, world=%d)", G, h->peer_world);
        for (int g = 0; g < h->peer_world; ++g) MPPIB_REQUIRE(h->peer_win[g] != nullptr, "mppib_finalize: peer %d is not open", g);
    }
    MPPIB_ON_DEVICE(h);
    return launch_finalize(h, partials, G, U, action_out, stats, (cudaStream_t)stream);
}

int32_t mppib_rollout_mapping_for_model(const MppibModel* model_h) {
    if (!model_h) return -1;
    MppibContext* c = new MppibContext();       // host arithmetic only: no device is touched
    memset(c, 0, sizeof(*c));
    c->model = *model_h;
    read_mapping_knobs(c);
    const int mapping = rollout_mapping(c);
    delete c;
    return mapping;
}

int32_t mppib_rollout_mapping(MppibHandle h) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    return rollout_mapping(h);
}

int64_t mppib_rollout_smem_bytes(const MppibModel* model_h) {
    if (!model_h) return -1;
    return (int64_t)rollout_smem_bytes(*model_h);
}

int32_t mppib_set_action_mirror(MppibHandle h, float* mirror) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    h->action_mirror = mirror;
    return 0;
}

int32_t mppib_set_distribution(MppibHandle h, float* dist) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    h->dist = dist;
    return 0;
}

int32_t mppib_set_smooth_state(MppibHandle h, float* state) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    h->smooth = state;
    return 0;
}

int32_t mppib_set_anneal(MppibHandle h, float* state, int32_t n_iterations) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    if (state == nullptr) {
        h->anneal = nullptr; h->anneal_n = 0; h->anneal_T = 0;
        return 0;
    }
    MPPIB_REQUIRE(n_iterations >= 1 && n_iterations <= MPPIB_MAX_ANNEAL, "mppib_set_anneal: n_iterations = %d out of range [1, %d]", n_iterations,
                  MPPIB_MAX_ANNEAL);
    if (int rc = check_exclusions(h->params, true, "mppib_set_anneal")) return rc;
    h->anneal = state; h->anneal_n = n_iterations; h->anneal_T = h->params.T;
    return 0;
}

int32_t mppib_set_spline(MppibHandle h, float* table, int32_t P, int32_t d) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    if (table == nullptr) {
        h->spline = nullptr; h->spline_T = h->spline_P = h->spline_d = h->spline_nu = 0;
        return 0;
    }
    MPPIB_REQUIRE(P > 0 && P == h->params.control_knots && d == h->params.spline_degree,
                  "mppib_set_spline: (P, d) = (%d, %d) does not match the parameter block's (control_knots, spline_degree) = (%d, %d)", P, d,
                  h->params.control_knots, h->params.spline_degree);
    h->spline = table; h->spline_T = h->params.T; h->spline_P = P; h->spline_d = d; h->spline_nu = h->model.nu;
    return 0;
}

int32_t mppib_set_constraint(MppibHandle h, const float* viol, float* cstate) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    if (viol == nullptr) {
        h->viol = nullptr; h->cstate = nullptr; h->viol_T = h->viol_K = 0;
        return 0;
    }
    MPPIB_REQUIRE(cstate != nullptr, "mppib_set_constraint: the constraint state (n_feasible, min V) is needed with a violation buffer");
    MPPIB_REQUIRE(h->params.constraint_mode, "mppib_set_constraint: the parameter block has constraint_mode = 0");
    MPPIB_REQUIRE(((uintptr_t)viol & 15) == 0, "mppib_set_constraint: viol must be 16-byte aligned");
    h->viol = viol; h->cstate = cstate; h->viol_T = h->params.T; h->viol_K = h->params.K;
    return 0;
}

int32_t mppib_set_temperature(MppibHandle h, float* state) {
    MPPIB_REQUIRE(h != nullptr, "null handle");
    h->temp = state;
    return 0;
}

int32_t mppib_temperature(MppibHandle h, const float* cost, const float* x, const float* U, float* row, int32_t solve, void* stream) {
    MPPIB_REQUIRE(h && cost && U && row && (x || h->params.mode != MPPIB_MODE_SIMPLE), "mppib_temperature: null argument");
    MPPIB_REQUIRE(h->params.lambda_ess, "mppib_temperature: the parameter block has lambda_ess = 0");
    if (int rc = check_temperature(h, "mppib_temperature")) return rc;
    if (solve && h->peer_world > 1)
        for (int g = 0; g < h->peer_world; ++g) MPPIB_REQUIRE(h->peer_win[g] != nullptr, "mppib_temperature: peer %d is not open", g);
    MPPIB_ON_DEVICE(h);
    return launch_temperature(h, cost, x, U, row, solve != 0, (cudaStream_t)stream);
}

int32_t mppib_temperature_solve(MppibHandle h, const float* rows, int32_t G, void* stream) {
    MPPIB_REQUIRE(h && rows && G >= 1, "mppib_temperature_solve: bad argument");
    MPPIB_REQUIRE(h->params.lambda_ess, "mppib_temperature_solve: the parameter block has lambda_ess = 0");
    if (int rc = check_temperature(h, "mppib_temperature_solve")) return rc;
    MPPIB_ON_DEVICE(h);
    return launch_temperature_solve(h, rows, G, (cudaStream_t)stream);
}

int32_t mppib_shift(MppibHandle h, float* U, uint32_t* plan_ctr, void* stream) {
    MPPIB_REQUIRE(h && U, "mppib_shift: null argument");
    if (int rc = check_anneal(h, "mppib_shift")) return rc;
    if (int rc = check_spline(h, "mppib_shift")) return rc;
    MPPIB_ON_DEVICE(h);
    return launch_shift(h, U, plan_ctr, (cudaStream_t)stream);
}

int32_t mppib_cost_pose(int64_t n, const float* a, int64_t a_si, int64_t a_sr, const float* b, int64_t b_si, int64_t b_sr, float w_pos, float w_ori,
                        float* cost, int32_t accumulate, void* stream) {
    MPPIB_REQUIRE(n >= 0 && a && cost && (b || w_pos == 0.f), "mppib_cost_pose: null argument");
    return launch_cost_pose(n, a, a_si, a_sr, b, b_si, b_sr, w_pos, w_ori, cost, accumulate, (cudaStream_t)stream);
}

}  // extern "C"
