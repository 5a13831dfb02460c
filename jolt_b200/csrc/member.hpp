// Internals shared by the sumcheck-member translation units (member.cu, resident.cu, capi.cu).
#pragma once
#include <cstring>
#include <ctime>
#include <vector>

#include "ctx.hpp"
#include "expr_pass.cuh"
#include "host_fr.hpp"
#include "poly_kernels.cuh"
#include "resident.cuh"

namespace jbi {

using jb::BindScalar;
using jb::HostFr;

inline uint64_t now_ns() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec;
}

inline BindScalar make_scalar(const uint64_t r[4], bool* hi4) {
    BindScalar s;
    for (int i = 0; i < 4; ++i) {
        s.w[2 * i] = (uint32_t)r[i];
        s.w[2 * i + 1] = (uint32_t)(r[i] >> 32);
    }
    *hi4 = (r[0] == 0 && r[1] == 0);
    return s;
}

inline bool canonical_fr(const uint64_t r[4]) { return !HostFr::geq_p(r); }

// The kernel-parameter form of `count` <= EQ_BLOCK_VARS coordinates (HOST limbs r) and an optional host scale.
inline jb::EqVars eq_vars(const uint64_t* r, size_t count, const uint64_t* scale) {
    jb::EqVars v;
    std::memset(&v, 0, sizeof v);
    for (size_t j = 0; j < count; ++j)
        for (int w = 0; w < 4; ++w) {
            v.r[j][2 * w] = (uint32_t)r[4 * j + w];
            v.r[j][2 * w + 1] = (uint32_t)(r[4 * j + w] >> 32);
        }
    if (scale) {
        v.has_scale = 1;
        for (int w = 0; w < 4; ++w) {
            v.scale[2 * w] = (uint32_t)scale[w];
            v.scale[2 * w + 1] = (uint32_t)(scale[w] >> 32);
        }
    }
    return v;
}

// Launches one round of a per-round sumcheck kernel over `pairs` pair indices: `kernel(args..., out)`, whose blocks
// each leave `values` partial sums in the context's partial buffer for the last block to fold. `kind` and `m` label
// the timed launch (jb_ctx::timing_begin), `what` names a launch error.
template <typename Kernel, typename... Args>
int launch_round(jb_ctx* c, Kernel kernel, int block, size_t smem, int per_sm, size_t pairs, int values, int kind, int m,
                 const char* what, jb::RoundOut out, const Args&... args) {
    const unsigned grid = launch_grid(c, pairs, block, per_sm);
    int st = c->ensure_partial((size_t)grid * values);
    if (st != JB_OK) return st;
    out.partial = c->d_partial;
    int tix = c->timing_begin(kind, pairs, m);
    // latency path: a round of <= 32 pairs runs as one warp (no barriers, no shared-memory stage)
    kernel<<<grid, pairs <= 32 ? 32u : (unsigned)block, smem, c->stream>>>(args..., out);
    c->timing_end(tix);
    c->launches++;
    return c->check(cudaGetLastError(), what);
}

// capi.cu
int bind_table(jb_ctx* c, Table& t, const uint64_t r[4], int order);  // Polynomial::bind_with_order on one table
int eq_build(jb_ctx* c, const uint64_t* r, size_t nvars, const uint64_t* scale, uint64_t* d_out);

// Accumulates the host time spent waiting for a round result (jb_ctx_diag).
struct WaitAcc {
    jb_ctx* c;
    uint64_t t0;
    explicit WaitAcc(jb_ctx* ctx) : c(ctx), t0(now_ns()) {}
    ~WaitAcc() {
        c->diag_wait_ns += now_ns() - t0;
        c->diag_waits++;
    }
};

}  // namespace jbi

// A source of an expression member before its bind (jb_member_create_expr_sources): what the source pass reads.
struct SourceCol {
    int type = JB_SOURCE_TABLE;
    int kind = 0;
    void* values = nullptr;    // member-owned copy of the column (COMPACT / ONE_HOT)
    uint64_t* eq = nullptr;    // ONE_HOT: eq(r_addr, .), K entries
    uint32_t K = 0;
};

// What a member proves, fixed when it is created. The kind decides which pass serves a round, how many tables the
// member reports and where their final values lie; eq weighting and index sharding are properties on top of it.
enum class MemberKind {
    Dense,       // a product or sum of products over field tables (also an expression that is exactly such a shape)
    Expr,        // the expression pass over tables or sources (ex)
    Product,     // the product of m <= 16 tables or sources (terms = 1) through product_round_kernel
    ReadWrite,   // read-write checking (rw): sparse rounds, then the expression pass over the remaining tables
    Booleanity,  // booleanity (bl): address rounds, then cycle rounds
};

// One ProveRounds member on the device (~ Box<dyn SumcheckKernel>): the relation
//   sum_x sum_{k<P} prod_{j<D} f_{kD+j}(x)       (degree D, T = D * P dense tables)
// optionally weighted by a split eq polynomial, optionally index-sharded over ranks.
struct jb_member {
    jb_ctx* ctx;
    MemberKind kind = MemberKind::Dense;
    std::vector<Table> tables;
    int m;       // D: factors per term = degree of the (unweighted) relation
    int terms = 1;  // P
    int order;
    size_t rounds;  // total (for a sharded member: local rounds + log2(world))
    size_t len;     // current (local) table length
    size_t rounds_done = 0;  // prove_round calls completed
    // index-sharded member (SURVEY 8e): this rank holds the contiguous block `rank` of the global
    // tables; rounds run with one all-reduce each until the shard is `gather_len` long, then the
    // shards are all-gathered into `tail`, which finishes the remaining rounds locally.
    bool sharded = false;
    size_t gather_len = 0;
    jb_member* tail = nullptr;
    bool gathered = false;  // the shards were gathered inside the resident kernel: the member continues un-sharded
    // split-eq member (GruenSplitEqPolynomial, crates/jolt-poly/src/split_eq.rs:159-447): the relation is
    // sum_x eq(w, x) prod_j f_j(x); eq is never materialised - per round the sweep is weighted by
    // E_out (x) E_in over the not-yet-current variables and the current variable's linear factor
    // l(t) = scalar * ((1 - w_cur) + t (2 w_cur - 1)) is multiplied in on the host.
    bool eq = false;
    size_t eq_n = 0, eq_split = 0;
    std::vector<uint64_t> eq_w;        // n elements, w[0] <-> most significant index bit
    uint64_t eq_scalar[4] = {0, 0, 0, 0};
    uint64_t* eq_tabs = nullptr;       // prefix tables Eo[k] (k <= split) then Ei[k] (k <= n-1-split), table k at 2^k - 1
    size_t eq_in_base = 0;             // element offset of the Ei family
    std::vector<size_t> eq_hi_off, eq_lo_off;  // HighToLow: element offsets of the suffix tables (see jb_eq_member_create)
    // resident service (resident.cuh): the launched kernel that serves this member's rounds from a mailbox
    ResidentRun* run = nullptr;
    int run_idx = 0;
    bool no_resident = false;  // a run of this member was stopped to make room for other work: stay on launches
    bool has_final = false;
    uint64_t final_vals[jb::JB_MAX_TABLES * 4];
    // lookahead (thin rounds, resident.cuh): the sums S0..S5 that determine round `look_round`'s polynomial as a
    // function of the challenge that round binds - harvested from the answer to the previous round's command
    bool look_ok = false;
    size_t look_round = 0;
    uint64_t look[6 * 4];
    // a round answered from lookahead sums with no command: its challenge is bound by the member's next command
    // (RES_ACT_BIND2_EVAL), or - when the run ends first - by launches as the run is released. len and the tables
    // do not include it.
    bool pend = false;
    uint64_t pend_r[4];
    // Expr (jb_member_create_expr): the summand is ex's weighted monomials over the tables (m = the largest monomial
    // degree, `terms` unused); also a ReadWrite member's address rounds
    jb::ExprParams ex;
    // an Expr or Product member over sources (jb_member_create_*_sources): until the sources are bound, src[j]
    // describes table j - a compact or one-hot source reads its member-owned column and its Table's buffer is where the
    // bind writes the len/2 field entries. Cleared (and the columns released) by the bind.
    std::vector<SourceCol> src;
    // ReadWrite (jb_member_create_read_write): the sparse cycle phase until the last cycle variable is bound, then the
    // expression pass over the A + 2 K-entry tables ra_0 .. ra_{A-1}, Val, inc (RwState::cycles); with p < t cycle
    // rounds first: p sparse cycle rounds, the sparse address rounds, then the eq-weighted expression pass over the
    // A + 2 tables over the remaining rows
    struct RwState* rw = nullptr;
    // Booleanity (jb_member_create_booleanity): its d tables live in bl, not in `tables`
    struct BoolState* bl = nullptr;
    int ntables() const;  // the tables the member reports (final_evals, export_table)
};

// A new member with the fields every kind sets, and rounds = log2(len) (len a power of two); null when out of memory.
jb_member* new_member(jb_ctx* c, MemberKind kind, int m, int terms, int order, size_t len);

// The split-eq weight tables of a round (e_out[y >> in_bits] * e_in[y & mask]).
struct EqWeights {
    const uint64_t* e_out;
    const uint64_t* e_in;
    int in_bits;
};

// read_write.cu ----------------------------------------------------------------------------------------------
constexpr int RW_MAX_ACCESSES = JB_RW_MAX_ACCESSES;
// The sparse phases of a read-write checking member: the bound K x T matrix as entries in two buffers that take turns
// as the input and the output of a bind. Per entry and buffer: key and row (u32), the field arrays ra_0 .. ra_{A-1},
// val, vs (Val before the row's block of cycles) and ve (Val after it). The cycle phase keeps the entries sorted by
// (row, key) and pairs rows; with p < t cycle rounds first the address phase then re-sorts them by (key, row) and pairs
// keys (by_key; vs is unused).
struct RwState {
    bool cycles = true;  // the sparse phases; cleared when the member's tables hold the expression pass's tables
    bool by_key = false; // the address phase of a mixed order (p < t)
    int A = 0, w = 0;
    uint64_t coeff[RW_MAX_ACCESSES][4];
    int d[RW_MAX_ACCESSES];
    size_t T = 0, K = 0;
    size_t p = 0;      // cycle rounds before the address rounds (t: every cycle round first)
    size_t kappa = 0;  // log2 K
    size_t rows = 0;  // groups of the bound matrix: rows (T >> cycle variables bound), or keys in the address phase
    size_t n = 0;     // live entries
    size_t cap = 0;   // entries a buffer holds: min(K, distinct address columns) * T, which no bind exceeds
    int cur = 0;      // the buffer holding the current matrix
    uint32_t* key[2] = {nullptr, nullptr};
    uint32_t* row[2] = {nullptr, nullptr};
    uint64_t* f[2] = {nullptr, nullptr};    // (A + 3) x cap field elements
    uint32_t* off[2] = {nullptr, nullptr};  // group offsets, groups + 1
    uint32_t* flag = nullptr;               // cap + 1: the scan input (the sort's input permutation)
    uint32_t* base = nullptr;               // cap + 1: the scan output (the sort's output permutation)
    void* scan_tmp = nullptr;               // the scan's and the sort's workspace
    size_t scan_bytes = 0;
    Table inc;   // inc(j) over the rows, bound alongside
    Table init;  // the K initial values, bound by the address rounds of a mixed order
};
// Checks and builds a read-write member without its eq factor (eq_setup adds it); nothing stays allocated on failure.
int rw_create(jb_ctx* c, const jb_rw_access* acc, size_t A, size_t w, int addr_kind, int addr_on_device, size_t T,
              size_t K, const jb_source* inc, const jb_source* init, const uint64_t* w_cycle, size_t nvars,
              const uint64_t* scale, size_t cycle_rounds_first, int order, jb_member** out);
// One cycle round: binds `bind` (if given), then the pass that leaves q(0), q(inf) in result slot ro.
int rw_cycle_round(jb_member* mem, const uint64_t* bind, const EqWeights& eqw, jb::RoundOut ro);
// Binds one cycle variable; after the last one the remaining row is scattered into the member's K-entry tables and
// the cycle-phase buffers are released.
int rw_cycle_bind(jb_member* mem, const uint64_t r[4]);
// Mixed order, after the p-th cycle bind: the entries re-sorted by (key, row) with their key offsets.
int rw_begin_keys(jb_member* mem);
// An address round's pass: leaves the unscaled q(0), q(1), q(inf) in result slot ro; eqw and w_low (the lowest row
// variable's coordinate) give the row weights eq(w[0 .. t - p), row).
int rw_key_pass(jb_member* mem, const EqWeights& eqw, const uint64_t* w_low, jb::RoundOut ro);
// Binds one address variable; after the last one the remaining key becomes the dense tables ra_a, Val, inc over the
// T / 2^p rows and the sparse buffers are released.
int rw_key_bind(jb_member* mem, const uint64_t r[4]);
void rw_release(jb_member* mem);

// booleanity.cu ----------------------------------------------------------------------------------------------
constexpr int BOOL_MAX_POLYS = JB_BOOL_MAX_POLYS;
// The state of a booleanity member. Address phase: G_i (bound linearly) and Q_i (bound by the squared rule) as d
// tables packed at the current length in gq[cur] (G then Q), the other buffer receiving the next bind; eq_rest holds
// eq over the address coordinates after the current one, one table per address round. Cycle phase: F = eq(rho_addr, .)
// and the member's copy of the columns until cycle round 1 binds them into h[0] (d tables at stride T / 2);
// LowToHigh binds alternate between h[0] and h[1] (stride T / 4), HighToLow binds h[0] in place.
struct BoolState {
    int d = 0, kind = 0, order = 0;
    size_t T = 0, K = 0, log_k = 0, log_t = 0;
    uint64_t coeff[BOOL_MAX_POLYS][4];
    std::vector<uint64_t> r_addr;  // log_k coordinates, r_addr[0] <-> MSB
    std::vector<uint64_t> rho;     // the address challenges bound so far, in binding order
    size_t klen = 0;               // address phase: current table length (0 once the cycle phase began)
    int gq_cur = 0;
    uint64_t* gq[2] = {nullptr, nullptr};  // 2 d K and 2 d K / 2 elements
    uint64_t* eq_rest = nullptr;           // K - 1 elements: round m's table at K - 2^(log_k - m)
    uint64_t* F = nullptr;                 // K elements
    void* cols = nullptr;                  // d x T addresses (member-owned), until cycle round 1
    size_t hlen = 0;                       // cycle phase: current table length (T while the columns are unbound)
    int h_cur = 0;
    uint64_t* h[2] = {nullptr, nullptr};
    size_t h_stride[2] = {0, 0};
};
// Checks and builds a booleanity member without its cycle eq factor (the caller adds it); nothing stays allocated on
// failure.
int bool_create(jb_ctx* c, const void* const* columns, size_t count, int kind, int on_device, size_t T, size_t K,
                const uint64_t* coeffs, const uint64_t* r_addr, const uint64_t* r_cycle, const uint64_t* scale,
                int order, jb_member** out);
// The address coordinate that address round m binds.
const uint64_t* bool_addr_coord(const BoolState& bl, size_t m);
// Address round m: binds `bind` (if given; the previous address variable) into G and Q, then the pass that leaves
// q(0), q(inf) in result slot ro.
int bool_address_pass(jb_member* mem, const uint64_t* bind, size_t m, jb::RoundOut ro);
// The end of the address phase: rho gets the last address challenge (if any), F = eq(rho_addr, .) is built and the
// address tables are released.
int bool_begin_cycles(jb_member* mem, const uint64_t* last_addr_challenge);
// A cycle round: binds `bind` (if given), then the pass that leaves q(0), q(inf) in result slot ro.
int bool_cycle_pass(jb_member* mem, const uint64_t* bind, const EqWeights& eqw, jb::RoundOut ro);
// The terminal bind (two entries per table left): a cycle variable, or the last address variable when T = 1.
int bool_finish(jb_member* mem, const uint64_t r[4]);
// Where ra_i's single entry lies once the member is fully bound.
const uint64_t* bool_final_entry(const jb_member* mem, int i);
void bool_release(jb_member* mem);
inline int jb_member::ntables() const { return kind == MemberKind::Booleanity ? bl->d : (int)tables.size(); }

// mle_eval.cu ------------------------------------------------------------------------------------------------
// G_p[k] = sum_{j: addr_p(j) = k} eq(r_cycle, j) for count device address columns into out[p] (K elements each);
// JB_ERR_INVALID (fail_bad_address) for an address >= K that is not none. Waits for the device.
int one_hot_pushforward_into(jb_ctx* c, const void* const* dev_columns, size_t count, int kind, size_t T, size_t K,
                             const uint64_t* r_cycle, uint64_t* const* out);

// product.cu -------------------------------------------------------------------------------------------------
// One round of a product member: in / out are the member's m table pointers as member_round prepared them (null in
// for a source read from its column); eqw: the split-eq weights (then skip1 is set). Rounds 0 and 1 read the sources.
int product_round(jb_ctx* c, const jb_member* mem, const uint64_t* const* in, uint64_t* const* out, const EqWeights* eqw,
                  bool skip1, size_t pairs, bool bind, bool hi4, const jb::BindScalar& s, jb::RoundOut ro);
// The terminal bind of a product member whose sources are still unbound (len = 2).
int product_finish(jb_member* mem, const uint64_t r[4]);

// sources.cu -------------------------------------------------------------------------------------------------
// The source pass of rounds 0 (bind == false) and 1 (bind: the sources are bound into their Tables' buffers, field
// tables as tp says). ex carries the round's points.
int sources_round(jb_ctx* c, const jb_member* mem, bool weighted, const jb::TablePtrs& tp, size_t pairs, bool bind,
                  const jb::BindScalar& s, const jb::ExprParams& ex, jb::RoundOut out);
// The terminal bind of a member whose sources are still unbound (len = 2): every table and source to one entry.
int sources_finish(jb_member* mem, const uint64_t r[4]);
// Releases the columns and eq tables of the sources (after their bind, or when the member is destroyed).
void sources_release(jb_member* mem);
// The one-hot eq table of a source and the check of its addresses.
int sources_one_hot_eq(jb_ctx* c, SourceCol& s, size_t len, const uint64_t* r_addr, size_t log_k, unsigned int* d_flag);

// resident.cu ------------------------------------------------------------------------------------------------
// Whether a resident kernel may serve the member's kind: Dense without split-eq weighting (resident_eligible also
// asks the member's current state).
inline bool resident_kind(const jb_member* mem) { return mem->kind == MemberKind::Dense && !mem->eq; }
// Starts a resident kernel serving `n` members (same D, P, order, same context; n <= RES_MAX_MEMBERS). Members
// must be plain (not eq / sharded-with-tail). `exchange`: the kernel may be asked to all-reduce member 0's sums
// over peer memory (sharded rounds). JB_ERR_UNSUPPORTED = not eligible (caller falls back to launches).
// first_len: entries of the largest pass a single-member run will be asked for (0 = the member's current length);
// may_evict: stop other runs of the context if the device cannot hold this one next to them (false:
// JB_ERR_UNSUPPORTED instead).
int resident_begin(jb_ctx* c, jb_member** mems, int n, uint64_t first_len = 0, bool may_evict = true);
// What a consumed command had asked of member i of the run.
struct ResConsumed {
    unsigned act = 0;       // RES_ACT_*
    bool thin = false;      // the answer carries the 8 thin sums (x 17 lanes) instead of K sums
    size_t round = 0;       // member-local round the command proved
    uint64_t nprime = 0;    // entries of the tables the round swept (after its bind)
};
// One launched resident_rounds_kernel and the members it serves.
struct ResidentRun {
    jb_ctx* c = nullptr;
    TailRes res;
    jb::ResMailbox* mb = nullptr;  // host view of the mailbox
    uint64_t seq = 0;          // commands posted
    uint64_t consumed = 0;     // answers consumed (<= seq <= consumed + 2: the mailbox is a ring of two)
    int n = 0;
    jb_member* mem[jb::RES_MAX_MEMBERS] = {nullptr};
    unsigned grid = 0;
    ResConsumed ring[2][jb::RES_MAX_MEMBERS];  // what command s (slot s & 1) asked of every member
    uint64_t ring_challenge[2][4];             // ... and the challenge it carried (to replay it if the kernel is lost)
    uint64_t ring_challenge2[2][4];            // ... and the one a RES_ACT_BIND2_EVAL binds first
    bool fuse = false;                         // staged run: large rounds may be folded into the next pass (res_fusable)
    bool ring_gather[2] = {false, false};      // ... and whether it was a gather (not replayable)
    std::vector<Table> deferred;               // shard buffers a gather made obsolete: freed when the run ends
    struct RoundInfo { int kind; uint64_t items; int m; };
    RoundInfo info[64];                       // what command s (< 64) asked for, for the device-timed pass log
    uint64_t host_post[64], host_recv[64];    // CLOCK_MONOTONIC ns (diagnostics)
    bool kernel_live = false;
    bool exclusive = false;  // holds more than half of the device's block slots: other kernels may starve
};

// The mailbox is a ring of two commands. post: actions[i] in RES_ACT_* (challenge may be null when no action binds);
// the host's view of the tables (len, ping-pong) advances at once - the device executes commands in order.
// consume: waits for the OLDEST unanswered command; `out` (may be null) receives n x RES_SLOT_U64 mailbox words per
// member (lanes, see resident.cuh; with `exchange` member 0's lanes are all-reduced over the ranks), `info` what
// the command had asked. The run is released when every member is fully bound and nothing is in flight (the run
// pointer is dead after that: check mem->run). round = drain + post + consume.
// gather (single-member run of an index-sharded member, action BIND_EVAL): bind, scatter the bound shard into every
// rank's arena and sweep the gathered tables; afterwards the member's tables ARE its arena views (len x world).
// RES_ACT_BIND2_EVAL binds challenge2 (the member's pending challenge, cleared here), then challenge; `look` sets
// RES_FLAG_LOOK (the command's EVAL actions are large passes that return lookahead sums).
int resident_post(ResidentRun* run, const unsigned* actions, const uint64_t* challenge, bool exchange, bool gather = false,
                  const uint64_t* challenge2 = nullptr, bool look = false);
bool resident_gather_fits(const jb_ctx* c, const jb_member* mem, uint64_t shard_len_after_bind);
int resident_consume(ResidentRun* run, uint64_t* out, ResConsumed* info);
int resident_inflight(const ResidentRun* run);
// resident_consume returns JB_RES_LOST when the kernel gave up waiting for commands (the host was held up for
// ~10 s: a debugger, a tool patching a module, an absorb callback that blocks) and exited WITHOUT executing the
// commands still in flight. The tables are consistent at the last executed round. resident_recover then replays
// the unexecuted commands' binds with ordinary launches (the host's view of the tables is exact again), releases the
// run and marks its members for one launch per round; the caller recomputes the current round's sums with an
// eval-only launch. A member never fails because its resident kernel went away.
constexpr int JB_RES_LOST = -1000;
int resident_recover(ResidentRun* run);
int resident_round(ResidentRun* run, const unsigned* actions, const uint64_t* challenge, bool exchange, uint64_t* out);
int resident_run_size(const ResidentRun* run);
// Stops the kernel (if it still runs), orders the context's stream after it and detaches the members.
void resident_end(ResidentRun* run, bool mark_no_resident);
bool resident_eligible(const jb_member* mem);
