/*
 * ssw_engine.cu -- host side of the batched aligner: planning, device buffers,
 * kernel launches and result assembly.  It is the batched equivalent of the
 * reference's ssw_align orchestrator (src/ssw.c:855-977):
 *
 *   P1  forward fill, byte semantics first when a byte profile exists, re-run
 *       with word semantics on overflow            (ssw.c:881-899)
 *   --  score <= 0 / flag gating                    (ssw.c:900-916)
 *   P2  reverse fill on the reversed query prefix with early termination
 *                                                   (ssw.c:919-936)
 *   P3  banded traceback + CIGAR re-scoring + retry (ssw.c:938-973)
 *
 * Nothing here computes alignments on the CPU; all DP work is in the kernels.
 */
#include <algorithm>
#include <exception>
#include <mutex>
#include <vector>
#include <string>
#include <string.h>
#include <math.h>
#include <functional>
#include <map>
#include <utility>

#include "ssw_common.cuh"
#include "ssw_host.h"
#include "ssw_fill.cuh"
#include "ssw_resolve.cuh"
#include "ssw_traceback.cuh"
#include "ssw_emul.cuh"
#include "ssw_grid.cuh"
#include "ssw_text.cuh"
#include "ssw_mark.cuh"
#include "ssw_hits.h"
#include "../../include/ssw_batch.h"

#include <chrono>
#include <memory>
#include <thread>
namespace {

static bool ssw_trace_on() { static int v = -1; if (v < 0) { const char* e = getenv("SSW_TRACE"); v = e && *e && *e != '0'; } return v != 0; }
struct Trace {
	std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
	void lap(const char* what) {
		if (!ssw_trace_on()) return;
		auto t1 = std::chrono::steady_clock::now();
		fprintf(stderr, "[libssw-b200 trace] %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(t1 - t0).count());
		t0 = t1;
	}
};

/* kernel instance = (lanes per group, rows per lane); rows covered = G*R.  Forward instances favour many rows per
 * lane (fewer shuffles and profile loads per cell).  `fwd`: a candidate of the automatic forward choice (pick_inst).
 * The index of an instance is its "inst" option value and the number earlier measurements quote: new ones are appended. */
struct Inst { int G, R; bool fwd; };
static constexpr Inst kInst[] = {
	{8, 4, true}, {8, 5, true}, {8, 8, true}, {8, 10, true}, {8, 16, true}, {8, 20, true},        /* 0..9: forward, by rows */
	{16, 16, true}, {16, 20, true}, {32, 16, true}, {32, 20, true},
	{32, 4, false}, {32, 5, false}, {32, 8, false}, {32, 10, false},                              /* 10..13: one alignment per warp (reverse pass, latency path) */
	{16, 19, true},                                                                               /* 14: forward, 304 rows (300 aa queries in word mode: 5 % fewer rows than (16,20)) */
	{8, 19, true},                                                                                /* 15: forward, 152 rows (150 bp reads on their word rows: 5 % fewer rows than (8,20)) */
};
static constexpr int kNumInst = (int)(sizeof(kInst) / sizeof(kInst[0]));
static int inst_rows(int inst) { return kInst[inst].G * kInst[inst].R; }

/* f(InstT<G, R>{}) with the (G, R) of instance `inst`: the one place where a runtime index becomes a kernel instance
 * (-1: no such instance) */
template <int G_, int R_> struct InstT { static constexpr int G = G_, R = R_; };
template <class F, size_t... I>
static int visit_inst(int inst, F&& f, std::index_sequence<I...>)
{
	int rc = -1;
	(void)((inst == (int)I && (rc = f(InstT<kInst[I].G, kInst[I].R>{}), true)) || ...);
	return rc;
}
template <class F>
static int visit_inst(int inst, F&& f) { return visit_inst(inst, f, std::make_index_sequence<kNumInst>{}); }

/* Tuning knobs ("ssw_engine_set_option"); every engine has its own copy (helper engines get their parent's). */
#define SSW_MAX_SLICES 8
/* A reference of at most this many columns is one item of the device-planned grid (one chunk from column 0, no warm-up).
 * Nothing in the fill or the resolve step depends on the length of an item (32-bit positions, one column-maximum word per
 * column); the bound is the tail of a launch, whose last item cannot be cut: 65,536 columns are a few milliseconds, and
 * no known protein is longer.  Longer references are chunked by the general path. */
#define SSW_GRID_MAX_REF 65536
struct SswOptions {
	int slices = 0;                 /* "slices": 0 automatic, 1 never slice a batch over helper engines, 2..8 forced (tests, measurements) */
	int slice_taper = 0;            /* "slice_taper": 0 equal slices; t in 1..99: every slice holds t % of the pairs of the one before it (the
	                                 * traceback of the last slice is not hidden under any fill: a short last slice shortens that tail) */
	int carve = 1;                  /* "carve": 1 = the kernels of the long-read phases (strip fills, traceback) ask for the largest shared-memory
	                                 * carve-out, so that their launches can share SMs (0: the driver's choice per launch; measurements) */
	int strip_parts = 0;            /* "parts": 0 automatic, 1 never split the strips of a task, 2/4 forced (tests) */
	int strip_super = SSW_STRIP_SUPER;   /* "super": columns per super-block of the strip kernel (tests) */
	int grid_min_pairs = 32768;     /* "grid_min": smaller grids use the general path */
	int64_t grid_split_pairs = (int64_t)4 << 20;   /* "grid_split": grids of at least this many pairs are cut into launch groups whose records are copied back while the next group computes */
	int grid_group_qp = 16;         /* "grid_group": smallest such group, in query pairs */
	int grid_arm = -1;              /* "grid_arm": best-cell rows of the device-planned grid are recorded in the last k columns of a reference only
	                                 * (pairs whose maximum lies earlier are re-done): -1 automatic (protein-like alphabets: padded query
	                                 * length / 4 + 64, switched off when a pilot group re-does more than 0.2 % of its pairs), 0 off, k > 0 fixed */
	int64_t latency_cols = (int64_t)5 << 19;   /* "latency_cols": passes over at most this many reference columns (2.6 M)
	                                            * use the 32-lane instances */
	int grid_order = 1;             /* "grid_order": 1 = the device-planned grid sweeps the references of a query pair longest first, so that the
	                                 * groups of a warp end together; 0 = in reference order (measurements) */
	int grid_max_ref = SSW_GRID_MAX_REF;   /* "grid_max_ref": longer references are not planned on the device (tests) */
	int64_t grid_tile_refs = 0;     /* "grid_tile_refs": at most this many references per grid tile of a search (0 automatic: tiles only where a
	                                 * grid has more than 2^31 - 1 pairs or one query pair's scratch exceeds the launch budget; tests, measurements) */
	int force_inst = -1;            /* "inst" (measurements): use this forward instance whenever it covers the query */
	int tb_maxbw = SSW_TBP_MAXBW;   /* "tb_maxbw": widest band handled by the shared-memory traceback kernel */
	int tb_spec = -1;               /* "tb_spec": 1 = band-doubling rounds of a task side by side (speculative kernel), 0 = one after the other, -1 = automatic (small batches) */
	int cm_block = -1;              /* "cm_block": -1 automatic, 0 one word per column always, 1 exact block maxima wherever chunking is
	                                 * possible (tests), 2 bounded block words (CM == 3) wherever chunking is possible (tests) */
	int64_t chunk = 0;              /* "chunk": reference chunk length of the fill kernel (0 automatic) */
	int64_t small_chunk = 0;        /* "small_chunk" (measurements): chunk length of launches too small to fill the device */
	int64_t cm_budget = 0;          /* "cm_budget_mb": cap of the column-maximum scratch per launch in bytes (0: half of the free memory; tests) */
};

/* every option of ssw_engine_set_option with the normalisation of its value (include/ssw_batch.h describes them) */
struct SswOptionDef { const char* name; void (*set)(SswOptions& o, int64_t v); };
static const SswOptionDef kOptions[] = {
	{"slices", [](SswOptions& o, int64_t v) { o.slices = v >= 1 && v <= SSW_MAX_SLICES ? (int)v : 0; }},
	{"slice_taper", [](SswOptions& o, int64_t v) { o.slice_taper = v >= 1 && v <= 99 ? (int)v : 0; }},
	{"carve", [](SswOptions& o, int64_t v) { o.carve = v != 0 ? 1 : 0; }},
	{"latency_cols", [](SswOptions& o, int64_t v) { o.latency_cols = v < 0 ? ((int64_t)5 << 19) : v; }},
	{"parts", [](SswOptions& o, int64_t v) { o.strip_parts = v == 1 || v == 2 || v == 4 ? (int)v : 0; }},
	{"small_chunk", [](SswOptions& o, int64_t v) { o.small_chunk = v < 0 ? 0 : (v + 3) / 4 * 4; }},
	{"chunk", [](SswOptions& o, int64_t v) { o.chunk = v < 0 ? 0 : (v + 3) / 4 * 4; }},
	{"cm_block", [](SswOptions& o, int64_t v) { o.cm_block = v < 0 ? -1 : (int)std::min<int64_t>(v, 2); }},
	{"cm_budget_mb", [](SswOptions& o, int64_t v) { o.cm_budget = v <= 0 ? 0 : v << 20; }},
	{"grid_split", [](SswOptions& o, int64_t v) { o.grid_split_pairs = v < 0 ? (int64_t)4 << 20 : v; }},
	{"grid_arm", [](SswOptions& o, int64_t v) { o.grid_arm = v < 0 ? -1 : (int)v; }},
	{"grid_group", [](SswOptions& o, int64_t v) { o.grid_group_qp = v < 1 ? 16 : (int)v; }},
	{"grid_min", [](SswOptions& o, int64_t v) { o.grid_min_pairs = v < 0 ? 32768 : (int)v; }},
	{"grid_order", [](SswOptions& o, int64_t v) { o.grid_order = v != 0 ? 1 : 0; }},
	{"grid_max_ref", [](SswOptions& o, int64_t v) { o.grid_max_ref = v < 1 ? SSW_GRID_MAX_REF : (int)std::min<int64_t>(v, SSW_GRID_MAX_REF); }},
	{"grid_tile_refs", [](SswOptions& o, int64_t v) { o.grid_tile_refs = v < 0 ? 0 : v; }},
	{"inst", [](SswOptions& o, int64_t v) { o.force_inst = (int)v; }},       /* index into kInst */
	{"super", [](SswOptions& o, int64_t v) { o.strip_super = v >= 64 ? (int)(v + 7) / 8 * 8 : SSW_STRIP_SUPER; }},
	{"tb_spec", [](SswOptions& o, int64_t v) { o.tb_spec = v < 0 ? -1 : (int)v; }},      /* > 1: on, rounds up to that many columns */
	{"tb_maxbw", [](SswOptions& o, int64_t v) { o.tb_maxbw = v < 0 ? SSW_TBP_MAXBW : (int)std::min<int64_t>(v, SSW_TBP_MAXBW); }},
};
static const SswOptionDef* find_option(const char* name)
{
	for (const SswOptionDef& d : kOptions) if (!strcmp(d.name, name)) return &d;
	return nullptr;
}

/* the forward (g32 false) or 32-lane (g32 true) instance with the fewest rows >= lp; -1: none covers lp */
static int fewest_rows(int lp, bool g32)
{
	int best = -1, best_rows = 0;
	for (int i = 0; i < kNumInst; ++i) {
		const int rows = inst_rows(i);
		if ((g32 ? kInst[i].G == 32 : kInst[i].fwd) && rows >= lp && (best < 0 || rows < best_rows)) { best = i; best_rows = rows; }
	}
	return best;
}
static int pick_inst(int lp, int force_inst)
{
	if (force_inst >= 0 && force_inst < kNumInst && inst_rows(force_inst) >= lp) return force_inst;   /* any instance, 10..13 included */
	return fewest_rows(lp, false);
}
/* reverse pass: one alignment per warp */
static int pick_inst_g32(int lp) { return fewest_rows(lp, true); }

}  // namespace

struct ssw_engine {
	int device = 0;
	std::string dev_name;
	int sm_count = 0;
	cudaStream_t stream = nullptr;

	/* resident sequences */
	int32_t n_q = 0, n_r = 0;
	std::vector<int64_t> q_off;      /* n_q + 1 */
	std::vector<int64_t> r_off;      /* offset of column 0 inside the padded device array */
	std::vector<int32_t> r_len;
	std::vector<int8_t> h_q, h_r;    /* host copies (codes), used to re-pad when the alphabet size changes */
	std::vector<int64_t> h_r_off;
	int padded_n = -1;               /* null letter currently stored in the reference pads */
	bool from_text = false;          /* sequences were translated on the device: no host copy to re-pad from */
	bool grid_arm_ok = true;         /* late arming paid off for the resident sequences so far (reset by set_sequences*) */
	int64_t cached_ref_len = -1;     /* ssw_engine_set_pair: length and content hash of the single resident reference (-1: none) */
	uint64_t cached_ref_hash = 0;
	SswDevBuf d_q, d_r, d_mat;
	/* query profiles (ssw_engine_set_sequences_pssm): d_q holds n scores per row and q_off counts rows; pssm_n is that n (0: query
	 * codes are resident).  Per query: the byte bias max(0, -min P) and the largest score, as ssw_init derives them from a matrix. */
	int pssm_n = 0;
	std::vector<int32_t> q_bias, q_max;
	bool self = false;               /* ssw_engine_set_sequences_self: the queries and the references are one set (ssw_engine_search_self) */

	/* scratch */
	SswDevBuf d_items, d_bests, d_alns, d_res, d_colmax, d_tb, d_bnd, d_park, d_emul, d_grid, d_out, d_sync;
	SswDevBuf d_hits;                                        /* ssw_engine_search: the n_q x k hit table of the grid path */
	SswDevBuf d_mark;                                        /* ssw_engine_mark_mismatch: tasks, input CIGARs, marked CIGARs */
	SswDevBuf d_rf_items, d_rf_bests, d_rf_blk, d_rf_cm;     /* block-maximum mode: re-fill items, their (unused) bests, first columns, column maxima */
	SswDevBuf d_bd_items, d_bd_bests, d_bd_cm, d_bd_cand, d_bd_cnt;   /* bounded block words: candidate re-fills, candidate lists, counts + offsets */
	int64_t last_cm_words = 0;                               /* column-maximum words of the last forward launch (ssw_engine_last_colmax) */
	SswStagedD2H staged;
	cudaStream_t side[3] = {nullptr, nullptr, nullptr};     /* traceback launches of different kernel shapes run side by side */
	ssw_engine* kids[SSW_MAX_SLICES] = {};                  /* helper engines of the sliced path (views of this engine's sequences) */
	bool is_kid = false;
	SswOptions opt;
	ssw_engine_timing timing;
	SswTimer t_total;
	SswLaps laps;                    /* per-phase kernel times, read once at the end of a call */
	std::vector<cudaEvent_t> grid_events;    /* one per launch group of the device-planned grid (records are copied back behind it) */
	int grid_event(size_t i, cudaEvent_t* out)
	{
		while (grid_events.size() <= i) {
			cudaEvent_t ev = nullptr;
			if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return -1;
			grid_events.push_back(ev);
		}
		*out = grid_events[i];
		return 0;
	}

	int upload_refs(int n);
	/* the matrix argument of the kernels: nullptr tells them that d_q holds query profiles */
	const int8_t* mat_arg() const { return pssm_n ? nullptr : d_mat.as<int8_t>(); }
	int run_fill(const std::vector<SswItem>& items, int inst, int dir, int cm_mode, int share, const ssw_batch_params& P, float* ms_acc);
};


/* ------------------------------------------------------------------------------------------- */
/* fill kernel dispatch                                                                          */
/* ------------------------------------------------------------------------------------------- */

struct FillPtrs { const SswItem* items; uint32_t* cm; SswItemBest* bests; bool arm = false; /* items carry late arming positions (grid path) */ };

/* Warps per CTA and dynamic shared memory of a fill launch with R rows per lane for an alphabet of n letters.  Per-warp
 * profiles (share == 0) can be large for big alphabets: fewer warps per CTA then.  A forward launch with a CTA-shared
 * profile takes 8 warps instead of 4 when that doubles the resident warps per SM (large alphabets: the profile, not the
 * registers, limits the CTAs per SM).  track == false (block mode, CM == 2, keeps no best cell): no snapshot area; the warp
 * count stays the one chosen with it, so that the planner's items per CTA do not depend on the column-maximum mode. */
struct FillShape { int warps; size_t smem; };
template <int R>
static FillShape fill_shape(int n, int share, int dir, bool track = true)
{
	const size_t prof = ssw_fill_smem_bytes<R>(n, 1), snap = ssw_snap_smem_bytes<R>(32);
	int warps = SSW_FILL_WARPS;
	if (!share) while (warps > 1 && (prof + snap) * warps > 200 * 1024) --warps;
	else if (dir > 0 && R >= 16) {
		const size_t sm = (size_t)227 * 1024, s4 = prof + snap * 4 + 1024, s8 = prof + snap * 8 + 1024;
		const int occ4 = (int)std::min<size_t>(SSW_FILL_MINB, sm / s4), occ8 = (int)std::min<size_t>(2, sm / s8);
		if (occ8 * 8 > occ4 * 4) warps = 8;
	}
	return FillShape{warps, (share ? prof : prof * warps) + (track ? snap * warps : 0)};       /* profile(s), then the best-cell snapshots */
}

/* items per CTA of a forward launch of instance `inst` with CTA-shared profiles */
static int fill_items_per_cta(int inst, int n)
{
	return visit_inst(inst, [n](auto t) { using T = decltype(t); return fill_shape<T::R>(n, 1, +1).warps * (32 / T::G); });
}

template <int G, int R, bool PSSM>
static int launch_fill_src(ssw_engine* e, const FillPtrs& fp, int n_items, int dir, int cm_mode, int share, const ssw_batch_params& P)
{
	const FillShape sh = fill_shape<R>(P.n, share, dir, !(dir > 0 && cm_mode >= 2));
	if (sh.smem > 220 * 1024) { fprintf(stderr, "[libssw-b200] alphabet of %d letters is too large for this query length\n", P.n); return -2; }
	const int per_cta = sh.warps * (32 / G);
	const int grid = (n_items + per_cta - 1) / per_cta;
	const int8_t* q = e->d_q.as<int8_t>();
	const int8_t* r = e->d_r.as<int8_t>();
	const int8_t* mat = e->mat_arg();
	auto go = [&](auto kern) {
		if (ssw_ensure_dyn_smem(reinterpret_cast<const void*>(kern), sh.smem)) return -1;
		ssw_launch(kern, dim3(grid), dim3(sh.warps * 32), sh.smem, e->stream, fp.items, n_items, q, r, mat, (int)P.n,
		           (int)P.gap_open, (int)P.gap_extend, fp.cm, fp.bests, share);
		SSW_CUDA_OK(cudaGetLastError());
		return 0;
	};
	if (dir < 0) {   /* reverse: one alignment per warp, early termination */
		if constexpr (G == 32) return go(ssw_fill_kernel<G, R, -1, 0, true, SSW_FILL_WARPS, false, PSSM>);
		return -2;
	}
	/* forward: column maxima per column or per block */
	if (sh.warps == 8) {
		if constexpr (R >= 16) {
			if (cm_mode == 2) return go(ssw_fill_kernel<G, R, 1, 2, false, 8, false, PSSM>);
			if (cm_mode == 3) return go(ssw_fill_kernel<G, R, 1, 3, false, 8, false, PSSM>);
			return fp.arm ? go(ssw_fill_kernel<G, R, 1, 1, false, 8, true, PSSM>) : go(ssw_fill_kernel<G, R, 1, 1, false, 8, false, PSSM>);
		}
		return -2;
	}
	if (cm_mode == 2) return go(ssw_fill_kernel<G, R, 1, 2, false, SSW_FILL_WARPS, false, PSSM>);
	if (cm_mode == 3) return go(ssw_fill_kernel<G, R, 1, 3, false, SSW_FILL_WARPS, false, PSSM>);
	return fp.arm ? go(ssw_fill_kernel<G, R, 1, 1, false, SSW_FILL_WARPS, true, PSSM>) : go(ssw_fill_kernel<G, R, 1, 1, false, SSW_FILL_WARPS, false, PSSM>);
}

/* the fill kernels' instances for query profiles (PSSM) or query codes */
template <int G, int R>
static int launch_fill(ssw_engine* e, const FillPtrs& fp, int n_items, int dir, int cm_mode, int share, const ssw_batch_params& P)
{
	return e->pssm_n ? launch_fill_src<G, R, true>(e, fp, n_items, dir, cm_mode, share, P) : launch_fill_src<G, R, false>(e, fp, n_items, dir, cm_mode, share, P);
}

static int dispatch_fill(ssw_engine* e, int inst, const FillPtrs& fp, int n_items, int dir, int cm_mode, int share, const ssw_batch_params& P)
{
	return visit_inst(inst, [&](auto t) { using T = decltype(t); return launch_fill<T::G, T::R>(e, fp, n_items, dir, cm_mode, share, P); });
}

int ssw_engine::run_fill(const std::vector<SswItem>& items, int inst, int dir, int cm_mode, int share, const ssw_batch_params& P, float* ms_acc)
{
	const int n_items = (int)items.size();
	if (n_items == 0) return 0;
	if (d_items.ensure(sizeof(SswItem) * items.size())) return -1;
	if (d_bests.ensure(sizeof(SswItemBest) * items.size())) return -1;
	Trace tr;
	SSW_CUDA_OK(cudaMemcpyAsync(d_items.p, items.data(), sizeof(SswItem) * items.size(), cudaMemcpyHostToDevice, stream));
	tr.lap("  fill: items h2d");
	laps.start(stream);
	const FillPtrs fp = {d_items.as<SswItem>(), d_colmax.as<uint32_t>(), d_bests.as<SswItemBest>()};
	const int rc = dispatch_fill(this, inst, fp, n_items, dir, cm_mode, share, P);
	tr.lap("  fill: launch");
	laps.stop(stream, ms_acc);
	tr.lap("  fill: wait");
	return rc;
}


/* resident CTAs per SM of the forward fill kernel of instance `inst` in CTA-shared-profile mode (block: with the shared
 * memory of a block-mode launch, which has no snapshot area) */
static int fill_occupancy(int inst, int n, bool block)
{
	static int cache[kNumInst][65][2];
	static std::mutex mu;
	if (inst < 0 || inst >= kNumInst || n < 0 || n > 64) return 1;
	std::lock_guard<std::mutex> lock(mu);
	int& occ = cache[inst][n][block ? 1 : 0];
	if (!occ) occ = std::max(1, visit_inst(inst, [n, block](auto t) {
		using T = decltype(t);
		const FillShape sh = fill_shape<T::R>(n, 1, +1, !block);
		auto kern = ssw_fill_kernel<T::G, T::R, 1, 2, false, SSW_FILL_WARPS, false>;
		if constexpr (T::R >= 16) if (sh.warps == 8) kern = ssw_fill_kernel<T::G, T::R, 1, 2, false, 8, false>;
		ssw_ensure_dyn_smem(reinterpret_cast<const void*>(kern), sh.smem);
		int blocks = 0;
		if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kern, sh.warps * 32, sh.smem) != cudaSuccess) blocks = 1;
		return blocks;
	}));
	return occ;
}

/* ------------------------------------------------------------------------------------------- */
/* engine life cycle                                                                              */
/* ------------------------------------------------------------------------------------------- */

extern "C" ssw_engine* ssw_engine_create(int device)
{
	int count = 0;
	if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
		fprintf(stderr, "[libssw-b200] no usable CUDA device: this library has no CPU compute path\n");
		return nullptr;
	}
	if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) device = 0; }
	if (device >= count || cudaSetDevice(device) != cudaSuccess) {
		fprintf(stderr, "[libssw-b200] cannot select CUDA device %d (of %d)\n", device, count);
		return nullptr;
	}
	cudaDeviceProp prop;
	if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return nullptr;
	ssw_engine* e = new ssw_engine();
	e->device = device;
	e->dev_name = prop.name;
	e->sm_count = prop.multiProcessorCount;
	if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) { delete e; return nullptr; }
	memset(&e->timing, 0, sizeof(e->timing));
	return e;
}

extern "C" void ssw_engine_destroy(ssw_engine* e)
{
	if (!e) return;
	cudaSetDevice(e->device);
	SswDevBuf* bufs[] = {&e->d_q, &e->d_r, &e->d_mat, &e->d_items, &e->d_bests, &e->d_alns, &e->d_res, &e->d_colmax, &e->d_tb, &e->d_bnd, &e->d_park, &e->d_emul, &e->d_grid, &e->d_out, &e->d_sync, &e->d_rf_items, &e->d_rf_bests, &e->d_rf_blk, &e->d_rf_cm, &e->d_mark, &e->d_hits,
	                     &e->d_bd_items, &e->d_bd_bests, &e->d_bd_cm, &e->d_bd_cand, &e->d_bd_cnt};
	for (SswDevBuf* b : bufs) b->release();
	for (ssw_engine*& k : e->kids) if (k) { ssw_engine_destroy(k); k = nullptr; }
	e->staged.release();
	for (cudaStream_t& st : e->side) if (st) { cudaStreamDestroy(st); st = nullptr; }
	for (cudaEvent_t ev : e->grid_events) if (ev) cudaEventDestroy(ev);
	if (e->stream) cudaStreamDestroy(e->stream);
	delete e;
}

extern "C" const char* ssw_engine_device_name(const ssw_engine* e) { return e ? e->dev_name.c_str() : ""; }

extern "C" int32_t ssw_device_count(void)
{
	int count = 0;
	return cudaGetDeviceCount(&count) == cudaSuccess && count > 0 ? count : 0;
}

extern "C" int ssw_engine_set_option(ssw_engine* e, const char* name, int64_t value)
{
	if (!name) return -1;
	if (!e) return ssw_default_engines_option(name, value);
	const SswOptionDef* d = find_option(name);
	if (!d) { fprintf(stderr, "[libssw-b200] unknown option '%s'\n", name); return -1; }
	d->set(e->opt, value);
	return 0;
}

bool ssw_engine_has_option(const char* name) { return find_option(name) != nullptr; }

extern "C" int ssw_engine_last_timing(const ssw_engine* e, ssw_engine_timing* t)
{
	if (!e || !t) return -1;
	*t = e->timing;
	return 0;
}

extern "C" int64_t ssw_engine_last_colmax(ssw_engine* e, uint32_t* out, int64_t n_words)
{
	if (!e || n_words < 0 || (n_words > 0 && !out)) return -1;
	const int64_t n = std::min(n_words, e->last_cm_words);
	if (n > 0) {
		SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
		SSW_CUDA_OK(cudaMemcpy(out, e->d_colmax.p, sizeof(uint32_t) * (size_t)n, cudaMemcpyDeviceToHost));
	}
	return e->last_cm_words;
}

/* References are stored as  [PAD x null] codes [PAD x null]  with null = n (scores as a dead letter), each block
 * 16-aligned; the fill kernels rely on those pads (col_lo / col_hi in ssw_fill.cuh).  Fills r_off with the offset of
 * column 0 of every reference and returns the length of the padded array. */
static int64_t ref_layout(const std::vector<int32_t>& r_len, std::vector<int64_t>& r_off)
{
	int64_t total = 0;
	r_off.resize(r_len.size());
	for (size_t i = 0; i < r_len.size(); ++i) {
		total += SSW_REF_PAD;
		r_off[i] = total;
		total += (int64_t)r_len[i] + SSW_REF_PAD;
		total = (total + 15) / 16 * 16;
	}
	return total + 2 * SSW_REF_PAD;
}

int ssw_engine::upload_refs(int n)
{
	if (padded_n == n && d_r.p) return 0;
	if (from_text) {
		fprintf(stderr, "[libssw-b200] sequences were set as text for an alphabet of %d letters; this call uses %d\n", padded_n, n);
		return -1;
	}
	const int64_t total = ref_layout(r_len, r_off);
	std::vector<int8_t> padded((size_t)total, (int8_t)n);
	for (int i = 0; i < n_r; ++i) memcpy(padded.data() + r_off[i], h_r.data() + h_r_off[i], (size_t)r_len[i]);
	if (d_r.ensure((size_t)total)) return -1;
	/* pageable source: the call returns once the bytes sit in the driver's staging buffer, so `padded` may go away and
	 * later work on the stream is ordered behind the copy -- no synchronisation needed */
	SSW_CUDA_OK(cudaMemcpyAsync(d_r.p, padded.data(), (size_t)total, cudaMemcpyHostToDevice, stream));
	padded_n = n;
	return 0;
}

/* Offsets must be non-decreasing and start at 0; device-side descriptors hold 32-bit query offsets and reference lengths. */
static int check_offsets(const char* what, int32_t n, const int64_t* off, int64_t limit_total, int64_t limit_each)
{
	if (n == 0) return 0;
	if (!off || off[0] != 0) { fprintf(stderr, "[libssw-b200] %s offsets must start at 0\n", what); return -1; }
	for (int32_t i = 0; i < n; ++i) {
		if (off[i + 1] < off[i]) { fprintf(stderr, "[libssw-b200] %s offsets are not non-decreasing at %d\n", what, i); return -1; }
		if (off[i + 1] - off[i] > limit_each) { fprintf(stderr, "[libssw-b200] %s %d is longer than %lld\n", what, i, (long long)limit_each); return -1; }
	}
	if (off[n] > limit_total) { fprintf(stderr, "[libssw-b200] %s hold %lld letters in total; the limit is %lld\n", what, (long long)off[n], (long long)limit_total); return -1; }
	return 0;
}
#define SSW_MAX_QUERY_LETTERS ((int64_t)0x7fffffff - 64)                        /* SswQuery.off is 32 bits */
#define SSW_MAX_REF_LEN ((int64_t)0x7fffffff - 4 * SSW_REF_PAD - 64)            /* SswItem.ref_len, scan positions */

/* pssm_n > 0: the queries are position-specific profiles of pssm_n scores per row (query_off counts rows); 0: query codes. */
static int set_sequences_impl(ssw_engine* e,
                              int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                              int32_t n_refs, const int8_t* refs, const int64_t* ref_off, int32_t pssm_n = 0)
{
	if (!e || n_queries < 0 || n_refs < 0 || (n_queries && (!queries || !query_off)) || (n_refs && (!refs || !ref_off))) return -1;
	if (pssm_n < 0 || pssm_n > 64) { fprintf(stderr, "[libssw-b200] profiles of %d letters: 1 .. 64 supported\n", pssm_n); return -1; }
	/* profiles: the banded traceback addresses a row's scores within its query in 32 bits */
	if (check_offsets("query", n_queries, query_off, SSW_MAX_QUERY_LETTERS, pssm_n ? 0x7fffffff / pssm_n - 64 : SSW_MAX_QUERY_LETTERS)) return -1;
	if (check_offsets("reference", n_refs, ref_off, (int64_t)1 << 46, SSW_MAX_REF_LEN)) return -1;
	SSW_CUDA_OK(cudaSetDevice(e->device));
	e->n_q = n_queries; e->n_r = n_refs;
	e->self = false;
	e->from_text = false;
	e->cached_ref_len = -1;
	e->grid_arm_ok = true;
	e->pssm_n = pssm_n;
	const int64_t width = pssm_n ? pssm_n : 1;
	const int64_t qb = (n_queries ? query_off[n_queries] : 0) * width, rb = n_refs ? ref_off[n_refs] : 0;
	if (n_queries) e->q_off.assign(query_off, query_off + n_queries + 1); else e->q_off.assign(1, 0);
	e->h_q.assign(queries, queries + qb);
	if (n_refs) e->h_r_off.assign(ref_off, ref_off + n_refs + 1); else e->h_r_off.assign(1, 0);
	e->h_r.assign(refs, refs + rb);
	e->r_len.resize(n_refs);
	for (int i = 0; i < n_refs; ++i) e->r_len[i] = (int32_t)(ref_off[i + 1] - ref_off[i]);
	e->q_bias.clear(); e->q_max.clear();
	if (pssm_n) {
		/* what ssw_init derives from the matrix of a profile (ssw.c:834-838): the byte bias, and the largest score for the word guard */
		e->q_bias.resize((size_t)n_queries); e->q_max.resize((size_t)n_queries);
		for (int32_t q = 0; q < n_queries; ++q) {
			int lo = 0, hi = 0;
			if (query_off[q + 1] > query_off[q]) { lo = 127; hi = -128; }
			for (int64_t i = query_off[q] * width; i < query_off[q + 1] * width; ++i) { lo = std::min<int>(lo, queries[i]); hi = std::max<int>(hi, queries[i]); }
			e->q_bias[q] = std::max(0, -lo); e->q_max[q] = hi;
		}
	}
	/* behind the last query a few zero bytes (profiles: two rows), so that no read of a row just past a query leaves the buffer */
	const size_t tail = pssm_n ? (size_t)(16 + 2 * pssm_n) : 16;
	if (e->d_q.ensure(e->h_q.size() + tail)) return -1;
	if (qb) SSW_CUDA_OK(cudaMemcpyAsync(e->d_q.p, e->h_q.data(), e->h_q.size(), cudaMemcpyHostToDevice, e->stream));
	if (pssm_n) SSW_CUDA_OK(cudaMemsetAsync(e->d_q.as<int8_t>() + qb, 0, tail, e->stream));
	e->padded_n = -1;           /* the null letter depends on the alphabet size given at align time */
	return 0;
}

extern "C" int ssw_engine_set_sequences(ssw_engine* e,
                                        int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                                        int32_t n_refs, const int8_t* refs, const int64_t* ref_off)
{
	try { return set_sequences_impl(e, n_queries, queries, query_off, n_refs, refs, ref_off); }
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_set_sequences: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_engine_set_sequences_pssm(ssw_engine* e,
                                             int32_t n_queries, const int8_t* pssm, const int64_t* query_off, int32_t n,
                                             int32_t n_refs, const int8_t* refs, const int64_t* ref_off)
{
	if (n < 1) { fprintf(stderr, "[libssw-b200] ssw_engine_set_sequences_pssm: profiles of %d letters: 1 .. 64 supported\n", n); return -1; }
	try { return set_sequences_impl(e, n_queries, pssm, query_off, n_refs, refs, ref_off, n); }
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_set_sequences_pssm: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_engine_set_sequences_self(ssw_engine* e, int32_t n, const int8_t* seqs, const int64_t* off)
{
	try {
		const int rc = set_sequences_impl(e, n, seqs, off, n, seqs, off);
		if (rc == 0) e->self = true;
		return rc;
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_set_sequences_self: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

/* One query against one reference, as ssw_align sees it.  The reference's consumers loop over many reads against one large
 * reference (main.c:462-532, ssw_cpp.cpp:336); when the bytes at `ref` are the ones already resident (same length, same 64-bit
 * content hash) only the query is uploaded -- no host copy, no re-padding, no H2D of the reference. */
extern "C" int ssw_engine_set_pair(ssw_engine* e, const int8_t* read, int32_t readLen, const int8_t* ref, int32_t refLen)
{
	if (!e || !read || !ref || readLen < 1 || refLen < 0) return -1;
	try {
		const uint64_t h = ssw_hash_bytes(ref, (size_t)refLen);
		const bool same = e->n_r == 1 && !e->from_text && e->cached_ref_len == (int64_t)refLen && e->cached_ref_hash == h && e->d_r.p;
		if (!same) {
			const int64_t qoff[2] = {0, readLen}, roff[2] = {0, refLen};
			const int rc = set_sequences_impl(e, 1, read, qoff, 1, ref, roff);
			if (rc) return rc;
			e->cached_ref_len = refLen; e->cached_ref_hash = h;
			return 0;
		}
		SSW_CUDA_OK(cudaSetDevice(e->device));
		e->n_q = 1;
		e->pssm_n = 0;
		e->self = false;
		e->q_off.assign(2, 0); e->q_off[1] = readLen;
		e->h_q.assign(read, read + readLen);
		if (e->d_q.ensure(e->h_q.size() + 16)) return -1;
		SSW_CUDA_OK(cudaMemcpyAsync(e->d_q.p, e->h_q.data(), e->h_q.size(), cudaMemcpyHostToDevice, e->stream));
		return 0;
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_set_pair: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

static int set_sequences_packed_impl(ssw_engine* e, int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                                     int32_t n_refs, const uint8_t* refs_packed, const int64_t* ref_off, int32_t bits, int32_t n)
{
	if (!e || (bits != 2 && bits != 4) || n < 1 || n > 64 || n_queries < 0 || n_refs < 0 || (n_queries && (!queries || !query_off)) ||
	    (n_refs && (!refs_packed || !ref_off)))
		return -1;
	if (check_offsets("query", n_queries, query_off, SSW_MAX_QUERY_LETTERS, SSW_MAX_QUERY_LETTERS)) return -1;
	if (check_offsets("reference", n_refs, ref_off, (int64_t)1 << 46, SSW_MAX_REF_LEN)) return -1;
	SSW_CUDA_OK(cudaSetDevice(e->device));
	e->cached_ref_len = -1;
	e->grid_arm_ok = true;
	e->pssm_n = 0;
	e->self = false;
	const int64_t qb = n_queries ? query_off[n_queries] : 0, rb = n_refs ? ref_off[n_refs] : 0;
	e->n_q = n_queries; e->n_r = n_refs;
	if (n_queries) e->q_off.assign(query_off, query_off + n_queries + 1); else e->q_off.assign(1, 0);
	e->h_q.assign(queries, queries + qb);
	e->h_r.clear(); e->h_r_off.clear();
	e->r_len.resize(n_refs);
	for (int i = 0; i < n_refs; ++i) e->r_len[i] = (int32_t)(ref_off[i + 1] - ref_off[i]);
	const int64_t total = ref_layout(e->r_len, e->r_off);
	const size_t pk = (size_t)((rb * bits + 7) / 8);
	const size_t o_ro = (pk + 255) / 256 * 256, o_rd = o_ro + 8 * (size_t)(n_refs + 1);
	if (e->d_grid.ensure(o_rd + 8 * (size_t)(n_refs + 1) + 256)) return -1;
	if (e->d_q.ensure((size_t)qb + 16)) return -1;
	if (e->d_r.ensure((size_t)total)) return -1;
	uint8_t* st = e->d_grid.as<uint8_t>();
	if (qb) SSW_CUDA_OK(cudaMemcpyAsync(e->d_q.p, e->h_q.data(), (size_t)qb, cudaMemcpyHostToDevice, e->stream));
	SSW_CUDA_OK(cudaMemsetAsync(e->d_r.p, n, (size_t)total, e->stream));          /* null letters everywhere, codes on top */
	if (n_refs && rb) {
		SSW_CUDA_OK(cudaMemcpyAsync(st, refs_packed, pk, cudaMemcpyHostToDevice, e->stream));
		SSW_CUDA_OK(cudaMemcpyAsync(st + o_ro, ref_off, 8 * (size_t)(n_refs + 1), cudaMemcpyHostToDevice, e->stream));
		SSW_CUDA_OK(cudaMemcpyAsync(st + o_rd, e->r_off.data(), 8 * (size_t)n_refs, cudaMemcpyHostToDevice, e->stream));
		const unsigned blocks = (unsigned)std::min<int64_t>((rb + 255) / 256, (int64_t)e->sm_count * 16);
		ssw_launch(ssw_unpack_kernel, dim3(blocks), dim3(256), 0, e->stream, rb, n_refs, bits, (const uint8_t*)st,
		           (const int64_t*)reinterpret_cast<int64_t*>(st + o_ro), (const int64_t*)reinterpret_cast<int64_t*>(st + o_rd), e->d_r.as<int8_t>());
		SSW_CUDA_OK(cudaGetLastError());
	}
	SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
	e->padded_n = n;
	e->from_text = true;        /* no unpacked host copy to re-pad from: the alphabet size is fixed by this call */
	return 0;
}

extern "C" int ssw_engine_set_sequences_packed(ssw_engine* e, int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                                               int32_t n_refs, const uint8_t* refs_packed, const int64_t* ref_off, int32_t bits, int32_t n)
{
	try { return set_sequences_packed_impl(e, n_queries, queries, query_off, n_refs, refs_packed, ref_off, bits, n); }
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_set_sequences_packed: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

static int set_sequences_text_impl(ssw_engine* e,
                                   int32_t n_queries, const char* queries, const int64_t* query_off,
                                   int32_t n_refs, const char* refs, const int64_t* ref_off,
                                   const int8_t* table, int32_t n, int32_t add_reverse_complement);
extern "C" int ssw_engine_set_sequences_text(ssw_engine* e,
                                             int32_t n_queries, const char* queries, const int64_t* query_off,
                                             int32_t n_refs, const char* refs, const int64_t* ref_off,
                                             const int8_t* table, int32_t n, int32_t add_reverse_complement)
{
	try { return set_sequences_text_impl(e, n_queries, queries, query_off, n_refs, refs, ref_off, table, n, add_reverse_complement); }
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_set_sequences_text: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}
static int set_sequences_text_impl(ssw_engine* e,
                                   int32_t n_queries, const char* queries, const int64_t* query_off,
                                   int32_t n_refs, const char* refs, const int64_t* ref_off,
                                   const int8_t* table, int32_t n, int32_t add_reverse_complement)
{
	if (!e || !table || n < 1 || n > 64 || n_queries < 0 || n_refs < 0 || (n_queries && (!queries || !query_off)) ||
	    (n_refs && (!refs || !ref_off)))
		return -1;
	const int rc = add_reverse_complement ? 1 : 0;
	if (check_offsets("query", n_queries, query_off, SSW_MAX_QUERY_LETTERS / (1 + rc), SSW_MAX_QUERY_LETTERS / (1 + rc))) return -1;
	if (check_offsets("reference", n_refs, ref_off, (int64_t)1 << 46, SSW_MAX_REF_LEN)) return -1;
	SSW_CUDA_OK(cudaSetDevice(e->device));
	e->cached_ref_len = -1;
	e->grid_arm_ok = true;
	e->pssm_n = 0;
	e->self = false;
	const int64_t qb = n_queries ? query_off[n_queries] : 0, rb = n_refs ? ref_off[n_refs] : 0;
	e->n_q = n_queries * (1 + rc); e->n_r = n_refs;
	if (n_queries) e->q_off.assign(query_off, query_off + n_queries + 1); else e->q_off.assign(1, 0);
	if (rc) for (int i = 1; i <= n_queries; ++i) e->q_off.push_back(qb + query_off[i]);
	e->h_q.clear(); e->h_r.clear(); e->h_r_off.clear();
	e->r_len.resize(n_refs);
	for (int i = 0; i < n_refs; ++i) e->r_len[i] = (int32_t)(ref_off[i + 1] - ref_off[i]);
	const int64_t total = ref_layout(e->r_len, e->r_off);
	/* staging: texts, offsets, destination offsets, table */
	const size_t o_qt = 0, o_rt = (size_t)(qb + 255) / 256 * 256, o_qo = o_rt + (size_t)(rb + 255) / 256 * 256;
	const size_t o_ro = o_qo + 8 * (size_t)(n_queries + 1), o_rd = o_ro + 8 * (size_t)(n_refs + 1), o_tab = o_rd + 8 * (size_t)(n_refs + 1);
	if (e->d_grid.ensure(o_tab + 128 + 256)) return -1;
	if (e->d_q.ensure((size_t)qb * (size_t)(1 + rc) + 16)) return -1;
	if (e->d_r.ensure((size_t)total)) return -1;
	uint8_t* st = e->d_grid.as<uint8_t>();
	if (qb) SSW_CUDA_OK(cudaMemcpyAsync(st + o_qt, queries, (size_t)qb, cudaMemcpyHostToDevice, e->stream));
	if (rb) SSW_CUDA_OK(cudaMemcpyAsync(st + o_rt, refs, (size_t)rb, cudaMemcpyHostToDevice, e->stream));
	if (n_queries) SSW_CUDA_OK(cudaMemcpyAsync(st + o_qo, query_off, 8 * (size_t)(n_queries + 1), cudaMemcpyHostToDevice, e->stream));
	if (n_refs) {
		SSW_CUDA_OK(cudaMemcpyAsync(st + o_ro, ref_off, 8 * (size_t)(n_refs + 1), cudaMemcpyHostToDevice, e->stream));
		SSW_CUDA_OK(cudaMemcpyAsync(st + o_rd, e->r_off.data(), 8 * (size_t)n_refs, cudaMemcpyHostToDevice, e->stream));
	}
	SSW_CUDA_OK(cudaMemcpyAsync(st + o_tab, table, 128, cudaMemcpyHostToDevice, e->stream));
	SSW_CUDA_OK(cudaMemsetAsync(e->d_r.p, n, (size_t)total, e->stream));          /* null letters everywhere, codes on top */
	SswTextArgs A;
	A.q_bytes = qb; A.r_bytes = rb; A.n_q = n_queries; A.n_r = n_refs; A.add_rc = rc; A.pad_ = 0;
	const int64_t work = std::max<int64_t>(qb, rb);
	if (work > 0) {
		const unsigned blocks = (unsigned)std::min<int64_t>((work + 255) / 256, (int64_t)e->sm_count * 16);
		ssw_launch(ssw_translate_kernel, dim3(blocks), dim3(256), 0, e->stream, A, (const uint8_t*)(st + o_qt),
		           (const int64_t*)reinterpret_cast<int64_t*>(st + o_qo), (const uint8_t*)(st + o_rt),
		           (const int64_t*)reinterpret_cast<int64_t*>(st + o_ro), (const int64_t*)reinterpret_cast<int64_t*>(st + o_rd),
		           (const int8_t*)reinterpret_cast<int8_t*>(st + o_tab), e->d_q.as<int8_t>(), e->d_r.as<int8_t>());
		SSW_CUDA_OK(cudaGetLastError());
	}
	SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
	e->padded_n = n;
	e->from_text = true;
	return 0;
}

/* ------------------------------------------------------------------------------------------- */
/* the batched ssw_align                                                                          */
/* ------------------------------------------------------------------------------------------- */

namespace {

struct Aln {            /* one requested pair while it moves through the phases */
	int32_t q, r;
	int32_t read_len, ref_len, mask_len;
	int32_t word;       /* semantics of the accepted forward result */
	SswFillResult fwd;
	int32_t rev_score, rev_pos, rev_row;
};

/* scoring context of one call.  With query profiles resident the bias and the limits are those of each query (q_bias / q_max
 * non-null); bias and max_mat are then the largest over the resident profiles, for the call-wide bounds. */
struct Sem {
	int bias, max_mat;
	int limit_byte;     /* 255 - bias: a byte-semantics score >= this overflows (ssw.c:329) */
	int limit_word;     /* 16-bit head-room guard */
	bool has_byte, has_word;
	const int32_t* q_bias = nullptr;
	const int32_t* q_max = nullptr;
	int bias_of(int32_t q) const { return q_bias ? q_bias[q] : bias; }
	int limit_byte_of(int32_t q) const { return q_bias ? 255 - q_bias[q] : limit_byte; }
	int limit_word_of(int32_t q) const { return q_max ? 32767 - std::max(q_max[q], 0) - 256 : limit_word; }
	int limit_of(int32_t q, int word) const { return word ? limit_word_of(q) : limit_byte_of(q); }
	int max_of(int32_t q) const { return q_max ? q_max[q] : max_mat; }
};

static inline int lp_of(int len, int word) { int g = word ? 8 : 16; return (len + g - 1) / g * g; }

/* Does a forward result obtained with semantics `word` have to be replaced by the other semantics?
 *   byte result that overflowed -> word (ssw.c:883-886)
 *   word result computed first because an overflow was predicted, but the score fits a byte -> byte */
static inline bool needs_other(const SswFillResult& r, int word, const Sem& S, bool word_first, int32_t q)
{
	if (!word) return r.overflow == 1 && S.has_word;
	return word_first && S.has_byte && r.overflow == 0 && r.score < S.limit_byte_of(q);
}

/* How the column maxima of the fill being resolved are stored (fill kernel CM mode), and -- block mode -- what the
 * re-fill of single blocks needs: a kernel instance that covers the rows of every alignment (those of the fill, or the
 * byte padding of alignments filled on their word rows: rows >= an item's lp are dead) and the scoring parameters. */
/* block: 0 one word per column, 1 exact block maxima (CM == 2), 2 bounded block words (CM == 3).  fill_inst: the instance of the
 * fill (bounded words: the pair-task of an alignment over the candidate cap re-runs with it).  colmax / items: the words and the
 * fill items the descriptors point into (nullptr: the engine's d_colmax / d_items). */
struct CmMode { int block; int inst; const ssw_batch_params* P; int fill_inst = -1; const uint32_t* colmax = nullptr; const SswItem* items = nullptr; };

/* Host side of a candidate stage of the bounded block words: read the per-alignment counts (-1: over the cap), turn them into
 * offsets on the device and mark the alignments over the cap.  Returns the number of candidates, -1 on an error. */
static int64_t bound_offsets(ssw_engine* e, size_t n_aln, const int32_t* d_cnt, int32_t* d_off, std::vector<char>& exact)
{
	std::vector<int32_t> cnt(n_aln), off(n_aln);
	if (cudaMemcpyAsync(cnt.data(), d_cnt, sizeof(int32_t) * n_aln, cudaMemcpyDeviceToHost, e->stream) != cudaSuccess ||
	    cudaStreamSynchronize(e->stream) != cudaSuccess) return -1;
	int64_t total = 0;
	for (size_t i = 0; i < n_aln; ++i) {
		off[i] = (int32_t)total;
		if (cnt[i] < 0) exact[i] = 1; else total += cnt[i];
	}
	if (total > INT32_MAX / SSW_CM_BLOCK) { fprintf(stderr, "[libssw-b200] too many candidate blocks in one resolve (%lld)\n", (long long)total); return -1; }
	if (cudaMemcpyAsync(d_off, off.data(), sizeof(int32_t) * n_aln, cudaMemcpyHostToDevice, e->stream) != cudaSuccess ||
	    cudaStreamSynchronize(e->stream) != cudaSuccess) return -1;     /* `off` is a local: wait for the copy */
	return total;
}

/* Launch the resolve kernel(s) over `descs` and fetch the results. */
static int run_resolve(ssw_engine* e, const std::vector<SswAlnDesc>& descs, bool second, std::vector<SswFillResult>& res, const CmMode* cm = nullptr)
{
	res.resize(descs.size());
	if (descs.empty()) return 0;
	if (e->d_alns.ensure(sizeof(SswAlnDesc) * descs.size())) return -1;
	if (e->d_res.ensure(sizeof(SswFillResult) * descs.size())) return -1;
	SSW_CUDA_OK(cudaMemcpyAsync(e->d_alns.p, descs.data(), sizeof(SswAlnDesc) * descs.size(), cudaMemcpyHostToDevice, e->stream));
	e->laps.start(e->stream);
	const int per = SSW_RESOLVE_THREADS / 32;
	const dim3 grid(((int)descs.size() + per - 1) / per);
	std::vector<char> exact;        /* bounded words: alignments over the candidate cap */
	if (cm && cm->block) {
		const uint32_t* colmax = cm->colmax ? cm->colmax : e->d_colmax.as<uint32_t>();
		const SswItem* items = cm->items ? cm->items : e->d_items.as<SswItem>();
		const SswAlnDesc* alns = e->d_alns.as<SswAlnDesc>();
		/* block words (the fill kept no item bests, so this runs whether or not the second best is wanted).  Exact maxima: stage 0
		 * (the first block holding the score) and its re-fill with best-cell tracking; bounded words: the C1 candidates and their
		 * re-fills with tracking.  Then stage 1 (the best cell + the blocks cut by the mask window, and the columns right of it of
		 * byte alignments filled on their word rows; exact maxima: the first block of the largest fully allowed block maximum,
		 * bounded words: the C2 candidates), re-fill of those ranges with one word per column, stage 2.  Scratch:
		 * SSW_REFILL_SLOTS items per alignment, then (exact maxima) one best-block item per alignment. */
		const size_t n_aln = descs.size(), n_rf = n_aln * SSW_REFILL_SLOTS;
		if (e->d_rf_items.ensure(sizeof(SswItem) * (n_rf + n_aln))) return -1;
		if (e->d_rf_bests.ensure(sizeof(SswItemBest) * (n_rf + n_aln))) return -1;
		if (e->d_rf_blk.ensure(sizeof(int32_t) * n_rf)) return -1;    /* first column of every re-filled range, -1: none */
		if (e->d_rf_cm.ensure(sizeof(uint32_t) * n_rf * SSW_CM_BLOCK + 64)) return -1;
		const FillPtrs fp = {e->d_rf_items.as<SswItem>(), e->d_rf_cm.as<uint32_t>(), e->d_rf_bests.as<SswItemBest>()};
		if (cm->block == 1) {
			ssw_launch(ssw_resolve_best_block_kernel<0>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, alns, (int)n_aln, colmax, items,
			           e->d_rf_items.as<SswItem>() + n_rf);
			SSW_CUDA_OK(cudaGetLastError());
			const FillPtrs fp_best = {e->d_rf_items.as<SswItem>() + n_rf, e->d_rf_cm.as<uint32_t>(), e->d_rf_bests.as<SswItemBest>() + n_rf};
			int rc = dispatch_fill(e, cm->inst, fp_best, (int)n_aln, +1, 1, 0, *cm->P);
			if (rc) return rc < 0 ? rc : -1;
			ssw_launch(ssw_resolve_blocks_kernel<false>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, alns, (int)n_aln,
			           (const SswItemBest*)e->d_rf_bests.as<SswItemBest>() + n_rf, colmax, items, e->d_res.as<SswFillResult>(),
			           e->d_rf_items.as<SswItem>(), e->d_rf_blk.as<int32_t>(), (const int32_t*)nullptr, (const int32_t*)nullptr,
			           SswBound{0, 0, 0}, (int32_t*)nullptr, (int32_t*)nullptr);
			SSW_CUDA_OK(cudaGetLastError());
			rc = dispatch_fill(e, cm->inst, fp, (int)n_rf, +1, 1, 0, *cm->P);
			if (rc) return rc < 0 ? rc : -1;
			ssw_launch(ssw_resolve_refill_kernel<0>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, alns, (int)n_aln,
			           (const int32_t*)e->d_rf_blk.as<int32_t>(), (const uint32_t*)e->d_rf_cm.as<uint32_t>(), e->d_res.as<SswFillResult>(),
			           (const int32_t*)nullptr, 0, (const int32_t*)nullptr, (const int32_t*)nullptr, (const uint32_t*)nullptr);
			e->timing.other_launches += 4;
		} else {
			const SswBound bd = {(int)cm->P->gap_open, (int)cm->P->gap_extend, SSW_BOUND_CAP};
			if (e->d_bd_cand.ensure(sizeof(int32_t) * n_aln * (size_t)bd.cap + 64)) return -1;
			if (e->d_bd_cnt.ensure(sizeof(int32_t) * 4 * n_aln)) return -1;
			int32_t* cnt1 = e->d_bd_cnt.as<int32_t>();
			int32_t* cnt2 = cnt1 + n_aln, *off1 = cnt2 + n_aln, *off2 = off1 + n_aln;
			int32_t* cand = e->d_bd_cand.as<int32_t>();
			exact.assign(n_aln, 0);
			ssw_launch(ssw_bound_best_kernel<0>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, alns, (int)n_aln, colmax, bd, cand, cnt1);
			SSW_CUDA_OK(cudaGetLastError());
			const int64_t n1 = bound_offsets(e, n_aln, cnt1, off1, exact);
			if (n1 < 0) return -1;
			if (e->d_bd_items.ensure(sizeof(SswItem) * (size_t)n1 + 64)) return -1;
			if (e->d_bd_bests.ensure(sizeof(SswItemBest) * (size_t)n1 + 64)) return -1;
			ssw_launch(ssw_bound_emit_kernel<0>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, alns, (int)n_aln, items, (const int32_t*)cand,
			           bd.cap, (const int32_t*)cnt1, (const int32_t*)off1, 0, e->d_bd_items.as<SswItem>());
			SSW_CUDA_OK(cudaGetLastError());
			const FillPtrs fp1 = {e->d_bd_items.as<SswItem>(), e->d_rf_cm.as<uint32_t>(), e->d_bd_bests.as<SswItemBest>()};
			int rc = n1 > 0 ? dispatch_fill(e, cm->inst, fp1, (int)n1, +1, 1, 0, *cm->P) : 0;
			if (rc) return rc < 0 ? rc : -1;
			ssw_launch(ssw_resolve_blocks_kernel<true>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, alns, (int)n_aln,
			           (const SswItemBest*)e->d_bd_bests.as<SswItemBest>(), colmax, items, e->d_res.as<SswFillResult>(),
			           e->d_rf_items.as<SswItem>(), e->d_rf_blk.as<int32_t>(), (const int32_t*)cnt1, (const int32_t*)off1, bd, cand, cnt2);
			SSW_CUDA_OK(cudaGetLastError());
			const int64_t n2 = bound_offsets(e, n_aln, cnt2, off2, exact);
			if (n2 < 0) return -1;
			if (e->d_bd_items.ensure(sizeof(SswItem) * (size_t)n2 + 64)) return -1;
			if (e->d_bd_bests.ensure(sizeof(SswItemBest) * (size_t)n2 + 64)) return -1;
			if (e->d_bd_cm.ensure(sizeof(uint32_t) * (size_t)n2 * SSW_CM_BLOCK + 64)) return -1;
			ssw_launch(ssw_bound_emit_kernel<0>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, alns, (int)n_aln, items, (const int32_t*)cand,
			           bd.cap, (const int32_t*)cnt2, (const int32_t*)off2, 1, e->d_bd_items.as<SswItem>());
			SSW_CUDA_OK(cudaGetLastError());
			rc = dispatch_fill(e, cm->inst, fp, (int)n_rf, +1, 1, 0, *cm->P);
			if (rc) return rc < 0 ? rc : -1;
			const FillPtrs fp2 = {e->d_bd_items.as<SswItem>(), e->d_bd_cm.as<uint32_t>(), e->d_bd_bests.as<SswItemBest>()};
			rc = n2 > 0 ? dispatch_fill(e, cm->inst, fp2, (int)n2, +1, 1, 0, *cm->P) : 0;
			if (rc) return rc < 0 ? rc : -1;
			ssw_launch(ssw_resolve_refill_kernel<0>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, alns, (int)n_aln,
			           (const int32_t*)e->d_rf_blk.as<int32_t>(), (const uint32_t*)e->d_rf_cm.as<uint32_t>(), e->d_res.as<SswFillResult>(),
			           (const int32_t*)cand, bd.cap, (const int32_t*)cnt2, (const int32_t*)off2, (const uint32_t*)e->d_bd_cm.as<uint32_t>());
			e->timing.other_launches += 6 + (n1 > 0 ? 1 : 0) + (n2 > 0 ? 1 : 0);
			e->timing.block_refills += n1 + n2;
		}
	} else if (second)
		ssw_launch(ssw_resolve_kernel<true>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, (const SswAlnDesc*)e->d_alns.as<SswAlnDesc>(),
		           (int)descs.size(), (const SswItemBest*)e->d_bests.as<SswItemBest>(), (const uint32_t*)e->d_colmax.as<uint32_t>(), e->d_res.as<SswFillResult>());
	else
		ssw_launch(ssw_resolve_kernel<false>, grid, dim3(SSW_RESOLVE_THREADS), 0, e->stream, (const SswAlnDesc*)e->d_alns.as<SswAlnDesc>(),
		           (int)descs.size(), (const SswItemBest*)e->d_bests.as<SswItemBest>(), (const uint32_t*)nullptr, e->d_res.as<SswFillResult>());
	SSW_CUDA_OK(cudaGetLastError());
	e->laps.stop(e->stream, &e->timing.resolve_ms);
	e->timing.other_launches += 1;
	SSW_CUDA_OK(cudaMemcpyAsync(res.data(), e->d_res.p, sizeof(SswFillResult) * descs.size(), cudaMemcpyDeviceToHost, e->stream));
	SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
	if (std::find(exact.begin(), exact.end(), 1) == exact.end()) return 0;

	/* Alignments over the candidate cap: their pair-tasks re-run with exact block maxima into rows of a scratch of their own (the
	 * bounded words stay as they are, for a second resolve of the same fill), and the alignments are resolved from those. */
	std::vector<int64_t> fb;
	for (size_t i = 0; i < exact.size(); ++i) if (exact[i]) fb.push_back((int64_t)i);
	std::vector<SswItem> fb_items;
	std::vector<SswAlnDesc> fb_descs;
	std::map<int32_t, int32_t> task;            /* first item of a pair-task -> its first item in the scratch */
	int64_t words = 0;
	const SswItem* items = cm->items ? cm->items : e->d_items.as<SswItem>();
	for (int64_t i : fb) {
		SswAlnDesc d = descs[(size_t)i];
		auto it = task.find(d.first_item);
		if (it == task.end()) {
			const size_t at = fb_items.size();
			fb_items.resize(at + (size_t)d.n_items);
			SSW_CUDA_OK(cudaMemcpy(fb_items.data() + at, items + d.first_item, sizeof(SswItem) * (size_t)d.n_items, cudaMemcpyDeviceToHost));
			for (size_t k = at; k < fb_items.size(); ++k) fb_items[k].cm_off = words;
			words += ((int64_t)d.ref_len / SSW_CM_BLOCK + 1 + 3) / 4 * 4;
			it = task.emplace(d.first_item, (int32_t)at).first;
		}
		d.cm_off = fb_items[(size_t)it->second].cm_off;
		d.first_item = it->second;
		fb_descs.push_back(d);
	}
	if (e->d_bd_items.ensure(sizeof(SswItem) * fb_items.size())) return -1;
	if (e->d_bd_cm.ensure(sizeof(uint32_t) * (size_t)words + 64)) return -1;
	SSW_CUDA_OK(cudaMemcpyAsync(e->d_bd_items.p, fb_items.data(), sizeof(SswItem) * fb_items.size(), cudaMemcpyHostToDevice, e->stream));
	e->laps.start(e->stream);
	const FillPtrs fpx = {e->d_bd_items.as<SswItem>(), e->d_bd_cm.as<uint32_t>(), e->d_rf_bests.as<SswItemBest>()};
	const int rc = dispatch_fill(e, cm->fill_inst, fpx, (int)fb_items.size(), +1, 2, 0, *cm->P);
	if (rc) return rc < 0 ? rc : -1;
	e->laps.stop(e->stream, &e->timing.resolve_ms);
	e->timing.other_launches += 1;
	e->timing.block_exact += (int64_t)fb.size();
	CmMode cx = *cm;
	cx.block = 1; cx.colmax = e->d_bd_cm.as<uint32_t>(); cx.items = e->d_bd_items.as<SswItem>();
	std::vector<SswFillResult> fb_res;
	if (run_resolve(e, fb_descs, second, fb_res, &cx)) return -1;
	for (size_t j = 0; j < fb.size(); ++j) res[(size_t)fb[j]] = fb_res[j];
	return 0;
}

/*
 * Forward bookkeeping shared by both fill kernels: resolve `descs` (semantics `word`), then, where the result must
 * be replaced by the other semantics (needs_other), either re-resolve on the same column maxima -- possible when
 * the rows it was filled on are the padding of the other semantics, i.e. the matrices are identical (the fill never
 * reads the semantics) -- or queue the alignment in `refill` for a fill with the other row count.
 * pad_reuse: byte alignments filled on their word rows (byte_pad > 0) count as filled on the word padding.
 */
static int resolve_forward(ssw_engine* e, std::vector<SswAlnDesc>& descs, const std::vector<int64_t>& desc_aln, std::vector<Aln>& alns,
                           int word, const Sem& S, bool word_first, std::vector<int64_t>* refill, const CmMode* cm = nullptr, bool dual = false,
                           bool pad_reuse = false)
{
	std::vector<SswFillResult> res;
	if (run_resolve(e, descs, true, res, cm)) return -1;
	if (dual) {
		/* descriptors come in pairs: (byte semantics, word semantics) of the same alignment, filled side by side in the two
		 * halves of one pair-task.  The reference takes the byte result unless it overflowed (ssw.c:881-886). */
		for (size_t i = 0; i + 1 < descs.size(); i += 2) {
			Aln& a = alns[desc_aln[i]];
			const bool over = res[i].overflow == 1;
			a.fwd = over ? res[i + 1] : res[i];
			a.word = over ? 1 : 0;
		}
		return 0;
	}
	std::vector<SswAlnDesc> alt;
	std::vector<int64_t> alt_aln;
	for (size_t i = 0; i < descs.size(); ++i) {
		Aln& a = alns[desc_aln[i]];
		a.fwd = res[i]; a.word = word;
		if (!needs_other(res[i], word, S, word_first, a.q)) continue;
		/* the rows the alignment was filled on: a byte alignment filled on its word rows (byte_pad > 0, DESIGN 2) is the
		 * word fill of its read, so its word result lies in the same column maxima and item bests */
		if (lp_of(a.read_len, word) - (pad_reuse ? descs[i].byte_pad : 0) == lp_of(a.read_len, !word)) {
			SswAlnDesc d = descs[i];
			d.word = !word;
			d.limit = S.limit_of(a.q, d.word);
			d.byte_pad = 0;             /* the byte-row columns right of the mask window matter to byte semantics only */
			alt.push_back(d);
			alt_aln.push_back(desc_aln[i]);
		} else if (refill) refill->push_back(desc_aln[i]);
	}
	if (!alt.empty()) {
		if (run_resolve(e, alt, true, res, cm)) return -1;
		for (size_t i = 0; i < alt.size(); ++i) { alns[alt_aln[i]].fwd = res[i]; alns[alt_aln[i]].word = alt[i].word; }
	}
	return 0;
}

/* ------------------------------------------------------------------------------------------- */
/* strip-pipelined fill for queries longer than one strip (ssw_fill_strips_kernel)               */
/* ------------------------------------------------------------------------------------------- */

struct StripReq {             /* one pair-task for the strip kernel */
	int64_t a, b;             /* indices into alns; b = -1: half B dead */
	SswQuery qa, qb;
	int32_t r, cend, p1, term;            /* forward: common reference r, p1 = its length; reverse: half A's window */
	int32_t r_b, cend_b, p1_b, term_b;    /* reverse: half B's reference, end column, scan length, score */
};

/* Launch the strip kernel over `reqs`; every launch hands its descriptors to `after` (resolve + merge). */
static int run_strips(ssw_engine* e, const ssw_batch_params& P, const std::vector<StripReq>& reqs, int dir, bool term,
                      const std::vector<Aln>& alns, float* ms_acc,
                      const std::function<int(std::vector<SswAlnDesc>&, const std::vector<int64_t>&)>& after)
{
	constexpr int R = SSW_STRIP_R;
	Trace tr;
	const int rows_per_strip = 32 * R;
	const size_t warp_smem = (size_t)(P.n + 1) * 32 * R * sizeof(uint32_t);
	/* one launch per distinct strip count (it fixes the CTA shape) */
	std::vector<size_t> order(reqs.size());
	for (size_t i = 0; i < reqs.size(); ++i) order[i] = i;
	auto strips_of = [&](const StripReq& q) { return (std::max(q.qa.lp, q.qb.lp) + rows_per_strip - 1) / rows_per_strip; };
	std::sort(order.begin(), order.end(), [&](size_t x, size_t y) {
		const int sx = strips_of(reqs[x]), sy = strips_of(reqs[y]);
		return sx != sy ? sx < sy : x < y;
	});
	size_t k = 0;
	while (k < order.size()) {
		const int n_strips = strips_of(reqs[order[k]]);
		/* warps per CTA: as many as shared memory allows, preferring a count that divides the strips evenly */
		const int nw_cap = (int)std::min<size_t>(SSW_STRIP_MAXW, (200 * 1024) / warp_smem);
		if (nw_cap < 1) { fprintf(stderr, "[libssw-b200] alphabet too large for the strip kernel\n"); return -2; }
		/* Forward fills may split the strips of a task over `parts` CTAs (see the kernel).  One CTA per SM, every CTA of a
		 * launch lasts about rounds x columns, so the launch lasts ceil(CTAs / SMs) x rounds: take the split that
		 * minimises it (config 5: 500 tasks of 32 strips -> 4 waves x 2 rounds unsplit, 7 waves x 1 round in two parts). */
		size_t n_same = 0;
		for (size_t kk = k; kk < order.size() && strips_of(reqs[order[kk]]) == n_strips; ++kk) ++n_same;
		int parts = 1, nw = 1;
		{
			double best_cost = 1e300;
			const bool may_split = dir > 0 && !term && e->opt.strip_parts != 1;
			const bool forced = may_split && e->opt.strip_parts > 1 && (n_strips + e->opt.strip_parts - 1) / e->opt.strip_parts >= 2;
			for (int pp = 1; pp <= (may_split ? 4 : 1); pp *= 2) {
				if (forced && pp != e->opt.strip_parts) continue;
				const int per = (n_strips + pp - 1) / pp;
				if (pp > 1 && per < 2) break;
				const int wmax = std::min(nw_cap, per);
				int wbest = wmax; double eff_best = 0;
				for (int w = wmax; w >= 1; --w) {
					const double eff = (double)per / (double)(((per + w - 1) / w) * w);
					if (eff > eff_best + 1e-9) { eff_best = eff; wbest = w; }
				}
				const double rounds = (double)((per + wbest - 1) / wbest);
				const double waves = ceil((double)(n_same * pp) / (double)e->sm_count);
				/* a CTA with few warps does not fill an SM: charge it as if it had at least 8 */
				/* a split CTA waits on its predecessor's progress word: charge it ~4 % more per round than an unsplit one */
				const double cost = waves * rounds * (wbest < 8 ? 8.0 / wbest : 1.0) * (pp > 1 ? 1.04 : 1.0);
				if (cost < best_cost - 1e-9) { best_cost = cost; parts = pp; nw = wbest; }
			}
		}
		std::vector<SswStripTask> tasks;
		std::vector<SswAlnDesc> descs;
		std::vector<int64_t> desc_aln;
		size_t cm_words = 0, bnd_words = 0, park_words = 0;
		int n_best = 0;
		const size_t free_b = ssw_free_device_bytes();
		const size_t budget = std::max<size_t>((size_t)256 << 20, ssw_budget_share(free_b + e->d_bnd.cap + e->d_colmax.cap));
		for (; k < order.size() && strips_of(reqs[order[k]]) == n_strips; ++k) {
			const StripReq& q = reqs[order[k]];
			SswStripTask T;
			memset(&T, 0, sizeof(T));
			T.qa = q.qa; T.qb = q.qb;
			T.ref_off = e->r_off[q.r]; T.ref_len = e->r_len[q.r]; T.cend = q.cend; T.p1 = q.p1; T.term_a = q.term;
			T.p1_a = q.p1; T.term_b = -1; T.ref_off_b = T.ref_off; T.cend_b = q.cend; T.p1_b = 0;
			if (dir < 0 && q.b >= 0) {
				T.ref_off_b = e->r_off[q.r_b]; T.cend_b = q.cend_b; T.p1_b = q.p1_b; T.term_b = q.term_b;
				T.p1 = std::max(q.p1, q.p1_b);
			}
			T.n_strips = n_strips;
			T.super = e->opt.strip_super;
			T.n_super = term ? std::max(1, (T.p1 + T.super - 1) / T.super) : 1;
			T.bnd_len = ((T.p1 + 7) / 8 * 8) + 2 * SSW_STRIP_BPAD + 64;
			const size_t need = 4 * (cm_words + bnd_words + park_words + 6 * (size_t)T.bnd_len + (size_t)T.p1 + 8);
			if (!tasks.empty() && need > budget) break;
			T.cm_off = dir > 0 ? (int64_t)cm_words : SSW_CM_NONE;
			T.bnd_off = (int64_t)bnd_words;
			T.park_off = (int64_t)park_words;
			T.first_best = n_best;
			if (dir > 0) cm_words += ((size_t)q.p1 + 7) / 8 * 8 + 8;
			bnd_words += 6 * (size_t)T.bnd_len;
			park_words += (size_t)n_strips * 32 * (2 * R + 3);
			for (int h = 0; h < (q.b >= 0 ? 2 : 1); ++h) {
				const Aln& X = alns[h ? q.b : q.a];
				SswAlnDesc d;
				memset(&d, 0, sizeof(d));
				d.first_item = n_best; d.n_items = n_strips * T.n_super; d.half = h;
				d.ref_len = dir > 0 ? T.ref_len : (h ? q.p1_b : q.p1);
				d.read_len = h ? q.qb.len : q.qa.len;
				d.word = 1; d.limit = 0x7fffffff; d.mask_len = X.mask_len; d.cm_off = T.cm_off; d.scan_all = 1;
				descs.push_back(d);
				desc_aln.push_back(h ? q.b : q.a);
			}
			n_best += n_strips * T.n_super;
			tasks.push_back(T);
		}
		tr.lap("strips: plan");
		if (e->d_items.ensure(sizeof(SswStripTask) * tasks.size())) return -1;
		if (e->d_bests.ensure(sizeof(SswItemBest) * (size_t)n_best)) return -1;
		if (e->d_colmax.ensure(cm_words * 4 + 64)) return -1;
		if (e->d_bnd.ensure(bnd_words * 4 + 64)) return -1;
		if (e->d_park.ensure(park_words * 4 + 64)) return -1;
		tr.lap("strips: ensure");
		SSW_CUDA_OK(cudaMemcpyAsync(e->d_items.p, tasks.data(), sizeof(SswStripTask) * tasks.size(), cudaMemcpyHostToDevice, e->stream));
		SSW_CUDA_OK(cudaMemsetAsync(e->d_bests.p, 0, sizeof(SswItemBest) * (size_t)n_best, e->stream));
		/* ticket counter + one progress word per (task, part) */
		std::vector<int> gsync(1 + tasks.size() * (size_t)parts, -0x40000000);
		gsync[0] = 0;
		if (e->d_sync.ensure(sizeof(int) * gsync.size())) return -1;
		SSW_CUDA_OK(cudaMemcpyAsync(e->d_sync.p, gsync.data(), sizeof(int) * gsync.size(), cudaMemcpyHostToDevice, e->stream));
		const size_t smem = (size_t)nw * warp_smem + sizeof(int) * (size_t)(n_strips + 4);
		tr.lap("strips: h2d + memset");
		e->laps.start(e->stream);
#define SSW_STRIPS_GO(DIR, TERM, SPLIT)                                                                                 \
		do {                                                                                                            \
			auto kern = e->pssm_n ? ssw_fill_strips_kernel<SSW_STRIP_R, DIR, TERM, SPLIT, true>                          \
			                      : ssw_fill_strips_kernel<SSW_STRIP_R, DIR, TERM, SPLIT, false>;                         \
			if (ssw_ensure_dyn_smem(reinterpret_cast<const void*>(kern), smem)) return -1;                              \
			if (e->opt.carve && ssw_prefer_max_smem(reinterpret_cast<const void*>(kern))) return -1;                    \
			ssw_launch(kern, dim3((unsigned)(tasks.size() * (size_t)parts)), dim3(nw * 32), smem, e->stream, (const SswStripTask*)e->d_items.as<SswStripTask>(), \
			           (const int8_t*)e->d_q.as<int8_t>(), (const int8_t*)e->d_r.as<int8_t>(), e->mat_arg(), (int)P.n, \
			           (int)P.gap_open, (int)P.gap_extend, e->d_colmax.as<uint32_t>(), e->d_bnd.as<uint32_t>(), e->d_park.as<uint32_t>(), \
			           e->d_bests.as<SswItemBest>(), parts, e->d_sync.as<int>());                                       \
		} while (0)
		if (dir > 0) { if (parts > 1) SSW_STRIPS_GO(1, false, true); else SSW_STRIPS_GO(1, false, false); }
		else SSW_STRIPS_GO(-1, true, false);
#undef SSW_STRIPS_GO
		SSW_CUDA_OK(cudaGetLastError());
		e->laps.stop(e->stream, ms_acc);
		if (dir > 0) e->timing.fill_forward_launches += 1; else e->timing.other_launches += 1;
		tr.lap("strips: kernel");
		const int rc = after(descs, desc_aln);
		if (rc) return rc;
		tr.lap("strips: resolve + merge");
	}
	return 0;
}

/*
 * One forward fill + bookkeeping over the alignments `sel` with semantics `word` (P1, ssw.c:881-899).
 * word_first: these alignments were given word semantics on a prediction; results whose score fits a byte are
 * replaced by byte semantics.  Alignments that need a fill with the other row count are appended to `refill`.
 */
static int forward_pass(ssw_engine* e, const ssw_batch_params& P, std::vector<Aln>& alns, const std::vector<int64_t>& sel,
                        int word, const Sem& S, bool word_first, std::vector<int64_t>* refill)
{
	if (sel.empty()) return 0;
	Trace tr;
	struct Key { int inst; int32_t r; int32_t q; int32_t lp; int64_t idx; };
	std::vector<Key> keys, long_keys;          /* long_keys: queries longer than one strip */
	/* A pass over few columns cannot fill the device whatever its layout, so its duration is the latency of one group's
	 * sweep: prefer 32 lanes with few rows each (a step is a chain of R dependent cell updates: (32,5) sweeps a 150 bp
	 * query ~4x faster than (8,20), which is the better shape once there is enough work).  This is what a one-pair
	 * ssw_align call gets. */
	int64_t pass_cols = 0;
	for (size_t i = 0; i < sel.size() && pass_cols <= e->opt.latency_cols; ++i) pass_cols += alns[sel[i]].ref_len;
	const bool latency = e->opt.force_inst < 0 && pass_cols <= e->opt.latency_cols;
	/* Byte semantics on the word rows (DESIGN 2): where the byte padding of a read adds pad rows to a word padding that
	 * already has one (length % 16 in 1..7; 150 bp: 152 rows instead of 160), the extra pad rows only raise column maxima
	 * to the H of the last word row a few columns earlier.  That changes neither the best cell nor the overflow test, and
	 * of the second-best scan only the 8 columns right of the mask window, which the block-mode resolve re-fills on the
	 * byte rows.  So it needs block maxima in every launch of the pass: batch layouts, long references or "cm_block" 1. */
	bool byte_rows = word == 0 && !latency && e->opt.cm_block != 0 && P.gap_extend > 0 && S.max_mat > 0;
	if (byte_rows && e->opt.cm_block < 0)
		for (size_t i = 0; i < sel.size() && byte_rows; ++i) if (alns[sel[i]].ref_len < 32768) byte_rows = false;
	auto fill_lp = [&](int len) {
		const int lp = lp_of(len, word);
		return byte_rows && len % 16 >= 1 && len % 16 <= 7 && pick_inst(lp, -1) >= 0 ? lp_of(len, 1) : lp;
	};
	for (size_t i = 0; i < sel.size(); ++i) {
		const Aln& a = alns[sel[i]];
		const int lp = fill_lp(a.read_len);
		int inst = latency ? pick_inst_g32(lp) : -1;
		if (inst < 0) inst = pick_inst(lp, e->opt.force_inst);
		(inst < 0 ? long_keys : keys).push_back(Key{inst < 0 ? 0 : inst, a.r, a.q, lp, sel[i]});
	}
	auto by_ref = [](const Key& x, const Key& y) {
		if (x.inst != y.inst) return x.inst < y.inst;
		if (x.r != y.r) return x.r < y.r;
		if (x.lp != y.lp) return x.lp < y.lp;
		if (x.q != y.q) return x.q < y.q;
		return x.idx < y.idx;
	};

	/* ---- long queries: strip-pipelined kernel, one CTA per pair-task ---- */
	if (!long_keys.empty()) {
		std::sort(long_keys.begin(), long_keys.end(), by_ref);
		std::vector<StripReq> reqs;
		for (size_t i = 0; i < long_keys.size();) {
			StripReq q;
			memset(&q, 0, sizeof(q));
			const Aln& A = alns[long_keys[i].idx];
			q.a = long_keys[i].idx; q.b = -1; q.r = A.r; q.cend = 0; q.p1 = A.ref_len; q.term = -1;
			q.qa.off = (int32_t)e->q_off[A.q]; q.qa.len = A.read_len; q.qa.lp = long_keys[i].lp; q.qa.rev = 0;
			++i;
			if (i < long_keys.size() && long_keys[i].r == A.r) {
				const Aln& B = alns[long_keys[i].idx];
				q.b = long_keys[i].idx;
				q.qb.off = (int32_t)e->q_off[B.q]; q.qb.len = B.read_len; q.qb.lp = long_keys[i].lp; q.qb.rev = 0;
				++i;
			}
			reqs.push_back(q);
			const int lpmax = std::max(q.qa.lp, q.qb.lp);
			e->timing.cells_forward += (int64_t)q.p1 * ((lpmax + 32 * SSW_STRIP_R - 1) / (32 * SSW_STRIP_R)) * 32 * SSW_STRIP_R * 2;
		}
		const int rc = run_strips(e, P, reqs, +1, false, alns, &e->timing.fill_forward_ms,
		                          [&](std::vector<SswAlnDesc>& descs, const std::vector<int64_t>& desc_aln) -> int {
			for (size_t j = 0; j < descs.size(); ++j) { descs[j].word = word; descs[j].limit = S.limit_of(alns[desc_aln[j]].q, word); }
			return resolve_forward(e, descs, desc_aln, alns, word, S, word_first, refill);
		});
		if (rc) return rc;
	}
	if (keys.empty()) return 0;

	/* ---- queries of one strip: pair-tasks = two alignments on the same reference ----
	 * Ordering is done with counting sorts (O(pairs)): a comparison sort of millions of keys costs more than the
	 * kernels for large grids.  rank[q] orders the distinct queries by (instance, padded length, id). */
	struct PT { int inst; int64_t a, b; int32_t r, qa, qb; };
	std::vector<PT> pts;
	/* Latency path with both profiles (a one-pair ssw_align with score_size 2): half B of a lone alignment's pair-task is
	 * idle, so it carries the SAME read with word semantics (other pad rows, other limit).  A read whose byte pass overflows
	 * (ssw.c:883-886) then costs one fill instead of two -- for free. */
	const bool dual = latency && word == 0 && !word_first && S.has_byte && S.has_word;
	if (dual) {
		std::sort(keys.begin(), keys.end(), by_ref);
		pts.reserve(keys.size());
		for (const Key& k : keys) { PT pt; pt.inst = k.inst; pt.a = k.idx; pt.b = k.idx; pt.r = k.r; pt.qa = k.q; pt.qb = k.q; pts.push_back(pt); }
	} else {
		std::vector<int32_t> qids;
		qids.reserve(keys.size());
		std::vector<int32_t> rank((size_t)e->n_q, -1), q_inst((size_t)e->n_q, 0);
		for (const Key& k : keys) if (rank[k.q] < 0) { rank[k.q] = 0; q_inst[k.q] = k.inst; qids.push_back(k.q); }
		std::sort(qids.begin(), qids.end(), [&](int32_t x, int32_t y) {
			if (q_inst[x] != q_inst[y]) return q_inst[x] < q_inst[y];
			const int lx = fill_lp((int)(e->q_off[x + 1] - e->q_off[x])), ly = fill_lp((int)(e->q_off[y + 1] - e->q_off[y]));
			return lx != ly ? lx < ly : x < y;
		});
		for (size_t i = 0; i < qids.size(); ++i) rank[qids[i]] = (int32_t)i;
		const size_t nq = qids.size();
		/* stable LSD: by rank, then by reference */
		std::vector<uint32_t> cnt(std::max<size_t>(nq, (size_t)e->n_r) + 1);
		std::vector<Key> tmp(keys.size());
		std::fill(cnt.begin(), cnt.end(), 0u);
		for (const Key& k : keys) ++cnt[(size_t)rank[k.q] + 1];
		for (size_t i = 1; i <= nq; ++i) cnt[i] += cnt[i - 1];
		for (const Key& k : keys) tmp[cnt[rank[k.q]]++] = k;
		std::fill(cnt.begin(), cnt.end(), 0u);
		for (const Key& k : tmp) ++cnt[(size_t)k.r + 1];
		for (size_t i = 1; i <= (size_t)e->n_r; ++i) cnt[i] += cnt[i - 1];
		for (const Key& k : tmp) keys[cnt[k.r]++] = k;
		/* keys are now ordered by (reference, instance, padded length, query): pair neighbours */
		pts.reserve(keys.size() / 2 + 1);
		for (size_t i = 0; i < keys.size();) {
			PT pt; pt.inst = keys[i].inst; pt.a = keys[i].idx; pt.b = -1; pt.r = keys[i].r; pt.qa = keys[i].q; pt.qb = -1;
			++i;
			if (i < keys.size() && keys[i].inst == pt.inst && keys[i].r == pt.r) { pt.b = keys[i].idx; pt.qb = keys[i].q; ++i; }
			pts.push_back(pt);
		}
		/* query-pair major order (stable by rank of the first query; references stay ascending): consecutive items
		 * then share their two queries, so a CTA needs one profile */
		std::vector<PT> ptmp(pts.size());
		std::fill(cnt.begin(), cnt.end(), 0u);
		for (const PT& t : pts) ++cnt[(size_t)rank[t.qa] + 1];
		for (size_t i = 1; i <= nq; ++i) cnt[i] += cnt[i - 1];
		for (const PT& t : pts) ptmp[cnt[rank[t.qa]]++] = t;
		pts.swap(ptmp);
	}
	tr.lap("forward: sort");
	const size_t free_b = ssw_free_device_bytes();
	size_t cm_budget_words = std::max<size_t>((size_t)1 << 22, ssw_budget_share(free_b + e->d_colmax.cap) / 4);
	if (e->opt.cm_budget > 0) cm_budget_words = std::max<size_t>(1024, (size_t)e->opt.cm_budget / 4);
	tr.lap("forward: memgetinfo");

	size_t k = 0;
	while (k < pts.size()) {
		/* one launch = one kernel instance, bounded by the column-maximum budget */
		const int inst = pts[k].inst;
		const int per_cta = fill_items_per_cta(inst, P.n);   /* items per CTA of a launch with CTA-shared profiles */
		size_t k_end = k, cm_words = 0;
		int64_t total_cols = 0;
		/* Column maxima: one word per column, or -- long references in a launch that fills the device -- one word per block of
		 * SSW_CM_BLOCK columns plus a re-fill of the three blocks per alignment whose single columns matter (ssw_resolve.cuh).
		 * The re-fill needs a bounded warm-up, i.e. the same condition as chunking. */
		/* Block words: exact block maxima ("cm_block" 1) or, by default, the bounded words of CM == 3 (DESIGN 2), which need
		 * gapE > 0 as chunking does. */
		bool block = e->opt.cm_block != 0 && P.gap_extend > 0 && S.max_mat > 0;
		const bool bounded = e->opt.cm_block != 1;
		if (block && e->opt.cm_block < 0) {
			if (latency) block = false;
			for (size_t i = k; block && i < pts.size() && pts[i].inst == inst; ++i) if (e->r_len[pts[i].r] < 32768) block = false;
		}
		auto cm_words_of = [&](int32_t ref_len) -> size_t {
			return block ? ((size_t)ref_len / SSW_CM_BLOCK + 1 + 3) / 4 * 4 : ((size_t)ref_len + 3) / 4 * 4;
		};
		while (k_end < pts.size() && pts[k_end].inst == inst) {
			const size_t words = cm_words_of(e->r_len[pts[k_end].r]);
			if (k_end > k && cm_words + words > cm_budget_words) break;
			cm_words += words;
			total_cols += e->r_len[pts[k_end].r];
			++k_end;
		}
		const int64_t target_items = (int64_t)e->sm_count * 32 * 8;
		const int64_t base_chunk = (total_cols / target_items + 3) / 4 * 4;

		/* chunk every pair-task; a multi-chunk pair-task gets a multiple of per_cta chunks so that its CTAs are full */
		struct Plan { int32_t n_chunks, chunk, warm; };
		std::vector<Plan> plan(k_end - k);
		int64_t live_items = 0, padded_items = 0;
		auto make_plan = [&](int64_t auto_chunk, double* warm_frac) {
			int64_t run_items = 0, cols = 0, warm_cols = 0;
			live_items = 0; padded_items = 0;
			for (size_t i = k; i < k_end; ++i) {
				const PT& pt = pts[i];
				const Aln& A = alns[pt.a];
				const Aln* B = pt.b >= 0 ? &alns[pt.b] : nullptr;
				const int32_t ref_len = e->r_len[pt.r];
				const int max_lp = std::max(lp_of(A.read_len, word), B ? lp_of(B->read_len, dual ? 1 : word) : 0);
				const int max_len = std::max(A.read_len, B ? B->read_len : 0);
				/* a path with positive score spans at most max_lp diagonal steps plus (total positive score)/gapE gap columns */
				int64_t warm = 0, chunk = ref_len;
				if (P.gap_extend > 0 && S.max_mat > 0) {
					warm = (int64_t)max_lp + ((int64_t)max_len * S.max_mat + P.gap_extend - 1) / P.gap_extend + 4;
					warm = (warm + 3) / 4 * 4;
					/* a launch too small to fill the device (one ssw_align call, the word re-fill of a few overflowed reads) is
					 * latency-bound: shorter chunks, at the price of more warm-up columns */
					if (e->opt.chunk > 0) chunk = block ? (e->opt.chunk + SSW_CM_BLOCK - 1) / SSW_CM_BLOCK * SSW_CM_BLOCK : e->opt.chunk;
					else if (latency) chunk = e->opt.small_chunk > 0 ? std::max<int64_t>(e->opt.small_chunk, 2 * warm) : std::max<int64_t>(1024, 2 * warm);   /* a lone call: the device is empty, its duration is one item's sweep */
					else if (base_chunk < 4096) chunk = e->opt.small_chunk > 0 ? std::max<int64_t>(e->opt.small_chunk, 2 * warm) : std::max<int64_t>(2048, 6 * warm);
					else chunk = std::max<int64_t>(std::max<int64_t>(4096, 16 * warm), auto_chunk);
				}
				int64_t n_chunks = chunk >= ref_len ? 1 : (ref_len + chunk - 1) / chunk;
				if (block) chunk = (chunk + SSW_CM_BLOCK - 1) / SSW_CM_BLOCK * SSW_CM_BLOCK;     /* chunks start at block boundaries */
				if (n_chunks > 1 && e->opt.chunk == 0) {
					n_chunks = (n_chunks + per_cta - 1) / per_cta * per_cta;
					chunk = ((ref_len + n_chunks - 1) / n_chunks + 3) / 4 * 4;
					if (block) chunk = (chunk + SSW_CM_BLOCK - 1) / SSW_CM_BLOCK * SSW_CM_BLOCK;
					n_chunks = (ref_len + chunk - 1) / chunk;
				}
				if (n_chunks == 1) chunk = std::max<int32_t>((ref_len + 3) / 4 * 4, 4);
				plan[i - k] = Plan{(int32_t)n_chunks, (int32_t)chunk, (int32_t)warm};
				live_items += n_chunks;
				cols += ref_len; warm_cols += (n_chunks - 1) * warm;
				const bool new_run = i == k || pts[i].qa != pts[i - 1].qa || pts[i].qb != pts[i - 1].qb;
				if (new_run) { padded_items += (run_items + per_cta - 1) / per_cta * per_cta; run_items = 0; }
				run_items += n_chunks;
			}
			padded_items += (run_items + per_cta - 1) / per_cta * per_cta;
			if (warm_frac) *warm_frac = cols > 0 ? (double)warm_cols / (double)cols : 0.0;
		};
		/* Wave quantisation: the CTAs of such a launch all take about the same time, so the launch lasts
		 * ceil(CTAs / resident CTAs) CTA-times.  Try chunk lengths around the default and keep the one with the best
		 * (fill of the last wave) x (1 - warm-up overhead). */
		int64_t auto_chunk = base_chunk;
		if (e->opt.chunk == 0 && base_chunk >= 4096) {
			const int occ = fill_occupancy(inst, P.n, block);
			const double slots = (double)e->sm_count * std::max(occ, 1);
			double best_eff = -1;
			for (int pct = 60; pct <= 150; pct += 5) {
				const int64_t c = (base_chunk * pct / 100 + 3) / 4 * 4;
				double wf = 0;
				make_plan(c, &wf);
				const double ctas = (double)((live_items + per_cta - 1) / per_cta);
				const double waves = ctas / slots;
				const double eff = (waves / ceil(waves - 1e-9)) / (1.0 + wf);
				if (eff > best_eff + 1e-6) { best_eff = eff; auto_chunk = c; }
			}
		}
		make_plan(auto_chunk, nullptr);
		const int share = padded_items * 100 <= live_items * 112 ? 1 : 0;

		std::vector<SswItem> items;
		std::vector<SswAlnDesc> descs;
		std::vector<int64_t> desc_aln;
		items.reserve((size_t)(share ? padded_items : live_items));
		int64_t cells = 0;
		int rf_lp = 0;          /* rows the block re-fill must cover: the byte padding of the alignments filled on their word rows */
		cm_words = 0;
		for (size_t i = k; i < k_end; ++i) {
			const PT& pt = pts[i];
			const Aln& A = alns[pt.a];
			const Aln* B = pt.b >= 0 ? &alns[pt.b] : nullptr;
			const int32_t ref_len = e->r_len[pt.r];
			const Plan& pl = plan[i - k];
			SswItem it;
			memset(&it, 0, sizeof(it));
			it.qa.off = (int32_t)e->q_off[A.q]; it.qa.len = A.read_len; it.qa.lp = fill_lp(A.read_len); it.qa.rev = 0;
			if (B) { it.qb.off = (int32_t)e->q_off[B->q]; it.qb.len = B->read_len; it.qb.lp = dual ? lp_of(B->read_len, 1) : fill_lp(B->read_len); it.qb.rev = 0; }
			it.ref_off = e->r_off[pt.r]; it.ref_len = ref_len; it.term_a = -1;
			if (share && i > k && (pts[i].qa != pts[i - 1].qa || pts[i].qb != pts[i - 1].qb)) {
				/* the queries change: fill the current CTA with dead items (empty range) of the previous queries */
				SswItem dead = items.back();
				dead.p0 = dead.p1 = 0; dead.warm = 0; dead.cm_off = SSW_CM_NONE;
				while (items.size() % (size_t)per_cta) items.push_back(dead);
			}
			const int first_item = (int)items.size();
			/* block mode: every item starts its sweep (p0 - warm) at a block boundary, which the block-mode fill relies on to
			 * find the blocks of all its lanes from the loop count alone (ssw_fill.cuh); a longer warm-up is just as exact */
			const int32_t warm = block ? (pl.warm + SSW_CM_BLOCK - 1) / SSW_CM_BLOCK * SSW_CM_BLOCK : pl.warm;
			for (int c = 0; c < pl.n_chunks; ++c) {
				it.p0 = (int32_t)((int64_t)c * pl.chunk);
				it.p1 = (int32_t)std::min<int64_t>(ref_len, (int64_t)(c + 1) * pl.chunk);
				it.warm = std::min(warm, it.p0);
				it.cm_off = (int64_t)cm_words;
				items.push_back(it);
				cells += (int64_t)(it.p1 - it.p0 + it.warm) * inst_rows(inst) * 2;
			}
			for (int h = 0; h < (B ? 2 : 1); ++h) {
				const Aln& X = h ? *B : A;
				SswAlnDesc d;
				memset(&d, 0, sizeof(d));
				d.first_item = first_item; d.n_items = pl.n_chunks; d.half = h; d.ref_len = ref_len; d.read_len = X.read_len;
				d.word = word; d.limit = S.limit_of(X.q, word); d.mask_len = X.mask_len; d.cm_off = (int64_t)cm_words; d.warm = pl.warm;
				d.byte_pad = lp_of(X.read_len, word) - fill_lp(X.read_len);
				rf_lp = std::max(rf_lp, lp_of(X.read_len, word));
				if (dual && h == 1) { d.word = 1; d.limit = S.limit_word_of(X.q); }
				descs.push_back(d);
				desc_aln.push_back(h ? pt.b : pt.a);
			}
			cm_words += cm_words_of(ref_len);
		}
		tr.lap("forward: plan");
		if (e->d_colmax.ensure(cm_words * 4 + 64)) return -1;
		if (e->run_fill(items, inst, +1, block ? (bounded ? 3 : 2) : 1, share, P, &e->timing.fill_forward_ms)) return -1;
		e->last_cm_words = (int64_t)cm_words;
		tr.lap("forward: fill (copy+kernel)");
		e->timing.fill_forward_launches += 1;
		e->timing.cells_forward += cells;
		const int rows = inst_rows(inst);
		const CmMode cm_mode = {block ? (bounded ? 2 : 1) : 0, rf_lp > rows ? pick_inst(rf_lp, -1) : inst, &P, inst};
		/* The word results of byte overflows filled on their word rows are resolved from this launch when it holds every
		 * pair-task of its kernel instance (the BASELINE shapes: config 3 is one launch per GPU, which then needs no second
		 * one).  Where the column-maximum budget cuts an instance into several launches, those overflows keep the word
		 * re-fill after the pass: that multi-launch path keeps the launch structure it had (budget launches + one re-fill),
		 * and the re-resolve has not been measured there. */
		const bool split = (k > 0 && pts[k - 1].inst == inst) || (k_end < pts.size() && pts[k_end].inst == inst);
		if (resolve_forward(e, descs, desc_aln, alns, word, S, word_first, refill, &cm_mode, dual, !split)) return -1;
		tr.lap("forward: resolve");
		k = k_end;
	}
	return 0;
}

/* Begin search (P2, ssw.c:919-936): one reverse item per alignment, early termination at score1. */
static int reverse_pass(ssw_engine* e, const ssw_batch_params& P, std::vector<Aln>& alns, const std::vector<int64_t>& sel)
{
	if (sel.empty()) return 0;
	struct Key { int inst; int64_t idx; };
	std::vector<Key> keys;
	std::vector<StripReq> long_reqs;
	std::vector<int64_t> long_sel;
	for (size_t i = 0; i < sel.size(); ++i) {
		const Aln& a = alns[sel[i]];
		const int inst = pick_inst_g32(lp_of(a.fwd.read + 1, a.word));
		if (inst >= 0) { keys.push_back(Key{inst, sel[i]}); continue; }
		long_sel.push_back(sel[i]);
	}
	/* long queries: two alignments per strip task (they need not share a reference: half B has its own letter stream),
	 * partners of similar padded length so that neither half drags many dead strips along */
	std::sort(long_sel.begin(), long_sel.end(), [&](int64_t x, int64_t y) {
		const int lx = lp_of(alns[x].fwd.read + 1, alns[x].word), ly = lp_of(alns[y].fwd.read + 1, alns[y].word);
		return lx != ly ? lx > ly : x < y;
	});
	for (size_t i = 0; i < long_sel.size(); i += 2) {
		const Aln& a = alns[long_sel[i]];
		StripReq q;
		memset(&q, 0, sizeof(q));
		q.a = long_sel[i]; q.b = -1; q.r = a.r; q.cend = a.fwd.ref; q.p1 = a.fwd.ref + 1; q.term = a.fwd.score;
		q.qa.off = (int32_t)e->q_off[a.q]; q.qa.len = a.fwd.read + 1; q.qa.lp = lp_of(q.qa.len, a.word); q.qa.rev = 1;
		if (i + 1 < long_sel.size()) {
			const Aln& b = alns[long_sel[i + 1]];
			q.b = long_sel[i + 1]; q.r_b = b.r; q.cend_b = b.fwd.ref; q.p1_b = b.fwd.ref + 1; q.term_b = b.fwd.score;
			q.qb.off = (int32_t)e->q_off[b.q]; q.qb.len = b.fwd.read + 1; q.qb.lp = lp_of(q.qb.len, b.word); q.qb.rev = 1;
		}
		long_reqs.push_back(q);
	}
	auto merge = [&](const std::vector<SswAlnDesc>& descs, const std::vector<int64_t>& desc_aln) -> int {
		std::vector<SswFillResult> res;
		if (run_resolve(e, descs, false, res)) return -1;
		for (size_t i = 0; i < descs.size(); ++i) {
			Aln& a = alns[desc_aln[i]];
			a.rev_score = res[i].score; a.rev_pos = res[i].ref; a.rev_row = res[i].read;
		}
		return 0;
	};
	if (!long_reqs.empty()) {
		const int rc = run_strips(e, P, long_reqs, -1, true, alns, &e->timing.fill_reverse_ms,
		                          [&](std::vector<SswAlnDesc>& descs, const std::vector<int64_t>& desc_aln) -> int { return merge(descs, desc_aln); });
		if (rc) return rc;
	}
	std::sort(keys.begin(), keys.end(), [](const Key& x, const Key& y) { return x.inst != y.inst ? x.inst < y.inst : x.idx < y.idx; });
	size_t k = 0;
	while (k < keys.size()) {
		const int inst = keys[k].inst;
		std::vector<SswItem> items;
		std::vector<SswAlnDesc> descs;
		std::vector<int64_t> desc_aln;
		for (; k < keys.size() && keys[k].inst == inst; ++k) {
			const Aln& a = alns[keys[k].idx];
			SswItem it;
			memset(&it, 0, sizeof(it));
			it.qa.off = (int32_t)e->q_off[a.q]; it.qa.len = a.fwd.read + 1; it.qa.lp = lp_of(it.qa.len, a.word); it.qa.rev = 1;
			it.ref_off = e->r_off[a.r]; it.ref_len = a.ref_len; it.cend = a.fwd.ref;
			it.p0 = 0; it.p1 = a.fwd.ref + 1; it.warm = 0; it.term_a = a.fwd.score; it.cm_off = SSW_CM_NONE;
			SswAlnDesc d;
			memset(&d, 0, sizeof(d));
			d.first_item = (int)items.size(); d.n_items = 1; d.half = 0; d.ref_len = it.p1; d.read_len = it.qa.len;
			d.word = 1; d.limit = 0x7fffffff; d.mask_len = 0; d.cm_off = SSW_CM_NONE;
			items.push_back(it);
			descs.push_back(d);
			desc_aln.push_back(keys[k].idx);
		}
		if (e->run_fill(items, inst, -1, 0, 0, P, &e->timing.fill_reverse_ms)) return -1;
		e->timing.other_launches += 1;
		if (merge(descs, desc_aln)) return -1;
	}
	return 0;
}


/* ------------------------------------------------------------------------------------------- */
/* layout-literal slow path (ssw_emul_kernel): gapO <= gapE, and word scores near saturation     */
/* ------------------------------------------------------------------------------------------- */

/* dir 0: forward fill of alns[sel] with semantics `word`; dir 1: begin search (reverse) of alns[sel]. */
static int emul_pass(ssw_engine* e, const ssw_batch_params& P, std::vector<Aln>& alns, const std::vector<int64_t>& sel,
                     int word, int dir, const Sem& S)
{
	if (sel.empty()) return 0;
	const size_t free_b = ssw_free_device_bytes();
	const size_t budget = std::max<size_t>((size_t)64 << 20, ssw_budget_share(free_b + e->d_emul.cap));
	size_t k = 0;
	while (k < sel.size()) {
		std::vector<SswEmulTask> tasks;
		std::vector<int64_t> task_aln;
		size_t state_words = 0, cm_elems = 0;
		for (; k < sel.size(); ++k) {
			const Aln& a = alns[sel[k]];
			const int w = dir ? a.word : word;
			const int L = w ? 8 : 16;
			SswEmulTask T;
			memset(&T, 0, sizeof(T));
			T.q_off = (int32_t)e->q_off[a.q];
			T.q_len = dir ? a.fwd.read + 1 : a.read_len;
			T.q_rev = dir;
			T.ref_len = dir ? a.fwd.ref + 1 : a.ref_len;
			T.ref_off = e->r_off[a.r];
			T.dir = dir; T.word = w;
			T.terminate = dir ? a.fwd.score : (w ? 65535 : 255);
			T.bias = S.bias_of(a.q); T.mask_len = a.mask_len;
			const size_t st = 4 * (size_t)((T.q_len + L - 1) / L) * L;
			const size_t cm = ((size_t)T.ref_len + 7) / 8 * 8;
			if (!tasks.empty() && 4 * (state_words + st) + 2 * (cm_elems + cm) > budget) break;
			T.state_off = (int64_t)state_words; T.cm_off = (int64_t)cm_elems;
			state_words += st; cm_elems += cm;
			tasks.push_back(T);
			task_aln.push_back(sel[k]);
		}
		const size_t off_cm = (state_words * 4 + 255) / 256 * 256;
		const size_t off_tasks = off_cm + (cm_elems * 2 + 255) / 256 * 256;
		const size_t off_res = off_tasks + (sizeof(SswEmulTask) * tasks.size() + 255) / 256 * 256;
		if (e->d_emul.ensure(off_res + sizeof(SswFillResult) * tasks.size())) return -1;
		uint8_t* base = e->d_emul.as<uint8_t>();
		SSW_CUDA_OK(cudaMemsetAsync(base + off_cm, 0, cm_elems * 2, e->stream));
		SSW_CUDA_OK(cudaMemcpyAsync(base + off_tasks, tasks.data(), sizeof(SswEmulTask) * tasks.size(), cudaMemcpyHostToDevice, e->stream));
		e->laps.start(e->stream);
		ssw_launch(ssw_emul_kernel, dim3(((int)tasks.size() + SSW_EMUL_WARPS - 1) / SSW_EMUL_WARPS), dim3(SSW_EMUL_THREADS), 0, e->stream,
		           (const SswEmulTask*)reinterpret_cast<SswEmulTask*>(base + off_tasks), (int)tasks.size(),
		           (const int8_t*)e->d_q.as<int8_t>(), (const int8_t*)e->d_r.as<int8_t>(), e->mat_arg(), (int)P.n,
		           (int)P.gap_open, (int)P.gap_extend, reinterpret_cast<int32_t*>(base), reinterpret_cast<uint16_t*>(base + off_cm),
		           reinterpret_cast<SswFillResult*>(base + off_res));
		SSW_CUDA_OK(cudaGetLastError());
		e->laps.stop(e->stream, dir ? &e->timing.fill_reverse_ms : &e->timing.fill_forward_ms);
		if (dir) e->timing.other_launches += 1; else e->timing.fill_forward_launches += 1;
		std::vector<SswFillResult> res(tasks.size());
		SSW_CUDA_OK(cudaMemcpyAsync(res.data(), base + off_res, sizeof(SswFillResult) * tasks.size(), cudaMemcpyDeviceToHost, e->stream));
		SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
		for (size_t i = 0; i < tasks.size(); ++i) {
			Aln& a = alns[task_aln[i]];
			if (dir) { a.rev_score = res[i].score; a.rev_pos = a.fwd.ref - res[i].ref; a.rev_row = res[i].read; }
			else { a.fwd = res[i]; a.word = word; }
		}
	}
	return 0;
}

/* ------------------------------------------------------------------------------------------- */
/* large grids, scores only: descriptors planned on the device (ssw_grid.cuh)                     */
/* ------------------------------------------------------------------------------------------- */


struct SearchHit { int32_t r; ssw_batch_result rec; };

/* Top-k search on the grid path (ssw_engine_search): a selection kernel replaces the emit kernel, and an n_q x k hit table on the
 * device replaces the n_pairs records.  Filled by grid_scores: each query's hits among the pairs that are final on the grid.
 * k == 0 is the threshold search (ssw_engine_search_all): a count and a compaction kernel replace the emit kernel, and every
 * hit of a launch group is copied back, in reference order, while the next group computes. */
struct GridSearch {
	int32_t k, min_score;                   /* min_score >= 1 */
	int64_t max_hits = 0;                   /* k == 0: more hits on the grid than this end the call (-2) */
	std::vector<int32_t> hit_ref, n_hits;   /* n_q * k, n_q */
	std::vector<ssw_batch_result> hits;     /* n_q * k */
	std::vector<std::vector<SearchHit>> rows;   /* k == 0: n_q rows of grid hits in ascending reference index (the caller's) */
	std::vector<uint8_t> q_on, r_on;        /* n_q, n_r: the grid path computed the pairs (q, r) with q_on[q] && r_on[r] */
	/* self-search (k == 0, one set resident as queries and references): rank[i] is sequence i's place in canonical order; only
	 * queries ranked in [rank_lo, rank_hi) are on the grid, and each only against the references ranked after it -- the pairs
	 * (q, r) with q_on[q] && r_on[r] && rank[r] > rank[q] */
	const int32_t* rank = nullptr;
	int32_t rank_lo = 0, rank_hi = 0;
};

/* Returns 1 when the grid path handled the batch (results filled -- or, with `gs`, the hit table; `redo` lists pairs to re-do
 * by the general path, numbered q * n_r + r), 0 when the batch is not eligible, < 0 on error.
 * An align (`results`) takes the grid as a whole or not at all.  A search (`gs`) takes the queries and the references that
 * qualify one by one and reports them in gs->q_on / r_on; every other pair is left to the caller.  A search's references are
 * cut into grid tiles (contiguous ranges of them), each run as a grid of its own, where the grid has more pairs than 32-bit
 * pair numbers hold or one query pair's scratch over all references exceeds the launch budget. */
static int grid_scores(ssw_engine* e, const ssw_batch_params& P, const Sem& S, int64_t n_pairs,
                       ssw_batch_result* results, std::vector<int64_t>* redo, GridSearch* gs = nullptr)
{
	if (n_pairs != (int64_t)e->n_q * e->n_r || n_pairs < e->opt.grid_min_pairs || (!gs && n_pairs > 0x7fffffff)) return 0;
	if (P.flag != 0 || P.gap_open <= P.gap_extend || e->opt.chunk != 0) return 0;
	if (!S.has_byte && !S.has_word) return 0;
	const int word = S.has_byte ? 0 : 1;
	const int n_q = e->n_q, n_r_all = e->n_r;
	/* The references of the grid, in ascending order of their index: the device's tables hold these n_r sequences only and
	 * number them 0 .. n_r - 1 (the selection kernel breaks ties by that number, which the ascending order keeps equivalent
	 * to the caller's index); rsel maps back. */
	std::vector<int32_t> rsel;
	for (int r = 0; r < n_r_all; ++r) if (e->r_len[r] <= e->opt.grid_max_ref) rsel.push_back(r);
	const int n_r = (int)rsel.size();
	/* after[q]: the first device number query q is paired with -- the references q needs are [after[q], n_r) -- and after[n_q]
	 * that of a missing second query.  Self-search: the references in canonical order instead (a tile is then a range of ranks),
	 * and after[q] the first device number ranked after sequence q.  The host sorts each row by index at the end. */
	const bool self = gs && gs->rank;
	std::vector<int32_t> after((size_t)n_q + 1, 0);
	if (self) {
		std::sort(rsel.begin(), rsel.end(), [&](int32_t x, int32_t y) { return gs->rank[x] < gs->rank[y]; });
		std::vector<int32_t> canon((size_t)n_q);
		for (int q = 0; q < n_q; ++q) canon[gs->rank[q]] = q;
		for (int t = 0, d = 0; t < n_q; ++t) {
			if (d < n_r && rsel[d] == canon[t]) ++d;
			after[canon[t]] = d;
		}
		after[n_q] = n_r;
	}
	/* The queries of the grid keep their index (the tables hold all of them; the others are in no query pair). */
	std::vector<SswGridQ> qt((size_t)n_q);
	std::vector<int> q_inst((size_t)n_q, -1);
	std::vector<int32_t> order;
	for (int q = 0; q < n_q; ++q) {
		const int len = (int)(e->q_off[q + 1] - e->q_off[q]);
		qt[q].off = (int32_t)e->q_off[q]; qt[q].len = len; qt[q].lp = lp_of(std::max(len, 1), word);
		qt[q].mask_len = P.mask_len < 0 ? len / 2 : P.mask_len;
		qt[q].limit = S.limit_of(q, word);
		if (len < 1) continue;
		if (self && (gs->rank[q] < gs->rank_lo || gs->rank[q] >= gs->rank_hi)) continue;
		if (S.has_byte && S.has_word && (int64_t)len * std::max(S.max_of(q), 0) >= 2 * (int64_t)S.limit_byte_of(q)) continue;   /* word-first prediction: general path */
		q_inst[q] = pick_inst(qt[q].lp, e->opt.force_inst);
		if (q_inst[q] >= 0) order.push_back(q);
	}
	const int n_qe = (int)order.size();
	if (!gs && (n_r != n_r_all || n_qe != n_q)) return 0;
	int64_t grid_pairs = 0;
	for (int32_t q : order) grid_pairs += n_r - after[q];
	if (n_qe == 0 || grid_pairs < std::max(e->opt.grid_min_pairs, 1)) return 0;
	Trace tr;
	/* self-search: query pairs of consecutive queries in canonical order within an instance, half a the earlier one */
	std::sort(order.begin(), order.end(), [&](int32_t x, int32_t y) {
		if (q_inst[x] != q_inst[y]) return q_inst[x] < q_inst[y];
		if (self) return gs->rank[x] < gs->rank[y];
		if (qt[x].lp != qt[y].lp) return qt[x].lp < qt[y].lp;
		return x < y;
	});
	/* static tables on the device: [qt][ref_off][ref_len][cm_prefix][perm]; the reference tables hold one grid tile at a time,
	 * at most all n_r references */
	const size_t o_qt = 0, o_roff = o_qt + (sizeof(SswGridQ) * n_q + 255) / 256 * 256, o_rlen = o_roff + (8 * (size_t)n_r + 255) / 256 * 256;
	const size_t o_cmp = o_rlen + (4 * (size_t)n_r + 255) / 256 * 256, o_perm = o_cmp + (8 * (size_t)n_r + 255) / 256 * 256;
	const size_t o_qp = o_perm + (4 * (size_t)n_r + 255) / 256 * 256;
	const size_t o_cnt = o_qp + (sizeof(SswGridQp) * (size_t)(n_q / 2 + 2) + 255) / 256 * 256, o_list = o_cnt + 256;
	const int32_t redo_cap = (int32_t)std::min<int64_t>((int64_t)n_qe * n_r, 1 << 22);
	/* threshold search: behind the redo list, the hit counts of a launch group's query slots and their exclusive prefix */
	const bool all = gs && gs->k == 0;
	const size_t n_slots = all ? 2 * (size_t)(n_q / 2 + 1) : 0;
	const size_t o_scnt = o_list + (4 * (size_t)redo_cap + 255) / 256 * 256, o_soff = o_scnt + (4 * n_slots + 255) / 256 * 256;
	if (e->d_grid.ensure(all ? o_soff + 8 * (n_slots + 1) : o_list + 4 * (size_t)redo_cap)) return -1;
	uint8_t* gb = e->d_grid.as<uint8_t>();
	SSW_CUDA_OK(cudaMemcpyAsync(gb + o_qt, qt.data(), sizeof(SswGridQ) * n_q, cudaMemcpyHostToDevice, e->stream));
	SSW_CUDA_OK(cudaMemsetAsync(gb + o_cnt, 0, 256, e->stream));
	/* search: [hits n_q*k][hit_ref n_q*k][n_hits n_q], every row written by the selection kernel of its query (first grid tile)
	 * or merged from a table of the same layout at o_tile (later tiles) */
	const size_t o_href = sizeof(ssw_batch_result) * (size_t)n_q * (gs ? gs->k : 0), o_nh = o_href + 4 * (size_t)n_q * (gs ? gs->k : 0);
	const size_t o_tile = o_nh + 4 * (size_t)n_q;
	if (all) {
		/* the hits of one launch group at a time, in e->d_hits (grown per group) */
	} else if (gs ? e->d_hits.ensure(o_tile) : e->d_out.ensure(sizeof(ssw_batch_result) * (size_t)n_pairs)) return -1;
	/* threshold search: the group whose hits are still on the device, and a copy that brings them to gs->rows.  The device buffer
	 * is written by the next group's compaction only after this copy has returned, so one buffer serves every group. */
	struct HitGroup { int64_t n = 0; std::vector<int64_t> off; std::vector<int32_t> q; int32_t r_lo = 0; cudaEvent_t ev = nullptr; };
	HitGroup pend;
	int64_t grid_hits = 0;
	if (all) gs->rows.assign((size_t)n_q, std::vector<SearchHit>());
	auto flush_hits = [&]() -> int {
		if (pend.n == 0) return 0;
		if (!e->side[0]) SSW_CUDA_OK(cudaStreamCreateWithFlags(&e->side[0], cudaStreamNonBlocking));
		SSW_CUDA_OK(cudaStreamWaitEvent(e->side[0], pend.ev, 0));
		std::vector<ssw_batch_result> h((size_t)pend.n);
		std::vector<int32_t> hr((size_t)pend.n);
		const size_t o_ref = (sizeof(ssw_batch_result) * (size_t)pend.n + 255) / 256 * 256;
		if (e->staged.copy(h.data(), e->d_hits.p, sizeof(ssw_batch_result) * (size_t)pend.n, e->side[0])) return -1;
		if (e->staged.copy(hr.data(), e->d_hits.as<uint8_t>() + o_ref, 4 * (size_t)pend.n, e->side[0])) return -1;
		for (size_t s = 0; s < pend.q.size(); ++s) {
			if (pend.q[s] < 0) continue;
			std::vector<SearchHit>& row = gs->rows[pend.q[s]];
			for (int64_t i = pend.off[s]; i < pend.off[s + 1]; ++i) row.push_back(SearchHit{rsel[pend.r_lo + hr[i]], h[i]});   /* rsel ascending: order kept */
		}
		pend = HitGroup();
		return 0;
	};

	const size_t free_b = ssw_free_device_bytes();
	const size_t budget = std::max<size_t>((size_t)256 << 20, ssw_budget_share(free_b + e->d_colmax.cap + e->d_items.cap + e->d_alns.cap + e->d_res.cap));
	tr.lap("grid: tables");
	/* Grid tiles of a search: the longest runs of references (in rsel order) with at most 2^31 - 1 pairs numbered q * n_rt + r
	 * (q: any resident query) and one query pair's scratch within the budget -- one tile wherever both hold for all references.
	 * An align is never cut. */
	std::vector<int32_t> tile_lo(1, 0);
	if (gs) {
		std::vector<int> per_ctas;                   /* items per CTA of the instances of the grid's queries */
		for (int32_t q : order) {
			const int c = fill_items_per_cta(q_inst[q], P.n);
			if (std::find(per_ctas.begin(), per_ctas.end(), c) == per_ctas.end()) per_ctas.push_back(c);
		}
		auto qp_bytes = [&](int64_t nr, int64_t cm_words) {   /* per_qp of the launch groups below, for the widest instance */
			size_t b = 0;
			for (int c : per_ctas)
				b = std::max(b, (size_t)cm_words * 4 + (size_t)((nr + c - 1) / c * c) * (sizeof(SswItem) + sizeof(SswItemBest)) + (size_t)nr * 2 * (sizeof(SswAlnDesc) + sizeof(SswFillResult)));
			return b;
		};
		int64_t cap = 0x7fffffff / n_q;
		if (e->opt.grid_tile_refs > 0) cap = std::min(cap, e->opt.grid_tile_refs);
		int64_t cm_words = 0;
		for (int r = 0; r < n_r; ++r) {
			const int64_t w = ((int64_t)e->r_len[rsel[r]] + 3) / 4 * 4, n = r - tile_lo.back();
			if (n > 0 && (n + 1 > cap || qp_bytes(n + 1, cm_words + w) > budget)) { tile_lo.push_back(r); cm_words = 0; }
			cm_words += w;
		}
	}
	tile_lo.push_back(n_r);
	const size_t n_tiles = tile_lo.size() - 1;
	if (gs && !all) {
		if (n_tiles > 1 && e->d_hits.ensure(o_tile + o_nh + 4 * (size_t)n_q)) return -1;
		SSW_CUDA_OK(cudaMemsetAsync(e->d_hits.as<uint8_t>() + o_nh, 0, 4 * (size_t)n_q, e->stream));   /* queries off the grid: no hits here */
	}
	/* The redo list holds the pairs of one tile, numbered on its tables; after each tile they are mapped to the caller's numbers.
	 * More than the list holds in any tile: the whole call goes through the general path (the overflows cannot be found). */
	bool redo_over = false;
	auto take_redo = [&](int32_t r_lo, int32_t n_rt) -> int {
		int32_t n_redo = 0;
		SSW_CUDA_OK(cudaMemcpyAsync(&n_redo, gb + o_cnt, 4, cudaMemcpyDeviceToHost, e->stream));
		SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
		if (n_redo > redo_cap) { redo_over = true; return 0; }
		if (n_redo) {
			std::vector<int32_t> list((size_t)n_redo);
			SSW_CUDA_OK(cudaMemcpy(list.data(), gb + o_list, 4 * (size_t)n_redo, cudaMemcpyDeviceToHost));
			for (int32_t p : list) redo->push_back((int64_t)(p / n_rt) * n_r_all + rsel[r_lo + p % n_rt]);
		}
		return 0;
	};
	struct GridGroup { cudaEvent_t ev; int32_t q_lo, q_n; bool contiguous; };
	std::vector<GridGroup> groups;
	/* Late arming of the best-cell bookkeeping (ssw_fill.cuh): rows are recorded in the last arm_tail columns of every
	 * reference only.  Automatic for protein-like alphabets, where the running maximum grows with every column and the
	 * maximum of a pair lies near the end of the reference; a small pilot group goes first and the rest of the grid is
	 * armed from column 0 again if more than 0.2 % of the pilot's pairs had to be re-done.  The pilot runs in the first tile. */
	bool arm_on = e->opt.grid_arm > 0 || (e->opt.grid_arm < 0 && P.n > 8 && e->grid_arm_ok);
	bool pilot_pending = arm_on && e->opt.grid_arm < 0;
	int64_t pilot_pairs = 0;
	/* The order in which a query pair's slots sweep a tile's references: ascending slot_key, stable.  Longest first: the groups
	 * of a warp run until the longest of their items is done, so neighbours of equal length waste no steps, and the longest
	 * items of a launch start first; references of equal length keep their order (a database of one length is launched exactly
	 * as without it).  Self-search: the canonical order reversed, so that the references a query pair needs, those ranked after
	 * its queries, are a prefix of its slots. */
	std::vector<int64_t> slot_key((size_t)n_r, 0);
	for (int r = 0; r < n_r; ++r) slot_key[r] = self ? -r : e->opt.grid_order ? -(int64_t)e->r_len[rsel[r]] : 0;
	for (size_t t = 0; t < n_tiles; ++t) {
		const int32_t r_lo = tile_lo[t], n_rt = tile_lo[t + 1] - r_lo;
		/* the tile's reference tables: its references numbered 0 .. n_rt - 1 (cm_prefix[n_rt]: the column-maximum words of all) */
		std::vector<int64_t> cm_prefix((size_t)n_rt + 1, 0), g_off((size_t)n_rt);
		std::vector<int32_t> g_len((size_t)n_rt), perm((size_t)n_rt);
		for (int r = 0; r < n_rt; ++r) {
			g_off[r] = e->r_off[rsel[r_lo + r]]; g_len[r] = e->r_len[rsel[r_lo + r]]; perm[r] = r;
			cm_prefix[r + 1] = cm_prefix[r] + ((int64_t)g_len[r] + 3) / 4 * 4;
		}
		std::stable_sort(perm.begin(), perm.end(), [&](int32_t x, int32_t y) { return slot_key[r_lo + x] < slot_key[r_lo + y]; });
		/* The planned sweep of a query pair whose live slots are the first m: useful columns useful_pre[m], and group-columns of
		 * the warps (groups per warp x the warp's longest item) planned_pre[s][m] with 2^s groups per warp (1, 2, 4). */
		std::vector<int64_t> useful_pre((size_t)n_rt + 1, 0), planned_pre[3];
		for (int rr = 0; rr < n_rt; ++rr) useful_pre[rr + 1] = useful_pre[rr] + g_len[perm[rr]];
		for (int s = 0; s < 3; ++s) {
			planned_pre[s].assign((size_t)n_rt + 1, 0);
			int64_t warps = 0;                       /* the warps that are complete in the first rr slots */
			int32_t longest = 0;                     /* the longest slot of the warp that is not */
			for (int rr = 0; rr < n_rt; ++rr) {
				longest = std::max(longest, g_len[perm[rr]]);
				planned_pre[s][rr + 1] = (warps + longest) << s;
				if (((rr + 1) & ((1 << s) - 1)) == 0) { warps += longest; longest = 0; }
			}
		}
		SSW_CUDA_OK(cudaMemcpyAsync(gb + o_roff, g_off.data(), 8 * (size_t)n_rt, cudaMemcpyHostToDevice, e->stream));
		SSW_CUDA_OK(cudaMemcpyAsync(gb + o_rlen, g_len.data(), 4 * (size_t)n_rt, cudaMemcpyHostToDevice, e->stream));
		SSW_CUDA_OK(cudaMemcpyAsync(gb + o_cmp, cm_prefix.data(), 8 * (size_t)n_rt, cudaMemcpyHostToDevice, e->stream));
		SSW_CUDA_OK(cudaMemcpyAsync(gb + o_perm, perm.data(), 4 * (size_t)n_rt, cudaMemcpyHostToDevice, e->stream));
		size_t k = 0;
		while (k < order.size()) {
			const int inst = q_inst[order[k]];
			const int per_cta = fill_items_per_cta(inst, P.n);
			/* query pairs of this launch: same instance, bounded by memory (their live scratch, below) */
			size_t max_qp = SIZE_MAX;
			/* large grids: several launch groups even when memory would allow one, so that the records of a finished group are
			 * copied to the host while the next group computes (115 MB of records per million pairs) */
			if ((int64_t)n_qe * n_r >= e->opt.grid_split_pairs)
				max_qp = std::min<size_t>(max_qp, std::max<size_t>((size_t)std::max(e->opt.grid_group_qp, 1), ((size_t)n_qe / 2 + 7) / 8));
			if (pilot_pending && (size_t)n_qe / 2 >= 16) max_qp = std::min<size_t>(max_qp, std::max<size_t>(2, (size_t)n_qe / 64));   /* the pilot: 1/32 of the queries */
			std::vector<SswGridQp> qps;                 /* the launch's query-pair table; n_qp + 1 entries once complete */
			int64_t n_items = 0, n_live = 0, cm_words = 0, pairs = 0, cols_useful = 0, cols_planned = 0;
			size_t bytes = 0;
			const int spw = kInst[inst].G == 32 ? 0 : kInst[inst].G == 16 ? 1 : 2;   /* log2 of the groups per warp */
			const size_t k_first = k;
			while (k < order.size() && q_inst[order[k]] == inst && qps.size() < max_qp) {
				SswGridQp s;
				const size_t k_pr = k;
				s.qa = order[k++]; s.qb = -1;
				if (k < order.size() && q_inst[order[k]] == inst) s.qb = order[k++];
				/* the tile's references each half needs, in tile numbers; a query pair with none is not launched */
				s.lo_a = std::min(std::max(after[s.qa] - r_lo, 0), n_rt);
				s.lo_b = std::min(std::max(after[s.qb < 0 ? n_q : s.qb] - r_lo, 0), n_rt);
				const int64_t m = n_rt - s.lo_a, m_pad = (m + per_cta - 1) / per_cta * per_cta, cm = cm_prefix[n_rt] - cm_prefix[s.lo_a];
				if (m == 0) continue;
				const size_t b = (size_t)cm * 4 + (size_t)m_pad * (sizeof(SswItem) + sizeof(SswItemBest)) + (size_t)m * 2 * (sizeof(SswAlnDesc) + sizeof(SswFillResult));
				if (!qps.empty() && bytes + b > budget) { k = k_pr; break; }
				bytes += b;
				s.item0 = n_items; s.desc0 = n_live; s.cm0 = cm_words;
				qps.push_back(s);
				n_items += m_pad; n_live += m; cm_words += cm; pairs += m + (n_rt - s.lo_b);
				cols_useful += useful_pre[m]; cols_planned += planned_pre[spw][m];
			}
			if (qps.empty()) continue;
			SswGridArgs A;
			A.n_qp = (int32_t)qps.size(); A.n_r = n_rt; A.word = word;
			A.arm_tail = 0;
			if (arm_on) {
				int lp_max = 0;
				for (const SswGridQp& s : qps) { lp_max = std::max(lp_max, qt[s.qa].lp); if (s.qb >= 0) lp_max = std::max(lp_max, qt[s.qb].lp); }
				A.arm_tail = e->opt.grid_arm > 0 ? e->opt.grid_arm : lp_max / 4 + 64;
			}
			qps.push_back(SswGridQp{-1, -1, n_rt, n_rt, n_items, n_live, cm_words});
			const int64_t n_desc = 2 * n_live;
			if (n_items > 0x7fffffff || n_desc > 0x7fffffff) return 0;
			if (e->d_items.ensure(sizeof(SswItem) * (size_t)n_items)) return -1;
			if (e->d_bests.ensure(sizeof(SswItemBest) * (size_t)n_items)) return -1;
			if (e->d_alns.ensure(sizeof(SswAlnDesc) * (size_t)n_desc)) return -1;
			if (e->d_res.ensure(sizeof(SswFillResult) * (size_t)n_desc)) return -1;
			if (e->d_colmax.ensure((size_t)cm_words * 4 + 64)) return -1;
			SSW_CUDA_OK(cudaMemcpyAsync(gb + o_qp, qps.data(), sizeof(SswGridQp) * qps.size(), cudaMemcpyHostToDevice, e->stream));
			const SswGridQp* d_qp = reinterpret_cast<const SswGridQp*>(gb + o_qp);
			e->laps.start(e->stream);
			ssw_launch(ssw_grid_plan_kernel, dim3((unsigned)((n_items + 255) / 256)), dim3(256), 0, e->stream, A,
			           d_qp, (const SswGridQ*)reinterpret_cast<SswGridQ*>(gb + o_qt),
			           (const int64_t*)reinterpret_cast<int64_t*>(gb + o_roff), (const int32_t*)reinterpret_cast<int32_t*>(gb + o_rlen),
			           (const int64_t*)reinterpret_cast<int64_t*>(gb + o_cmp), (const int32_t*)reinterpret_cast<int32_t*>(gb + o_perm),
			           e->d_items.as<SswItem>(), e->d_alns.as<SswAlnDesc>());
			SSW_CUDA_OK(cudaGetLastError());
			e->laps.stop(e->stream, &e->timing.resolve_ms);
			e->timing.other_launches += 1;
			/* fill (items are already on the device) */
			{
				e->laps.start(e->stream);
				FillPtrs fp = {e->d_items.as<SswItem>(), e->d_colmax.as<uint32_t>(), e->d_bests.as<SswItemBest>()};
				fp.arm = A.arm_tail > 0;
				const int rc = dispatch_fill(e, inst, fp, (int)n_items, +1, 1, 1, P);
				if (rc) return rc < 0 ? rc : -1;
				e->laps.stop(e->stream, &e->timing.fill_forward_ms);
				e->timing.fill_forward_launches += 1;
				e->timing.cells_forward += cm_words * inst_rows(inst) * 2;
				e->timing.grid_cols_useful += cols_useful;
				e->timing.grid_cols_planned += cols_planned;
			}
			e->laps.start(e->stream);
			{
				const int per = SSW_RESOLVE_THREADS / 32;
				ssw_launch(ssw_resolve_kernel<true>, dim3((unsigned)((n_desc + per - 1) / per)), dim3(SSW_RESOLVE_THREADS), 0, e->stream,
				           (const SswAlnDesc*)e->d_alns.as<SswAlnDesc>(), (int)n_desc, (const SswItemBest*)e->d_bests.as<SswItemBest>(),
				           (const uint32_t*)e->d_colmax.as<uint32_t>(), e->d_res.as<SswFillResult>());
				if (!gs)
					ssw_launch(ssw_grid_emit_kernel, dim3((unsigned)((n_desc + 255) / 256)), dim3(256), 0, e->stream, A,
					           d_qp, (const SswGridQ*)reinterpret_cast<SswGridQ*>(gb + o_qt),
					           (const SswFillResult*)e->d_res.as<SswFillResult>(), e->d_out.as<ssw_batch_result>(),
					           reinterpret_cast<int32_t*>(gb + o_list), reinterpret_cast<int32_t*>(gb + o_cnt), redo_cap);
				else if (all)
					ssw_launch(ssw_grid_count_kernel, dim3((unsigned)(2 * A.n_qp)), dim3(SSW_SELECT_THREADS), 0, e->stream, A,
					           d_qp, (const SswGridQ*)reinterpret_cast<SswGridQ*>(gb + o_qt),
					           (const SswFillResult*)e->d_res.as<SswFillResult>(), gs->min_score, reinterpret_cast<int32_t*>(gb + o_scnt),
					           reinterpret_cast<int32_t*>(gb + o_list), reinterpret_cast<int32_t*>(gb + o_cnt), redo_cap);
				else {
					/* the first tile selects into the running table; a later tile into the tile table, merged into the running one */
					uint8_t* hb = e->d_hits.as<uint8_t>(), *tb = hb + (t ? o_tile : 0);
					ssw_launch(ssw_grid_select_kernel, dim3((unsigned)(2 * A.n_qp)), dim3(SSW_SELECT_THREADS), 0, e->stream, A,
					           d_qp, (const SswGridQ*)reinterpret_cast<SswGridQ*>(gb + o_qt),
					           (const SswFillResult*)e->d_res.as<SswFillResult>(), gs->k, gs->min_score,
					           reinterpret_cast<int32_t*>(tb + o_href), reinterpret_cast<ssw_batch_result*>(tb), reinterpret_cast<int32_t*>(tb + o_nh),
					           reinterpret_cast<int32_t*>(gb + o_list), reinterpret_cast<int32_t*>(gb + o_cnt), redo_cap);
					if (t) {
						ssw_launch(ssw_grid_merge_kernel, dim3((unsigned)(2 * A.n_qp)), dim3(SSW_SELECT_THREADS), 0, e->stream,
						           d_qp, gs->k, r_lo,
						           reinterpret_cast<int32_t*>(hb + o_href), reinterpret_cast<ssw_batch_result*>(hb), reinterpret_cast<int32_t*>(hb + o_nh),
						           (const int32_t*)reinterpret_cast<int32_t*>(tb + o_href), (const ssw_batch_result*)reinterpret_cast<ssw_batch_result*>(tb),
						           (const int32_t*)reinterpret_cast<int32_t*>(tb + o_nh));
						e->timing.other_launches += 1;
					}
				}
				SSW_CUDA_OK(cudaGetLastError());
			}
			e->laps.stop(e->stream, &e->timing.resolve_ms);
			e->timing.other_launches += 2;
			/* the group's records are final once its emit kernel has run: remember the event and, when the group's queries are a
			 * contiguous ascending range (equal-length queries: `order` is the identity), the slice of records they own */
			GridGroup gg;
			if (e->grid_event(groups.size(), &gg.ev)) return -1;
			SSW_CUDA_OK(cudaEventRecord(gg.ev, e->stream));
			gg.q_lo = order[k_first]; gg.q_n = (int32_t)(k - k_first); gg.contiguous = true;
			for (size_t i = k_first; i < k; ++i) if (order[i] != gg.q_lo + (int32_t)(i - k_first)) gg.contiguous = false;
			groups.push_back(gg);
			if (pilot_pending) {
				/* how many of the pilot's pairs must be re-done?  (byte overflows count too: either way the grid path does not pay off) */
				pilot_pending = false;
				int32_t n_now = 0;
				SSW_CUDA_OK(cudaMemcpyAsync(&n_now, gb + o_cnt, 4, cudaMemcpyDeviceToHost, e->stream));
				SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
				pilot_pairs = pairs;
				if ((int64_t)n_now * 500 > pilot_pairs) {    /* a re-done pair costs ~400x what arming saves per pair */
					/* arming does not pay for these sequences: forget the pilot (its re-do list too) and run its queries again,
					 * armed from column 0, as the first regular group -- 1/32 of the grid is computed twice, nothing goes through
					 * the general path */
					arm_on = false; e->grid_arm_ok = false;
					SSW_CUDA_OK(cudaMemsetAsync(gb + o_cnt, 0, 256, e->stream));
					groups.pop_back();
					k = k_first;
					tr.lap("grid: pilot group rejected");
					continue;
				}
			}
			if (all) {
				/* the previous group's hits come back while this group computes; then this group's counts, the one synchronisation
				 * per group, and its compaction at their prefix */
				if (flush_hits()) return -1;
				HitGroup hg;
				std::vector<int32_t> sn((size_t)2 * A.n_qp);
				SSW_CUDA_OK(cudaMemcpyAsync(sn.data(), gb + o_scnt, 4 * sn.size(), cudaMemcpyDeviceToHost, e->stream));
				SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
				hg.off.assign(sn.size() + 1, 0); hg.q.resize(sn.size()); hg.r_lo = r_lo;
				for (size_t s = 0; s < sn.size(); ++s) { hg.q[s] = s & 1 ? qps[s / 2].qb : qps[s / 2].qa; hg.off[s + 1] = hg.off[s] + sn[s]; }
				hg.n = hg.off.back();
				grid_hits += hg.n;
				if (grid_hits > gs->max_hits) return -2;
				if (hg.n > 0) {
					const size_t o_ref = (sizeof(ssw_batch_result) * (size_t)hg.n + 255) / 256 * 256;
					if (e->d_hits.ensure(o_ref + 4 * (size_t)hg.n)) return -1;
					uint8_t* hb = e->d_hits.as<uint8_t>();
					SSW_CUDA_OK(cudaMemcpyAsync(gb + o_soff, hg.off.data(), 8 * hg.off.size(), cudaMemcpyHostToDevice, e->stream));
					e->laps.start(e->stream);
					ssw_launch(ssw_grid_compact_kernel, dim3((unsigned)(2 * A.n_qp)), dim3(SSW_SELECT_THREADS), 0, e->stream, A,
					           d_qp, (const SswGridQ*)reinterpret_cast<SswGridQ*>(gb + o_qt),
					           (const SswFillResult*)e->d_res.as<SswFillResult>(), gs->min_score, (const int64_t*)reinterpret_cast<int64_t*>(gb + o_soff),
					           reinterpret_cast<int32_t*>(hb + o_ref), reinterpret_cast<ssw_batch_result*>(hb));
					SSW_CUDA_OK(cudaGetLastError());
					e->laps.stop(e->stream, &e->timing.resolve_ms);
					e->timing.other_launches += 1;
					hg.ev = groups.back().ev;
					SSW_CUDA_OK(cudaEventRecord(hg.ev, e->stream));
				}
				pend = std::move(hg);
			}
			tr.lap("grid: launch group");
		}
		if (t + 1 < n_tiles) {
			if (take_redo(r_lo, n_rt)) return -1;
			if (redo_over) return 0;
			SSW_CUDA_OK(cudaMemsetAsync(gb + o_cnt, 0, 256, e->stream));
		}
	}
	/* every launch is queued; bring the records back group by group on the copy stream while later groups still compute */
	bool all_contiguous = !groups.empty();
	for (const GridGroup& gg : groups) if (!gg.contiguous) all_contiguous = false;
	if (all) {
		if (flush_hits()) return -1;                 /* the last group's hits */
		if (self)                                    /* rows came in canonical order */
			for (std::vector<SearchHit>& v : gs->rows) std::sort(v.begin(), v.end(), [](const SearchHit& a, const SearchHit& b) { return a.r < b.r; });
	} else if (gs) {
		/* the hit table in one copy (rows of a rejected pilot group were overwritten by their second run) */
		std::vector<uint8_t> h(o_nh + 4 * (size_t)n_q);
		if (e->staged.copy(h.data(), e->d_hits.p, h.size(), e->stream)) return -1;
		gs->hits.resize((size_t)n_q * gs->k); gs->hit_ref.resize((size_t)n_q * gs->k); gs->n_hits.resize((size_t)n_q);
		memcpy(gs->hits.data(), h.data(), o_href);
		memcpy(gs->hit_ref.data(), h.data() + o_href, o_nh - o_href);
		memcpy(gs->n_hits.data(), h.data() + o_nh, 4 * (size_t)n_q);
		for (int32_t q : order)
			for (int32_t i = 0; i < gs->n_hits[q]; ++i) { int32_t& r = gs->hit_ref[(size_t)q * gs->k + i]; r = rsel[r]; }
	}
	if (gs) {
		gs->q_on.assign((size_t)n_q, 0); gs->r_on.assign((size_t)n_r_all, 0);
		for (int32_t q : order) gs->q_on[q] = 1;
		for (int32_t r : rsel) gs->r_on[r] = 1;
	} else if (all_contiguous && groups.size() > 1) {
		if (!e->side[0]) SSW_CUDA_OK(cudaStreamCreateWithFlags(&e->side[0], cudaStreamNonBlocking));
		for (const GridGroup& gg : groups) {
			SSW_CUDA_OK(cudaStreamWaitEvent(e->side[0], gg.ev, 0));
			const size_t first = (size_t)gg.q_lo * (size_t)n_r, cnt = (size_t)gg.q_n * (size_t)n_r;
			if (e->staged.copy(results + first, e->d_out.as<ssw_batch_result>() + first, sizeof(ssw_batch_result) * cnt, e->side[0])) return -1;
		}
	} else if (e->staged.copy(results, e->d_out.p, sizeof(ssw_batch_result) * (size_t)n_pairs, e->stream)) return -1;
	if (take_redo(tile_lo[n_tiles - 1], n_r - tile_lo[n_tiles - 1])) return -1;
	if (redo_over) return 0;
	std::sort(redo->begin(), redo->end());
	tr.lap("grid: results d2h");
	return 1;
}

}  // namespace

/* The general path: any pair list, any flag. */
static int align_general(ssw_engine* e, const ssw_batch_params& P, const Sem& S,
                         int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                         ssw_batch_result* results, uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used)
{
	/* gapO <= gapE: the reference's result depends on its SIMD layout (lazy-F exit); use the lane-literal kernel */
	const bool literal = P.gap_open <= P.gap_extend;
	Trace phase;

	std::vector<Aln> alns((size_t)n_pairs);
	for (int64_t p = 0; p < n_pairs; ++p) {
		Aln& a = alns[p];
		a.q = pair_query ? pair_query[p] : (int32_t)(p / e->n_r);
		a.r = pair_ref ? pair_ref[p] : (int32_t)(p % e->n_r);
		if (a.q < 0 || a.q >= e->n_q || a.r < 0 || a.r >= e->n_r) { fprintf(stderr, "[libssw-b200] pair %lld out of range\n", (long long)p); return -1; }
		a.read_len = (int32_t)(e->q_off[a.q + 1] - e->q_off[a.q]);
		a.ref_len = e->r_len[a.r];
		a.mask_len = P.mask_len < 0 ? a.read_len / 2 : P.mask_len;
		a.word = 0; a.rev_score = 0; a.rev_pos = 0; a.rev_row = 0;
		memset(&a.fwd, 0, sizeof(a.fwd));
		if (a.read_len < 1) { fprintf(stderr, "[libssw-b200] pair %lld: empty query\n", (long long)p); return -1; }
	}
	if (!S.has_byte && !S.has_word) {
		fprintf(stderr, "Please call the function ssw_init before ssw_align.\n");
		for (int64_t p = 0; p < n_pairs; ++p) { memset(&results[p], 0, sizeof(results[p])); results[p].status = 1; results[p].cigar_off = -1; }
		return 0;
	}

	/* ---- P1 (ssw.c:881-899).  The reference tries byte semantics first and re-runs with word semantics on
	 * overflow.  The outcome only depends on the final score, so where a byte overflow is certain to be likely
	 * (the query could score twice the byte limit) word semantics are tried first; either way a result that the
	 * other semantics must replace is re-resolved on the same matrix or, if the pad rows differ, re-filled. ---- */
	std::vector<int64_t> byte_first, word_first, refill_word, refill_byte;
	for (int64_t p = 0; p < n_pairs; ++p) {
		const bool predict = S.has_byte && S.has_word && (int64_t)alns[p].read_len * std::max(S.max_of(alns[p].q), 0) >= 2 * (int64_t)S.limit_byte_of(alns[p].q);
		if (!S.has_byte || predict) word_first.push_back(p); else byte_first.push_back(p);
	}
	int rc = 0;
	if (literal) {
		std::vector<int64_t> all((size_t)n_pairs), redo;
		for (int64_t p = 0; p < n_pairs; ++p) all[p] = p;
		rc = emul_pass(e, P, alns, all, S.has_byte ? 0 : 1, 0, S);
		if (rc) return rc;
		if (S.has_byte && S.has_word) {
			for (int64_t p = 0; p < n_pairs; ++p) if (alns[p].fwd.overflow == 1) redo.push_back(p);
			rc = emul_pass(e, P, alns, redo, 1, 0, S);
			if (rc) return rc;
			e->timing.byte_overflows = (int64_t)redo.size();
		}
	} else {
		rc = forward_pass(e, P, alns, byte_first, 0, S, false, &refill_word);
		if (rc) return rc;
		rc = forward_pass(e, P, alns, word_first, 1, S, S.has_byte, &refill_byte);
		if (rc) return rc;
		rc = forward_pass(e, P, alns, refill_word, 1, S, false, nullptr);
		if (rc) return rc;
		rc = forward_pass(e, P, alns, refill_byte, 0, S, false, nullptr);
		if (rc) return rc;
		/* word scores within reach of the 16-bit saturation of the reference (ssw.c:483): literal kernel */
		std::vector<int64_t> sat;
		for (int64_t p = 0; p < n_pairs; ++p) if (alns[p].fwd.overflow == 2) sat.push_back(p);
		rc = emul_pass(e, P, alns, sat, 1, 0, S);
		if (rc) return rc;
	}
	for (int64_t p = 0; p < n_pairs; ++p)
		if (alns[p].fwd.overflow == 3) { fprintf(stderr, "[libssw-b200] internal: unarmed best cell outside the grid path\n"); return -1; }
	std::vector<uint8_t> null_result((size_t)n_pairs, 0);
	for (int64_t p = 0; p < n_pairs; ++p) {
		const Aln& a = alns[p];
		if (a.word == 0 && a.fwd.overflow == 1) { null_result[p] = 1; continue; }    /* byte overflow without a word profile (ssw.c:887-890) */
		if (!literal && a.word == 1 && S.has_byte && a.fwd.score >= S.limit_byte_of(a.q)) e->timing.byte_overflows += 1;
	}

	phase.lap("general: forward passes");
	/* ---- gating (ssw.c:900-916) and P2 ---- */
	std::vector<int64_t> need_begin;
	for (int64_t p = 0; p < n_pairs; ++p) {
		const Aln& a = alns[p];
		if (null_result[p] || a.fwd.score <= 0) continue;
		if (P.flag == 0 || (P.flag == 2 && a.fwd.score < P.filters)) continue;
		need_begin.push_back(p);
	}
	{
		/* begin search: literal kernel where the forward result came from it (saturating scores) or the regime demands it */
		std::vector<int64_t> rev_fast, rev_lit;
		for (int64_t p : need_begin) (literal || alns[p].fwd.score >= S.limit_word_of(alns[p].q) ? rev_lit : rev_fast).push_back(p);
		rc = reverse_pass(e, P, alns, rev_fast);
		if (rc) return rc;
		rc = emul_pass(e, P, alns, rev_lit, 1, 1, S);
		if (rc) return rc;
	}

	phase.lap("general: reverse passes");
	/* ---- assemble the fixed-size records ---- */
	std::vector<uint8_t> has_begin((size_t)n_pairs, 0);
	for (int64_t p : need_begin) has_begin[p] = 1;
	std::vector<SswTbTask> tb;
	std::vector<int64_t> tb_pair;
	for (int64_t p = 0; p < n_pairs; ++p) {
		const Aln& a = alns[p];
		ssw_batch_result& r = results[p];
		memset(&r, 0, sizeof(r));
		r.ref_begin1 = -1; r.read_begin1 = -1; r.cigar_off = -1;
		if (null_result[p]) {
			fprintf(stderr, "Please set 2 to the score_size parameter of the function ssw_init, otherwise the alignment results will be incorrect.\n");
			r.status = 1;
			continue;
		}
		if (a.fwd.score <= 0) continue;                                   /* ssw.c:900-903 */
		r.score1 = (uint16_t)a.fwd.score; r.ref_end1 = a.fwd.ref; r.read_end1 = a.fwd.read;
		if (a.mask_len >= 15) { r.score2 = (uint16_t)a.fwd.score2; r.ref_end2 = a.fwd.ref2; }
		else { r.score2 = 0; r.ref_end2 = -1; }
		if (!has_begin[p]) continue;
		r.ref_begin1 = a.fwd.ref - a.rev_pos;                              /* scan index 0 == column ref_end1 */
		r.read_begin1 = a.fwd.read - a.rev_row;                            /* ssw.c:929-930 */
		if (a.fwd.score > a.rev_score) {
			fprintf(stderr, "Warning: The alignment path of one pair of sequences may miss a small part. [ssw.c ssw_align]\n");
			r.flag = 2;
		}
		if ((7 & P.flag) == 0 || ((2 & P.flag) != 0 && r.score1 < P.filters) ||
		    ((4 & P.flag) != 0 && (r.ref_end1 - r.ref_begin1 > P.filterd || r.read_end1 - r.read_begin1 > P.filterd)))
			continue;                                                      /* ssw.c:938 */
		SswTbTask t;
		memset(&t, 0, sizeof(t));
		t.ref_off = e->r_off[a.r] + r.ref_begin1;
		t.read_off = (e->q_off[a.q] + r.read_begin1) * (e->pssm_n ? e->pssm_n : 1);
		t.ref_len = r.ref_end1 - r.ref_begin1 + 1;
		t.read_len = r.read_end1 - r.read_begin1 + 1;
		t.score = r.score1;
		tb.push_back(t);
		tb_pair.push_back(p);
	}

	phase.lap("general: records");
	/* ---- P3 ---- */
	if (!tb.empty()) {
		rc = ssw_traceback_run(e->stream, e->side, tb, e->d_q.as<int8_t>(), e->d_r.as<int8_t>(), e->mat_arg(), P.n,
		                       P.gap_open, P.gap_extend, &e->d_tb, &e->timing.traceback_ms, &e->timing.other_launches, e->opt.tb_maxbw, e->opt.carve != 0, e->opt.tb_spec,
		                       [&](size_t i, const uint32_t* words, int32_t len, int failed) -> int {
			ssw_batch_result& r = results[tb_pair[i]];
			if (failed) { r.flag = 1; return 0; }                           /* ssw.c:968 */
			if (!cigar_pool || *pool_used + len > pool_cap) { fprintf(stderr, "[libssw-b200] CIGAR pool too small\n"); return -1; }
			if (*pool_used + len > 0x7fffffff) { fprintf(stderr, "[libssw-b200] more than 2^31 CIGAR words in one batch: split the batch\n"); return -1; }
			r.cigar_off = (int32_t)*pool_used; r.cigar_len = len;
			memcpy(cigar_pool + *pool_used, words, sizeof(uint32_t) * (size_t)len);
			*pool_used += len;
			return 0;
		});
		if (rc) return rc;
	}
	phase.lap("general: traceback");
	return 0;
}

/* The scoring source of a call: a matrix (params->mat) with sequences resident, none (NULL, params->n = the profiles' n) with query
 * profiles resident.  Prints why not and returns false. */
static bool scoring_args_ok(const ssw_engine* e, const ssw_batch_params* params, const char* what)
{
	if (!e || !params) { fprintf(stderr, "[libssw-b200] %s: no engine or no parameters\n", what); return false; }
	if (e->pssm_n && params->mat) { fprintf(stderr, "[libssw-b200] %s: query profiles are resident: params->mat must be NULL\n", what); return false; }
	if (e->pssm_n && params->n != e->pssm_n) {
		fprintf(stderr, "[libssw-b200] %s: the resident query profiles have %d letters, params->n is %d\n", what, e->pssm_n, params->n);
		return false;
	}
	if (!e->pssm_n && !params->mat) { fprintf(stderr, "[libssw-b200] %s: no scoring matrix (params->mat is NULL) and no query profiles resident\n", what); return false; }
	return true;
}

/* scoring matrix on the device and the semantics it implies: bias = |min(mat)| for byte semantics (ssw.c:834-838).  Query profiles:
 * each query has its own bias and limits (taken at upload); bias and max_mat are their largest values, for the call-wide bounds. */
static int prepare_scoring(ssw_engine* e, const ssw_batch_params& P, Sem* out)
{
	Sem& S = *out;
	S.has_byte = P.score_size == 0 || P.score_size == 2;
	S.has_word = P.score_size == 1 || P.score_size == 2;
	if (e->pssm_n) {
		S.bias = 0; S.max_mat = -128;
		for (int32_t q = 0; q < e->n_q; ++q) { S.bias = std::max(S.bias, e->q_bias[q]); S.max_mat = std::max(S.max_mat, e->q_max[q]); }
		S.limit_byte = 255 - S.bias;
		S.limit_word = 32767 - std::max(S.max_mat, 0) - 256;
		S.q_bias = e->q_bias.data(); S.q_max = e->q_max.data();
		return e->upload_refs(P.n);
	}
	S.bias = 0; S.max_mat = -128;
	for (int i = 0; i < P.n * P.n; ++i) { if (P.mat[i] < S.bias) S.bias = P.mat[i]; if (P.mat[i] > S.max_mat) S.max_mat = P.mat[i]; }
	S.bias = S.bias < 0 ? -S.bias : S.bias;
	S.limit_byte = 255 - S.bias;
	S.limit_word = 32767 - std::max(S.max_mat, 0) - 256;
	if (e->d_mat.ensure((size_t)P.n * P.n + 16)) return -1;
	SSW_CUDA_OK(cudaMemcpyAsync(e->d_mat.p, P.mat, (size_t)P.n * P.n, cudaMemcpyHostToDevice, e->stream));
	return e->upload_refs(P.n);
}

static int engine_align_impl(ssw_engine* e, const ssw_batch_params* params,
                             int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                             ssw_batch_result* results,
                             uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used)
{
	if (!scoring_args_ok(e, params, "ssw_engine_align") || n_pairs < 0 || (n_pairs && !results)) return -1;
	if (n_pairs > 0 && (e->n_q <= 0 || e->n_r <= 0)) { fprintf(stderr, "[libssw-b200] ssw_engine_align: no resident sequences\n"); return -1; }
	const ssw_batch_params& P = *params;
	if (P.n < 1 || P.n > 64) { fprintf(stderr, "[libssw-b200] alphabet size %d not supported (1..64)\n", P.n); return -1; }
	if ((pair_query == nullptr) != (pair_ref == nullptr)) return -1;
	int64_t pool_used_local = 0;
	if (!pool_used) pool_used = &pool_used_local;
	*pool_used = 0;
	SSW_CUDA_OK(cudaSetDevice(e->device));
	memset(&e->timing, 0, sizeof(e->timing));
	e->laps.laps.clear(); e->laps.used = 0;            /* a call that failed half-way leaves its laps behind */
	if (n_pairs == 0) return 0;
	e->t_total.start(e->stream);

	Sem S;
	if (prepare_scoring(e, P, &S)) return -1;

	int rc = 0;
	/* Long reads with CIGARs: the banded traceback is a set of long serial chains that leaves most of the device idle, and
	 * the strip fills before it are throughput-bound.  The batch is cut into slices that run on helper engines (own stream
	 * and scratch, views of this engine's sequences) from as many host threads, so that one slice's traceback runs under
	 * the fills of the others.  A fill CTA takes all registers of an SM, so the
	 * overlap is by SMs, not by issue slots: traceback CTAs move in where fill CTAs retire. */
	{
		int slices = 1;
		bool auto_slices = false;
		if (!e->is_kid && e->opt.slices != 1 && (P.flag & 7) != 0 && P.gap_open > P.gap_extend) {
			int64_t qsum = 0;
			const int64_t probe = std::min<int64_t>(n_pairs, 64);
			for (int64_t p = 0; p < probe; ++p) { const int32_t q = pair_query ? pair_query[p] : (int32_t)(p / e->n_r); if (q >= 0 && q < e->n_q) qsum += e->q_off[q + 1] - e->q_off[q]; }
			if (e->opt.slices > 1) slices = e->opt.slices;
			else if (n_pairs >= 96 && qsum / probe >= 2000) { slices = n_pairs >= 512 ? 6 : 3; auto_slices = true; }
			slices = (int)std::min<int64_t>(slices, n_pairs);
		}
		if (slices > 1) {
			SSW_CUDA_OK(cudaStreamSynchronize(e->stream));          /* sequences, matrix and padded references are in place */
			std::vector<int32_t> pq_all, pr_all;
			if (!pair_query) {
				pq_all.resize((size_t)n_pairs); pr_all.resize((size_t)n_pairs);
				for (int64_t p = 0; p < n_pairs; ++p) { pq_all[p] = (int32_t)(p / e->n_r); pr_all[p] = (int32_t)(p % e->n_r); }
				pair_query = pq_all.data(); pair_ref = pr_all.data();
			}
			/* pool: worst-case sized, most of it never touched -- uninitialised storage, not a zero-filled vector */
			struct Slice { int64_t lo, hi, used, cap; int rc; std::unique_ptr<uint32_t[]> pool; };
			std::vector<Slice> sl((size_t)slices);
			/* slice boundaries: equal parts, or every slice `slice_taper` % of the one before it */
			std::vector<int64_t> cut((size_t)slices + 1, 0);
			{
				std::vector<double> w((size_t)slices, 1.0);
				/* automatic: six slices, each 80 % of the one before it (the last slice's traceback is not hidden under any fill,
				 * so it is the smallest) */
				const int taper = e->opt.slice_taper > 0 ? e->opt.slice_taper : (auto_slices && slices == 6 ? 80 : 0);
				if (taper > 0) for (int k = 1; k < slices; ++k) w[k] = w[k - 1] * (double)taper / 100.0;
				double tot = 0, acc = 0;
				for (double x : w) tot += x;
				for (int k = 0; k < slices; ++k) {
					acc += w[k];
					cut[k + 1] = k + 1 == slices ? n_pairs : std::max<int64_t>(cut[k] + 1, std::min<int64_t>(n_pairs - (slices - 1 - k), (int64_t)((double)n_pairs * acc / tot)));
				}
			}
			for (int k = 0; k < slices; ++k) {
				Slice& s = sl[k];
				s.lo = cut[k]; s.hi = cut[k + 1]; s.used = 0; s.rc = 0;
				int64_t cap = 0;
				for (int64_t p = s.lo; p < s.hi; ++p) {
					const int32_t q = pair_query[p], r = pair_ref[p];
					if (q < 0 || q >= e->n_q || r < 0 || r >= e->n_r) { fprintf(stderr, "[libssw-b200] pair %lld out of range\n", (long long)p); return -1; }
					const int64_t ql = e->q_off[q + 1] - e->q_off[q];
					cap += ql + std::min<int64_t>(e->r_len[r], ql + ql * 127 / std::max<int>(P.gap_extend, 1)) + 4;
				}
				s.cap = cap + 8;
				s.pool.reset(new uint32_t[(size_t)s.cap]);
				ssw_engine*& kid = e->kids[k];
				if (!kid) { kid = ssw_engine_create(e->device); if (!kid) return -1; kid->is_kid = true; }
				kid->n_q = e->n_q; kid->n_r = e->n_r; kid->q_off = e->q_off; kid->r_off = e->r_off; kid->r_len = e->r_len;
				kid->padded_n = e->padded_n; kid->from_text = true;     /* no host copy: the padded references are the parent's */
				kid->d_q.borrow(e->d_q); kid->d_r.borrow(e->d_r);
				kid->pssm_n = e->pssm_n; kid->q_bias = e->q_bias; kid->q_max = e->q_max;
				kid->opt = e->opt;
			}
			auto work = [&](int k) {
				Slice& s = sl[k];
				s.rc = ssw_engine_align(e->kids[k], params, s.hi - s.lo, pair_query + s.lo, pair_ref + s.lo, results + s.lo,
				                        s.pool.get(), s.cap, &s.used);
			};
#ifdef SSW_CPU_EMU
			for (int k = 0; k < slices; ++k) work(k);               /* the emulator's fibers are not thread-safe */
#else
			{
				std::vector<std::thread> th;
				for (int k = 1; k < slices; ++k) th.emplace_back(work, k);
				work(0);
				for (std::thread& t : th) t.join();
			}
			SSW_CUDA_OK(cudaSetDevice(e->device));
#endif
			for (int k = 0; k < slices; ++k) {
				Slice& s = sl[k];
				if (s.rc) return s.rc;
				if (s.used > 0) {
					if (!cigar_pool || *pool_used + s.used > pool_cap) { fprintf(stderr, "[libssw-b200] CIGAR pool too small\n"); return -1; }
					if (*pool_used + s.used > 0x7fffffff) { fprintf(stderr, "[libssw-b200] more than 2^31 CIGAR words in one batch: split the batch\n"); return -1; }
					memcpy(cigar_pool + *pool_used, s.pool.get(), sizeof(uint32_t) * (size_t)s.used);
					for (int64_t p = s.lo; p < s.hi; ++p) if (results[p].cigar_off >= 0) results[p].cigar_off += (int32_t)*pool_used;
					*pool_used += s.used;
				}
				const ssw_engine_timing& t = e->kids[k]->timing;
				e->timing.fill_forward_ms += t.fill_forward_ms; e->timing.resolve_ms += t.resolve_ms;
				e->timing.fill_reverse_ms += t.fill_reverse_ms; e->timing.traceback_ms += t.traceback_ms;
				e->timing.fill_forward_launches += t.fill_forward_launches; e->timing.other_launches += t.other_launches;
				e->timing.cells_forward += t.cells_forward; e->timing.byte_overflows += t.byte_overflows;
				e->timing.block_refills += t.block_refills; e->timing.block_exact += t.block_exact;
			}
			e->timing.total_ms = e->t_total.stop(e->stream);
			e->laps.collect();
			return 0;
		}
	}
	std::vector<int64_t> redo;
	const int grid = pair_query ? 0 : grid_scores(e, P, S, n_pairs, results, &redo);
	if (grid < 0) return grid;
	if (grid == 1) {
		/* the device-planned grid handled everything except byte overflows: those pairs go through the general path */
		if (!redo.empty()) {
			std::vector<int32_t> pq(redo.size()), pr(redo.size());
			for (size_t i = 0; i < redo.size(); ++i) { pq[i] = (int32_t)(redo[i] / e->n_r); pr[i] = (int32_t)(redo[i] % e->n_r); }
			std::vector<ssw_batch_result> sub(redo.size());
			const ssw_engine_timing keep = e->timing;
			rc = align_general(e, P, S, (int64_t)redo.size(), pq.data(), pr.data(), sub.data(), cigar_pool, pool_cap, pool_used);
			if (rc) return rc;
			for (size_t i = 0; i < redo.size(); ++i) results[redo[i]] = sub[i];
			e->timing.byte_overflows = keep.byte_overflows + (int64_t)redo.size();
		}
	} else {
		rc = align_general(e, P, S, n_pairs, pair_query, pair_ref, results, cigar_pool, pool_cap, pool_used);
		if (rc) return rc;
	}
	e->timing.total_ms = e->t_total.stop(e->stream);
	e->laps.collect();
	return 0;
}

extern "C" int ssw_engine_align(ssw_engine* e, const ssw_batch_params* params,
                                int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                                ssw_batch_result* results,
                                uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used)
{
	/* nothing may unwind through the C ABI (std::bad_alloc from the planners' vectors, std::length_error, ...) */
	try { SswBusyGuard busy(e ? e->device : 0); return engine_align_impl(e, params, n_pairs, pair_query, pair_ref, results, cigar_pool, pool_cap, pool_used); }
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_align: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

/* ------------------------------------------------------------------------------------------- */
/* top-k search over the full grid                                                               */
/* ------------------------------------------------------------------------------------------- */

/* the rank order of ssw_engine_search: status-1 pairs first (their score is at least the byte limit), then score1 descending,
 * then reference ascending -- a total order, so the k best do not depend on how the grid was cut */
static bool hit_before(const SearchHit& a, const SearchHit& b)
{
	if (a.rec.status != b.rec.status) return a.rec.status > b.rec.status;
	if (a.rec.score1 != b.rec.score1) return a.rec.score1 > b.rec.score1;
	return a.r < b.r;
}
static bool is_hit(const ssw_batch_result& o, int32_t min_score) { return o.status == 1 || o.score1 >= min_score; }

/* the first k of v in rank order, sorted */
static void keep_best(std::vector<SearchHit>& v, int32_t k)
{
	if ((int64_t)v.size() > k) { std::partial_sort(v.begin(), v.begin() + k, v.end(), hit_before); v.resize((size_t)k); }
	else std::sort(v.begin(), v.end(), hit_before);
}

/* general path of a search: pairs per block of whole queries */
#define SSW_SEARCH_BLOCK_PAIRS ((int64_t)1 << 22)

/* worst-case CIGAR words of one pair (the bound of the device groups): a path has at most query span + reference span + 2
 * words, and a positive-scoring path cannot delete more than query length * max score / gap_extend bases */
static int64_t cigar_words_bound(int64_t ql, int64_t rl, int gap_extend)
{
	int64_t span = rl;
	if (gap_extend > 0) { const int64_t b = ql + ql * 127 / gap_extend; if (b < span) span = b; }
	return ql + span + 4;
}

static bool ref_before(const SearchHit& a, const SearchHit& b) { return a.r < b.r; }

/* The triangle of a self-search: the pairs (canon[i], canon[j]) with lo <= i < hi and j > i, where canon lists the sequences in
 * canonical order (length, then index, ascending) and rank is its inverse. */
struct SelfTri { std::vector<int32_t> rank, canon; int32_t lo, hi; };

/* The rows of a search over the full grid, shared by the top-k search (keep = k: a row holds its k best hits in rank order)
 * and the threshold search (keep = 0: every hit, in ascending reference index).  The grid path takes what it can; the pairs
 * it re-does and the pairs it leaves over run through the general path and are merged into their rows (disjoint sets, so a
 * merge of sorted lists); with a flag, the caller's params run once more on the kept pairs only, their CIGARs going to
 * cigar_pool or, with own_pool, to a pool sized for them.  keep = 0 and more than max_hits hits: -2. */
static int search_rows(ssw_engine* e, const ssw_batch_params& P, int32_t keep, int32_t min_score, int64_t max_hits,
                       std::vector<std::vector<SearchHit>>& best, uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used,
                       std::vector<uint32_t>* own_pool, const SelfTri* tri = nullptr)
{
	int64_t no_pool = 0;
	SSW_CUDA_OK(cudaSetDevice(e->device));
	memset(&e->timing, 0, sizeof(e->timing));
	e->laps.laps.clear(); e->laps.used = 0;
	e->t_total.start(e->stream);
	Sem S;
	if (prepare_scoring(e, P, &S)) return -1;
	const int32_t n_q = e->n_q, n_r = e->n_r, thr = std::max(min_score, 1);
	/* the ranking runs on flag-0 records: score1, the ends and the second best do not depend on the flag */
	ssw_batch_params P0 = P;
	P0.flag = 0;
	best.assign((size_t)n_q, std::vector<SearchHit>());
	int64_t n_kept = 0;                              /* keep = 0: the hits so far */
	/* a row after a merge: its k best in rank order, or -- a sorted row followed by sorted additions -- one merge by reference */
	auto settle = [&](int32_t q) {
		std::vector<SearchHit>& v = best[q];
		if (keep > 0) keep_best(v, keep);
		else {
			const auto mid = std::is_sorted_until(v.begin(), v.end(), ref_before);
			if (tri) std::sort(mid, v.end(), ref_before);      /* a self-search adds a row's pairs in canonical order */
			std::inplace_merge(v.begin(), mid, v.end(), ref_before);
		}
	};
	GridSearch gs;
	gs.k = keep; gs.min_score = thr; gs.max_hits = max_hits;
	if (tri) { gs.rank = tri->rank.data(); gs.rank_lo = tri->lo; gs.rank_hi = tri->hi; }
	std::vector<int64_t> redo;
	int rc = grid_scores(e, P0, S, (int64_t)n_q * n_r, nullptr, &redo, &gs);
	if (rc < 0) return rc;
	if (rc == 1) {
		if (keep > 0) {
			for (int32_t q = 0; q < n_q; ++q)
				for (int32_t i = 0; i < gs.n_hits[q]; ++i) best[q].push_back(SearchHit{gs.hit_ref[(size_t)q * keep + i], gs.hits[(size_t)q * keep + i]});
		} else {
			best.swap(gs.rows);
			for (const std::vector<SearchHit>& v : best) n_kept += (int64_t)v.size();
		}
		/* pairs the grid left to the general path, merged per query: the k best of all pairs are the k best of the grid's k best
		 * and the re-done pairs, whatever the reason of the re-do */
		if (!redo.empty()) {
			std::vector<int32_t> pq(redo.size()), pr(redo.size());
			for (size_t i = 0; i < redo.size(); ++i) { pq[i] = (int32_t)(redo[i] / n_r); pr[i] = (int32_t)(redo[i] % n_r); }
			std::vector<ssw_batch_result> sub(redo.size());
			const ssw_engine_timing keep_t = e->timing;
			rc = align_general(e, P0, S, (int64_t)redo.size(), pq.data(), pr.data(), sub.data(), nullptr, 0, &no_pool);
			if (rc) return rc;
			e->timing.byte_overflows = keep_t.byte_overflows + (int64_t)redo.size();
			for (size_t i = 0; i < redo.size(); ++i) if (is_hit(sub[i], thr)) { best[pq[i]].push_back(SearchHit{pr[i], sub[i]}); ++n_kept; }
			if (keep == 0 && n_kept > max_hits) return -2;
			for (int32_t q = 0; q < n_q; ++q) settle(q);
		}
	} else {
		gs.q_on.assign((size_t)n_q, 0); gs.r_on.assign((size_t)n_r, 0);       /* no grid: every pair is left over */
	}
	/* The pairs the grid did not take -- a query off the grid against every reference, a query on it against the references off
	 * it -- go through the general path in blocks of whole queries and are merged per query in the same way; the selection of
	 * these is on the host.  Memory is bounded by a block.  A self-search takes its queries in canonical order, each against the
	 * references ranked after it only. */
	std::vector<int32_t> r_off_grid;
	for (int32_t r = 0; r < n_r; ++r) if (!gs.r_on[r]) r_off_grid.push_back(r);
	std::vector<int32_t> pq, pr;
	std::vector<ssw_batch_result> rec;
	const int32_t i_end = tri ? tri->hi : n_q;
	auto q_at = [&](int32_t i) { return tri ? tri->canon[i] : i; };
	for (int32_t q0 = tri ? tri->lo : 0; q0 < i_end;) {
		int32_t q1 = q0;
		pq.clear(); pr.clear();
		for (; q1 < i_end; ++q1) {
			const int32_t q = q_at(q1);
			const int64_t row = gs.q_on[q] ? (int64_t)r_off_grid.size() : tri ? n_r - 1 - q1 : n_r;
			if (q1 > q0 && (int64_t)pq.size() + row > SSW_SEARCH_BLOCK_PAIRS) break;
			if (gs.q_on[q]) { for (int32_t r : r_off_grid) if (!tri || tri->rank[r] > q1) { pq.push_back(q); pr.push_back(r); } }
			else if (tri) {
				/* an empty sequence comes first in canonical order and is the query of all its pairs: it aligns nowhere (score 0),
				 * so none of them is a hit, and none is computed */
				if (e->q_off[q + 1] > e->q_off[q]) for (int32_t j = q1 + 1; j < n_r; ++j) { pq.push_back(q); pr.push_back(tri->canon[j]); }
			}
			else for (int32_t r = 0; r < n_r; ++r) { pq.push_back(q); pr.push_back(r); }
		}
		const int64_t m = (int64_t)pq.size();
		if (m > 0) {
			rec.resize((size_t)m);
			const int64_t over = e->timing.byte_overflows;
			e->timing.byte_overflows = 0;
			rc = align_general(e, P0, S, m, pq.data(), pr.data(), rec.data(), nullptr, 0, &no_pool);
			if (rc) return rc;
			e->timing.byte_overflows += over;
			e->timing.leftover_pairs += m;
			for (int64_t i = 0; i < m; ++i) if (is_hit(rec[i], thr)) { best[pq[i]].push_back(SearchHit{pr[i], rec[i]}); ++n_kept; }
			if (keep == 0 && n_kept > max_hits) return -2;
			for (int32_t i = q0; i < q1; ++i) settle(q_at(i));
		}
		q0 = q1;
	}
	/* the caller's flag: begins and CIGARs of the kept hits only */
	if (P.flag != 0) {
		std::vector<int32_t> hq, hr;
		for (int32_t q = 0; q < n_q; ++q) for (const SearchHit& h : best[q]) { hq.push_back(q); hr.push_back(h.r); }
		if (!hq.empty()) {
			std::unique_ptr<uint32_t[]> own;
			if (own_pool && (P.flag & 7)) {
				pool_cap = 8;
				for (size_t i = 0; i < hq.size(); ++i)
					pool_cap += cigar_words_bound(e->q_off[hq[i] + 1] - e->q_off[hq[i]], e->r_len[hr[i]], P.gap_extend);
				own.reset(new uint32_t[(size_t)pool_cap]);      /* worst-case sized and mostly untouched: uninitialised storage */
				cigar_pool = own.get();
			}
			std::vector<ssw_batch_result> rec(hq.size());
			const int64_t over = e->timing.byte_overflows;
			rc = align_general(e, P, S, (int64_t)hq.size(), hq.data(), hr.data(), rec.data(), cigar_pool, pool_cap, pool_used);
			if (rc) return rc;
			e->timing.byte_overflows = over;
			size_t j = 0;
			for (int32_t q = 0; q < n_q; ++q) for (SearchHit& h : best[q]) h.rec = rec[j++];
			if (own) own_pool->assign(own.get(), own.get() + *pool_used);
		}
	}
	e->timing.total_ms = e->t_total.stop(e->stream);
	e->laps.collect();
	return 0;
}

static int engine_search_impl(ssw_engine* e, const ssw_batch_params* params, int32_t k, int32_t min_score,
                              int32_t* hit_ref, ssw_batch_result* hits, int32_t* n_hits,
                              uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used)
{
	if (!scoring_args_ok(e, params, "ssw_engine_search")) return -1;
	if (k < 1 || k > SSW_SEARCH_MAX_K) { fprintf(stderr, "[libssw-b200] ssw_engine_search: k = %d outside 1 .. %d\n", k, SSW_SEARCH_MAX_K); return -1; }
	if (!hit_ref || !hits || !n_hits) { fprintf(stderr, "[libssw-b200] ssw_engine_search: NULL output array\n"); return -1; }
	if (e->n_q <= 0 || e->n_r <= 0) { fprintf(stderr, "[libssw-b200] ssw_engine_search: no resident sequences\n"); return -1; }
	const ssw_batch_params& P = *params;
	if (P.n < 1 || P.n > 64) { fprintf(stderr, "[libssw-b200] alphabet size %d not supported (1..64)\n", P.n); return -1; }
	int64_t pool_used_local = 0;
	if (!pool_used) pool_used = &pool_used_local;
	*pool_used = 0;
	std::vector<std::vector<SearchHit>> best;
	const int rc = search_rows(e, P, k, min_score, 0, best, cigar_pool, pool_cap, pool_used, nullptr);
	if (rc) return rc;
	ssw_batch_result none;
	memset(&none, 0, sizeof(none));
	none.ref_begin1 = -1; none.read_begin1 = -1; none.cigar_off = -1;
	for (int32_t q = 0; q < e->n_q; ++q) {
		const std::vector<SearchHit>& v = best[q];
		n_hits[q] = (int32_t)v.size();
		for (int32_t i = 0; i < k; ++i) {
			const bool used = i < (int32_t)v.size();
			hit_ref[(size_t)q * k + i] = used ? v[i].r : -1;
			hits[(size_t)q * k + i] = used ? v[i].rec : none;
		}
	}
	return 0;
}

extern "C" int ssw_engine_search(ssw_engine* e, const ssw_batch_params* params, int32_t k, int32_t min_score,
                                 int32_t* hit_ref, ssw_batch_result* hits, int32_t* n_hits,
                                 uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used)
{
	try { SswBusyGuard busy(e ? e->device : 0); return engine_search_impl(e, params, k, min_score, hit_ref, hits, n_hits, cigar_pool, pool_cap, pool_used); }
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_search: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

/* ------------------------------------------------------------------------------------------- */
/* threshold search over the full grid: every hit, as a CSR matrix in pair order                  */
/* ------------------------------------------------------------------------------------------- */

/* the rows of search_rows as the CSR matrix of a hit set (pool already in place); empties the rows */
static void fill_hit_set(std::vector<std::vector<SearchHit>>& best, ssw_hit_set* s)
{
	s->n_rows = (int32_t)best.size();
	s->row_off.assign(best.size() + 1, 0);
	for (size_t q = 0; q < best.size(); ++q) s->row_off[q + 1] = s->row_off[q] + (int64_t)best[q].size();
	const size_t n = (size_t)s->row_off.back();
	s->hit_ref.resize(n); s->hits.resize(n);
	size_t j = 0;
	for (std::vector<SearchHit>& v : best) {
		for (const SearchHit& h : v) { s->hit_ref[j] = h.r; s->hits[j] = h.rec; ++j; }
		std::vector<SearchHit>().swap(v);
	}
}

static int engine_search_all_impl(ssw_engine* e, const ssw_batch_params* params, int32_t min_score, int64_t max_hits, ssw_hit_set** out)
{
	if (!out) { fprintf(stderr, "[libssw-b200] ssw_engine_search_all: NULL output\n"); return -1; }
	*out = nullptr;
	if (!scoring_args_ok(e, params, "ssw_engine_search_all")) return -1;
	if (max_hits < 0) { fprintf(stderr, "[libssw-b200] ssw_engine_search_all: max_hits = %lld is negative\n", (long long)max_hits); return -1; }
	if (e->n_q <= 0 || e->n_r <= 0) { fprintf(stderr, "[libssw-b200] ssw_engine_search_all: no resident sequences\n"); return -1; }
	const ssw_batch_params& P = *params;
	if (P.n < 1 || P.n > 64) { fprintf(stderr, "[libssw-b200] alphabet size %d not supported (1..64)\n", P.n); return -1; }
	std::unique_ptr<ssw_hit_set> s(new ssw_hit_set());
	std::vector<std::vector<SearchHit>> best;
	int64_t used = 0;
	const int rc = search_rows(e, P, 0, min_score, max_hits, best, nullptr, 0, &used, &s->pool);
	if (rc == -2) fprintf(stderr, "[libssw-b200] ssw_engine_search_all: more than max_hits = %lld hits\n", (long long)max_hits);
	if (rc) return rc;
	fill_hit_set(best, s.get());
	*out = s.release();
	return 0;
}

extern "C" int ssw_engine_search_all(ssw_engine* e, const ssw_batch_params* params, int32_t min_score, int64_t max_hits, ssw_hit_set** out)
{
	if (out) *out = nullptr;
	try { SswBusyGuard busy(e ? e->device : 0); return engine_search_all_impl(e, params, min_score, max_hits, out); }
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_search_all: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

/* ------------------------------------------------------------------------------------------- */
/* self-search: every pair of one set above a threshold, each unordered pair computed once        */
/* ------------------------------------------------------------------------------------------- */

/* With a symmetric matrix and gap_open > gap_extend the score of a pair does not depend on which sequence is the query, so the
 * pair {i, j} is computed once, as query = the earlier of the two in canonical order (length, then index, ascending).  The
 * queries ranked in [rank_lo, rank_hi) only (the device groups' share); rows of the others stay empty. */
int ssw_engine_search_self_ranks(ssw_engine* e, const ssw_batch_params* params, int32_t min_score, int64_t max_hits,
                                 int32_t rank_lo, int32_t rank_hi, ssw_hit_set** out)
{
	if (out) *out = nullptr;
	try {
		SswBusyGuard busy(e ? e->device : 0);
		if (!out) { fprintf(stderr, "[libssw-b200] ssw_engine_search_self: NULL output\n"); return -1; }
		if (!e || !params) { fprintf(stderr, "[libssw-b200] ssw_engine_search_self: no engine or no parameters\n"); return -1; }
		if (!e->self) { fprintf(stderr, "[libssw-b200] ssw_engine_search_self: the resident sequences were not set by ssw_engine_set_sequences_self\n"); return -1; }
		const ssw_batch_params& P = *params;
		if (!P.mat) { fprintf(stderr, "[libssw-b200] ssw_engine_search_self: no scoring matrix (params->mat is NULL)\n"); return -1; }
		if (P.n < 1 || P.n > 64) { fprintf(stderr, "[libssw-b200] alphabet size %d not supported (1..64)\n", P.n); return -1; }
		if (max_hits < 0) { fprintf(stderr, "[libssw-b200] ssw_engine_search_self: max_hits = %lld is negative\n", (long long)max_hits); return -1; }
		if (P.gap_open <= P.gap_extend) {
			fprintf(stderr, "[libssw-b200] ssw_engine_search_self: gap_open %d <= gap_extend %d: scores are not symmetric\n", P.gap_open, P.gap_extend);
			return -1;
		}
		for (int a = 0; a < P.n; ++a)
			for (int b = 0; b < a; ++b)
				if (P.mat[a * P.n + b] != P.mat[b * P.n + a]) {
					fprintf(stderr, "[libssw-b200] ssw_engine_search_self: the matrix is not symmetric (%d, %d)\n", a, b);
					return -1;
				}
		const int32_t n = e->n_q;
		SelfTri tri;
		tri.canon.resize((size_t)n); tri.rank.resize((size_t)n);
		for (int32_t i = 0; i < n; ++i) tri.canon[i] = i;
		std::sort(tri.canon.begin(), tri.canon.end(), [&](int32_t x, int32_t y) { return e->r_len[x] != e->r_len[y] ? e->r_len[x] < e->r_len[y] : x < y; });
		for (int32_t t = 0; t < n; ++t) tri.rank[tri.canon[t]] = t;
		tri.lo = std::max(rank_lo, 0); tri.hi = std::min(rank_hi, n);
		std::unique_ptr<ssw_hit_set> s(new ssw_hit_set());
		std::vector<std::vector<SearchHit>> best((size_t)n);
		if (tri.lo < tri.hi) {
			int64_t used = 0;
			const int rc = search_rows(e, P, 0, min_score, max_hits, best, nullptr, 0, &used, &s->pool, &tri);
			if (rc == -2) fprintf(stderr, "[libssw-b200] ssw_engine_search_self: more than max_hits = %lld hits\n", (long long)max_hits);
			if (rc) return rc;
		}
		fill_hit_set(best, s.get());
		*out = s.release();
		return 0;
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_search_self: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_engine_search_self(ssw_engine* e, const ssw_batch_params* params, int32_t min_score, int64_t max_hits, ssw_hit_set** out)
{
	return ssw_engine_search_self_ranks(e, params, min_score, max_hits, 0, e ? e->n_q : 0, out);
}

extern "C" int ssw_hit_set_view(const ssw_hit_set* s, ssw_hit_view* v)
{
	if (!s || !v) { fprintf(stderr, "[libssw-b200] ssw_hit_set_view: NULL argument\n"); return -1; }
	v->n_rows = s->n_rows;
	v->n_hits = (int64_t)s->hits.size();
	v->row_off = s->row_off.data();
	v->hit_ref = s->hit_ref.empty() ? nullptr : s->hit_ref.data();
	v->hits = s->hits.empty() ? nullptr : s->hits.data();
	v->cigar_pool = s->pool.empty() ? nullptr : s->pool.data();
	v->pool_used = (int64_t)s->pool.size();
	return 0;
}

extern "C" void ssw_hit_set_destroy(ssw_hit_set* s) { delete s; }

/* mark_mismatch (ssw.c:1019-1074) for the CIGARs of a batch, on the device (ssw_mark.cuh) */
static int mark_mismatch_impl(ssw_engine* e, int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                              ssw_batch_result* results, const uint32_t* cigar_pool, int64_t pool_used,
                              uint32_t* out_pool, int64_t out_cap, int64_t* out_used, int32_t* nm)
{
	if (!e || n_pairs < 0 || (n_pairs && !results) || !out_used) return -1;
	if ((pair_query == nullptr) != (pair_ref == nullptr)) return -1;
	*out_used = 0;
	if (e->pssm_n) { fprintf(stderr, "[libssw-b200] ssw_engine_mark_mismatch: query profiles are resident: there are no query letters to compare\n"); return -1; }
	if (n_pairs > 0 && (e->n_q <= 0 || e->n_r <= 0)) return -1;
	SSW_CUDA_OK(cudaSetDevice(e->device));
	std::vector<SswMarkTask> tasks;
	std::vector<int64_t> owner;
	for (int64_t p = 0; p < n_pairs; ++p) {
		if (nm) nm[p] = 0;
		const ssw_batch_result& r = results[p];
		if (r.status || r.cigar_off < 0 || r.cigar_len <= 0) continue;
		const int32_t q = pair_query ? pair_query[p] : (int32_t)(p / e->n_r), rr = pair_ref ? pair_ref[p] : (int32_t)(p % e->n_r);
		if (q < 0 || q >= e->n_q || rr < 0 || rr >= e->n_r || !cigar_pool || (int64_t)r.cigar_off + r.cigar_len > pool_used) return -1;
		SswMarkTask t;
		memset(&t, 0, sizeof(t));
		t.ref_off = e->r_off[rr] + r.ref_begin1;
		t.read_off = e->q_off[q];
		t.cig_off = r.cigar_off; t.cig_len = r.cigar_len;
		t.read_len = (int32_t)(e->q_off[q + 1] - e->q_off[q]); t.read_begin1 = r.read_begin1; t.read_end1 = r.read_end1;
		tasks.push_back(t);
		owner.push_back(p);
	}
	if (tasks.empty()) return 0;
	const size_t o_in = (sizeof(SswMarkTask) * tasks.size() + 255) / 256 * 256;
	const size_t in_bytes = ((size_t)pool_used * 4 + 255) / 256 * 256;
	if (e->d_mark.ensure(o_in + in_bytes + 256)) return -1;
	uint8_t* base = e->d_mark.as<uint8_t>();
	SswMarkTask* d_tasks = reinterpret_cast<SswMarkTask*>(base);
	uint32_t* d_in = reinterpret_cast<uint32_t*>(base + o_in);
	SSW_CUDA_OK(cudaMemcpyAsync(d_tasks, tasks.data(), sizeof(SswMarkTask) * tasks.size(), cudaMemcpyHostToDevice, e->stream));
	SSW_CUDA_OK(cudaMemcpyAsync(d_in, cigar_pool, (size_t)pool_used * 4, cudaMemcpyHostToDevice, e->stream));
	const dim3 grid((unsigned)((tasks.size() + SSW_MARK_THREADS / 32 - 1) / (SSW_MARK_THREADS / 32)));
	ssw_launch(ssw_mark_kernel<false>, grid, dim3(SSW_MARK_THREADS), 0, e->stream, d_tasks, (int)tasks.size(), (const int8_t*)e->d_q.as<int8_t>(),
	           (const int8_t*)e->d_r.as<int8_t>(), (const uint32_t*)d_in, (uint32_t*)nullptr);
	SSW_CUDA_OK(cudaGetLastError());
	SSW_CUDA_OK(cudaMemcpyAsync(tasks.data(), d_tasks, sizeof(SswMarkTask) * tasks.size(), cudaMemcpyDeviceToHost, e->stream));
	SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
	int64_t total = 0;
	for (SswMarkTask& t : tasks) { t.out_off = total; total += t.out_len; }
	if (total > out_cap || total > 0x7fffffff || !out_pool) { fprintf(stderr, "[libssw-b200] marked CIGAR pool too small (%lld words needed)\n", (long long)total); return -1; }
	/* the output words go behind the input words */
	const size_t o_out = o_in + in_bytes;
	if (e->d_mark.cap < o_out + (size_t)total * 4 + 256) {
		/* grow without losing the inputs: simplest is to re-stage them */
		if (e->d_mark.ensure(o_out + (size_t)total * 4 + 256)) return -1;
		base = e->d_mark.as<uint8_t>();
		d_tasks = reinterpret_cast<SswMarkTask*>(base);
		d_in = reinterpret_cast<uint32_t*>(base + o_in);
		SSW_CUDA_OK(cudaMemcpyAsync(d_in, cigar_pool, (size_t)pool_used * 4, cudaMemcpyHostToDevice, e->stream));
	}
	uint32_t* d_out = reinterpret_cast<uint32_t*>(base + o_out);
	SSW_CUDA_OK(cudaMemcpyAsync(d_tasks, tasks.data(), sizeof(SswMarkTask) * tasks.size(), cudaMemcpyHostToDevice, e->stream));
	ssw_launch(ssw_mark_kernel<true>, grid, dim3(SSW_MARK_THREADS), 0, e->stream, d_tasks, (int)tasks.size(), (const int8_t*)e->d_q.as<int8_t>(),
	           (const int8_t*)e->d_r.as<int8_t>(), (const uint32_t*)d_in, d_out);
	SSW_CUDA_OK(cudaGetLastError());
	SSW_CUDA_OK(cudaMemcpyAsync(out_pool, d_out, (size_t)total * 4, cudaMemcpyDeviceToHost, e->stream));
	SSW_CUDA_OK(cudaStreamSynchronize(e->stream));
	for (size_t i = 0; i < tasks.size(); ++i) {
		ssw_batch_result& r = results[owner[i]];
		r.cigar_off = (int32_t)tasks[i].out_off; r.cigar_len = tasks[i].out_len;
		if (nm) nm[owner[i]] = tasks[i].nm;
	}
	*out_used = total;
	return 0;
}

extern "C" int ssw_engine_mark_mismatch(ssw_engine* e, int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                                        ssw_batch_result* results, const uint32_t* cigar_pool, int64_t pool_used,
                                        uint32_t* out_pool, int64_t out_cap, int64_t* out_used, int32_t* nm)
{
	try { return mark_mismatch_impl(e, n_pairs, pair_query, pair_ref, results, cigar_pool, pool_used, out_pool, out_cap, out_used, nm); }
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_engine_mark_mismatch: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}
