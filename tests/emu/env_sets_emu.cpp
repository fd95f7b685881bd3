// env_sets_emu.cpp -- TEST HARNESS: the parameter-set-indexed drivers of the plan chain's stages either side of the QP,
// and the (set, class) segment sort of the device dispatch, compiled with plain g++ (-DPQP_HOST_EMU) into a library of
// its own (tests/emu/sets_emu.py).  Every path looks its set up as the kernels of pqp_env.cu do -- pqp::param_of on a
// pqp::ParamTable built with pqp::make_param_row, a count and an optional per-path index -- and then runs through the
// map-indexed driver of env_maps_emu.cpp with that set's params.  An index outside the sets gives n_valid = 0 (bounds)
// or n_kept / n_out = 0 and ok = 0 (tails, when they check collisions), the path's states left as they came.
// Never linked into libpqp.so.
#include "env_maps_emu.cpp"
#include "../../path_optimizer_b200/csrc/pqp_dispatch.h"

struct EmuSets {
    ParamTable<PQP_MAX_PARAM_SETS> table;
    EmuSets(const pqp_params *sets, int n_sets, const int32_t *index) {
        table.n = n_sets;
        table.index = index;
        for (int s = 0; s < n_sets; ++s) table.row[s] = make_param_row(sets[s]);
    }
    // params of path b's set, NULL when its index is outside the sets
    const pqp_params *of(const pqp_params *sets, int b) const {
        const ParamRow *r = param_of(table, b);
        return r ? sets + (r - table.row) : nullptr;
    }
};

static const int32_t *at(const int32_t *index, int b) { return index ? index + b : nullptr; }

extern "C" {

void env_emu_update_bounds_sets(const pqp_params *sets, int n_sets, const int32_t *set_index,
                                const pqp_distance_map *maps, int n_maps, const int32_t *map_index, int mode, int batch,
                                const int32_t *n_points, const pqp_state *ref, const int32_t *n_knots, const double *knots,
                                const double *xc, const double *yc, pqp_station_bounds *out, int32_t *n_valid) {
    const EmuSets es(sets, n_sets, set_index);
    const bool improved = mode == PQP_BOUNDS_IMPROVED;
    int off = 0, koff = 0;
    for (int b = 0; b < batch; ++b) {
        const pqp_params *p = es.of(sets, b);
        if (!p) n_valid[b] = 0;
        else
            env_emu_update_bounds_maps(p, maps, n_maps, at(map_index, b), mode, 1, n_points + b, ref + off,
                                       improved ? n_knots + b : nullptr, improved ? knots + koff : nullptr,
                                       improved ? xc + 4 * (size_t)koff : nullptr,
                                       improved ? yc + 4 * (size_t)koff : nullptr, out + off, n_valid + b);
        off += n_points[b];
        if (improved) koff += n_knots[b];
    }
}

void env_emu_finish_raw_sets(const pqp_params *sets, int n_sets, const int32_t *set_index, const pqp_distance_map *maps,
                             int n_maps, const int32_t *map_index, int batch, const int32_t *n_points, pqp_state *paths,
                             int collision_check, int32_t *n_kept, int32_t *ok) {
    const EmuSets es(sets, n_sets, set_index);
    int off = 0;
    for (int b = 0; b < batch; ++b) {
        // without a collision check the set is not read (the kernel does not look it up)
        const pqp_params *p = collision_check ? es.of(sets, b) : sets;
        if (!p) { n_kept[b] = 0; ok[b] = 0; }
        else env_emu_finish_raw_maps(p, maps, n_maps, at(map_index, b), 1, n_points + b, paths + off, collision_check,
                                     n_kept + b, ok + b);
        off += n_points[b];
    }
}

void env_emu_densify_sets(const pqp_params *sets, int n_sets, const int32_t *set_index, const pqp_distance_map *maps,
                          int n_maps, const int32_t *map_index, int batch, const int32_t *n_points, const pqp_state *paths,
                          double spacing, int collision_check, int max_out, pqp_state *out_all, int32_t *n_out,
                          int32_t *ok) {
    const EmuSets es(sets, n_sets, set_index);
    int off = 0;
    for (int b = 0; b < batch; ++b) {
        const pqp_params *p = collision_check ? es.of(sets, b) : sets;
        if (!p) { n_out[b] = 0; ok[b] = 0; }
        else
            env_emu_densify_maps(p, maps, n_maps, at(map_index, b), 1, n_points + b, paths + off, spacing,
                                 collision_check, max_out, out_all + (size_t)b * max_out, n_out + b, ok + b);
        off += n_points[b];
    }
}

// The device dispatch's sort with a set index (pqp_dispatch_kernel in pqp_capi.cu), serially: every path's class from
// the table, its key pqp::dispatch_key, a histogram over the keys, its exclusive prefix and the scatter into order
// segments of `batch` entries each (segment set * nv + class, pre-filled with `batch`).  A path whose set lies outside
// [0, n_sets) or whose class is -1 gets key -1 and no entry.  order: [n_sets * nv * batch]; key: [batch].
void sets_dispatch_emu(const int8_t *table, int ncols, int formulation, int v0, int nv, int n_sets, int batch,
                       const int32_t *n_points, const int32_t *offsets, const pqp_state *ref, const int32_t *set_index,
                       int max_n, int min_keep, int max_keep, int32_t *order, int32_t *key) {
    const int nb = n_sets * nv * ncols;
    std::vector<int32_t> hist((size_t)nb, 0), base((size_t)n_sets * nv, 0);
    for (size_t i = 0; i < (size_t)n_sets * nv * batch; ++i) order[i] = batch;
    for (int b = 0; b < batch; ++b) {
        const int n = n_points[b];
        const int s = set_index ? set_index[b] : 0;
        const bool set_ok = s >= 0 && s < n_sets;
        const int keep = set_ok ? keep_control_steps(formulation, ref + offsets[b], n) : 0;
        const int v = set_ok ? dispatch_class(table, ncols, formulation, n, keep, max_n, min_keep, max_keep) : -1;
        key[b] = v >= 0 ? dispatch_key(s, v - v0, nv, ncols, n) : -1;
        if (key[b] >= 0) hist[key[b]]++;
    }
    int run = 0;
    for (int i = 0; i < nb; ++i) { const int c = hist[i]; hist[i] = run; run += c; }
    for (int r = 0; r < n_sets * nv; ++r) base[r] = hist[(size_t)r * ncols];
    for (int b = 0; b < batch; ++b) {
        if (key[b] < 0) continue;
        const int r = key[b] / ncols;
        order[(size_t)r * batch + (hist[key[b]]++ - base[r])] = b;
    }
}

}  // extern "C"
