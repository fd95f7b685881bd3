// env_sets_emu.cpp -- TEST HARNESS: the parameter-set-indexed drivers of the plan chain's stages either side of the QP,
// and the device dispatch's sort (dispatch_emu.cpp), compiled with plain g++ (-DPQP_HOST_EMU) into a library of
// its own (tests/emu/sets_emu.py).  Every path looks its set up as the kernels of pqp_env.cu do -- pqp::param_of on a
// pqp::ParamTable built with pqp::make_param_row, a count and an optional per-path index -- and then runs through the
// map-indexed driver of env_maps_emu.cpp with that set's params.  An index outside the sets gives n_valid = 0 (bounds)
// or n_kept / n_out = 0 and ok = 0 (tails, when they check collisions), the path's states left as they came.
// Never linked into libpqp.so.
#include "env_maps_emu.cpp"
#include "dispatch_emu.cpp"

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

}  // extern "C"
