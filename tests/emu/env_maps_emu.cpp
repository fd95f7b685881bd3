// env_maps_emu.cpp -- TEST HARNESS: the map-indexed drivers of the plan chain's stages either side of the QP, compiled
// with plain g++ (-DPQP_HOST_EMU) into a library of its own (tests/emu/maps_emu.py).  Every path is looked up as the
// kernels of pqp_env.cu look it up -- pqp::map_of on a descriptor table with a count and an optional per-path index,
// the map set of pqp_set_maps / pqp_plan_batch_maps -- and then runs through the single-map driver of env_emu.cpp on
// its own map.  An index outside the set gives n_valid = 0 (bounds) or n_kept / n_out = 0 and ok = 0 (tails, when they
// check collisions), the path's states left as they came.  Never linked into libpqp.so.
#include "env_emu.cpp"

struct EmuMapSet {
    std::vector<MapView> views;
    int32_t count;
    MapTable table;
    EmuMapSet(const pqp_distance_map *maps, int n_maps, const int32_t *index) : count(n_maps) {
        for (int m = 0; m < n_maps; ++m) views.push_back(view_of(maps + m));
        table = MapTable{views.data(), &count, index};
    }
    // descriptor of path b's map, NULL when its index is outside the set
    const pqp_distance_map *of(const pqp_distance_map *maps, int b) const {
        const MapView *mp = map_of(table, b);
        return mp ? maps + (mp - views.data()) : nullptr;
    }
};

extern "C" {

void env_emu_update_bounds_maps(const pqp_params *prm, const pqp_distance_map *maps, int n_maps, const int32_t *map_index,
                                int mode, int batch, const int32_t *n_points, const pqp_state *ref, const int32_t *n_knots,
                                const double *knots, const double *xc, const double *yc, pqp_station_bounds *out,
                                int32_t *n_valid) {
    const EmuMapSet set(maps, n_maps, map_index);
    const bool improved = mode == PQP_BOUNDS_IMPROVED;
    int off = 0, koff = 0;
    for (int b = 0; b < batch; ++b) {
        const pqp_distance_map *m = set.of(maps, b);
        if (!m) n_valid[b] = 0;
        else
            env_emu_update_bounds(prm, m, mode, 1, n_points + b, ref + off, improved ? n_knots + b : nullptr,
                                  improved ? knots + koff : nullptr, improved ? xc + 4 * (size_t)koff : nullptr,
                                  improved ? yc + 4 * (size_t)koff : nullptr, out + off, n_valid + b);
        off += n_points[b];
        if (improved) koff += n_knots[b];
    }
}

void env_emu_finish_raw_maps(const pqp_params *prm, const pqp_distance_map *maps, int n_maps, const int32_t *map_index,
                             int batch, const int32_t *n_points, pqp_state *paths, int collision_check, int32_t *n_kept,
                             int32_t *ok) {
    const EmuMapSet set(maps, n_maps, map_index);
    int off = 0;
    for (int b = 0; b < batch; ++b) {
        // without a collision check the map is not read (the kernel does not look it up)
        const pqp_distance_map *m = collision_check ? set.of(maps, b) : maps;
        if (!m) { n_kept[b] = 0; ok[b] = 0; }
        else env_emu_finish_raw(prm, m, 1, n_points + b, paths + off, collision_check, n_kept + b, ok + b);
        off += n_points[b];
    }
}

void env_emu_densify_maps(const pqp_params *prm, const pqp_distance_map *maps, int n_maps, const int32_t *map_index,
                          int batch, const int32_t *n_points, const pqp_state *paths, double spacing, int collision_check,
                          int max_out, pqp_state *out_all, int32_t *n_out, int32_t *ok) {
    const EmuMapSet set(maps, n_maps, map_index);
    int off = 0;
    for (int b = 0; b < batch; ++b) {
        const pqp_distance_map *m = collision_check ? set.of(maps, b) : maps;
        if (!m) { n_out[b] = 0; ok[b] = 0; }
        else
            env_emu_densify(prm, m, 1, n_points + b, paths + off, spacing, collision_check, max_out,
                            out_all + (size_t)b * max_out, n_out + b, ok + b);
        off += n_points[b];
    }
}

}  // extern "C"
