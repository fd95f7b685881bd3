// planner_maps_driver.cpp -- C++ driver over include/pqp_planner.hpp (needs a GPU): a PathOptimizerGpu built from
// several maps and the batched solveWithoutSmoothing with one map index per reference (simple bounds, raw output).
// Written for tests/test_gpu_multi_map.py, which compares what it writes with PathPlanner.plan(..., map_index).
//   planner_maps_driver <in.bin> <out.bin>
// in : int32 n_maps; per map: int32 rows, cols; double res, cx, cy; float dist[rows*cols];
//      int32 B; int32 n[B]; int32 map_index[B]; State ref[sumN]; double veh[B][4]
// out: int32 n_out[B]; int32 ok[B]; int32 status[B]; State paths (concatenated, n_out each)
#include <cstdio>
#include <vector>

#include "../../include/pqp_planner.hpp"

int main(int argc, char **argv) {
    if (argc < 3) return 2;
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    int32_t n_maps = 0;
    if (fread(&n_maps, 4, 1, f) != 1 || n_maps < 1) return 2;
    std::vector<pqp::DistanceMap> maps(n_maps);
    for (pqp::DistanceMap &map : maps) {
        int32_t dims[2];
        double geo[3];
        if (fread(dims, 4, 2, f) != 2 || fread(geo, 8, 3, f) != 3) return 2;
        map.rows = dims[0]; map.cols = dims[1]; map.resolution = geo[0]; map.center_x = geo[1]; map.center_y = geo[2];
        map.distance.resize((size_t)map.rows * map.cols);
        if (fread(map.distance.data(), 4, map.distance.size(), f) != map.distance.size()) return 2;
    }
    int32_t B = 0;
    if (fread(&B, 4, 1, f) != 1) return 2;
    std::vector<int32_t> n(B), map_index(B);
    if (fread(n.data(), 4, B, f) != (size_t)B || fread(map_index.data(), 4, B, f) != (size_t)B) return 2;
    std::vector<std::vector<pqp::State>> refs(B);
    size_t total = 0;
    for (int b = 0; b < B; ++b) {
        refs[b].resize(n[b]);
        if (fread(refs[b].data(), sizeof(pqp::State), n[b], f) != (size_t)n[b]) return 2;
        total += n[b];
    }
    std::vector<pqp::VehicleStateView> veh(B);
    if (fread(veh.data(), sizeof(pqp::VehicleStateView), B, f) != (size_t)B) return 2;
    fclose(f);

    auto po = pqp::PathOptimizerGpu::create(maps, B, (int)total);
    if (!po) return 4;
    std::vector<std::vector<pqp::State>> out;
    std::vector<char> ok;
    std::vector<int32_t> status;
    if (!po->solveWithoutSmoothing(refs, veh, map_index, &out, &ok, nullptr, nullptr, &status)) return 5;

    FILE *g = fopen(argv[2], "wb");
    if (!g) return 2;
    for (int b = 0; b < B; ++b) { const int32_t v = (int32_t)out[b].size(); fwrite(&v, 4, 1, g); }
    for (int b = 0; b < B; ++b) { const int32_t v = ok[b]; fwrite(&v, 4, 1, g); }
    fwrite(status.data(), 4, B, g);
    for (int b = 0; b < B; ++b) fwrite(out[b].data(), sizeof(pqp::State), out[b].size(), g);
    fclose(g);
    return 0;
}
