// Host-side scene object behind the C ABI (rb_scene).  Mirrors what Scene::Scene builds in the reference
// (src/scene.cpp:63-307) with GPU-native replacements: GPU LBVH instead of Embree/OptiX Prime, stream-ordered
// pool allocations instead of cudaMallocManaged buffers.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "rb_types.cuh"

// Timing events owned by a scene and reused by every rb_render call on it.
struct EventPool {
    std::vector<cudaEvent_t> ev;
    bool ensure(size_t n) {
        while (ev.size() < n) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) return false;
            ev.push_back(e);
        }
        return true;
    }
    void destroy() {
        for (cudaEvent_t e : ev) cudaEventDestroy(e);
        ev.clear();
    }
};

// Device tables owned by a scene, one slot each.  scene_table() keeps a slot's buffer when the requested size is unchanged and otherwise
// frees it in stream order and allocates a new one, so an update that rebuilds a table replaces it instead of adding to it.
enum SceneSlot {
    SS_SHAPES, SS_MATERIALS, SS_BVH_NODES, SS_BVH_TRIS, SS_LIGHTS, SS_LIGHT_PMF, SS_LIGHT_CDF, SS_LIGHT_AREAS, SS_AREA_POOL, SS_AREA_OFFSETS,
    SS_LIGHT_AUX, SS_EDGES, SS_PRIM_PMF, SS_PRIM_CDF, SS_EDGE_NODES, SS_COUNT
};
struct SceneBuffer {
    void* p = nullptr;
    size_t bytes = 0;
};

struct rb_scene {
    int device = 0;
    int gpu_index = -1;      // as in the descriptor of the build
    cudaStream_t stream = 0; // stream of the last build or update: builds, rb_scene_set_camera and the frees of rb_scene_destroy
    EventPool events;
    DevScene dev;   // passed by value to kernels
    rb_camera cam;  // host copy of the descriptor camera
    SceneBuffer bufs[SS_COUNT]; // device tables owned by the scene
    std::vector<rb_shape> shapes;
    std::vector<rb_material> materials;
    std::vector<DevLight> lights;
    std::vector<int> light_offsets; // [lights + 1]: first entry of every light in the area-CDF pool, then the pool size
    int max_generic_texture_dimension = 0;
    int has_envmap = 0;
    // partition (multi-GPU)
    int part = 0, num_parts = 1, rows_per_stripe = 16;
    // stats of the last render
    int last_launches = 0;
    float last_kernel_ms = 0.f;
    float last_stage_ms[4] = {0.f, 0.f, 0.f, 0.f}; // k_forward, backward bands, k_primary_edge, k_finish_camera
    float last_bwd_ms[3] = {0.f, 0.f, 0.f};        // inside the bands: k_bwd_trace (+ work lists), boundary stage (pick, sort by edge, shade), k_bwd_sweep
    double last_path_vertices = 0, last_primary_hits = 0;
    size_t last_exact_bytes = 0; // exact accumulators of the last deterministic backward pass (0 otherwise)
    int num_edge_nodes = 0; // records of the secondary-edge trees (dev.edge_nodes)
    bool edge_list_on_device = false;   // this scene's edge list was built by rb_edge_list.cu (else on the host)
    bool host_tables = false;           // ... and its camera-dependent tables on the host, from host_edges
    bool camera_tables_as_built = true; // the camera-dependent tables are on the side the build chose (not rb_scene_set_camera's device)
    bool incomplete = false;            // the last build / update / camera change failed part-way: rb_render refuses the scene
    std::vector<Edge> host_edges;
    // timings of the last build or update (ms, host clock) for reporting
    float build_ms_bvh = 0.f, build_ms_lights = 0.f, build_ms_edges = 0.f;
};

void rb_set_error(const std::string& msg);
#define RB_CUDA_OK(expr)                                                                                       \
    do {                                                                                                       \
        cudaError_t _e = (expr);                                                                               \
        if (_e != cudaSuccess) {                                                                               \
            rb_set_error(std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " + __FILE__ + ":" +      \
                         std::to_string(__LINE__) + " (" #expr ")");                                           \
            return 1;                                                                                          \
        }                                                                                                      \
    } while (0)

// tables embedded into the shared object (rb_tables.cpp)
extern "C" const unsigned char rb_sobol_table_begin[];
extern "C" const unsigned char rb_sobol_table_end[];
extern "C" const unsigned char rb_ltc_table_begin[];
extern "C" const unsigned char rb_ltc_table_end[];

int scene_buffer(rb_scene* sc, SceneSlot slot, size_t bytes, cudaStream_t stream, void** out); // rb_scene.cu
template <typename T>
int scene_table(rb_scene* sc, SceneSlot slot, size_t count, cudaStream_t stream, T** out) {
    void* p = nullptr;
    if (scene_buffer(sc, slot, (count > 0 ? count : 1) * sizeof(T), stream, &p)) return 1;
    *out = (T*)p;
    return 0;
}

int rb_build_bvh(rb_scene* sc, cudaStream_t stream);
int rb_build_lights(rb_scene* sc, bool geometry, cudaStream_t stream); // rb_light_build.cu
int rb_light_status(const rb_scene* sc, cudaStream_t stream, int* status);
int rb_build_edges(rb_scene* sc, cudaStream_t stream);
int rb_build_edge_list_gpu(rb_scene* sc, cudaStream_t stream);  // rb_edge_list.cu
int rb_build_edge_trees_gpu(rb_scene* sc, cudaStream_t stream); // rb_edge_tree.cu
int rb_build_primary_edge_cdf_gpu(rb_scene* sc, cudaStream_t stream);
