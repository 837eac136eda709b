// tray_exec.hpp — C++ host side above the C ABI (include/trb.h), shaped like the reference's Rust interface for
// this path so a tray_rust user finds the same names with the same argument meaning:
//
//   tray::FrameInfo      film::FrameInfo        /root/reference/src/film/mod.rs:26-36
//   tray::Config         exec::Config           src/exec/mod.rs:17-37        (+ seed: the reference seeds from the OS)
//   tray::RenderTarget   film::RenderTarget     src/film/render_target.rs    (RGBW f32 film, get_renderf32 layout)
//   tray::Scene          scene::Scene           src/scene.rs:93-182          (load_file, update_frame)
//   tray::Exec           trait exec::Exec       src/exec/mod.rs:41-49
//   tray::B200           replaces exec::MultiThreaded (src/exec/multithreaded.rs) on one GPU / one rank
//
// Where the reference panics, these throw tray::Error carrying the trb_status. Header-only; link with libtrb.so.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>
#include "trb.h"

namespace tray {

struct Error : std::runtime_error {
    trb_status status;
    Error(trb_status s, const std::string& m) : std::runtime_error(m), status(s) {}
};
inline void check(trb_status s) { if (s != TRB_OK) throw Error(s, trb_last_error()); }

struct FrameInfo { size_t frames = 1; float time = 0.f; size_t start = 0, end = 0; };

struct Adaptive { uint32_t min_spp = 0, max_spp = 0; }; // sampler::Adaptive (sampler/adaptive.rs); rounded up to powers of two

struct Config {
    std::string out_path, scene_file;
    size_t spp = 0;                          // 0: the scene's film.samples
    uint32_t num_threads = 0;                // accepted for signature compatibility; the GPU decides
    FrameInfo frame_info;
    size_t current_frame = 0;
    std::pair<size_t, size_t> select_blocks{0, 0}; // (start, count) into the Morton-sorted 8x8 block list; count 0 = all
    uint32_t seed = 1;
    bool adaptive = false;                   // false: LowDiscrepancy at spp; true: the Adaptive sampler below (spp unused)
    Adaptive sampler;
};

class RenderTarget {
  public:
    RenderTarget(size_t w, size_t h) : width_(w), height_(h), pixels_(w * h * 4, 0.f) {
        if (w % 2 || h % 2) throw Error(TRB_INVALID_ARG, "Image not evenly divided by blocks of (2, 2)"); // render_target.rs:43-45
    }
    std::pair<size_t, size_t> dimensions() const { return {width_, height_}; }
    void clear() { std::fill(pixels_.begin(), pixels_.end(), 0.f); }
    const std::vector<float>& get_renderf32() const { return pixels_; }    // render_target.rs:243-265
    float* data() { return pixels_.data(); }
    void add_pixels(const float* p) { for (size_t i = 0; i < pixels_.size(); ++i) pixels_[i] += p[i]; } // film/image.rs:21-33
  private:
    size_t width_, height_;
    std::vector<float> pixels_;
};

class Scene {
  public:
    // Scene::load_file (scene.rs:101). width/height/spp > 0 override the film section.
    static Scene load_file(const std::string& path, int device = 0, uint32_t width = 0, uint32_t height = 0, uint32_t spp = 0) {
        trb_scene* s = nullptr;
        check(trb_scene_load_json(path.c_str(), width, height, spp, device, &s));
        return Scene(s);
    }
    static Scene from_desc(const trb_scene_desc& d, int device = 0) { trb_scene* s = nullptr; check(trb_scene_create(&d, device, &s)); return Scene(s); }
    Scene(Scene&& o) noexcept : s_(o.s_) { o.s_ = nullptr; }
    Scene(const Scene&) = delete;
    ~Scene() { trb_scene_destroy(s_); }
    void update_frame(size_t frame, float start, float end) { check(trb_scene_update_frame(s_, (uint32_t)frame, start, end)); } // scene.rs:152
    // the scene's cameras and objects replaced in place; meshes, materials and textures stay built (trb_scene_replace_objects)
    void replace_objects(const trb_scene_objects& objects) { check(trb_scene_replace_objects(s_, &objects)); }
    // the scene's meshes added, removed, reordered and rebuilt in place, with the object section too when `objects` is given
    // (trb_scene_replace_meshes)
    void replace_meshes(const trb_scene_meshes& meshes, const trb_scene_objects* objects = nullptr) {
        check(trb_scene_replace_meshes(s_, &meshes, objects));
    }
    // the scene's film and / or integrator replaced in place; a null pointer keeps the current one (trb_scene_replace_settings)
    void replace_settings(const trb_film* film, const trb_integrator* integrator = nullptr) {
        check(trb_scene_replace_settings(s_, film, integrator));
    }
    // the scene's materials, MERL tables, textures and images replaced in place, with the object section too when `objects` is given
    // (trb_scene_replace_materials)
    void replace_materials(const trb_scene_materials& materials, const trb_scene_objects* objects = nullptr) {
        check(trb_scene_replace_materials(s_, &materials, objects));
    }
    RenderTarget make_render_target() const { uint32_t w, h; check(trb_scene_info(s_, &w, &h, nullptr, nullptr, nullptr, nullptr)); return RenderTarget(w, h); }
    uint32_t spp() const { uint32_t v; check(trb_scene_info(s_, nullptr, nullptr, &v, nullptr, nullptr, nullptr)); return v; }
    trb_scene* handle() const { return s_; }
  private:
    explicit Scene(trb_scene* s) : s_(s) {}
    trb_scene* s_;
};

struct Exec { // trait Exec (exec/mod.rs:41-49)
    virtual ~Exec() = default;
    virtual void render(Scene& scene, RenderTarget& rt, const Config& config) = 0;
};

class B200 : public Exec {
  public:
    trb_stats last_stats{};
    std::vector<uint32_t> last_pixel_spp; // Adaptive: samples per pixel (width * height, zero outside the selected blocks)
    void render(Scene& scene, RenderTarget& rt, const Config& c) override {
        trb_render_cfg cfg{};
        cfg.block_start = (uint32_t)c.select_blocks.first; cfg.block_count = (uint32_t)c.select_blocks.second;
        cfg.current_frame = (uint32_t)c.current_frame; cfg.seed = c.seed;
        if (c.adaptive) {
            const trb_adaptive ad{c.sampler.min_spp, c.sampler.max_spp};
            const auto d = rt.dimensions();
            last_pixel_spp.assign(d.first * d.second, 0u);
            check(trb_render_adaptive(scene.handle(), &cfg, &ad, rt.data(), last_pixel_spp.data(), &last_stats));
            return;
        }
        last_pixel_spp.clear();
        cfg.spp = (uint32_t)c.spp;
        check(trb_render(scene.handle(), &cfg, rt.data(), &last_stats)); // includes Scene::update_frame, like MultiThreaded::render
    }
};

inline std::vector<uint8_t> get_render(Scene& scene, RenderTarget& rt) { // RenderTarget::get_render (render_target.rs:185-210)
    auto d = rt.dimensions();
    std::vector<uint8_t> out(d.first * d.second * 3);
    check(trb_film_to_srgb8(scene.handle(), rt.data(), out.data()));
    return out;
}

} // namespace tray
