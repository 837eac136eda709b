// trb_tray — the `tray_rust` program (src/main.rs) over the C ABI, with the reference's three modes:
//
//   trb_tray <scenefile> [-o <path>] [-n <number>] [--start-frame <n>] [--end-frame <n>] [--seed S] [--spp N] [--device D | --devices LIST]
//            [--denoise] [--denoise-temporal [--temporal-gradients]] [--denoise-moments [--moment-gradients]] [--denoise-variance]
//            [--denoise-variance-temporal [--variance-gradients]] [--adaptive MIN MAX]
//   trb_tray <scenefile> --master <workers>... [-o <path>] [--start-frame <n>] [--end-frame <n>]
//   trb_tray --worker [-n <number>] [--port P] [--seed S] [--spp N] [--device D | --devices LIST]
//
// Single node (main.rs:56-109): Scene::load_file, then for every frame of the inclusive range Exec::render (trb_render, which
// includes update_frame), RenderTarget::get_render (trb_film_to_srgb8), write the image, clear the film.
// Master (main.rs:111-146, exec/distrib/master.rs): reads the film section on the host only (no GPU needed), splits the Morton
// block list B / W blocks per worker with the remainder on the last (master.rs:88-93, 217-224), connects to every worker, sends
// each its Instructions, then collects Frames from all workers in one poll loop and adds each into its frame's image
// (Image::add_blocks, film/image.rs:36-50) in arrival order. When all W workers have reported a frame it is converted
// (Image::get_srgb8 == trb_host_film_to_srgb8) and written.
// Worker: trb_worker's code (trb_distrib.hpp).
//
// Extensions over the reference: --seed, --spp and --device mean what they mean for trb_worker; --denoise renders every frame as two
// half-sample renders with AOVs and writes the denoised image (trb_denoise; single node, path integrator, 2 spp or more, refused
// before anything renders otherwise: the wire format carries no AOVs); --denoise-temporal renders the frames in order with one
// history and seed (S + frame) mod 2^32, denoising each with trb_denoise_temporal (refused where --denoise is, and with --denoise);
// --temporal-gradients, only with --denoise-temporal, denoises with trb_denoise_temporal_gradient at the frame's seed; --denoise-moments
// renders each frame once with AOVs (1 spp allowed), in order, with one history and seed (S + frame) mod 2^32, denoising it with
// trb_denoise_moments (single node, path integrator, refused with the other denoise flags); --moment-gradients, only with
// --denoise-moments, denoises with trb_denoise_moments_gradient at the frame's seed; --adaptive MIN MAX renders each frame with the
// Adaptive sampler (trb_render_adaptive), or with --denoise-moments by trb_render_adaptive_aov and the moment call (single node, path
// integrator; refused with --spp, since the sampler owns the schedule, and with --denoise, --denoise-temporal and --temporal-gradients,
// which need two half sample ranges); --denoise-variance renders each frame once with AOVs and the lum_w film (trb_render_aov_lum, or
// with --adaptive trb_render_adaptive_aov_lum) and denoises it with trb_denoise_variance (single node on one GPU, path integrator, 2
// samples per pixel or more, refused with the other denoise flags, --devices, --master and --worker); --denoise-variance-temporal
// renders the frames in order the same way, frame k with seed (S + k) mod 2^32, and denoises each with trb_denoise_variance_temporal
// and one history (refused where --denoise-variance is, and with --denoise-variance); --variance-gradients, only with
// --denoise-variance-temporal, denoises with trb_denoise_variance_temporal_gradient at the frame's seed; --devices 0,1,2,3 renders each frame on a trb_group of those GPUs in place of one --device:
// plain and --adaptive frames by trb_group_render(_adaptive), every denoise mode by the group's AOV renders (trb_group_render_aov,
// trb_group_render_adaptive_aov) and the denoise call on replica 0, which holds the history; with --worker the master's block range
// is rendered by trb_group_render, in the same Frames (refused with --device, with --master, and for an empty, malformed or
// duplicate list, before anything renders); a worker address is host[:port],
// a bare host meaning port 63234; -n is accepted and ignored. Output: -o without an extension is a directory (created, one level;
// frames go to frame%05d.png inside), with an extension one file rewritten by every frame, none means ./. PNG (stored deflate
// blocks) and binary PPM are written; JPEG is not built.
// Where the reference master panics, hangs or silently misbehaves (a worker it cannot reach, a worker that hangs up early, a
// malformed or out-of-range Frame, more workers than blocks), trb_tray exits with status 1 and a message naming the worker and
// the frame. Without a CUDA device, single-node mode exits with status 3, like trb_worker.
#include <netdb.h>
#include <poll.h>
#include <sys/stat.h>
#include <algorithm>
#include <cctype>
#include <cerrno>
#include <chrono>
#include <cstdarg>
#include <memory>
#include "trb_distrib.hpp"
#include "../../include/tray_exec.hpp"

namespace {

const char* USAGE =
    "Usage:\n"
    "    trb_tray <scenefile> [-o <path>] [-n <number>] [--start-frame <number>] [--end-frame <number>] [--seed S] [--spp N]\n"
    "             [--device D | --devices LIST] [--denoise | --denoise-temporal [--temporal-gradients] | --denoise-moments [--moment-gradients]\n"
    "             | --denoise-variance | --denoise-variance-temporal [--variance-gradients]]\n"
    "             [--adaptive MIN MAX]\n"
    "    trb_tray <scenefile> --master <workers>... [-o <path>] [--start-frame <number>] [--end-frame <number>]\n"
    "    trb_tray --worker [-n <number>] [--port P] [--seed S] [--spp N] [--device D | --devices LIST]\n"
    "    trb_tray (-h | --help)\n"
    "\n"
    "Options:\n"
    "  -o <path>               Output file (.png or .ppm) or directory (frames written as frame<#####>.png). Default './'.\n"
    "  -n <number>             Accepted for compatibility with tray_rust; the GPU decides its own parallelism.\n"
    "  --start-frame <number>  First frame to render, of the inclusive range [start, end]. Default: the scene's film.start_frame.\n"
    "  --end-frame <number>    Last frame to render, of the inclusive range [start, end]. Default: the scene's film.end_frame.\n"
    "  --master                Drive the workers in <workers>... (host or host:port, default port 63234) and save the frames.\n"
    "  --worker                Listen for a master and render the blocks it assigns (the same program as trb_worker).\n"
    "  --seed S                Random seed of the render (default 1).\n"
    "  --spp N                 Samples per pixel, overriding the scene's film.samples.\n"
    "  --device D              CUDA device to render on (default 0).\n"
    "  --devices LIST          Render each frame on all the CUDA devices of the comma-separated LIST (e.g. 0,1,2,3): the image is\n"
    "                          split between them and their films summed; every --denoise mode denoises on the first. Not with\n"
    "                          --device or --master (with --master pass it to each worker).\n"
    "  --denoise               Render each frame's samples as two halves with albedo, normal and depth, and write the denoised\n"
    "                          image. Single node only, path integrator, at least 2 samples per pixel.\n"
    "  --denoise-temporal      As --denoise, accumulating each pixel's history over the frame range through the scene's motion;\n"
    "                          frame k is rendered with seed S + k.\n"
    "  --temporal-gradients    With --denoise-temporal only: re-shade a sample of each 3x3 pixel block of the previous frame in\n"
    "                          this one and shorten the history where the lighting changed (animated lights). Single node only.\n"
    "  --denoise-moments       Render each frame once with albedo, normal and depth (1 sample per pixel is enough) and denoise it\n"
    "                          with a history of luminance moments over the frame range; frame k is rendered with seed S + k.\n"
    "                          Single node only, path integrator.\n"
    "  --moment-gradients      With --denoise-moments only: re-shade a sample of each 3x3 pixel block of the previous frame in\n"
    "                          this one and shorten the moment history where the lighting changed. Single node only.\n"
    "  --denoise-variance      Render each frame once with albedo, normal, depth and the luminance moments of its samples, and\n"
    "                          denoise it with the variance of each pixel's own samples. Single node on one --device, path\n"
    "                          integrator, at least 2 samples per pixel (with --adaptive: MIN at least 2).\n"
    "  --denoise-variance-temporal  As --denoise-variance, carrying each pixel's variance through a history over the frame range;\n"
    "                          frame k is rendered with seed S + k.\n"
    "  --variance-gradients    With --denoise-variance-temporal only: re-shade a sample of each 3x3 pixel block of the previous frame\n"
    "                          in this one and shorten the history where the lighting changed.\n"
    "  --adaptive MIN MAX      Render with the Adaptive sampler: MIN samples per pixel, then more in rounds while a pixel's samples\n"
    "                          disagree, up to MAX (both rounded up to powers of two). With --denoise-moments each frame is also\n"
    "                          rendered with albedo, normal and depth and denoised by the moment denoiser.\n"
    "                          Single node only, path integrator; not with --spp, --denoise or --denoise-temporal.\n"
    "  -h, --help              Show this message.\n";

int die(const char* fmt, ...) {
    std::fputs("trb_tray: ", stderr);
    va_list ap; va_start(ap, fmt); std::vfprintf(stderr, fmt, ap); va_end(ap);
    std::fputc('\n', stderr);
    return 1;
}

double seconds_since(std::chrono::steady_clock::time_point t0) { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); }

bool parse_u64(const char* s, uint64_t& v) {
    if (!s || !*s || *s == '-') return false;
    char* e = nullptr; errno = 0;
    const unsigned long long x = std::strtoull(s, &e, 10);
    if (errno || *e) return false;
    v = x; return true;
}

// -o: PathBuf::extension decides between a directory and one file (main.rs:60-73, 88-91)
struct OutPath {
    std::string path = "./";
    bool is_dir = true;
    bool ppm = false;
    std::string file_for(uint64_t frame) const {
        if (!is_dir) return path;
        char name[32]; std::snprintf(name, sizeof name, "frame%05llu.png", (unsigned long long)frame);
        return path + (path.back() == '/' ? "" : "/") + name;
    }
};

// Path::extension: the part of the last component after its last '.', unless that dot starts the name; "." and ".." have none
bool path_extension(const std::string& p, std::string& ext) {
    size_t end = p.size();
    while (end > 1 && p[end - 1] == '/') --end;
    const size_t slash = p.rfind('/', end - 1);
    const std::string name = p.substr(slash == std::string::npos ? 0 : slash + 1, end - (slash == std::string::npos ? 0 : slash + 1));
    if (name.empty() || name == "." || name == "..") return false;
    const size_t dot = name.rfind('.');
    if (dot == std::string::npos || dot == 0) return false;
    ext = name.substr(dot + 1);
    return true;
}

// Checked before any scene load: an output the program cannot write is refused up front, where the reference renders every frame
// and then prints "Error saving image" for each.
bool resolve_out_path(const char* o, OutPath& out) {
    if (!o) return true;
    out.path = o;
    std::string ext;
    out.is_dir = !path_extension(out.path, ext);
    if (out.is_dir) return true;
    for (char& c : ext) c = (char)std::tolower((unsigned char)c);
    if (ext == "png") return true;
    if (ext == "ppm") { out.ppm = true; return true; }
    if (ext == "jpg" || ext == "jpeg") die("cannot write '%s': JPEG output is not built; use .png or .ppm", o);
    else die("cannot write '%s': unsupported image format '.%s'; use .png or .ppm", o, ext.c_str());
    return false;
}

// std::fs::create_dir of the -o directory: one level; an existing one is fine
bool create_out_dir(const OutPath& out, bool given) {
    if (!given || !out.is_dir) return true;
    if (::mkdir(out.path.c_str(), 0777) == 0 || errno == EEXIST) return true;
    die("failed to create output directory '%s': %s", out.path.c_str(), std::strerror(errno));
    return false;
}

// image::save_buffer(path, img, w, h, image::RGB(8)) for the two formats that are built
bool save_image(const OutPath& out, const std::string& file, const uint8_t* rgb8, uint32_t w, uint32_t h) {
    if (!out.ppm) {
        if (trb_write_png(file.c_str(), rgb8, w, h) == TRB_OK) return true;
        die("Error saving image '%s': %s", file.c_str(), trb_last_error());
        return false;
    }
    FILE* f = std::fopen(file.c_str(), "wb");
    bool ok = f != nullptr;
    if (ok) {
        ok = std::fprintf(f, "P6\n%u %u\n255\n", w, h) > 0 && std::fwrite(rgb8, 1, (size_t)w * h * 3, f) == (size_t)w * h * 3;
        ok = std::fclose(f) == 0 && ok;
    }
    if (!ok) die("Error saving image '%s': %s", file.c_str(), std::strerror(errno));
    return ok;
}

struct Args {
    std::string scene;
    std::vector<std::string> workers;
    const char* out = nullptr;
    bool master = false, has_start = false, has_end = false, has_seed = false, has_spp = false, has_device = false, denoise = false,
         denoise_temporal = false, temporal_gradients = false, denoise_moments = false, moment_gradients = false, adaptive = false,
         denoise_variance = false, denoise_variance_temporal = false, variance_gradients = false;
    uint64_t start = 0, end = 0, seed = 1, spp = 0, device = 0, ad_min = 0, ad_max = 0;
    std::vector<int> devices; // --devices; empty: one --device
};

// scene description (host only): the film section, frame range overrides applied
struct Desc {
    trb_scene_desc* d = nullptr;
    ~Desc() { if (d) trb_desc_free(d); }
};

bool load_desc(const Args& a, uint32_t spp, Desc& desc, uint64_t& start, uint64_t& end) {
    const trb_status rc = trb_desc_load_json(a.scene.c_str(), 0, 0, spp, &desc.d);
    if (rc != TRB_OK) { die("cannot load scene '%s': %s", a.scene.c_str(), trb_last_error()); return false; }
    start = a.has_start ? a.start : desc.d->film.start_frame;
    end = a.has_end ? a.end : desc.d->film.end_frame;
    if (end < start) { die("end frame %llu is before start frame %llu", (unsigned long long)end, (unsigned long long)start); return false; }
    if (end > UINT32_MAX) { die("end frame %llu does not fit the renderer's 32-bit frame index", (unsigned long long)end); return false; }
    return true;
}

uint32_t pow2_at_least(uint32_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }

// Where a frame renders: one scene (--device), or a group of GPUs (--devices) whose renders reduce to replica 0. `scene` is the
// scene that converts and denoises: the one scene, or the group's replica 0, which also holds the denoise history.
struct Renderer {
    trb_scene* scene = nullptr;
    trb_group* group = nullptr;
    trb_status aov(const trb_render_cfg* cfg, float* film, const trb_aov_film* aov) const {
        return group ? trb_group_render_aov(group, cfg, film, aov, nullptr) : trb_render_aov(scene, cfg, film, aov, nullptr);
    }
    trb_status adaptive_aov(const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, const trb_aov_film* aov) const {
        return group ? trb_group_render_adaptive_aov(group, cfg, ad, film, aov, nullptr, nullptr)
                     : trb_render_adaptive_aov(scene, cfg, ad, film, aov, nullptr, nullptr);
    }
};

// --denoise: samples [0, n/2) and [n/2, n) of the frame into two films, the AOVs over both, then trb_denoise (DESIGN.md §4 "Denoising");
// --denoise-temporal: the same with trb_denoise_temporal and the history of the frames before (DESIGN.md §4 "Temporal denoising")
struct DenoisedFrame {
    std::vector<float> a, b, albedo, normal, out;
    std::vector<uint64_t> nearest;
    explicit DenoisedFrame(size_t npx) : a(npx * 4), b(npx * 4), albedo(npx * 4), normal(npx * 4), out(npx * 4), nearest(npx) {}
    void render(const Renderer& r, uint32_t spp, uint32_t seed, uint32_t frame, trb_denoise_history* history = nullptr, bool gradients = false) {
        trb_scene* s = r.scene;
        std::fill(a.begin(), a.end(), 0.0f); std::fill(b.begin(), b.end(), 0.0f);
        std::fill(albedo.begin(), albedo.end(), 0.0f); std::fill(normal.begin(), normal.end(), 0.0f);
        std::fill(nearest.begin(), nearest.end(), ~0ull);
        trb_render_cfg cfg{};
        cfg.spp = spp; cfg.seed = seed; cfg.current_frame = frame; cfg.sample_count = spp / 2;
        const trb_aov_film aov{albedo.data(), normal.data(), nearest.data()};
        tray::check(r.aov(&cfg, a.data(), &aov)); // includes Scene::update_frame
        cfg.sample_first = spp / 2; cfg.flags = TRB_RENDER_NO_UPDATE;
        tray::check(r.aov(&cfg, b.data(), &aov));
        const trb_denoise_input in{a.data(), b.data(), albedo.data(), normal.data(), nearest.data()};
        if (history && gradients) {
            const trb_denoise_gradient_output o{out.data(), nullptr, nullptr, nullptr};
            tray::check(trb_denoise_temporal_gradient(s, history, &in, nullptr, seed, &o));
        } else if (history) {
            const trb_denoise_temporal_output o{out.data(), nullptr, nullptr};
            tray::check(trb_denoise_temporal(s, history, &in, nullptr, &o));
        } else {
            tray::check(trb_denoise(s, &in, nullptr, out.data()));
        }
    }
};

// --denoise-moments: the frame's whole sample range into one film with its AOVs, then trb_denoise_moments with the history of the
// frames before (DESIGN.md §4 "Moment denoising"); --moment-gradients: trb_denoise_moments_gradient at the frame's seed instead
// (DESIGN.md §4 "Moment gradients")
struct MomentsFrame {
    std::vector<float> colour, albedo, normal, out;
    std::vector<uint64_t> nearest;
    explicit MomentsFrame(size_t npx) : colour(npx * 4), albedo(npx * 4), normal(npx * 4), out(npx * 4), nearest(npx) {}
    // ad: the Adaptive sampler in place of LowDiscrepancy at spp (trb_render_adaptive_aov; DESIGN.md §4 "Adaptive AOVs"), or nullptr
    void render(const Renderer& r, uint32_t spp, uint32_t seed, uint32_t frame, trb_denoise_history* history, bool gradients, const trb_adaptive* ad) {
        trb_scene* s = r.scene;
        std::fill(colour.begin(), colour.end(), 0.0f);
        std::fill(albedo.begin(), albedo.end(), 0.0f); std::fill(normal.begin(), normal.end(), 0.0f);
        std::fill(nearest.begin(), nearest.end(), ~0ull);
        trb_render_cfg cfg{};
        cfg.spp = spp; cfg.seed = seed; cfg.current_frame = frame;
        const trb_aov_film aov{albedo.data(), normal.data(), nearest.data()};
        if (ad) { cfg.spp = 0; tray::check(r.adaptive_aov(&cfg, ad, colour.data(), &aov)); } // includes Scene::update_frame
        else tray::check(r.aov(&cfg, colour.data(), &aov)); // includes Scene::update_frame
        const trb_denoise_frame in{colour.data(), albedo.data(), normal.data(), nearest.data()};
        if (gradients) {
            const trb_denoise_moments_gradient_output o{out.data(), nullptr, nullptr, nullptr, nullptr};
            tray::check(trb_denoise_moments_gradient(s, history, &in, nullptr, seed, &o));
        } else {
            const trb_denoise_moments_output o{out.data(), nullptr, nullptr, nullptr};
            tray::check(trb_denoise_moments(s, history, &in, nullptr, &o));
        }
    }
};

// --denoise-variance: the frame's whole sample range into one film with its AOVs and the lum_w film, then trb_denoise_variance
// (DESIGN.md §4 "Sample variance"); with ad, the Adaptive sampler's render (trb_render_adaptive_aov_lum) in place of LowDiscrepancy.
// --denoise-variance-temporal: the same with trb_denoise_variance_temporal and the history of the frames before, or with
// --variance-gradients trb_denoise_variance_temporal_gradient at the frame's seed (DESIGN.md §4 "Variance temporal denoising")
struct VarianceFrame {
    std::vector<float> colour, albedo, normal, lum, out;
    std::vector<uint64_t> nearest;
    explicit VarianceFrame(size_t npx) : colour(npx * 4), albedo(npx * 4), normal(npx * 4), lum(npx * 4), out(npx * 4), nearest(npx) {}
    void render(trb_scene* s, uint32_t spp, uint32_t seed, uint32_t frame, const trb_adaptive* ad, trb_denoise_history* history = nullptr,
                bool gradients = false) {
        for (std::vector<float>* v : {&colour, &albedo, &normal, &lum}) std::fill(v->begin(), v->end(), 0.0f);
        std::fill(nearest.begin(), nearest.end(), ~0ull);
        trb_render_cfg cfg{};
        cfg.spp = ad ? 0 : spp; cfg.seed = seed; cfg.current_frame = frame;
        const trb_aov_film aov{albedo.data(), normal.data(), nearest.data()};
        if (ad) tray::check(trb_render_adaptive_aov_lum(s, &cfg, ad, colour.data(), &aov, lum.data(), nullptr, nullptr)); // includes Scene::update_frame
        else tray::check(trb_render_aov_lum(s, &cfg, colour.data(), &aov, lum.data(), nullptr));
        const trb_denoise_frame in{colour.data(), albedo.data(), normal.data(), nearest.data()};
        if (history && gradients) {
            const trb_denoise_moments_gradient_output o{out.data(), nullptr, nullptr, nullptr, nullptr};
            tray::check(trb_denoise_variance_temporal_gradient(s, history, &in, lum.data(), nullptr, seed, &o));
        } else if (history) {
            const trb_denoise_moments_output o{out.data(), nullptr, nullptr, nullptr};
            tray::check(trb_denoise_variance_temporal(s, history, &in, lum.data(), nullptr, &o));
        } else {
            tray::check(trb_denoise_variance(s, &in, lum.data(), nullptr, out.data(), nullptr));
        }
    }
};

// ---- single node (main.rs:56-109) -------------------------------------------------------------------------------------------
int single_node(const Args& a, const OutPath& out) {
    Desc desc;
    uint64_t start = 0, end = 0;
    if (!load_desc(a, (uint32_t)a.spp, desc, start, end)) return 1;
    const uint32_t spp = pow2_at_least(std::max(1u, desc.d->film.samples));
    const bool denoise = a.denoise || a.denoise_temporal;
    const char* flag = a.denoise_temporal ? "--denoise-temporal" : "--denoise";
    if (denoise && desc.d->integrator.type != TRB_INTEGRATOR_PATH)
        return die("%s needs the path integrator: the scene's integrator renders no albedo, normal or depth", flag);
    if (denoise && spp < 2) return die("%s needs at least 2 samples per pixel (two half renders); the scene has %u", flag, spp);
    if (a.denoise_moments && desc.d->integrator.type != TRB_INTEGRATOR_PATH)
        return die("--denoise-moments needs the path integrator: the scene's integrator renders no albedo, normal or depth");
    if (a.adaptive && desc.d->integrator.type != TRB_INTEGRATOR_PATH)
        return die("--adaptive needs the path integrator: the Adaptive sampler is built for it only");
    const bool variance = a.denoise_variance || a.denoise_variance_temporal;
    const char* vflag = a.denoise_variance_temporal ? "--denoise-variance-temporal" : "--denoise-variance";
    if (variance && desc.d->integrator.type != TRB_INTEGRATOR_PATH)
        return die("%s needs the path integrator: the scene's integrator renders no albedo, normal or depth", vflag);
    if (variance && !a.adaptive && spp < 2)
        return die("%s needs at least 2 samples per pixel (a variance of one sample is undefined); the scene has %u", vflag, spp);
    const trb_adaptive ad{(uint32_t)a.ad_min, (uint32_t)a.ad_max};
    try {
        std::unique_ptr<tray::Scene> one;
        std::unique_ptr<trb_group, void (*)(trb_group*)> group(nullptr, trb_group_destroy);
        if (a.devices.empty()) {
            one.reset(new tray::Scene(tray::Scene::from_desc(*desc.d, (int)a.device)));
        } else {
            trb_group* g = nullptr;
            tray::check(trb_group_create(desc.d, a.devices.data(), (int)a.devices.size(), &g));
            group.reset(g);
        }
        trb_desc_free(desc.d); desc.d = nullptr;
        const Renderer rd{one ? one->handle() : trb_group_scene(group.get(), 0), group.get()};
        uint32_t width = 0, height = 0;
        tray::check(trb_scene_info(rd.scene, &width, &height, nullptr, nullptr, nullptr, nullptr));
        tray::RenderTarget rt(width, height);
        const auto dim = rt.dimensions();
        tray::B200 exec;
        tray::Config config;
        config.seed = (uint32_t)a.seed;
        config.adaptive = a.adaptive;
        config.sampler = tray::Adaptive{ad.min_spp, ad.max_spp};
        const auto scene_start = std::chrono::steady_clock::now();
        std::unique_ptr<DenoisedFrame> dn;
        if (denoise) dn.reset(new DenoisedFrame((size_t)dim.first * dim.second));
        trb_denoise_history* history = nullptr;
        std::unique_ptr<MomentsFrame> mf;
        if (a.denoise_moments) mf.reset(new MomentsFrame((size_t)dim.first * dim.second));
        std::unique_ptr<VarianceFrame> vf;
        if (variance) vf.reset(new VarianceFrame((size_t)dim.first * dim.second));
        if (a.denoise_temporal || a.denoise_moments || a.denoise_variance_temporal) tray::check(trb_denoise_history_create(rd.scene, &history));
        const std::unique_ptr<trb_denoise_history, trb_status (*)(trb_denoise_history*)> history_owner(history, trb_denoise_history_destroy);
        for (uint64_t i = start; i <= end; ++i) {
            config.current_frame = i;
            std::vector<uint8_t> img;
            if (vf) {
                if (history) vf->render(rd.scene, spp, (uint32_t)(config.seed + i), (uint32_t)i, a.adaptive ? &ad : nullptr, history, a.variance_gradients);
                else vf->render(rd.scene, spp, config.seed, (uint32_t)i, a.adaptive ? &ad : nullptr);
                img.resize((size_t)dim.first * dim.second * 3);
                tray::check(trb_film_to_srgb8(rd.scene, vf->out.data(), img.data()));
            } else if (mf) {
                mf->render(rd, spp, (uint32_t)(config.seed + i), (uint32_t)i, history, a.moment_gradients, a.adaptive ? &ad : nullptr);
                img.resize((size_t)dim.first * dim.second * 3);
                tray::check(trb_film_to_srgb8(rd.scene, mf->out.data(), img.data()));
            } else if (dn) {
                if (history) dn->render(rd, spp, (uint32_t)(config.seed + i), (uint32_t)i, history, a.temporal_gradients);
                else dn->render(rd, spp, config.seed, (uint32_t)i);
                img.resize((size_t)dim.first * dim.second * 3);
                tray::check(trb_film_to_srgb8(rd.scene, dn->out.data(), img.data()));
            } else if (one) {
                exec.render(*one, rt, config);
                img = tray::get_render(*one, rt);
            } else { // B200::render's calls on the group
                trb_render_cfg cfg{};
                cfg.current_frame = (uint32_t)i; cfg.seed = config.seed;
                std::vector<uint32_t> pixel_spp(a.adaptive ? (size_t)dim.first * dim.second : 0);
                if (a.adaptive) tray::check(trb_group_render_adaptive(group.get(), &cfg, &ad, rt.data(), pixel_spp.data(), nullptr));
                else tray::check(trb_group_render(group.get(), &cfg, rt.data(), nullptr));
                img.resize((size_t)dim.first * dim.second * 3);
                tray::check(trb_film_to_srgb8(rd.scene, rt.data(), img.data()));
            }
            const std::string file = out.file_for(i);
            if (!save_image(out, file, img.data(), (uint32_t)dim.first, (uint32_t)dim.second)) return 1;
            rt.clear();
            std::printf("Frame %llu: rendered to '%s'\n--------------------\n", (unsigned long long)i, file.c_str());
            std::fflush(stdout);
        }
        std::printf("Rendering entire sequence took %.4fs\n", seconds_since(scene_start));
    } catch (const tray::Error& e) {
        std::fprintf(stderr, "trb_tray: status %d: %s\n", (int)e.status, e.what());
        return e.status == TRB_NO_DEVICE ? 3 : 1;
    }
    return 0;
}

// ---- master (main.rs:111-146, exec/distrib/master.rs) -----------------------------------------------------------------------
struct WorkerConn {
    std::string name;             // host:port, as the messages print it
    int fd = -1;
    std::vector<uint8_t> buf;     // the Frame being read
    size_t got = 0;
    uint64_t expected = 8;        // the size header first, then the Frame's encoded_size
    std::vector<bool> reported;   // per frame of the range
    uint64_t n_reported = 0;
};

struct DistributedFrame {         // master.rs:24-46
    std::vector<float> render;    // RGBW; empty until the first worker reports and after the frame is written
    size_t num_reporting = 0;
    std::chrono::steady_clock::time_point first_tile_recv;
};

struct Master {
    std::vector<WorkerConn> workers;
    ~Master() { for (WorkerConn& w : workers) if (w.fd >= 0) ::close(w.fd); }
};

// host[:port]; a bare host means exec::distrib::worker::PORT
bool parse_worker(const std::string& s, std::string& host, std::string& port) {
    port = std::to_string(trb_distrib::PORT);
    if (std::count(s.begin(), s.end(), ':') == 1) {
        host = s.substr(0, s.find(':')); port = s.substr(s.find(':') + 1);
    } else {
        host = s;
    }
    uint64_t p = 0;
    return !host.empty() && parse_u64(port.c_str(), p) && p > 0 && p < 65536;
}

int connect_worker(const std::string& host, const std::string& port, std::string& err) {
    addrinfo hints{}, *res = nullptr;
    hints.ai_family = AF_UNSPEC; hints.ai_socktype = SOCK_STREAM;
    const int g = ::getaddrinfo(host.c_str(), port.c_str(), &hints, &res);
    if (g != 0) { err = ::gai_strerror(g); return -1; }
    int fd = -1;
    err = "no address";
    for (addrinfo* ai = res; ai; ai = ai->ai_next) {
        fd = ::socket(ai->ai_family, ai->ai_socktype | SOCK_CLOEXEC, ai->ai_protocol);
        if (fd < 0) { err = std::strerror(errno); continue; }
        if (::connect(fd, ai->ai_addr, ai->ai_addrlen) == 0) break;
        err = std::strerror(errno);
        ::close(fd); fd = -1;
    }
    ::freeaddrinfo(res);
    return fd;
}

// which frame a message about worker `w` is about
std::string frame_of(const WorkerConn& w, uint64_t start, uint64_t n_frames) {
    char s[96];
    if (w.got >= 16) { uint64_t f; std::memcpy(&f, &w.buf[8], 8); std::snprintf(s, sizeof s, "frame %llu", (unsigned long long)f); return s; }
    for (uint64_t k = 0; k < n_frames; ++k)
        if (!w.reported[k]) { std::snprintf(s, sizeof s, "frame %llu (its next unreported frame)", (unsigned long long)(start + k)); return s; }
    return "after its last frame";
}

int master_node(const Args& a, const OutPath& out) {
    Desc desc;
    uint64_t start = 0, end = 0;
    if (!load_desc(a, 0, desc, start, end)) return 1;
    const uint32_t w = desc.d->film.width, h = desc.d->film.height;
    trb_desc_free(desc.d); desc.d = nullptr;
    if (w == 0 || h == 0 || w % 8 || h % 8) return die("image %ux%u is not evenly divided by blocks of (8, 8)", w, h); // block_queue.rs:29-31
    const uint64_t n_frames = end - start + 1;
    const uint64_t n_workers = a.workers.size();
    const uint64_t n_blocks = (uint64_t)(w / 8) * (h / 8);
    // block_count 0 means "all blocks" to a worker (block_queue.rs:39), so an idle worker would render the whole image again
    if (n_workers > n_blocks) return die("%llu workers for %llu blocks: every worker needs at least one 8x8 block", (unsigned long long)n_workers, (unsigned long long)n_blocks);
    const uint64_t blocks_per_worker = n_blocks / n_workers, blocks_remainder = n_blocks % n_workers; // master.rs:91-93
    const uint64_t max_frame_bytes = trb_distrib::FRAME_HEADER_BYTES + 32ull * w * h; // 1x1 blocks over the whole image, each 16 + 16 bytes

    Master m;
    m.workers.resize(n_workers);
    const auto scene_start = std::chrono::steady_clock::now();
    for (uint64_t i = 0; i < n_workers; ++i) { // connect to every worker before sending anything (master.rs:99-113)
        std::string host, port, err;
        WorkerConn& wc = m.workers[i];
        if (!parse_worker(a.workers[i], host, port)) return die("bad worker address '%s': use host or host:port", a.workers[i].c_str());
        wc.name = host + ":" + port;
        wc.reported.assign(n_frames, false);
        wc.fd = connect_worker(host, port, err);
        if (wc.fd < 0) return die("failed to contact worker %s: %s", wc.name.c_str(), err.c_str());
    }
    for (uint64_t i = 0; i < n_workers; ++i) { // master.rs:217-229
        const uint64_t b_start = i * blocks_per_worker;
        const uint64_t b_count = i == n_workers - 1 ? blocks_per_worker + blocks_remainder : blocks_per_worker;
        const std::vector<uint8_t> bytes = trb_distrib::encode_instructions(a.scene, start, end, b_start, b_count);
        if (!trb_distrib::write_all(m.workers[i].fd, bytes.data(), bytes.size()))
            return die("failed to send instructions to worker %s: %s", m.workers[i].name.c_str(), std::strerror(errno));
    }

    std::vector<DistributedFrame> frames(n_frames);
    std::vector<uint8_t> rgb8((size_t)w * h * 3);
    uint64_t n_written = 0;
    while (n_written < n_frames) {
        std::vector<pollfd> pfd;
        std::vector<size_t> who;
        for (size_t i = 0; i < m.workers.size(); ++i)
            if (m.workers[i].fd >= 0) { pfd.push_back(pollfd{m.workers[i].fd, POLLIN, 0}); who.push_back(i); }
        if (::poll(pfd.data(), pfd.size(), -1) < 0) {
            if (errno == EINTR) continue;
            return die("poll: %s", std::strerror(errno));
        }
        for (size_t k = 0; k < pfd.size(); ++k) {
            if (!pfd[k].revents) continue;
            WorkerConn& wc = m.workers[who[k]];
            if (wc.buf.size() < wc.expected) wc.buf.resize((size_t)wc.expected);
            const ssize_t r = ::read(wc.fd, &wc.buf[wc.got], (size_t)(wc.expected - wc.got));
            if (r < 0 && (errno == EINTR || errno == EAGAIN)) continue;
            if (r <= 0) {
                const std::string why = r < 0 ? std::strerror(errno) : "connection closed";
                if (wc.got) return die("worker %s hung up in the middle of %s (%zu of %llu bytes received): %s", wc.name.c_str(),
                                       frame_of(wc, start, n_frames).c_str(), wc.got, (unsigned long long)wc.expected, why.c_str());
                return die("worker %s hung up before %s, having sent %llu of %llu frames: %s", wc.name.c_str(), frame_of(wc, start, n_frames).c_str(),
                           (unsigned long long)wc.n_reported, (unsigned long long)n_frames, why.c_str());
            }
            wc.got += (size_t)r;
            if (wc.got < wc.expected) continue;
            if (wc.expected == 8) { // the size header (master.rs:249-262)
                std::memcpy(&wc.expected, wc.buf.data(), 8);
                if (wc.expected < trb_distrib::FRAME_HEADER_BYTES || wc.expected > max_frame_bytes)
                    return die("worker %s sent an implausible Frame size %llu for %s (a %ux%u image's Frames hold %llu to %llu bytes)", wc.name.c_str(),
                               (unsigned long long)wc.expected, frame_of(wc, start, n_frames).c_str(), w, h,
                               (unsigned long long)trb_distrib::FRAME_HEADER_BYTES, (unsigned long long)max_frame_bytes);
                continue;
            }
            trb_distrib::Frame f;
            const std::string bad = trb_distrib::decode_frame(wc.buf, f);
            const std::string what = frame_of(wc, start, n_frames);
            if (!bad.empty()) return die("worker %s, %s: %s", wc.name.c_str(), what.c_str(), bad.c_str());
            if (f.frame < start || f.frame > end)
                return die("worker %s reported %s, outside the range [%llu, %llu]", wc.name.c_str(), what.c_str(), (unsigned long long)start, (unsigned long long)end);
            const uint64_t fi = f.frame - start;
            if (wc.reported[fi]) return die("worker %s reported %s twice", wc.name.c_str(), what.c_str());
            if (f.block_w == 0 || f.block_h == 0 || f.block_w > w || f.block_h > h)
                return die("worker %s, %s: block size (%llu, %llu) does not fit the %ux%u image", wc.name.c_str(), what.c_str(),
                           (unsigned long long)f.block_w, (unsigned long long)f.block_h, w, h);
            const uint64_t n_fb = f.blocks.size() / 2, stride = f.block_w * f.block_h * 4;
            if (f.pixels.size() != n_fb * stride)
                return die("worker %s, %s: %zu pixel floats for %llu blocks of (%llu, %llu), expected %llu", wc.name.c_str(), what.c_str(), f.pixels.size(),
                           (unsigned long long)n_fb, (unsigned long long)f.block_w, (unsigned long long)f.block_h, (unsigned long long)(n_fb * stride));
            for (uint64_t b = 0; b < n_fb; ++b) {
                const uint64_t x0 = f.blocks[2 * b], y0 = f.blocks[2 * b + 1];
                if (x0 > w - f.block_w || y0 > h - f.block_h)
                    return die("worker %s, %s: block (%llu, %llu) of size (%llu, %llu) lies outside the %ux%u image", wc.name.c_str(), what.c_str(),
                               (unsigned long long)x0, (unsigned long long)y0, (unsigned long long)f.block_w, (unsigned long long)f.block_h, w, h);
            }
            DistributedFrame& df = frames[fi];
            if (df.num_reporting == 0) { df.render.assign((size_t)w * h * 4, 0.0f); df.first_tile_recv = std::chrono::steady_clock::now(); }
            for (uint64_t b = 0; b < n_fb; ++b) { // Image::add_blocks (film/image.rs:36-50)
                const float* px = &f.pixels[b * stride];
                for (uint64_t by = 0; by < f.block_h; ++by)
                    for (uint64_t bx = 0; bx < f.block_w; ++bx) {
                        float* c = &df.render[4 * ((f.blocks[2 * b + 1] + by) * w + f.blocks[2 * b] + bx)];
                        const float* p = &px[4 * (by * f.block_w + bx)];
                        for (int i = 0; i < 4; ++i) c[i] += p[i];
                    }
            }
            wc.reported[fi] = true; ++wc.n_reported;
            wc.buf.clear(); wc.got = 0; wc.expected = 8;
            if (wc.n_reported == n_frames) { ::close(wc.fd); wc.fd = -1; } // its last frame: the reference worker exits now
            if (++df.num_reporting < n_workers) continue;
            const double render_time = seconds_since(df.first_tile_recv); // master.rs:130-146
            const std::string file = out.file_for(f.frame);
            trb_host_film_to_srgb8(w, h, df.render.data(), rgb8.data());
            if (!save_image(out, file, rgb8.data(), w, h)) return 1;
            std::printf("Frame %llu: time between receiving first and last tile %.4fs\n", (unsigned long long)f.frame, render_time);
            std::printf("Frame %llu: rendered to '%s'\n--------------------\n", (unsigned long long)f.frame, file.c_str());
            std::fflush(stdout);
            std::vector<float>().swap(df.render);
            ++n_written;
        }
    }
    std::printf("Rendering entire sequence took %.4fs\n", seconds_since(scene_start));
    return 0;
}

} // namespace

int main(int argc, char** argv) {
    bool worker = false, denoise = false, denoise_temporal = false, temporal_gradients = false, denoise_moments = false,
         moment_gradients = false, adaptive = false, denoise_variance = false, denoise_variance_temporal = false, variance_gradients = false;
    for (int i = 1; i < argc; ++i) {
        worker = worker || std::strcmp(argv[i], "--worker") == 0;
        temporal_gradients = temporal_gradients || std::strcmp(argv[i], "--temporal-gradients") == 0;
        denoise = denoise || std::strcmp(argv[i], "--denoise") == 0;
        denoise_temporal = denoise_temporal || std::strcmp(argv[i], "--denoise-temporal") == 0;
        denoise_moments = denoise_moments || std::strcmp(argv[i], "--denoise-moments") == 0;
        moment_gradients = moment_gradients || std::strcmp(argv[i], "--moment-gradients") == 0;
        adaptive = adaptive || std::strcmp(argv[i], "--adaptive") == 0;
        denoise_variance = denoise_variance || std::strcmp(argv[i], "--denoise-variance") == 0;
        denoise_variance_temporal = denoise_variance_temporal || std::strcmp(argv[i], "--denoise-variance-temporal") == 0;
        variance_gradients = variance_gradients || std::strcmp(argv[i], "--variance-gradients") == 0;
    }
    if (worker && adaptive) return die("--adaptive is not available with --worker: the wire format carries no sampler");
    if (worker && denoise) return die("--denoise is not available with --worker: the wire format carries no albedo, normal or depth");
    if (worker && denoise_temporal)
        return die("--denoise-temporal is not available with --worker: the wire format carries no albedo, normal or depth");
    if (worker && temporal_gradients)
        return die("--temporal-gradients is not available with --worker: the wire format carries no albedo, normal or depth");
    if (worker && denoise_moments)
        return die("--denoise-moments is not available with --worker: the wire format carries no albedo, normal or depth");
    if (worker && moment_gradients)
        return die("--moment-gradients is not available with --worker: the wire format carries no albedo, normal or depth");
    if (worker && denoise_variance)
        return die("--denoise-variance is not available with --worker: the wire format carries no albedo, normal or depth");
    if (worker && denoise_variance_temporal)
        return die("--denoise-variance-temporal is not available with --worker: the wire format carries no albedo, normal or depth");
    if (worker && variance_gradients)
        return die("--variance-gradients is not available with --worker: the wire format carries no albedo, normal or depth");
    if (worker) return trb_distrib::worker_main(argc, argv);
    Args a;
    bool have_scene = false;
    for (int i = 1; i < argc; ++i) {
        const std::string s = argv[i];
        const char* v = i + 1 < argc ? argv[i + 1] : nullptr;
        auto number = [&](uint64_t& x, bool& has) {
            if (!parse_u64(v, x)) { die("%s needs a non-negative integer", s.c_str()); return false; }
            has = true; ++i; return true;
        };
        bool ok = true, unused = false;
        if (s == "-h" || s == "--help") { std::fputs(USAGE, stdout); return 0; }
        else if (s == "-o") { if (!v) return die("-o needs a path"); a.out = v; ++i; }
        else if (s == "-n") { uint64_t n; ok = number(n, unused); }
        else if (s == "--start-frame") ok = number(a.start, a.has_start);
        else if (s == "--end-frame") ok = number(a.end, a.has_end);
        else if (s == "--seed") ok = number(a.seed, a.has_seed) && a.seed <= UINT32_MAX;
        else if (s == "--spp") ok = number(a.spp, a.has_spp) && a.spp <= UINT32_MAX;
        else if (s == "--device") ok = number(a.device, a.has_device) && a.device <= INT32_MAX;
        else if (s == "--devices") {
            const std::string bad = trb_distrib::parse_devices(v, a.devices);
            if (!bad.empty()) return die("%s", bad.c_str());
            ++i;
        }
        else if (s == "--master") a.master = true;
        else if (s == "--denoise") a.denoise = true;
        else if (s == "--denoise-temporal") a.denoise_temporal = true;
        else if (s == "--temporal-gradients") a.temporal_gradients = true;
        else if (s == "--denoise-moments") a.denoise_moments = true;
        else if (s == "--moment-gradients") a.moment_gradients = true;
        else if (s == "--denoise-variance") a.denoise_variance = true;
        else if (s == "--denoise-variance-temporal") a.denoise_variance_temporal = true;
        else if (s == "--variance-gradients") a.variance_gradients = true;
        else if (s == "--adaptive") { // two numbers: MIN MAX
            const char* v2 = i + 2 < argc ? argv[i + 2] : nullptr;
            ok = parse_u64(v, a.ad_min) && parse_u64(v2, a.ad_max) && a.ad_min <= UINT32_MAX && a.ad_max <= UINT32_MAX;
            if (!ok) die("--adaptive needs two non-negative integers: MIN MAX");
            a.adaptive = true; i += 2;
        }
        else if (!s.empty() && s[0] == '-') { std::fputs(USAGE, stderr); return 2; }
        else if (!have_scene) { a.scene = s; have_scene = true; }
        else a.workers.push_back(s);
        if (!ok) { std::fputs(USAGE, stderr); return 2; }
    }
    if (!have_scene) { std::fputs(USAGE, stderr); return 2; }
    if (a.master && a.workers.empty()) return die("--master needs at least one worker address");
    if (!a.master && !a.workers.empty()) return die("unexpected argument '%s' (worker addresses follow --master)", a.workers[0].c_str());
    if (a.master && !a.devices.empty()) return die("--devices is a worker's option with --master: pass it to each worker");
    if (a.has_device && !a.devices.empty()) return die("--devices and --device exclude each other: list every GPU in --devices");
    if (a.master && (a.has_seed || a.has_spp || a.has_device)) return die("--seed, --spp and --device are the workers' options: pass them to each worker");
    if (a.master && a.denoise_moments)
        return die("--denoise-moments is not available with --master: the wire format carries no albedo, normal or depth");
    if (a.denoise_moments && (a.denoise || a.denoise_temporal || a.temporal_gradients))
        return die("--denoise-moments excludes --denoise, --denoise-temporal and --temporal-gradients: choose one denoiser");
    if (a.master && a.moment_gradients)
        return die("--moment-gradients is not available with --master: the wire format carries no albedo, normal or depth");
    if (a.moment_gradients && !a.denoise_moments) return die("--moment-gradients needs --denoise-moments");
    if (a.master && a.denoise) return die("--denoise is not available with --master: the wire format carries no albedo, normal or depth");
    if (a.denoise && a.has_spp && a.spp < 2) return die("--denoise needs at least 2 samples per pixel (two half renders)");
    if (a.denoise && a.denoise_temporal) return die("--denoise and --denoise-temporal exclude each other: choose one");
    if (a.master && a.denoise_temporal)
        return die("--denoise-temporal is not available with --master: the wire format carries no albedo, normal or depth");
    if (a.master && a.temporal_gradients)
        return die("--temporal-gradients is not available with --master: the wire format carries no albedo, normal or depth");
    if (a.temporal_gradients && !a.denoise_temporal) return die("--temporal-gradients needs --denoise-temporal");
    if (a.denoise_temporal && a.has_spp && a.spp < 2) return die("--denoise-temporal needs at least 2 samples per pixel (two half renders)");
    if (a.master && a.adaptive) return die("--adaptive is not available with --master: the wire format carries no sampler");
    if (a.adaptive && a.has_spp) return die("--adaptive excludes --spp: the Adaptive sampler owns the sample schedule");
    if (a.adaptive && (a.denoise || a.denoise_temporal || a.temporal_gradients))
        return die("--adaptive excludes --denoise, --denoise-temporal and --temporal-gradients: they need two half sample ranges; use --denoise-moments");
    if (a.adaptive) {
        const trb_adaptive ad{(uint32_t)a.ad_min, (uint32_t)a.ad_max};
        if (trb_adaptive_schedule(&ad, nullptr, nullptr, nullptr, nullptr) != TRB_OK) return die("--adaptive %llu %llu: %s", (unsigned long long)a.ad_min,
                                                                                                (unsigned long long)a.ad_max, trb_last_error());
    }
    if (a.master && a.variance_gradients)
        return die("--variance-gradients is not available with --master: the wire format carries no albedo, normal or depth");
    if (a.variance_gradients && !a.denoise_variance_temporal) return die("--variance-gradients needs --denoise-variance-temporal");
    if (a.denoise_variance_temporal) {
        if (a.master)
            return die("--denoise-variance-temporal is not available with --master: the wire format carries no albedo, normal or depth");
        if (!a.devices.empty()) return die("--denoise-variance-temporal renders on one GPU: use --device, not --devices");
        if (a.denoise || a.denoise_temporal || a.temporal_gradients || a.denoise_moments || a.moment_gradients || a.denoise_variance)
            return die("--denoise-variance-temporal excludes --denoise, --denoise-temporal, --temporal-gradients, --denoise-moments, "
                       "--moment-gradients and --denoise-variance: choose one denoiser");
        // --spp 0 keeps the scene's film.samples, as in every mode; single_node checks that value once the scene is read
        if (a.has_spp && a.spp == 1)
            return die("--denoise-variance-temporal needs at least 2 samples per pixel (a variance of one sample is undefined)");
        if (a.adaptive) {
            const trb_adaptive ad{(uint32_t)a.ad_min, (uint32_t)a.ad_max};
            uint32_t mn = 0;
            if (trb_adaptive_schedule(&ad, &mn, nullptr, nullptr, nullptr) == TRB_OK && mn < 2)
                return die("--denoise-variance-temporal needs --adaptive MIN of at least 2 samples per pixel; MIN rounds to %u", mn);
        }
    }
    if (a.denoise_variance) {
        if (a.master) return die("--denoise-variance is not available with --master: the wire format carries no albedo, normal or depth");
        if (!a.devices.empty()) return die("--denoise-variance renders on one GPU: use --device, not --devices");
        if (a.denoise || a.denoise_temporal || a.temporal_gradients || a.denoise_moments || a.moment_gradients)
            return die("--denoise-variance excludes --denoise, --denoise-temporal, --temporal-gradients, --denoise-moments and --moment-gradients: choose one denoiser");
        // --spp 0 keeps the scene's film.samples, as in every mode; single_node checks that value once the scene is read
        if (a.has_spp && a.spp == 1) return die("--denoise-variance needs at least 2 samples per pixel (a variance of one sample is undefined)");
        if (a.adaptive) {
            const trb_adaptive ad{(uint32_t)a.ad_min, (uint32_t)a.ad_max};
            uint32_t mn = 0;
            if (trb_adaptive_schedule(&ad, &mn, nullptr, nullptr, nullptr) == TRB_OK && mn < 2)
                return die("--denoise-variance needs --adaptive MIN of at least 2 samples per pixel; MIN rounds to %u", mn);
        }
    }
    if (a.has_start && a.has_end && a.end < a.start)
        return die("end frame %llu is before start frame %llu", (unsigned long long)a.end, (unsigned long long)a.start);
    OutPath out;
    if (!resolve_out_path(a.out, out) || !create_out_dir(out, a.out != nullptr)) return 1;
    return a.master ? master_node(a, out) : single_node(a, out);
}
