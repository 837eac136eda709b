// trb_distrib.hpp — exec::distrib (src/exec/distrib/mod.rs, worker.rs) over the C ABI: the bincode wire format of the master's
// `Instructions` and the worker's `Frame`, and the worker loop (worker.rs:37-89, main.rs:148-166). trb_worker and trb_tray (in both
// --worker and --master mode) include this one header, so there is one copy of the format.
//
// bincode 0.x "Infinite" encoding: little-endian, u64 lengths, usize as u64, tuples and structs inline.
//   Instructions (mod.rs:51-72):  encoded_size u64 | scene: u64 len + utf-8 | frames (u64, u64) | block_start u64 | block_count u64
//   Frame        (mod.rs:76-100): encoded_size u64 | frame u64 | block_size (u64, u64) | blocks: u64 n + n x (u64, u64)
//                                 | pixels: u64 n + n x f32
// encoded_size is the size of the whole message, itself included; the reader reads it first, then the rest.
#pragma once
#include <arpa/inet.h>
#include <netinet/in.h>
#include <sys/socket.h>
#include <unistd.h>
#include <cctype>
#include <cerrno>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/trb.h"

namespace trb_distrib {

constexpr int PORT = 63234;               // exec::distrib::worker::PORT (worker.rs:16)
constexpr uint64_t FRAME_HEADER_BYTES = 48; // encoded_size, frame, block_size, blocks.len(), pixels.len()

inline bool read_all(int fd, void* dst, size_t n) {
    uint8_t* p = static_cast<uint8_t*>(dst);
    while (n) { const ssize_t r = ::read(fd, p, n); if (r <= 0) return false; p += r; n -= (size_t)r; }
    return true;
}
// MSG_NOSIGNAL: a peer that has gone away is a failed write, not a SIGPIPE
inline bool write_all(int fd, const void* src, size_t n) {
    const uint8_t* p = static_cast<const uint8_t*>(src);
    while (n) { const ssize_t r = ::send(fd, p, n, MSG_NOSIGNAL); if (r <= 0) return false; p += r; n -= (size_t)r; }
    return true;
}
inline uint64_t get_u64(const std::vector<uint8_t>& b, size_t& o) { uint64_t v = 0; if (o + 8 <= b.size()) std::memcpy(&v, &b[o], 8); o += 8; return v; } // x86-64: little-endian
inline void put_u64(std::vector<uint8_t>& b, uint64_t v) { const size_t o = b.size(); b.resize(o + 8); std::memcpy(&b[o], &v, 8); }

// --devices: a comma-separated list of distinct CUDA device ordinals ("0,1,2,3"). Returns an empty string, or what is wrong with it.
inline std::string parse_devices(const char* s, std::vector<int>& out) {
    out.clear();
    if (!s || !*s) return "--devices needs a comma-separated list of device ordinals, e.g. 0,1,2,3";
    const std::string bad = std::string("malformed --devices list '") + s + "': use device ordinals separated by commas, e.g. 0,1,2,3";
    for (const char* p = s;; ++p) {
        if (!std::isdigit((unsigned char)*p)) return bad;
        char* e = nullptr; errno = 0;
        const unsigned long v = std::strtoul(p, &e, 10);
        if (errno || v > 0x7fffffffu) return bad;
        for (int d : out) if (d == (int)v) return std::string("--devices lists device ") + std::to_string(v) + " twice";
        out.push_back((int)v);
        if (!*e) return "";
        if (*e != ',') return bad;
        p = e;
    }
}

struct Instructions { uint64_t encoded_size = 0; std::string scene; uint64_t frame_start = 0, frame_end = 0, block_start = 0, block_count = 0; };

// Instructions::new + bincode::serialize (mod.rs:63-72, master.rs:217-229)
inline std::vector<uint8_t> encode_instructions(const std::string& scene, uint64_t frame_start, uint64_t frame_end, uint64_t block_start, uint64_t block_count) {
    std::vector<uint8_t> out;
    put_u64(out, 8 + 8 + scene.size() + 32);
    put_u64(out, scene.size());
    out.insert(out.end(), scene.begin(), scene.end());
    put_u64(out, frame_start); put_u64(out, frame_end); put_u64(out, block_start); put_u64(out, block_count);
    return out;
}

inline bool decode_instructions(const std::vector<uint8_t>& buf, Instructions& in) {
    size_t o = 0;
    in.encoded_size = get_u64(buf, o);
    const uint64_t len = get_u64(buf, o);
    if (o + len + 32 > buf.size()) return false;
    in.scene.assign(reinterpret_cast<const char*>(&buf[o]), (size_t)len); o += (size_t)len;
    in.frame_start = get_u64(buf, o); in.frame_end = get_u64(buf, o);
    in.block_start = get_u64(buf, o); in.block_count = get_u64(buf, o);
    return o == buf.size();
}

struct Frame {
    uint64_t encoded_size = 0, frame = 0, block_w = 0, block_h = 0;
    std::vector<uint64_t> blocks; // (x, y) of each block's first pixel, interleaved
    std::vector<float> pixels;    // block_w * block_h RGBW pixels per block, row-major within the block
};

// RenderTarget::get_rendered_blocks (film/render_target.rs:215-241) + Frame::new + bincode::serialize: the 2x2 lock blocks whose
// four weights are all non-zero, row-major over the block grid, 16 floats RGBW per block.
inline std::vector<uint8_t> encode_frame(uint64_t frame, const float* film, uint32_t w, uint32_t h) {
    std::vector<uint64_t> blocks;
    std::vector<float> pixels;
    for (uint32_t by = 0; by < h / 2; ++by)
        for (uint32_t bx = 0; bx < w / 2; ++bx) {
            bool all = true;
            for (uint32_t y = 0; y < 2; ++y) for (uint32_t x = 0; x < 2; ++x) all = all && film[4 * ((size_t)(2 * by + y) * w + 2 * bx + x) + 3] != 0.0f;
            if (!all) continue;
            blocks.push_back(2 * bx); blocks.push_back(2 * by);
            for (uint32_t y = 0; y < 2; ++y) for (uint32_t x = 0; x < 2; ++x) { const float* c = &film[4 * ((size_t)(2 * by + y) * w + 2 * bx + x)]; pixels.insert(pixels.end(), c, c + 4); }
        }
    std::vector<uint8_t> out;
    const uint64_t size = FRAME_HEADER_BYTES + 8 * blocks.size() + 4 * pixels.size(); // == bincode::serialized_size(&frame)
    put_u64(out, size); put_u64(out, frame); put_u64(out, 2); put_u64(out, 2);
    put_u64(out, blocks.size() / 2);
    for (uint64_t v : blocks) put_u64(out, v);
    put_u64(out, pixels.size());
    const size_t o = out.size();
    out.resize(o + 4 * pixels.size());
    if (!pixels.empty()) std::memcpy(&out[o], pixels.data(), 4 * pixels.size());
    return out;
}

// bincode::deserialize::<Frame>. Returns an empty string, or what is wrong with the bytes. Only the encoding is checked here: whether
// the blocks fit an image is the reader's question.
inline std::string decode_frame(const std::vector<uint8_t>& buf, Frame& f) {
    if (buf.size() < FRAME_HEADER_BYTES) return "a Frame of " + std::to_string(buf.size()) + " bytes is shorter than its fixed fields";
    size_t o = 0;
    f.encoded_size = get_u64(buf, o); f.frame = get_u64(buf, o); f.block_w = get_u64(buf, o); f.block_h = get_u64(buf, o);
    const uint64_t nb = get_u64(buf, o);
    if (nb > (buf.size() - o - 8) / 16) return "the Frame lists " + std::to_string(nb) + " blocks, more than its " + std::to_string(buf.size()) + " bytes hold";
    f.blocks.resize(2 * (size_t)nb);
    if (nb) std::memcpy(f.blocks.data(), &buf[o], 16 * (size_t)nb);
    o += 16 * (size_t)nb;
    const uint64_t np = get_u64(buf, o);
    if (np != (buf.size() - o) / 4 || (buf.size() - o) % 4)
        return "the Frame's " + std::to_string(np) + " pixel floats do not fill the " + std::to_string(buf.size() - o) + " bytes after its block list";
    f.pixels.resize((size_t)np);
    if (np) std::memcpy(f.pixels.data(), &buf[o], 4 * (size_t)np);
    if (f.encoded_size != buf.size()) return "the Frame's encoded_size " + std::to_string(f.encoded_size) + " is not its length " + std::to_string(buf.size());
    return "";
}

// `tray_rust --worker` (main.rs:148-166, worker.rs:37-89): listens on `port`, accepts ONE connection, reads the Instructions,
// Scene::load_file(instructions.scene), then for every frame of the inclusive range renders blocks
// [block_start, block_start + block_count) of the Morton list (trb_render: Exec::render with select_blocks, including
// update_frame), sends the Frame and clears the film. Exits after the last frame. With --devices the blocks are rendered by a
// trb_group of those GPUs (trb_group_render: the range sharded over them, one film reduce); the Frames are the same message.
//   [--worker] [-n N] [--port P] [--device D | --devices D0,D1,...] [--seed S] [--spp N]
// No CPU fallback: without a CUDA device the scene load fails with TRB_NO_DEVICE and the worker exits with status 3.
inline int worker_main(int argc, char** argv) {
    int port = PORT, device = 0;
    uint32_t seed = 1, spp = 0;
    bool has_device = false;
    std::vector<int> devices;
    for (int i = 1; i < argc; ++i) {
        const std::string a = argv[i];
        if (a == "--port" && i + 1 < argc) port = std::atoi(argv[++i]);
        else if (a == "--device" && i + 1 < argc) { device = std::atoi(argv[++i]); has_device = true; }
        else if (a == "--devices") {
            const std::string bad = parse_devices(i + 1 < argc ? argv[i + 1] : nullptr, devices);
            if (!bad.empty()) { std::fprintf(stderr, "%s\n", bad.c_str()); return 2; }
            ++i;
        }
        else if (a == "--seed" && i + 1 < argc) seed = (uint32_t)std::strtoul(argv[++i], nullptr, 0);
        else if (a == "--spp" && i + 1 < argc) spp = (uint32_t)std::strtoul(argv[++i], nullptr, 0);
        else if (a == "--worker" || a == "-n") { if (a == "-n") ++i; } // accepted for command-line compatibility with `tray_rust --worker [-n threads]`
        else { std::fprintf(stderr, "usage: %s [--worker] [--port P] [--device D | --devices D0,D1,...] [--seed S] [--spp N]\n", argv[0]); return 2; }
    }
    if (has_device && !devices.empty()) { std::fprintf(stderr, "--devices and --device exclude each other: list every GPU in --devices\n"); return 2; }
    const int lfd = ::socket(AF_INET, SOCK_STREAM, 0);
    int one = 1;
    ::setsockopt(lfd, SOL_SOCKET, SO_REUSEADDR, &one, sizeof one);
    sockaddr_in addr{};
    addr.sin_family = AF_INET; addr.sin_addr.s_addr = htonl(INADDR_ANY); addr.sin_port = htons((uint16_t)port);
    if (lfd < 0 || ::bind(lfd, reinterpret_cast<sockaddr*>(&addr), sizeof addr) != 0 || ::listen(lfd, 1) != 0) { std::perror("Worker failed to get port"); return 1; }
    std::printf("Worker listening for master on %d\n", port); std::fflush(stdout);
    const int fd = ::accept(lfd, nullptr, nullptr);
    if (fd < 0) { std::perror("Error accepting"); return 1; }
    std::vector<uint8_t> buf(8);
    if (!read_all(fd, buf.data(), 8)) { std::fprintf(stderr, "Failed to read from master\n"); return 1; }
    uint64_t expected = 0; std::memcpy(&expected, buf.data(), 8);
    if (expected < 48 || expected > (1u << 20)) { std::fprintf(stderr, "implausible instruction size %llu\n", (unsigned long long)expected); return 1; }
    buf.resize((size_t)expected);
    if (!read_all(fd, buf.data() + 8, (size_t)expected - 8)) { std::fprintf(stderr, "Failed to read from master\n"); return 1; }
    Instructions in;
    if (!decode_instructions(buf, in)) { std::fprintf(stderr, "malformed instructions\n"); return 1; }
    std::printf("Received instructions: Instructions { encoded_size: %llu, scene: \"%s\", frames: (%llu, %llu), block_start: %llu, block_count: %llu }\n",
                (unsigned long long)in.encoded_size, in.scene.c_str(), (unsigned long long)in.frame_start, (unsigned long long)in.frame_end,
                (unsigned long long)in.block_start, (unsigned long long)in.block_count);
    trb_scene* scene = nullptr;
    trb_group* group = nullptr;
    trb_status rc = devices.empty() ? trb_scene_load_json(in.scene.c_str(), 0, 0, spp, device, &scene) // Scene::load_file(&instructions.scene) (worker.rs:39)
                                    : trb_group_load_json(in.scene.c_str(), 0, 0, spp, devices.data(), (int)devices.size(), &group);
    if (rc != TRB_OK) {
        std::fprintf(stderr, "%s status %d: %s\n", devices.empty() ? "trb_scene_load_json" : "trb_group_load_json", (int)rc, trb_last_error());
        return rc == TRB_NO_DEVICE ? 3 : 1;
    }
    if (group) scene = trb_group_scene(group, 0);
    uint32_t w = 0, h = 0;
    trb_scene_info(scene, &w, &h, nullptr, nullptr, nullptr, nullptr);
    std::vector<float> film((size_t)w * h * 4);
    for (uint64_t frame = in.frame_start; frame <= in.frame_end; ++frame) { // main.rs:157-163
        std::fill(film.begin(), film.end(), 0.0f);                            // render_target.clear()
        trb_render_cfg cfg{};
        cfg.block_start = (uint32_t)in.block_start; cfg.block_count = (uint32_t)in.block_count; cfg.current_frame = (uint32_t)frame; cfg.seed = seed;
        trb_stats st{};
        rc = group ? trb_group_render(group, &cfg, film.data(), &st) : trb_render(scene, &cfg, film.data(), &st);
        if (rc != TRB_OK) { std::fprintf(stderr, "%s status %d: %s\n", group ? "trb_group_render" : "trb_render", (int)rc, trb_last_error()); return 1; }
        const std::vector<uint8_t> bytes = encode_frame(frame, film.data(), w, h);
        if (!write_all(fd, bytes.data(), bytes.size())) { std::fprintf(stderr, "Failed to send frame to the master\n"); return 1; }
        std::printf("Frame %llu: rendering took %.4fs\n--------------------\n", (unsigned long long)frame, st.kernel_ms * 1e-3);
        std::fflush(stdout);
    }
    if (group) trb_group_destroy(group);
    else trb_scene_destroy(scene);
    ::close(fd); ::close(lfd);
    return 0;
}

} // namespace trb_distrib
