// trb_worker — a wire-compatible replacement for `tray_rust --worker` (SURVEY 8f N2) that renders on an H100 through the C ABI.
//
// It speaks the reference master's protocol unchanged, so an unmodified `tray_rust scene.json --master host...` (or
// `trb_tray scene.json --master host...`) can drive it:
//   * listens on exec::distrib::worker::PORT = 63234 (src/exec/distrib/worker.rs:16), accepts ONE connection (worker.rs:60-89);
//   * reads `Instructions` (src/exec/distrib/mod.rs:51-72);
//   * Scene::load_file(instructions.scene), then for every frame of the inclusive range: Exec::render with
//     select_blocks = (block_start, block_count) (worker.rs:37-50, main.rs:148-166) == trb_render, and sends a `Frame`
//     (mod.rs:76-100) holding RenderTarget::get_rendered_blocks (film/render_target.rs:215-241); then clears the film (main.rs:161).
//   * exits after the last frame, like the reference worker.
// The wire format and the loop are trb_distrib.hpp's, shared with trb_tray.
//
//   trb_worker [--port P] [--device D] [--seed S] [--spp N]
// No CPU fallback: without a CUDA device the scene load fails with TRB_NO_DEVICE and the worker exits non-zero.
#include "trb_distrib.hpp"

int main(int argc, char** argv) { return trb_distrib::worker_main(argc, argv); }
