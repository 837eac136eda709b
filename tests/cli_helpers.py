"""Shared by test_cli_cpu.py and test_cli_gpu.py: the exec::distrib wire format written out in Python (mod.rs:51-100), image
readers for what trb_tray writes, and child-process handling that never leaves a process behind."""
import ctypes as C
import os
import queue
import socket
import struct
import subprocess
import threading
import time
import zlib

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENES = os.path.join(REPO, "tests", "golden", "scenes")
CORNELL = os.path.join(SCENES, "c1_cornell_box.json")
C5 = os.path.join(SCENES, "c5_tr15_like.json")
LIB = os.path.join(REPO, "tray_rust_b200", "lib")
TRAY = os.path.join(LIB, "trb_tray")
WORKER = os.path.join(LIB, "trb_worker")
TIMEOUT = 120


def build_programs():
    """conftest builds libtrb.so, and build_trb returns early when it is current: build the programs here as well."""
    import __graft_entry__ as g
    g.build_trb()
    g.build_worker()
    g.build_tray()


def encode_instructions(scene, frames, block_start, block_count):
    s = scene.encode()
    body = struct.pack("<Q", len(s)) + s + struct.pack("<QQQQ", frames[0], frames[1], block_start, block_count)
    return struct.pack("<Q", 8 + len(body)) + body


def encode_frame(frame, blocks, pixels, block_size=(2, 2), encoded_size=None):
    blocks = np.asarray(blocks, np.uint64).reshape(-1, 2)
    pixels = np.asarray(pixels, np.float32).reshape(-1)
    body = struct.pack("<QQQQ", frame, block_size[0], block_size[1], len(blocks)) + blocks.astype("<u8").tobytes()
    body += struct.pack("<Q", len(pixels)) + pixels.astype("<f4").tobytes()
    return struct.pack("<Q", 8 + len(body) if encoded_size is None else encoded_size) + body


def decode_frame(buf):
    size, frame, bw, bh, nb = struct.unpack_from("<QQQQQ", buf, 0)
    o = 40
    blocks = np.frombuffer(buf, "<u8", 2 * nb, o).reshape(-1, 2); o += 16 * nb
    (npx,) = struct.unpack_from("<Q", buf, o); o += 8
    pixels = np.frombuffer(buf, "<f4", npx, o); o += 4 * npx
    assert size == len(buf) == o
    return frame, (bw, bh), blocks, pixels


def recv_exact(sock, n):
    out = b""
    while len(out) < n:
        chunk = sock.recv(n - len(out))
        if not chunk:
            break
        out += chunk
    return out


def recv_message(sock):
    """One size-prefixed bincode message (Instructions or Frame)."""
    head = recv_exact(sock, 8)
    assert len(head) == 8
    (size,) = struct.unpack("<Q", head)
    return head + recv_exact(sock, size - 8)


def read_png(path):
    raw = open(path, "rb").read()
    assert raw[:8] == b"\x89PNG\r\n\x1a\n"
    o, chunks = 8, {}
    while o < len(raw):
        (n,) = struct.unpack(">I", raw[o:o + 4])
        chunks.setdefault(raw[o + 4:o + 8], []).append(raw[o + 8:o + 8 + n])
        o += 12 + n
    w, h = struct.unpack(">II", chunks[b"IHDR"][0][:8])
    scan = np.frombuffer(zlib.decompress(b"".join(chunks[b"IDAT"])), np.uint8).reshape(h, 1 + 3 * w)
    assert (scan[:, 0] == 0).all()
    return scan[:, 1:].reshape(h, w, 3)


def read_ppm(path):
    raw = open(path, "rb").read()
    magic, dims, maxval, rest = raw.split(b"\n", 3)
    assert magic == b"P6" and maxval == b"255"
    w, h = map(int, dims.split())
    return np.frombuffer(rest, np.uint8).reshape(h, w, 3)


def special_film(rng, h, w):
    """Random RGBW plus the edges of the conversion: weight <= 0, NaN and infinities, huge values, the 0.0031308 knee."""
    film = rng.uniform(-0.2, 3.0, size=(h, w, 4)).astype(np.float32)
    flat = film.reshape(-1, 4)
    n = len(flat)
    specials = np.array([0.0, -0.0, -1.0, np.nan, np.inf, -np.inf, 3e38, 1e-40, 0.0031308, np.nextafter(np.float32(0.0031308), 1),
                         np.nextafter(np.float32(0.0031308), 0), 1.0, np.nextafter(np.float32(1), 2)], np.float32)
    pick = rng.integers(0, n, size=n // 4)
    flat[pick, rng.integers(0, 4, size=len(pick))] = specials[rng.integers(0, len(specials), size=len(pick))]
    knee = rng.integers(0, n, size=n // 8)  # colour / weight right at the knee
    flat[knee, 3] = 1.0
    flat[knee, :3] = np.float32(0.0031308) + rng.integers(-4, 5, size=(len(knee), 3)).astype(np.float32) * np.float32(2.3e-10)
    return film


def free_port():
    """A port the kernel just handed out and that is closed again: nothing listens on it."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def listener():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    s.listen(1)
    s.settimeout(TIMEOUT)
    return s


def load_desc(path, width=0, height=0, spp=0):
    """trb_desc_load_json (host only). The caller frees it with free_desc."""
    from tray_rust_b200 import _ffi as F
    lib = F.load_trb()
    d = C.POINTER(F.SceneDesc)()
    assert lib.trb_desc_load_json(path.encode(), width, height, spp, C.byref(d)) == F.TRB_OK, lib.trb_last_error()
    return d


def free_desc(d):
    from tray_rust_b200 import _ffi as F
    F.load_trb().trb_desc_free(d)


class Proc:
    """A child process whose stdout is read line by line on a thread, so a test can wait for one line with a timeout."""

    def __init__(self, args, cwd=REPO):
        self.p = subprocess.Popen(args, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        self.lines = queue.Queue()
        self.out = []
        self.t = threading.Thread(target=self._pump, daemon=True)
        self.t.start()

    def _pump(self):
        for line in self.p.stdout:
            self.out.append(line)
            self.lines.put(line)
        self.lines.put(None)

    def wait_line(self, text, timeout=TIMEOUT):
        end = time.monotonic() + timeout
        while True:
            line = self.lines.get(timeout=max(0.0, end - time.monotonic()))
            assert line is not None, "process ended before printing %r: %s" % (text, self.p.stderr.read())
            if text in line:
                return line

    def finish(self, timeout=TIMEOUT):
        """Wait for the exit; returns (returncode, stdout, stderr)."""
        err = self.p.stderr.read() if self.p.wait(timeout=timeout) is not None else ""
        self.t.join(timeout=10)
        return self.p.returncode, "".join(self.out), err

    def kill(self):
        if self.p.poll() is None:
            self.p.kill()
        try:
            self.p.wait(timeout=30)
        finally:
            for f in (self.p.stdout, self.p.stderr):
                f.close()
