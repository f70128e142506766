"""The on-disk cache of decoded images (``data_pipeline.DecodedCache``, ``load_pairs(cache=)``,
``load_inputs(cache=)``, ``--decoded_cache``), without a GPU: the maps equal ``decode_image`` bit for
bit for every pixel format and channel layout; a warm open decodes nothing and takes no process
memory, where the in-memory load takes the dataset's size; every invalid entry is rebuilt, alone;
read-only caches; two processes building one cache; two gloo ranks splitting the decoding; the
CLI flag and the pipelines' keyword."""
import mmap
import os
import shutil
import socket
import struct
import warnings
import zlib

import cv2
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from hdrnet_b200 import data_pipeline as dp
from hdrnet_b200.checkpoint import crc32c
from hdrnet_b200.bin import train

DC = dp.DecodedCache


def _png_grey_alpha(path, grey, alpha):
    """An 8-bit grey + alpha PNG (colour type 4), which cv2.imwrite cannot write."""
    H, W = grey.shape
    rows = b"".join(b"\0" + np.stack([grey, alpha], axis=2)[y].tobytes() for y in range(H))

    def chunk(kind, data):
        return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data))

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 4, 0, 0, 0))
                + chunk(b"IDAT", zlib.compress(rows)) + chunk(b"IEND", b""))


def _sources(root):
    """One file per pixel format and channel layout, of odd and non-square sizes."""
    rng = np.random.RandomState(0)
    os.makedirs(root, exist_ok=True)
    files = {
        "rgb_u8.png": rng.randint(0, 256, (37, 53, 3)).astype(np.uint8),
        "rgb_u16.png": rng.randint(0, 65536, (29, 41, 3)).astype(np.uint16),
        "grey_u8.png": rng.randint(0, 256, (31, 17)).astype(np.uint8),
        "grey_u16.png": rng.randint(0, 65536, (19, 23)).astype(np.uint16),
        "rgba_u8.png": rng.randint(0, 256, (21, 33, 4)).astype(np.uint8),
        "rgba_u16.png": rng.randint(0, 65536, (25, 13, 4)).astype(np.uint16),
        "rgb_f32.tiff": rng.rand(27, 39, 3).astype(np.float32),
        "grey_f32.tiff": rng.rand(15, 43).astype(np.float32),
    }
    paths = []
    for name, im in files.items():
        assert cv2.imwrite(os.path.join(root, name), im)
        paths.append(os.path.join(root, name))
    ga = os.path.join(root, "grey_alpha_u8.png")
    _png_grey_alpha(ga, rng.randint(0, 256, (23, 35)).astype(np.uint8), rng.randint(0, 256, (23, 35)).astype(np.uint8))
    paths.append(ga)
    return paths


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.asarray(a).tobytes() == np.asarray(b).tobytes()


def test_maps_equal_decode_image_bit_for_bit(tmp_path):
    paths = _sources(str(tmp_path / "src"))
    cache = DC(tmp_path / "cache")
    maps = cache.open(paths, nthreads=3)
    assert cache.built == len(paths) and cache.valid == 0
    assert {m.dtype for m in maps} == {np.dtype(np.uint8), np.dtype(np.uint16), np.dtype(np.float32)}
    for p, m in zip(paths, maps):
        want = dp.decode_image(p)
        assert isinstance(m, np.memmap) and _same(m, want), p
        assert m.offset == DC.HEADER_BYTES and m.offset % mmap.PAGESIZE == 0
        assert os.path.samefile(m.filename, cache.entry_path(p))
        assert os.path.getsize(cache.entry_path(p)) == DC.HEADER_BYTES + want.nbytes
    assert cache.nbytes == sum(m.nbytes for m in maps)
    # the entry name: 32 hex digits of the absolute path's SHA-256, the same for a relative path
    name = os.path.basename(cache.entry_path(paths[0]))
    assert len(name) == 35 and name.endswith(".px") and int(name[:32], 16) >= 0
    rel = os.path.relpath(paths[0])
    assert cache.entry_path(rel) == cache.entry_path(paths[0])
    # the maps are writable to numpy and torch (copy-on-write), so torch does not warn; nothing is written
    before = open(cache.entry_path(paths[0]), "rb").read()
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        t = torch.from_numpy(maps[0].reshape(-1).view(np.uint8))
        assert t.numel() == maps[0].nbytes
        maps[0][0, 0, 0] ^= 1
    del t, maps
    assert open(cache.entry_path(paths[0]), "rb").read() == before
    # duplicates in the list share one entry
    again = DC(tmp_path / "cache").open([paths[1], paths[1]])
    assert _same(again[0], again[1])


def _dataset(root, n=6, H=600, W=800):
    """n pairs: uint16 inputs, uint8 targets, PNGs without compression."""
    rng = np.random.RandomState(1)
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    names = []
    for i in range(n):
        name = f"im{i}.png"
        assert cv2.imwrite(str(root / "input" / name), rng.randint(0, 65536, (H + i, W, 3)).astype(np.uint16),
                           [cv2.IMWRITE_PNG_COMPRESSION, 0])
        assert cv2.imwrite(str(root / "output" / name), rng.randint(0, 256, (H + i, W, 3)).astype(np.uint8),
                           [cv2.IMWRITE_PNG_COMPRESSION, 0])
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


def rss_anon():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("RssAnon:"):
                return int(line.split()[1]) * 1024
    return None                              # not reported by this kernel


def _fail(*args, **kwargs):
    raise AssertionError("decoded although every entry is valid")


def _load_in_fresh_process(data, cache, q):
    """Load ``data`` (through ``cache`` when given, with decoding patched to fail) in a process of
    its own, whose heap holds no memory freed earlier; report the RssAnon it grew by."""
    if cache is not None:
        dp.decode_image = _fail
        cv2.imread = _fail
        cache = DC(cache)
    before = rss_anon()
    names, ins, outs, _ = dp.load_pairs(data, 2, cache=cache)
    dp.check_pairs(names, ins, outs, data, (512, 512), rotate=True)
    grown = None if before is None else rss_anon() - before
    q.put((grown, [a.shape[:2] for a in ins], [bytes(np.asarray(a)) for a in ins + outs],
           None if cache is None else (cache.valid, cache.built, cache.nbytes)))


def _fresh(data, cache):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_load_in_fresh_process, args=(data, cache, q))
    p.start()
    try:
        return q.get(timeout=120)
    finally:
        p.join(timeout=60)


def test_warm_open_decodes_nothing_and_takes_no_process_memory(tmp_path):
    if rss_anon() is None:
        pytest.skip("this kernel does not report RssAnon in /proc/self/status")
    data = _dataset(tmp_path / "data")
    cold = DC(tmp_path / "cache")
    names, ins, outs, _ = dp.load_pairs(str(data), 2, cache=cold)
    want = [bytes(np.asarray(a)) for a in ins + outs]
    decoded = sum(a.nbytes for a in ins + outs)
    assert cold.built == 2 * len(names) and cold.valid == 0
    del ins, outs

    grown, sizes, got, counts = _fresh(str(data / "filelist.txt"), str(tmp_path / "cache"))
    assert counts == (2 * len(names), 0, decoded)
    assert grown < 4 << 20, f"a warm open grew RssAnon by {grown} bytes"
    assert sizes == [(600 + i, 800) for i in range(6)]
    assert got == want
    grown_ram, _, got, _ = _fresh(str(data), None)
    assert grown_ram >= decoded, f"the in-memory load grew RssAnon by {grown_ram} < {decoded} bytes"
    assert got == want
    print(f"MEASURE RssAnon growth for a {decoded}-byte dataset: warm open {grown}, in memory {grown_ram}")


def _stamp(path):
    st = os.stat(path)
    return st.st_ino, st.st_mtime_ns


def _rewrite_header(entry, **fields):
    """Rewrite ``entry``'s header with ``fields`` changed and a CRC that matches them."""
    with open(entry, "r+b") as f:
        head = f.read(DC.HEADER_BYTES)
        keys = ("magic", "version", "fmt", "H", "W", "size", "mtime_ns", "n")
        vals = dict(zip(keys, DC._HEAD.unpack_from(head)))
        path = head[DC._HEAD.size:DC._HEAD.size + vals["n"]]
        vals.update(fields)
        body = DC._HEAD.pack(*(vals[k] for k in keys)) + path
        f.seek(0)
        f.write(body + struct.pack("<I", crc32c(body)))


def _flip(entry, offset):
    with open(entry, "r+b") as f:
        f.seek(offset)
        b = f.read(1)
        f.seek(offset)
        f.write(bytes([b[0] ^ 0x10]))


def _damage(kind, cache, paths, i):
    entry = cache.entry_path(paths[i])
    src = paths[i]
    if kind == "truncated":
        os.truncate(entry, os.path.getsize(entry) - 1)
    elif kind == "longer":
        with open(entry, "ab") as f:
            f.write(b"\0")
    elif kind == "header byte":
        _flip(entry, 21)                     # inside H
    elif kind == "magic":
        _flip(entry, 0)
    elif kind == "crc":
        n = DC._HEAD.unpack_from(open(entry, "rb").read(DC._HEAD.size))[-1]
        _flip(entry, DC._HEAD.size + n)
    elif kind == "padding":
        _flip(entry, DC.HEADER_BYTES - 1)
    elif kind == "future version":
        _rewrite_header(entry, version=DC.VERSION + 1)
    elif kind == "touched source":
        st = os.stat(src)
        os.utime(src, ns=(st.st_atime_ns, st.st_mtime_ns + 1_000_000))
    elif kind == "source size":
        st = os.stat(src)
        with open(src, "ab") as f:
            f.write(b"\0")                   # cv2 ignores bytes after IEND; the mtime is put back
        os.utime(src, ns=(st.st_atime_ns, st.st_mtime_ns))
        assert os.stat(src).st_size == st.st_size + 1
    elif kind == "another path":
        shutil.copyfile(cache.entry_path(paths[i + 1]), entry)
    elif kind == "removed":
        os.unlink(entry)
    else:
        raise AssertionError(kind)


DAMAGE = ["truncated", "longer", "header byte", "magic", "crc", "padding", "future version", "touched source",
          "source size", "another path", "removed"]


@pytest.mark.parametrize("kind", DAMAGE)
def test_an_invalid_entry_is_rebuilt_alone(tmp_path, kind):
    paths = _sources(str(tmp_path / "src"))
    DC(tmp_path / "cache").open(paths)
    cache = DC(tmp_path / "cache")
    i = 2
    _damage(kind, cache, paths, i)
    assert cache.entry(paths[i]) is None
    stamps = {p: _stamp(cache.entry_path(p)) for p in paths if p != paths[i]}
    maps = cache.open(paths, nthreads=2)
    assert cache.built == 1 and cache.valid == len(paths) - 1
    assert cache.entry(paths[i]) is not None
    for p, m in zip(paths, maps):
        assert _same(m, dp.decode_image(p)), p
    assert {p: _stamp(cache.entry_path(p)) for p in stamps} == stamps
    assert not [f for f in os.listdir(tmp_path / "cache") if not f.endswith(".px")]


def test_leftover_temporary_files_are_not_entries(tmp_path):
    paths = _sources(str(tmp_path / "src"))[:2]
    cache = DC(tmp_path / "cache")
    os.makedirs(cache.directory)
    entry = cache.entry_path(paths[0])
    with open(os.path.join(cache.directory, f".{os.path.basename(entry)}.1.2.tmp"), "wb") as f:
        f.write(b"partial")
    cache.open(paths)
    assert cache.built == 2 and _same(np.memmap(entry, mode="r", dtype=np.uint8, offset=DC.HEADER_BYTES,
                                                shape=(37, 53, 3)), dp.decode_image(paths[0]))


@pytest.mark.skipif(os.geteuid() == 0, reason="root may write to a read-only directory")
def test_read_only_cache(tmp_path):
    paths = _sources(str(tmp_path / "src"))
    d = tmp_path / "cache"
    DC(d).open(paths)
    os.chmod(d, 0o555)
    try:
        cache = DC(d)
        maps = cache.open(paths)
        assert cache.valid == len(paths) and cache.built == 0
        assert all(_same(m, dp.decode_image(p)) for p, m in zip(paths, maps))
        os.chmod(d, 0o755)
        os.unlink(cache.entry_path(paths[3]))
        os.chmod(d, 0o555)
        with pytest.raises(PermissionError, match=str(d)):
            DC(d).open(paths)
    finally:
        os.chmod(d, 0o755)


def _builder(root, paths, go, q):
    go.wait(60)
    maps = DC(root).open(paths, nthreads=2)
    q.put([bytes(np.asarray(m)) for m in maps])


def test_two_processes_build_one_cache_at_once(tmp_path):
    paths = _sources(str(tmp_path / "src"))
    ctx = mp.get_context("spawn")
    q, go = ctx.Queue(), ctx.Event()
    procs = [ctx.Process(target=_builder, args=(str(tmp_path / "cache"), paths, go, q)) for _ in range(2)]
    for p in procs:
        p.start()
    go.set()
    try:
        got = [q.get(timeout=120) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=60)
    assert all(p.exitcode == 0 for p in procs)
    want = [bytes(dp.decode_image(p)) for p in paths]
    assert got[0] == want and got[1] == want
    assert sorted(os.listdir(tmp_path / "cache")) == sorted(os.path.basename(DC(tmp_path / "cache").entry_path(p))
                                                           for p in paths)
    cache = DC(tmp_path / "cache")
    assert all(cache.entry(p) is not None for p in paths)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank(rank, world, port, train_dir, eval_dir, cache_dir, q):
    from hdrnet_b200 import parallel
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    parallel.init_distributed("gloo")
    try:
        decoded = []
        real = dp.decode_image

        def counting(path):
            decoded.append(os.path.relpath(path, os.path.dirname(train_dir)))
            return real(path)

        dp.decode_image = counting
        names, ins, outs, _ = dp.load_pairs(train_dir, 2, cache=cache_dir)
        train_decoded = list(decoded)
        _, evals, _ = dp.load_inputs(eval_dir, 1, cache=cache_dir)
        again = dp.load_pairs(train_dir, 2, cache=cache_dir)        # warm: nothing more
        q.put((rank, train_decoded, decoded[len(train_decoded):],
               [bytes(np.asarray(a)) for a in ins + outs + evals + again[1] + again[2]]))
    finally:
        parallel.finalize()


def test_two_gloo_ranks_split_the_decoding(tmp_path):
    data = _dataset(tmp_path / "train", n=5, H=40, W=56)
    ev = _dataset(tmp_path / "eval", n=3, H=48, W=52)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank, args=(r, 2, port, str(data), str(ev), str(tmp_path / "cache"), q))
             for r in range(2)]
    for p in procs:
        p.start()
    try:
        results = sorted((q.get(timeout=180) for _ in procs), key=lambda r: r[0])
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join(timeout=10)
    assert all(p.exitcode == 0 for p in procs)
    (_, t0, e0, a0), (_, t1, e1, a1) = results
    # the 10 training files in file-list order (input, output per name), alternately per rank
    order = [f"train/{sub}/im{i}.png" for i in range(5) for sub in ("input", "output")]
    assert sorted(t0) == sorted(order[0::2]) and sorted(t1) == sorted(order[1::2])
    # the eval set's 3 inputs, decoded once over the ranks; the warm reopen decodes nothing
    assert sorted(e0 + e1) == [f"eval/input/im{i}.png" for i in range(3)] and len(e0) == 2 and len(e1) == 1
    assert a0 == a1
    _, ins, outs, _ = dp.load_pairs(str(data))
    _, evals, _ = dp.load_inputs(str(ev))
    assert a0 == [bytes(a) for a in ins + outs + evals + ins + outs]


# ---- the CLI flag and the pipelines' keyword -------------------------------------------------------
def test_flag_parses_and_is_not_a_model_parameter():
    parser = train.build_parser()
    args = parser.parse_args(["ckpt", "data"])
    assert args.decoded_cache is None
    args = parser.parse_args(["ckpt", "data", "--decoded_cache", "/some/dir"])
    assert args.decoded_cache == "/some/dir"
    params = train.model_params(parser, args)
    assert "decoded_cache" not in params and "/some/dir" not in str(params)
    group = [g for g in parser._action_groups if g.title == "data pipeline"][0]
    assert "decoded_cache" in [a.dest for a in group._group_actions]


class _Loaded(Exception):
    pass


@pytest.mark.parametrize("pipeline", ["ImageFilesDataPipeline", "UnsharpMaskDataPipeline"])
def test_pipelines_pass_the_cache_to_the_loader(monkeypatch, tmp_path, pipeline):
    calls = []

    def loader(*args, **kwargs):
        calls.append((args, kwargs))
        raise _Loaded

    monkeypatch.setattr(dp, "load_inputs" if pipeline == "UnsharpMaskDataPipeline" else "load_pairs", loader)
    kw = {"blur_sigma": 2.0, "sharpen": 1.0} if pipeline == "UnsharpMaskDataPipeline" else {}
    cls = getattr(dp, pipeline)
    with pytest.raises(_Loaded):
        cls("data", batch_size=2, nthreads=3, **kw)
    with pytest.raises(_Loaded):
        cls("data", batch_size=2, nthreads=3, decoded_cache=str(tmp_path / "c"), **kw)
    (a0, k0), (a1, k1) = calls
    assert a0 == ("data", 3) and k0 == {}                    # without the keyword: today's call
    assert a1 == ("data", 3) and isinstance(k1["cache"], dp.DecodedCache)
    assert k1["cache"].directory == str(tmp_path / "c")
