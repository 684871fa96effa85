"""Small run of every model and entry point for compute-sanitizer (memcheck / racecheck):
compute-sanitizer --tool memcheck python tools/sanitizer_workload.py"""
import os, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "ais-catcher_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import aisgpu, aissynth
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mode_x_util
import __graft_entry__ as g

g.smoke()
fs, N, B = 1536000, 16384, 3
xs = np.stack([aissynth.random_stream(fs, N * 4, 300 + s)[0] for s in range(B)])
for model in (aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2):
    for taps in (False, True):  # without taps the back end runs over two streams
        eng = aisgpu.Engine(model=model, sample_rate=fs, n_streams=B, max_chunk=N, taps=taps)
        n = 0
        for c in range(4):
            eng.submit(np.ascontiguousarray(xs[:, c * N:(c + 1) * N]), N)
        n += len(eng.poll())
        eng.close()
        print("model", model, "taps", taps, "messages", n)
for fmt, nodd in ((aisgpu.FMT_CF32, 64 * 257), (aisgpu.FMT_CU8, 64 * 131)):  # block lengths with no power-of-two lane split: uneven sub-segments, spare lanes
    xo = np.stack([aissynth.random_stream(fs, nodd * 3, 350 + s)[0] for s in range(5)])
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, fmt=fmt, n_streams=5, max_chunk=nodd)
    for c in range(3):
        blk = np.ascontiguousarray(xo[:, c * nodd:(c + 1) * nodd])
        eng.submit(np.stack([aissynth.to_cu8(r) for r in blk]) if fmt == aisgpu.FMT_CU8 else blk, nodd)
    print("odd block", nodd, "fmt", fmt, "messages", len(eng.poll()))
    eng.close()
import edge_signals  # silence, exact-zero gaps and clipped traffic beside ordinary rows, CF32 and CU8
for model in (aisgpu.MODEL_STANDARD, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_V2):
    for fmt in (aisgpu.FMT_CF32, aisgpu.FMT_CU8):
        rows = [edge_signals.make(k, fs, N * 4, 800 + i, fmt, submit=N, granule=64)[0] for i, k in enumerate(("silence", "gaps", "clipped"))]
        rows.insert(1, mode_x_util.to_raw(xs[0], fmt)[0])
        rows.insert(3, mode_x_util.to_raw(xs[1], fmt)[0])
        per = 1 if fmt == aisgpu.FMT_CF32 else 2
        eng = aisgpu.Engine(model=model, sample_rate=fs, fmt=fmt, n_streams=5, max_chunk=N)
        for c in range(4):
            eng.submit(np.stack([r[c * N * per:(c + 1) * N * per] for r in rows]), N)
        print("edge rows model", model, "fmt", fmt, "messages", len(eng.poll()))
        eng.close()
eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=6000000, n_streams=2, max_chunk=32768)  # resampler pre-stage
x6 = np.stack([aissynth.random_stream(6000000, 32768 * 3, 400 + s)[0] for s in range(2)])
for c in range(3):
    eng.submit(np.ascontiguousarray(x6[:, c * 32768:(c + 1) * 32768]), 32768)
print("6 MSPS messages", len(eng.poll()))
eng.close()
for fs_x, fmt, model in ((192000, aisgpu.FMT_CS16, aisgpu.MODEL_CHALLENGER), (12000, aisgpu.FMT_CF32, aisgpu.MODEL_DEFAULT)):  # single-channel mode, odd batch
    nx = 64 * 37
    xx = [mode_x_util.x_stream(fs_x, nx * 3, 500 + s)[0] for s in range(3)]
    eng = aisgpu.Engine(model=model, sample_rate=fs_x, fmt=fmt, n_streams=3, max_chunk=nx, channel_mode=aisgpu.MODE_X)
    for c in range(3):
        blk = [x[c * nx:(c + 1) * nx] for x in xx]
        if fmt == aisgpu.FMT_CS16:
            blk = [np.clip(np.round(np.stack([b.real, b.imag], 1).ravel() * 32767.0), -32768, 32767).astype(np.int16) for b in blk]
        eng.submit(np.stack(blk), nx)
    print("X mode", fs_x, "messages", len(eng.poll()))
    eng.close()
import disc_util
for fs_d, fmt in ((48000, aisgpu.FMT_CS16), (44100, aisgpu.FMT_CF32)):  # FM-discriminator input (-m 3); 44100 through the Upsample pre-stage
    nd = 64 * 69
    xd = [disc_util.stream_input(fs_d, nd * 3, 600 + s, fmt)[0] for s in range(3)]
    eng = aisgpu.Engine(model=aisgpu.MODEL_DISCRIMINATOR, sample_rate=fs_d, fmt=fmt, n_streams=3, max_chunk=nd)
    per = 1 if fmt == aisgpu.FMT_CF32 else 2
    for c in range(3):
        eng.submit(np.stack([x[c * nd * per:(c + 1) * nd * per] for x in xd]), nd)
    print("-m 3", fs_d, "messages", len(eng.poll()))
    eng.close()
sched = [320, 1536, 1472, 16384 + 64, 64, 16384 - 64, 64 * 1017]  # one engine, the submit length changing (tiled <-> streaming)
xv = np.stack([aissynth.random_stream(fs, sum(sched), 700 + s)[0] for s in range(B)])
eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=max(sched))
o = 0
for n in sched:
    eng.submit(np.ascontiguousarray(xv[:, o:o + n]), n)
    o += n
print("length schedule messages", len(eng.poll()))
eng.close()
import torch  # CU8 device batch with padded rows (N + 2, N + 6: not a multiple of 8 bytes) and a base 2 samples in
cu = np.stack([aissynth.to_cu8(x) for x in xs])
eng = aisgpu.Engine(model=aisgpu.MODEL_STANDARD, sample_rate=fs, fmt=aisgpu.FMT_CU8, n_streams=B, max_chunk=N, host_staging=False)
for c, (stride, off) in enumerate(((N + 2, 0), (N + 6, 4), (N + 2, 4), (N + 6, 0))):
    host = np.zeros(off + B * stride * 2, np.uint8)
    for s in range(B):
        host[off + s * stride * 2:off + s * stride * 2 + N * 2] = cu[s, c * N * 2:(c + 1) * N * 2]
    dev = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    eng.submit_device(dev.data_ptr() + off, stride, N)
    eng.sync()
    del dev
print("padded-stride CU8 device batch messages", len(eng.poll()))
eng.close()
with tempfile.TemporaryDirectory() as d:  # file feeder, CU8, ragged lengths, FP_DS integer front end
    paths = []
    for s in range(2):
        p = os.path.join(d, "r%d.cu8" % s)
        aissynth.to_cu8(xs[s][:N * 3 - 100 * s]).tofile(p)
        paths.append(p)
    eng = aisgpu.Engine(model=aisgpu.MODEL_STANDARD, sample_rate=fs, fmt=aisgpu.FMT_CU8, n_streams=2, max_chunk=N, fp_ds=True)
    msgs, nb = eng.feed_files(paths, N)
    print("feeder blocks", nb, "messages", len(msgs))
    eng.close()
eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=N)  # engine group: one front end, three back ends
mem = [eng.attach(model=aisgpu.MODEL_STANDARD), eng.attach(model=aisgpu.MODEL_V2)]
for c in range(3):
    eng.submit(np.stack([x[c * N:(c + 1) * N] for x in xs]), N)
    if c == 1:
        mem.pop(0).close()  # a member destroyed mid-run
print("group messages", len(eng.poll()), len(mem[0].poll()))
mem[0].close()
eng.close()
print("sanitizer workload done")
