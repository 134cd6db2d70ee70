"""Where the time of one tile of the BN = 256 tensor-core GEMM goes: per-tile timestamps from a traced build.

Compiles the GEMM unit cn_gemm_tc.cu (with cn_host_util.cpp, the error plumbing it links against) with -DCN_GEMM_TRACE
(the repository's nvcc flags otherwise) into a separate library in a temporary directory; the default build has no
trace code.  In the traced build consumer warp 0 of every CTA records, for each tile, %globaltimer at the tile start,
at the first pass of a full barrier (operands landed), at the end of the main loop and at the end of the epilogue (the moment it handed the tile's last output box to TMA), counts its failed
polls of the full barriers, and counts the waits for a staging buffer whose previous box TMA had not yet read
(cn_gemm_tc.cuh, TC_TRACE_REC).

The three per-human GEMMs run through cn_internal_gemm_tc_ex at the shapes of tools/policy_stage_times.py (N = 4096,
H = 20, the same detected-human draw, so Mc = 17 119 rows at seed 0), with their rollout epilogues: embed2 ReLU into a
split fp16 output, qkv no activation into fp32, outproj ReLU into fp32.  Printed per GEMM: the median over tiles and
calls of the first wait, the main loop, the epilogue and the whole tile (microseconds), the median failed polls per
tile, the mean per tile of the staging-buffer waits that blocked and of the SM clock cycles (thousands) spent in all
staging waits, and the median kernel span (first tile start to last epilogue end).

    python tools/gemm_tile_trace.py [--lib traced.so] [--build-only --out traced.so] [--reps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

CSRC = os.path.join(REPO, "crowdnav_prediction_attngraph_b200", "csrc")
CAP = 16            # tile records per CTA (the busiest CTA runs 7 qkv tiles at Mc = 17 119)
REC = 7             # fields per record (TC_TRACE_REC)
# (name, K, N, act, output) of the per-human GEMMs as the rollout launches them
GEMMS = [("embed2", 128, 512, 1, "f16"), ("qkv", 512, 1536, 0, "f32"), ("outproj", 512, 256, 1, "f32")]


def build(out):
    from __graft_entry__ import ARCH, COMMON
    cmd = (["nvcc"] + ARCH + COMMON + ["-DCN_GEMM_TRACE", "-shared", "-o", out,
                                        os.path.join(CSRC, "cn_gemm_tc.cu"), os.path.join(CSRC, "cn_host_util.cpp")])
    subprocess.check_call(cmd)
    return out


def rollout_rows(envs, humans, seed):
    """compacted rows of tools/policy_stage_times.py: Binomial(H, 0.21) detected humans per environment, at least 1"""
    import torch
    g = torch.Generator().manual_seed(seed)
    return int((torch.rand(envs, humans, generator=g) < 0.21).sum(1).clamp_min(1).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="a traced library built earlier (default: build one now)")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--out", default=None, help="with --build-only: where to write the traced library")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--humans", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if a.build_only:
        if not a.out:
            raise SystemExit("--build-only needs --out")
        print("built", build(a.out))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gemm_tile_trace.py needs a CUDA device")
    tmp = None
    path = a.lib
    if path is None:
        tmp = tempfile.TemporaryDirectory()
        path = build(os.path.join(tmp.name, "libcn_gemm_trace.so"))
    lib = C.CDLL(os.path.abspath(path))
    lib.cn_last_error.restype = C.c_char_p
    lib.cn_internal_gemm_trace.argtypes = [C.c_void_p, C.c_int]
    lib.cn_internal_gemm_tc_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_int, C.c_int, C.c_int]
    M = rollout_rows(a.envs, a.humans, a.seed)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dev = torch.device("cuda:0")
    trace = torch.zeros(sms * CAP * REC, dtype=torch.int64, device=dev)
    lib.cn_internal_gemm_trace(trace.data_ptr(), CAP)
    g = torch.Generator().manual_seed(a.seed)
    result = dict(card=torch.cuda.get_device_name(0), rows=M, gemms={})
    print("card: %s, rows Mc = %d, %d traced calls per GEMM after %d warm-up" % (result["card"], M, a.reps, a.warmup))
    print("%-8s %6s %9s %9s %9s %9s %9s %7s %8s %8s %9s" % ("gemm", "tiles", "max/CTA", "wait1 us", "loop us", "epi us",
                                                          "tile us", "polls", "stwaits", "stw kclk", "span us"))
    for name, K, N, act, out in GEMMS:
        A = torch.relu(torch.randn(M, K, generator=g)).to(dev)
        W = (torch.randn(N, K, generator=g) * 0.05).to(dev)
        b = torch.randn(N, generator=g).to(dev)
        c32 = torch.empty(M, N, device=dev) if out == "f32" else None
        hi = torch.empty(M, N, dtype=torch.float16, device=dev) if out == "f16" else None
        lo = torch.empty_like(hi) if hi is not None else None
        p = lambda t: t.data_ptr() if t is not None else None
        waits, loops, epis, tiles, polls, spans, st_waits, st_clk = [], [], [], [], [], [], [], []
        for i in range(a.warmup + a.reps):
            trace.zero_()
            rc = lib.cn_internal_gemm_tc_ex(p(A), p(W), p(b), p(c32), M, N, K, act, 256, None, None, 0, 0, p(hi), p(lo),
                                            N if hi is not None else 0, 0, 0)
            if rc:
                raise SystemExit("cn_internal_gemm_tc_ex: %s" % lib.cn_last_error().decode())
            if i < a.warmup:
                continue
            r = trace.view(sms, CAP, REC).cpu()
            used = r[:, :, 3] != 0
            rec = r[used]
            if rec.shape[0] == 0:
                raise SystemExit("%s wrote no tile records: is %s a CN_GEMM_TRACE build?" % (name, path))
            waits += ((rec[:, 1] - rec[:, 0]) / 1e3).tolist()
            loops += ((rec[:, 2] - rec[:, 1]) / 1e3).tolist()
            epis += ((rec[:, 3] - rec[:, 2]) / 1e3).tolist()
            tiles += ((rec[:, 3] - rec[:, 0]) / 1e3).tolist()
            polls += rec[:, 4].tolist()
            st_waits += rec[:, 5].tolist()
            st_clk += rec[:, 6].tolist()
            spans.append(float(rec[:, 3].max() - rec[:, 0].min()) / 1e3)
        n_tiles = -(-M // 128) * (N // 256)
        med = dict(tiles=n_tiles, max_tiles_per_cta=-(-n_tiles // sms), wait1_us=statistics.median(waits),
                   loop_us=statistics.median(loops), epilogue_us=statistics.median(epis),
                   tile_us=statistics.median(tiles), polls=statistics.median(polls),
                   staging_waits=statistics.mean(st_waits), staging_wait_kclk=statistics.mean(st_clk) / 1e3,
                   span_us=statistics.median(spans))
        result["gemms"][name] = {k: round(v, 3) if isinstance(v, float) else v for k, v in med.items()}
        print("%-8s %6d %9d %9.2f %9.2f %9.2f %9.2f %7.0f %8.2f %8.2f %9.1f" % (
            name, n_tiles, med["max_tiles_per_cta"], med["wait1_us"], med["loop_us"], med["epilogue_us"],
            med["tile_us"], med["polls"], med["staging_waits"], med["staging_wait_kclk"], med["span_us"]))
    lib.cn_internal_gemm_trace(None, 0)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
