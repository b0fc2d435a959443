"""Random scenarios through the C-ABI of the EMULATED library (tests/emu/build_emu_lib.py, ideally the
--asan build) against the oracle: every index kind (FLAT, IVF-Flat, 8- and 4-bit IVF-PQ, IVF-SQ fp16
and 8-bit, FastScan, IVF-PQR, and the ",RFlat" refinement over each of its bases), odd dimensions
and list counts, empty and tiny shards, adds in random chunks with searches in between, k larger than the shard, nprobe
larger than nlist, nq = 0, invalid ids in reconstruct, and the experimental kernel variants picked
at random.  Ids and distance bits must match the oracle in every scenario.

    DFX_EMU_LIB=$(python tests/emu/build_emu_lib.py --asan) LD_PRELOAD=$(g++ -print-file-name=libasan.so) \\
    ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 python tests/emu/fuzz_against_oracle.py <seed> <seconds>
"""
import sys, os, time, traceback, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from distributed_faiss_b200 import engine
engine.LIB_PATH = os.environ['DFX_EMU_LIB']; engine._lib = None
from oracle import oracle as O
from tests import oracle_pq_fs, oracle_pqr, oracle_rflat
E = engine
kinds = {"flat": E.KIND_FLAT, "ivf_flat": E.KIND_IVF_FLAT, "ivf_pq": E.KIND_IVF_PQ, "ivf_sq": E.KIND_IVF_SQ16,
         "ivf_pq4": E.KIND_IVF_PQ, "ivf_sq8": E.KIND_IVF_SQ8, "ivf_pq_fs": E.KIND_IVF_PQ_FS, "ivf_pqr": E.KIND_IVF_PQR}
kinds.update({"rflat_" + b: kinds[b] for b in ("ivf_pq", "ivf_pq_fs", "ivf_sq8", "ivf_sq")})
L2_ONLY = ("ivf_pq_fs", "ivf_pqr", "rflat_")   # kinds (prefixes) without an inner-product form


def make_oracle(kind, d, metric, nlist, M, M2):
    if kind.startswith("rflat_"):
        return oracle_rflat.make_rflat(kind[len("rflat_"):], d, nlist, M, coarse_metric=metric)
    if kind == "ivf_pq4":
        return O.make_index("ivf_pq", d, metric=metric, nlist=nlist, M=M, nbits=4)
    if kind == "ivf_pqr":
        return oracle_pqr.OracleIVFPQR(d, nlist, M, M2, coarse_metric=metric)
    return oracle_pq_fs.make_index(kind, d, metric=metric, nlist=nlist, M=M)


seed0 = int(sys.argv[1]) if len(sys.argv) > 1 else 0
budget = float(sys.argv[2]) if len(sys.argv) > 2 else 300
t0 = time.time(); it = 0; fails = 0
while time.time() - t0 < budget:
    rs = np.random.RandomState(seed0 + it); it += 1
    kind = rs.choice(list(kinds))
    d = int(rs.choice([4, 8, 32, 64, 96, 128]))
    metric = int(rs.randint(0, 2))
    nlist = int(rs.randint(1, 20)); M = 0; M2 = 0
    if kind.startswith(L2_ONLY): metric = E.METRIC_L2
    nbits = 4 if kind in ("ivf_pq4", "ivf_pq_fs", "rflat_ivf_pq_fs") else 8
    if kind in ("ivf_pq", "rflat_ivf_pq", "ivf_pqr"):
        Ms = [m for m in (4, 8, 16, 24, 32, 64) if d % m == 0 and m <= d]
        M = int(rs.choice(Ms))
    elif nbits == 4:   # 4-bit codes: M a multiple of 8
        d = max(d, 8)
        M = int(rs.choice([m for m in (8, 16, 24, 32, 64) if d % m == 0]))
    if kind == "ivf_pqr":   # M2 = 12 at d = 96 gives a generic dsub2
        M2 = int(rs.choice([m for m in (4, 8, 12, 16, 32) if d % m == 0]))
    n = int(rs.choice([0, 1, 31, 33, 200, 600]))
    desc = f"seed={seed0+it-1} kind={kind} d={d} metric={metric} nlist={nlist} M={M} M2={M2} n={n}"
    try:
        x = rs.randn(max(n, 1), d).astype(np.float32)[:n]
        if n > 40: x[-20:] = x[:20]
        o = make_oracle(kind, d, metric, nlist, M, M2)
        g = E.GpuIndex(kinds[kind], d, metric, nlist=nlist, pq_m=M, pq_nbits=nbits, refine_m=M2,
                       refine_flat=kind.startswith("rflat_"))
        if kind != "flat":
            xt = rs.randn(max(300, nlist * 3), d).astype(np.float32)
            o.train_niter = 2
            o.train(xt)
            if kind in ("ivf_pq", "ivf_pqr") and M == 32 and rs.rand() < 0.5:
                g.set_param("interleaved", int(rs.randint(0, 2)))
            if kind in ("ivf_flat", "ivf_sq", "ivf_sq8") and rs.rand() < 0.5: g.set_param("rows_inflight", 8)
        # ship the trained (empty) state, then add on both sides in the same chunks
        if kind != "flat":
            g.set_state(o.get_state())
        cuts = sorted(set([0, n] + [int(c) for c in rs.randint(0, n + 1, size=2)]))
        for a, b in zip(cuts[:-1], cuts[1:]):
            if b > a:
                o.add(x[a:b]); g.add(x[a:b])
            if rs.rand() < 0.3 and o.ntotal > 0:   # search between adds
                q = rs.randn(2, d).astype(np.float32); kk = int(rs.randint(1, 12))
                if kind != "flat":
                    npb = int(rs.randint(1, nlist + 3)); o.nprobe = min(npb, nlist); g.nprobe = npb
                Do, Io = o.search(q, kk); Dg, Ig = g.search(q, kk)
                assert np.array_equal(Ig, Io) and Dg.tobytes() == Do.tobytes(), "mid-add search mismatch"
        assert g.ntotal == o.ntotal == n
        for nq in (0, 1, 5):
            q = rs.randn(nq, d).astype(np.float32)
            if nq and n: q[0] = x[rs.randint(0, n)]
            k = int(rs.choice([1, 3, 10, 40, 130]))
            if kind != "flat":
                npb = int(rs.randint(1, nlist + 3)); o.nprobe = min(npb, nlist); g.nprobe = npb
            Dg, Ig = g.search(q, k)
            if nq:
                Do, Io = o.search(q, k)
                assert np.array_equal(Ig, Io), f"ids differ nq={nq} k={k}"
                fin = np.isfinite(Do)
                assert Dg[fin].tobytes() == Do[fin].tobytes(), f"distances differ nq={nq} k={k}"
        if n:
            ids = np.array([0, n - 1, -1, n + 5, int(rs.randint(0, n))], dtype=np.int64)
            Rg = g.reconstruct_rows(ids)
            assert np.isnan(Rg[2]).all() and np.isnan(Rg[3]).all()
            if kind != "flat":
                Ro = o.reconstruct_rows(ids[[0, 1, 4]])
                assert np.allclose(Rg[[0, 1, 4]], Ro, rtol=0, atol=1e-5)
            else:
                assert np.array_equal(Rg[[0, 1, 4]], x[ids[[0, 1, 4]]])
        st = g.get_state()
        del g
    except Exception as e:
        fails += 1
        print("FAIL", desc, "->", repr(e)[:300]); traceback.print_exc(limit=2)
        if fails > 5: break
print(f"fuzz done: {it} scenarios, {fails} failures, {time.time()-t0:.0f}s")
sys.exit(1 if fails else 0)
