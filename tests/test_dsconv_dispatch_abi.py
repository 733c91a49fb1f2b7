"""The fused DS conv's dispatch table, restated in plain Python and checked against the library's eligibility entry points.

``expected`` says, for one request, whether the fused DS conv (csrc/dsconv_fused.cu) takes it and, if so, which kernel runs
it, at which N_TILE and patch width PW, in how many channel passes.  It restates ``ds_select`` (with ``pick_pw``), which both
launches and the ``smaat_dsconv_*_eligible`` entry points ask.  Two facts come from compiled shared-memory sizes and cannot be
restated: whether an instance stages its output (DsCfg::ST_BUFS > 0, which the max-pool and the CBAM pools read back) and how
many classes' OutConv weights it keeps (DsCfg::MAX_CLASSES).  They are probed per instance and pinned in INSTANCES, so that a
change to the rings shows up here as a diff.

``SPACE`` is every combination of the axes below; the CPU test asserts that the library agrees with ``expected`` on each
(host logic only: fake, 16-byte aligned addresses that are never dereferenced).  ``CELLS`` is the subset that
tests/test_gpu_dsconv_dispatch.py runs on the GPU: chosen greedily from ``SPACE`` so that every (kernel, N_TILE, k, PW,
precision, A form, epilogue) that ``expected`` can reach has a cell, and so that each kernel also meets every geometry,
input form, stride form, Cout and class count with each epilogue; plus a few large images for the persistent scheduler.
"""
import itertools
import math
import random

import pytest

import smaat_unet_b200 as S

A = 1 << 20                       # fake, 16-byte aligned address
DECLINED = "declined"
MAX_CLS = 32                      # DS_MAX_CLASSES
MIN_CLS = 21                      # DS_MIN_CLASSES: the classes a paired tile keeps beside its rings
PREC = ("tf32", "tf32x3", "bf16", "bf16maps")       # bf16maps: bf16 operands and bf16 activations in HBM
MODE_CODE = {"tf32": 1, "tf32x3": 2, "bf16": 3, "bf16maps": 3}
AFORMS = ("regs", "smem")                           # the register A form ('auto' takes it) or wgmma reading A from shared memory
EPILOGUES = ("relu", "linear", "stats", "outconv", "classify", "maxpool", "gate", "pools")
BACT_EPILOGUES = ("relu", "linear", "outconv", "classify", "maxpool", "gate")   # the bf16-activation route has no stats or pools
KS = (1, 2, 3, 4)
COUTS = (8, 24, 64, 96, 128, 136, 200, 256, 384, 512, 4, 640)
CLASSES = (1, 21, 22, 23, 32, 33)
# name -> (H, W): the patch width pick_pw takes, and whether the patch rows ceil(H / PH) are even
GEOMS = {
    "pw32": (32, 64),             # PW 32, 8 patch rows
    "pw32-odd": (28, 64),         # PW 32, 7 patch rows
    "pw32-partial": (30, 52),     # PW 32, partial last column; 8 patch rows, the last one partial (a partial last pair)
    "pw16": (32, 48),             # PW 16, 4 patch rows
    "pw16-odd": (40, 40),         # PW 16, 5 patch rows, partial last column
    "pw16-72": (72, 72),          # PW 16, 9 patch rows
    "refused": (36, 36),          # pick_pw: both widths waste more than 1.35
    "w-odd4": (32, 50),           # W not a multiple of 4
}
# large images: more tiles than SMs and a tile count that is not a multiple of the grid (GPU cells only)
BIG = {"big144": (144, 144, 2), "big288": (288, 288, 1)}
# name -> (C0, C1): plain input or the virtual concat [x0, x1]; C0 % (32 / k) decides the concat's eligibility
INPUTS = {"plain24": (24, 0), "plain32": (32, 0), "plain6": (6, 0), "cat32+16": (32, 16), "cat16+24": (16, 24),
          "cat8+8": (8, 8), "cat12+4": (12, 4)}
# x's batch stride: dense, a channel slice of a wider tensor, or one that TMA cannot take (fake addresses only)
STRIDES = ("dense", "slice", "bad4", "bad8")


def pick_pw(H, W):
    """csrc/dsconv_fused.cu pick_pw: the patch width that wastes fewer MMA rows, 0 when both waste more than 1.35."""
    best, pw = 1e9, 0
    for c in (32, 16):
        ph = 128 // c
        waste = (math.ceil(W / c) * c / W) * (math.ceil(H / ph) * ph / H)
        if waste < best - 1e-9:
            best, pw = waste, c
    return pw if best <= 1.35 else 0


def bstride(C, H, W, form):
    """x's batch stride in elements: dense, a slice of 7 more channels, or 2 / 4 past a multiple of 4 / 8."""
    return {"dense": C * H * W, "slice": (C + 7) * H * W, "bad4": C * H * W + 2, "bad8": C * H * W + 4}[form]


# (N_TILE, k, PW, precision, A form) -> (staged, max_classes): DsCfg::ST_BUFS > 0 and DsCfg::MAX_CLASSES of the single-tile
# instance, probed from the library (test_instances_are_pinned) and pinned here
INSTANCES = {
    (64, 1, 16, "tf32", "regs"): (True, 32), (64, 1, 16, "tf32", "smem"): (True, 32),
    (64, 1, 16, "tf32x3", "regs"): (True, 32), (64, 1, 16, "tf32x3", "smem"): (False, 32),
    (64, 1, 16, "bf16", "regs"): (True, 32), (64, 1, 16, "bf16maps", "regs"): (True, 32),
    (64, 1, 32, "tf32", "regs"): (True, 32), (64, 1, 32, "tf32", "smem"): (True, 32),
    (64, 1, 32, "tf32x3", "regs"): (True, 32), (64, 1, 32, "tf32x3", "smem"): (False, 32),
    (64, 1, 32, "bf16", "regs"): (True, 32), (64, 1, 32, "bf16maps", "regs"): (True, 32),
    (64, 2, 16, "tf32", "regs"): (True, 32), (64, 2, 16, "tf32", "smem"): (True, 32),
    (64, 2, 16, "tf32x3", "regs"): (True, 32), (64, 2, 16, "tf32x3", "smem"): (True, 32),
    (64, 2, 16, "bf16", "regs"): (True, 32), (64, 2, 16, "bf16maps", "regs"): (True, 32),
    (64, 2, 32, "tf32", "regs"): (True, 32), (64, 2, 32, "tf32", "smem"): (True, 32),
    (64, 2, 32, "tf32x3", "regs"): (True, 32), (64, 2, 32, "tf32x3", "smem"): (True, 32),
    (64, 2, 32, "bf16", "regs"): (True, 32), (64, 2, 32, "bf16maps", "regs"): (True, 32),
    (64, 4, 16, "tf32", "regs"): (True, 32), (64, 4, 16, "tf32x3", "regs"): (True, 29),
    (64, 4, 16, "bf16", "regs"): (True, 32), (64, 4, 32, "tf32", "regs"): (True, 32),
    (64, 4, 32, "tf32x3", "regs"): (True, 29), (64, 4, 32, "bf16", "regs"): (True, 32),
    (128, 1, 16, "tf32", "regs"): (True, 26), (128, 1, 16, "tf32", "smem"): (True, 26),
    (128, 1, 16, "tf32x3", "regs"): (False, 26), (128, 1, 16, "tf32x3", "smem"): (True, 26),
    (128, 1, 16, "bf16", "regs"): (True, 32), (128, 1, 16, "bf16maps", "regs"): (True, 32),
    (128, 1, 32, "tf32", "regs"): (True, 26), (128, 1, 32, "tf32", "smem"): (True, 26),
    (128, 1, 32, "tf32x3", "regs"): (False, 26), (128, 1, 32, "tf32x3", "smem"): (True, 26),
    (128, 1, 32, "bf16", "regs"): (True, 32), (128, 1, 32, "bf16maps", "regs"): (True, 22),
    (128, 2, 16, "tf32", "regs"): (True, 22), (128, 2, 16, "tf32", "smem"): (True, 22),
    (128, 2, 16, "tf32x3", "regs"): (True, 22), (128, 2, 16, "tf32x3", "smem"): (True, 22),
    (128, 2, 16, "bf16", "regs"): (True, 22), (128, 2, 16, "bf16maps", "regs"): (True, 32),
    (128, 2, 32, "tf32", "regs"): (True, 22), (128, 2, 32, "tf32", "smem"): (True, 22),
    (128, 2, 32, "tf32x3", "regs"): (True, 22), (128, 2, 32, "tf32x3", "smem"): (True, 22),
    (128, 2, 32, "bf16", "regs"): (True, 22), (128, 2, 32, "bf16maps", "regs"): (True, 32),
    (128, 4, 16, "tf32", "regs"): (True, 32), (128, 4, 16, "tf32x3", "regs"): (True, 32),
    (128, 4, 16, "bf16", "regs"): (True, 32), (128, 4, 32, "tf32", "regs"): (True, 32),
    (128, 4, 32, "tf32x3", "regs"): (True, 32), (128, 4, 32, "bf16", "regs"): (True, 32),
}


def expected(C0, C1, bs0, bs1, H, W, k, Cout, mode, impl, wide_on, bact, epilogue, ncls, pair_on=True):
    """What the fused DS conv does with one request: DECLINED, or (kernel, N_TILE, PW, channel passes).

    mode 'tf32' | 'tf32x3' | 'bf16'; bact: bf16 activations (mode 'bf16' only); impl 'regs' | 'smem'; wide_on / pair_on:
    smaat_set_dsconv_wide / smaat_set_dsconv_pair; epilogue one of EPILOGUES; ncls the classes of 'classify'."""
    assert not bact or (mode == "bf16" and epilogue in BACT_EPILOGUES)
    a_smem, bf16 = impl == "smem", mode == "bf16"
    head, stats = epilogue in ("outconv", "classify"), epilogue == "stats"
    # ds_select: the shape, stride, alignment, k, mode and A-form rules
    if k not in (1, 2, 4) or (k == 4 and a_smem) or (bf16 and a_smem):
        return DECLINED
    if bact and (k == 4 or W % 8 or bs0 % 8 or (C1 and bs1 % 8)):
        return DECLINED
    if Cout < 8 or Cout > 512 or (Cout > 128 and (stats or head)):
        return DECLINED
    wide = wide_on and 128 < Cout <= 256 and k == 2 and not a_smem and not bf16 and not head
    if Cout > 128 and Cout % 128 and not wide:
        return DECLINED
    if W % 4 or bs0 % 4 or (C1 and (bs1 % 4 or C0 % (32 // k))):
        return DECLINED
    if k * (C0 + C1) % 4 and not bact:
        return DECLINED
    pw = pick_pw(H, W)
    if not pw:
        return DECLINED
    # the epilogue's limits: eligibility asks the instance that runs.  The single tile's pinned values stand for a pair or a
    # wide tile: both keep the staged epilogue (static_asserts), as do the single tiles they replace (INSTANCES); a pair takes
    # class launches of up to MIN_CLS classes, which every instance keeps; a wide tile takes no head
    n_tile = 128 if Cout > 64 else 64
    staged, max_cls = INSTANCES[(n_tile, k, pw, "bf16maps" if bact else mode, impl)]
    if epilogue in ("maxpool", "pools") and not staged:
        return DECLINED
    if epilogue == "classify" and ncls > min(max_cls, MAX_CLS):
        return DECLINED
    # ds_select: which instance runs it, wide, else pair, else the single tile
    if wide:
        return "dsconv_wide_kernel", 128, pw, 1
    pair = (pair_on and n_tile == 64 and k in (2, 4) and not a_smem and not bf16 and math.ceil(H / (128 // pw)) % 2 == 0
            and (ncls if epilogue == "classify" else 0) <= MIN_CLS)
    if pair:
        return "dsconv_pair_kernel", 64, pw, 1
    name = ("dsconv_bf16act_kernel" if bact else "dsconv_bf16_kernel" if bf16 else "dsconv_kpl4_kernel" if k == 4
            else "dsconv_fused_kernel")
    return name, n_tile, pw, math.ceil(Cout / n_tile)


# ------------------------------------------------------------------------------------------------------------- the space
def _cell(prec, impl, wide_on, k, Cout, inp, geom, stride, epilogue, ncls):
    C0, C1 = INPUTS[inp]
    H, W, B = BIG[geom] if geom in BIG else GEOMS[geom] + (2,)
    c = dict(prec=prec, impl=impl, wide_on=wide_on, k=k, Cout=Cout, inp=inp, C0=C0, C1=C1, geom=geom, H=H, W=W, B=B,
             stride=stride, bs0=bstride(C0, H, W, stride), bs1=bstride(C1, H, W, stride) if C1 else 0, epilogue=epilogue,
             ncls=ncls if epilogue == "classify" else 0)
    c["mode"] = "bf16" if prec == "bf16maps" else prec
    c["bact"] = prec == "bf16maps"
    c["want"] = _expected(c)
    c["id"] = (f"{prec}-{impl}{'' if wide_on else '-nowide'}-k{k}-N{Cout}-{inp}-{geom}-{stride}-{epilogue}"
               f"{c['ncls'] if epilogue == 'classify' else ''}")
    return c


def _expected(c, **kw):
    a = dict(c, **kw)
    return expected(a["C0"], a["C1"], a["bs0"], a["bs1"], a["H"], a["W"], a["k"], a["Cout"], a["mode"], a["impl"], a["wide_on"],
                    a["bact"], a["epilogue"], a["ncls"])


def _space(geoms):
    for prec, impl, wide_on, k, Cout, inp, geom, stride, epi in itertools.product(
            PREC, AFORMS, (True, False), KS, COUTS, INPUTS, geoms, STRIDES, EPILOGUES):
        if prec == "bf16maps" and epi not in BACT_EPILOGUES:
            continue
        if not wide_on and not 128 < Cout <= 256:      # the switch only matters there
            continue
        for ncls in (_classes(prec, impl, k, Cout, geom) if epi == "classify" else (0,)):
            yield _cell(prec, impl, wide_on, k, Cout, inp, geom, stride, epi, ncls)


def _classes(prec, impl, k, Cout, geom):
    """CLASSES, and the largest count the request's instance takes and the next one up."""
    H, W = BIG[geom][:2] if geom in BIG else GEOMS[geom]
    inst = INSTANCES.get((128 if Cout > 64 else 64, k, pick_pw(H, W), prec, impl))
    return sorted(set(CLASSES) | ({inst[1], inst[1] + 1} if inst else set()))


SPACE = list(_space(GEOMS))


def combo(c):
    """The coverage key: (kernel, N_TILE, k, PW, precision, A form, epilogue)."""
    kern, nt, pw, _ = c["want"]
    return kern, nt, c["k"], pw, c["prec"], c["impl"], c["epilogue"]


REACHABLE = sorted({combo(c) for c in SPACE if c["want"] != DECLINED})


def _families(c):
    """The keys a GPU cell covers: the coverage combination, and each kernel (or the decline) against the other axes."""
    if c["want"] == DECLINED:
        keys = [("declined", c["prec"], c["impl"], c["epilogue"])]
        if c["epilogue"] == "classify" and _expected(c, ncls=1) != DECLINED:      # declined for its class count
            keys.append(("classes", c["k"], 128 if c["Cout"] > 64 else 64, pick_pw(c["H"], c["W"]), c["prec"], c["impl"], c["ncls"]))
        return keys
    kern, nt, pw, npass = c["want"]
    if c["geom"] in BIG:
        return [(kern, c["geom"])]
    e = c["epilogue"]
    keys = [combo(c), (kern, e, c["geom"]), (kern, e, c["inp"]), (kern, e, c["stride"], c["y_slice"]), (kern, e, c["Cout"]),
            (kern, c["k"], c["prec"], c["impl"], "x0 slice" if c["stride"] == "slice" else "x0 dense")]
    if e == "classify":
        keys += [("classes", c["k"], nt, pw, c["prec"], c["impl"], c["ncls"]), (kern, "classes", c["ncls"])]
    return keys


def _gpu_cells():
    """CELLS: a greedy cover of the families over SPACE's small, GPU-sized cells (Cout <= 512, strides TMA takes), in a seeded
    order so that the axes mix."""
    pool = [c for c in SPACE if c["stride"] in ("dense", "slice") and c["geom"] != "w-odd4" or c["want"] == DECLINED]
    pool += [c for c in _space(BIG) if c["stride"] == "dense" and c["want"] != DECLINED and c["inp"] == "cat32+16"]
    pool = [dict(c) for c in pool if 8 <= c["Cout"] <= 512 and c["k"] in (1, 2, 4) and c["stride"] != "bad8"]
    rng = random.Random(2024)
    rng.shuffle(pool)
    for i, c in enumerate(pool):
        c["y_slice"] = bool(i % 2)                       # y as a channel slice of a wider buffer, or dense
    seen, cells = set(), []
    for c in pool:
        new = [key for key in _families(c) if key not in seen]
        if new:
            seen.update(new)
            cells.append(c)
    return sorted(cells, key=lambda c: c["id"])


CELLS = _gpu_cells()


# ================================================================================================================= tests
def _lib():
    try:
        return S._lib.load()
    except (OSError, RuntimeError) as e:
        pytest.skip(f"the library is not built: {e}")


def _entry(lib, c):
    """What the library's eligibility entry point for the cell's epilogue answers (1 / 0)."""
    x1 = A if c["C1"] else None
    args = (A, c["C0"], c["bs0"], x1, c["C1"], c["bs1"], A, c["H"], c["W"], c["k"], c["Cout"])
    m, e = MODE_CODE[c["prec"]], c["epilogue"]
    if c["bact"]:
        if e == "maxpool":
            return lib.smaat_dsconv_maxpool_bf16_eligible(*args)
        return lib.smaat_dsconv_bf16_eligible(*args, {"outconv": 1, "classify": c["ncls"]}.get(e, 0))
    if e in ("relu", "linear", "stats"):
        ok = lib.smaat_dsconv_eligible2(*args, int(e == "stats"))
        # eligible2 does not know the mode: 'bf16' has register-form instances only (ops.dsconv_takes asks both)
        return ok and (m != 3 or lib.smaat_dsconv_cbam_eligible(*args, m, 0, 0))
    if e in ("outconv", "classify"):
        return lib.smaat_dsconv_classify_eligible(*args, 1 if e == "outconv" else c["ncls"], m)
    if e == "maxpool":
        return lib.smaat_dsconv_maxpool_eligible(*args, m)
    return lib.smaat_dsconv_cbam_eligible(*args, m, int(e == "gate"), int(e == "pools"))


def _switches(lib, impl, wide_on):
    assert lib.smaat_set_dsconv_impl({"regs": 2, "smem": 1}[impl]) == 0
    assert lib.smaat_set_dsconv_wide(int(wide_on)) == 0


def _restore(lib):
    assert lib.smaat_set_dsconv_impl(0) == 0 and lib.smaat_set_dsconv_wide(1) == 0


def test_pick_pw_restatement():
    assert [pick_pw(*GEOMS[g]) for g in GEOMS] == [32, 32, 32, 16, 16, 16, 0, 32]
    assert pick_pw(288, 288) == 32 and pick_pw(144, 144) == 16 and pick_pw(72, 72) == 16
    # the waste limit: 1.35 passes, just above it does not (36 x 36 wastes 1.48 at PW 16; 24 x 40 wastes 1.333 at PW 16)
    assert pick_pw(24, 40) == 16 and pick_pw(16, 56) == 32


def test_library_agrees_with_expected_in_every_cell():
    lib = _lib()
    bad = []
    try:
        for (impl, wide_on), cells in itertools.groupby(sorted(SPACE, key=lambda c: (c["impl"], c["wide_on"])),
                                                         key=lambda c: (c["impl"], c["wide_on"])):
            _switches(lib, impl, wide_on)
            for c in cells:
                got = bool(_entry(lib, c))
                if got != (c["want"] != DECLINED):
                    bad.append(f"{c['id']}: library {'takes' if got else 'declines'}, expected {c['want']}")
    finally:
        _restore(lib)
    print(f"{len(SPACE)} cells, {sum(c['want'] != DECLINED for c in SPACE)} taken")
    assert not bad, f"{len(bad)} of {len(SPACE)} cells differ, e.g.\n" + "\n".join(bad[:20])


def _probe(lib, n_tile, k, pw, prec, impl):
    H, W = GEOMS["pw32-odd" if pw == 32 else "pw16-odd"]
    Cout = n_tile
    args = (A, 32, 32 * H * W, None, 0, 0, A, H, W, k, Cout)
    _switches(lib, impl, True)
    if prec == "bf16maps":
        if not lib.smaat_dsconv_bf16_eligible(*args, 0):
            return None
        staged = bool(lib.smaat_dsconv_maxpool_bf16_eligible(*args))
        ks = [K for K in range(1, MAX_CLS + 2) if lib.smaat_dsconv_bf16_eligible(*args, K)]
    else:
        m = MODE_CODE[prec]
        if not lib.smaat_dsconv_cbam_eligible(*args, m, 1, 0):
            return None
        staged = bool(lib.smaat_dsconv_maxpool_eligible(*args, m))
        ks = [K for K in range(1, MAX_CLS + 2) if lib.smaat_dsconv_classify_eligible(*args, K, m)]
    assert ks == list(range(1, len(ks) + 1)), f"the class counts taken are not 1..max: {ks}"
    return staged, len(ks)


def test_instances_are_pinned():
    """Probe each single-tile instance's staged epilogue and largest class count; they must equal INSTANCES."""
    lib = _lib()
    got = {}
    try:
        for key in itertools.product((64, 128), (1, 2, 4), (16, 32), PREC, AFORMS):
            r = _probe(lib, *key)
            if r is not None:
                got[key] = r
    finally:
        _restore(lib)
    assert got == INSTANCES, "\n".join(f"{k}: probed {got.get(k)}, pinned {INSTANCES.get(k)}" for k in sorted(set(got) | set(INSTANCES))
                                       if got.get(k) != INSTANCES.get(k))
    # every instance keeps a 21-class model's weights, so that the paired tile (which keeps 21) never takes fewer than its
    # single tile
    assert min(v[1] for v in INSTANCES.values()) >= MIN_CLS


def test_every_reachable_combination_has_a_gpu_cell():
    have = {combo(c) for c in CELLS if c["want"] != DECLINED}
    missing = [r for r in REACHABLE if r not in have]
    kernels = sorted({r[0] for r in REACHABLE})
    print(f"{len(REACHABLE)} reachable (kernel, N_TILE, k, PW, precision, A form, epilogue) combinations over {kernels}; "
          f"{len(CELLS)} GPU cells ({sum(c['want'] == DECLINED for c in CELLS)} declined)")
    assert not missing, f"{len(missing)} combinations without a cell: {missing[:10]}"
    assert len(kernels) == 6
    # the cells the table was built to reach
    def has(**kw):
        return any(all(c.get(k) == v if not callable(v) else v(c.get(k)) for k, v in kw.items()) for c in CELLS)
    pair = lambda w: w != DECLINED and w[0] == "dsconv_pair_kernel"
    wide = lambda w: w != DECLINED and w[0] == "dsconv_wide_kernel"
    assert has(want=lambda w: pair(w) and w[2] == 16, k=4, epilogue="pools")
    assert has(want=lambda w: wide(w) and w[2] == 16, epilogue="gate", inp="cat32+16")
    for Cout in (384, 512):
        for e in ("gate", "pools", "maxpool"):
            assert has(Cout=Cout, epilogue=e, want=lambda w: w != DECLINED and w[3] == Cout // 128)
    for kern in (pair, wide):
        assert has(want=kern, y_slice=True) and has(want=kern, stride="slice")
        assert has(want=kern, geom="big144") or has(want=kern, geom="big288")
    for key, (staged, mx) in INSTANCES.items():
        n_tile, k, pw, prec, impl = key
        for K in (mx, mx + 1):
            assert any(c["epilogue"] == "classify" and c["ncls"] == K and c["k"] == k and (c["Cout"] > 64) == (n_tile == 128)
                       and c["prec"] == prec and c["impl"] == impl and pick_pw(c["H"], c["W"]) == pw for c in CELLS), (key, K)
