"""Cases of the lossless-transform tests (tests/test_transform.py) and of tools/make_golden.py --transform.

Every source is written by the repository's CPU oracle, so a GPU run needs no reference binary; the expected outputs
in tests/golden/transform_golden.json come from the reference's own jpegtran on those sources."""
import hashlib
import struct

import numpy as np

SAMPLINGS = {"gray": ["-grayscale"], "444": ["-sample", "1x1"], "422": ["-sample", "2x1"], "440": ["-sample", "1x2"],
             "420": ["-sample", "2x2"], "3x2": ["-sample", "3x2"]}
SIZES = [(227, 149), (33, 17), (17, 9), (1, 1), (8, 300), (256, 128)]
TRANSFORMS = [[], ["-flip", "horizontal"], ["-flip", "vertical"], ["-transpose"], ["-transverse"],
              ["-rotate", "90"], ["-rotate", "180"], ["-rotate", "270"]]
# the re-encode switches, spread over the main matrix
REENCODE = [[], ["-optimize"], ["-progressive"], ["-revert"], ["-restart", "1"]]

CROPS = ["64x48+0+0", "64x48+16+16", "64x48+5+3", "100x60+17+9", "50x40-0-0", "50x40-7-5", "64fx48f+5+3", "64x48f+17+9",
         "60rx40+3+3", "+16+8", "x40+0+100", "227x149+0+0", "27x49+200+100", "1x1+226+148"]
CROP_COMBOS = [["-rotate", "90", "-crop", "64x48+16+16"], ["-rotate", "180", "-crop", "50x40+33+21"],
               ["-rotate", "270", "-crop", "64x48+5+3"], ["-flip", "horizontal", "-crop", "64x48+16+8"],
               ["-flip", "vertical", "-crop", "64x48+16+8"], ["-transverse", "-crop", "40x40+9+9"],
               ["-transpose", "-crop", "30x70+0+0"], ["-crop", "64x48+16+16", "-grayscale"],
               ["-rotate", "90", "-trim", "-crop", "100x100+20+20"]]
OTHER = [["-grayscale"], ["-grayscale", "-rotate", "270"], ["-perfect", "-rotate", "90"], ["-perfect", "-transverse"],
         ["-perfect", "-flip", "horizontal", "-optimize"]]
# the reference refuses these (its message, or exit status 1 from its switch parser)
REFUSALS = [("227x149_420", ["-crop", "10x10+230+0"]), ("227x149_420", ["-crop", "0x10+0+0"]),
            ("227x149_420", ["-rotate", "90", "-crop", "300x10+0+0"]), ("227x149_420", ["-perfect", "-rotate", "90"]),
            ("227x149_420", ["-perfect", "-flip", "horizontal"]), ("227x149_420", ["-rotate", "45"]),
            ("227x149_420", ["-rotate", "90", "-flip", "horizontal"]), ("227x149_420", ["-crop", "10y10"]),
            ("lumasub_420", ["-grayscale"])]


def source_ids():
    ids = [f"{w}x{h}_{s}" for s in SAMPLINGS for (w, h) in SIZES]
    return ids + ["227x149_420_restart", "227x149_422_restart3B", "lumasub_420", "q50_420", "q90_420", "q75_420_dqt", "prog_420",
                  "baseline12"]


def _params(sid):
    import mozjpeg_b200 as mj
    if sid == "lumasub_420":                          # luma below the largest factors: -grayscale is refused
        p = mj.params_from_switches(["-revert", "-sample", "2x2"], 64, 48, 3)
        for ci, (h, v) in enumerate([(1, 1), (2, 2), (1, 1)]):
            p.comp_info[ci].h_samp_factor, p.comp_info[ci].v_samp_factor = h, v
        return p
    size, samp = sid.split("_")[:2]
    w, h = map(int, size.split("x")) if size[0].isdigit() else (227, 149)
    sw = ["-revert", *SAMPLINGS.get(samp, SAMPLINGS["420"])]
    if sid.endswith("_restart"):
        sw += ["-restart", "1"]
    if sid.endswith("_restart3B"):
        sw += ["-restart", "3B"]
    if size.startswith("q"):
        sw = ["-revert", "-quality", size[1:3], "-sample", "2x2"]
    if sid == "prog_420":
        sw = ["-revert", "-progressive", "-sample", "2x2"]
    p = mj.params_from_switches(sw, w, h, 3)
    if sid == "q75_420_dqt":                          # tables that differ between rows and columns
        for s in range(2):
            for k in range(64):
                p.quant_tbl[s][k] = 2 + (k % 8) * 3 + (k // 8) + s
    return p


def source(sid):
    """(file bytes, per component (hib, wib, 64) int16 natural-order planes the oracle quantized)"""
    from oracle import oracle as O
    if sid == "baseline12":                           # 12-bit 4:2:0, 120x72 (tests/decode_cases.py)
        import decode_cases as D
        return D.extra_source(sid), None
    p = _params(sid)
    seed = sum(map(ord, sid)) % 97
    r = O.oracle_encode(p, O.synth_image(seed, p.image_width, p.image_height), want_debug=True)
    d = r.dbg
    return r.jpeg, [np.ascontiguousarray(d["final"][ci][:d["hib"][ci], :d["wib"][ci]]) for ci in range(d["ncomp"])]


def main_matrix():
    """(case id, source id, switches): every transform with and without -trim on every sequential source"""
    out = []
    for i, sid in enumerate(f"{w}x{h}_{s}" for s in SAMPLINGS for (w, h) in SIZES):
        for j, tr in enumerate(TRANSFORMS):
            for trim in (0, 1):
                sw = tr + (["-trim"] if trim else []) + REENCODE[(i + j + trim) % len(REENCODE)]
                out.append((f"{sid}:{'_'.join(a.lstrip('-') for a in sw)}", sid, sw))
    return out


def other_cases():
    out = []
    for c in CROPS:
        out.append(("crop_" + c, "227x149_420", ["-crop", c]))
    for c in ["64x48+16+16", "50x40-7-5", "27x49+200+100"]:
        out.append(("crop422_" + c, "227x149_422", ["-crop", c]))
        out.append(("cropgray_" + c, "227x149_gray", ["-crop", c]))
    for k, sw in enumerate(CROP_COMBOS):
        out.append((f"cropx{k}", "227x149_420" if k % 2 == 0 else "227x149_3x2", sw))
    for k, sw in enumerate(OTHER):
        out.append((f"other{k}", "256x128_420" if "-perfect" in sw else "227x149_420", sw))
    out.append(("gray444", "227x149_444", ["-grayscale", "-optimize"]))
    for sw in (["-rotate", "90"], ["-flip", "horizontal", "-crop", "64x40+9+9"], ["-transverse", "-trim", "-progressive"]):
        out.append((f"baseline12:{'_'.join(a.lstrip('-') for a in sw)}", "baseline12", sw))
    for sid in ("227x149_420_restart", "227x149_422_restart3B"):
        for sw in (["-rotate", "90"], ["-flip", "vertical", "-restart", "2"], ["-transverse", "-crop", "64x48+8+8"]):
            out.append((f"{sid}:{'_'.join(a.lstrip('-') for a in sw)}", sid, sw))
    return out


def mixed_ids():
    """same geometry, different DQTs: one -rotate 90 batch"""
    return ["q50_420", "227x149_420", "q90_420", "q75_420_dqt"]


def md5(b: bytes) -> str:
    return hashlib.md5(b).hexdigest()


def sof_dqt(jpeg: bytes):
    """(width, height, [(id, h, v, Tq)], md5 of the component slots' tables in natural order) from the file's SOF and
    DQT segments"""
    from mozjpeg_b200 import jpegtran as T
    r = T.parse_source(jpeg)
    comps = [(r.component_id[i], r.h_samp_factor[i], r.v_samp_factor[i], r.quant_tbl_no[i]) for i in range(r.num_components)]
    return r.image_width, r.image_height, comps, tables_md5([list(r.quant_tbl[c[3]]) for c in comps])


def tables_md5(tables) -> str:
    m = hashlib.md5()
    for t in tables:
        m.update(struct.pack("<64H", *t))
    return m.hexdigest()
