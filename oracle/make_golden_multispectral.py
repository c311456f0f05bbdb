"""Generate tests/golden/multispectral_edges.npz from the UNMODIFIED reference band-index kernels.

TEST INFRASTRUCTURE (needs a checkout of the reference, like make_golden.py; the existing golden files are not
touched).  Every output comes from the reference's Numba CPU kernels `_normalized_ratio_cpu`, `_savi_cpu`,
`_evi_cpu`, `_arvi_cpu`, `_gci_cpu`, `_sipi_cpu` and `_ebbi_cpu` (multispectral.py), called on float32 bands of
one row, as the public functions call them after `.astype('f4')`.

* `special`: for each kernel, every combination of band values from {+-0, +-min subnormal, +-FLT_MIN, +-1,
  +-0.5, +-FLT_MAX, +-inf, NaN}, plus band values that make the denominator exactly zero (a = -b, nir = red,
  nir + red = -L, nir + 6 red - 7.5 blue + 1 = 0, nir + 2 red + blue = 0, green = +-0, swir + tir = 0 and < 0).
* `random`: seeded bands over mixed magnitudes (1e-30 .. 1e30, random signs), reflectances in [0, 1), pairs
  within a few float32 ulps of each other (so differences cancel) and integer-valued uint16 counts.  savi runs
  at L in {-1, -0.5, 0, 0.3, 1}.
* `savi_type`: savi with the soil factor in every scalar type the public function accepts.  Numba types
  `nir + red + soil_factor` after the soil factor: float32 for np.float32, np.int8, np.int16, np.uint8, np.bool_
  and Python bool, float64 for Python float and int, np.float64, np.int32, np.int64 and the wider unsigned
  types (np.uint16 included, although NumPy would promote float32 + uint16 to float32).
* `evi_type`: evi with np.float32, np.int8 and Python int soil factor and gain, gain 0 and L = +-1.

Each case stores its kernel, a label, its scalars as (type name, value) and its bands and output, flattened
into one table (offsets in `off`).  The file is written with fixed zip timestamps, so a second run writes the
same bytes.

Usage:  XRS_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_multispectral.py
"""
import io
import itertools
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402

OUT_DIR = os.path.join(os.path.dirname(HERE), "tests", "golden")

F32 = np.finfo(np.float32)
SPECIAL = [0.0, -0.0, float(F32.smallest_subnormal), -float(F32.smallest_subnormal), float(F32.tiny),
           -float(F32.tiny), 1.0, -1.0, 0.5, -0.5, float(F32.max), -float(F32.max), np.inf, -np.inf, np.nan]

# kernel -> (number of bands, band values that make its denominator exactly zero at the default scalars)
KERNELS = {
    "normalized_ratio": (2, [(0.3, -0.3), (-1e-30, 1e-30), (1e30, -1e30), (123.456, -123.456),
                             (float(F32.max), -float(F32.max)), (-float(F32.smallest_subnormal),
                                                                 float(F32.smallest_subnormal))]),
    "savi": (2, [(-0.25, -0.75), (-1.0, 0.0), (0.5, -1.5), (-0.0, -1.0)]),
    "evi": (3, [(0.875, 0.0, 0.25), (-1.0, 0.0, 0.0), (-7.0, 1.0, 0.0), (6.5, 0.0, 1.0), (-1.0, -0.0, -0.0)]),
    "arvi": (3, [(1.0, -1.0, 1.0), (-3.0, 1.0, 1.0), (0.5, 0.25, -1.0), (0.0, -0.0, 0.0)]),
    "gci": (2, [(0.3, 0.0), (0.3, -0.0), (-2.0, 0.0), (0.0, -0.0), (np.inf, 0.0), (np.nan, -0.0)]),
    "sipi": (3, [(0.3, 0.3, 0.1), (-2.0, -2.0, 5.0), (0.0, -0.0, 1.0), (1e30, 1e30, 1e30)]),
    "ebbi": (3, [(0.1, 0.3, -0.3), (0.1, 0.0, 0.0), (0.1, -0.0, 0.0), (0.2, -0.0, -0.0), (0.1, -1.0, 0.5),
                 (-0.4, 1e-30, -1.0)]),
}

SOIL_VALUES = [-1.0, -0.5, 0.0, 0.3, 1.0]
# every soil-factor type savi accepts -> the values of SOIL_VALUES it can hold
SAVI_TYPES = {
    "float": SOIL_VALUES, "int": [-1, 0, 1], "bool": [False, True],
    "float64": SOIL_VALUES, "float32": SOIL_VALUES,
    "int8": [-1, 0, 1], "int16": [-1, 0, 1], "int32": [-1, 0, 1], "int64": [-1, 0, 1],
    "uint8": [0, 1], "uint16": [0, 1], "uint32": [0, 1], "uint64": [0, 1], "bool_": [False, True],
}
# (c1, c2, soil_factor, gain) as (type name, value)
EVI_TYPED = [
    (("float", 6.0), ("float", 7.5), ("float32", 1.0), ("float32", 2.5)),
    (("float", 6.0), ("float", 7.5), ("float32", 0.3), ("float32", 2.5)),
    (("float", 6.0), ("float", 7.5), ("float32", -1.0), ("float32", 0.5)),
    (("float", 6.0), ("float", 7.5), ("int8", 1), ("int8", 2)),
    (("float", 6.0), ("float", 7.5), ("int8", -1), ("int8", 3)),
    (("int", 6), ("int", 7), ("int", 1), ("int", 2)),
    (("float", 6.0), ("float", 7.5), ("float", 1.0), ("float", 0.0)),
    (("float", 6.0), ("float", 7.5), ("float", -1.0), ("float", 2.5)),
    (("float", 6.0), ("float", 7.5), ("float", 0.5), ("float", 2.5)),
]


def scalar(kind, v):
    """The scalar of type `kind`: 'float', 'int', 'bool' (Python) or a NumPy scalar type name."""
    if kind in ("float", "int", "bool"):
        return {"float": float, "int": int, "bool": bool}[kind](v)
    return getattr(np, kind)(v)


def random_bands(rng, nb, n=1024):
    """nb float32 bands of 4 n cells: mixed magnitudes, reflectances, near-equal pairs, uint16 counts."""
    mixed = rng.choice([-1.0, 1.0], (nb, n)) * 10.0 ** rng.uniform(-30, 30, (nb, n))
    refl = rng.random((nb, n))
    base = rng.uniform(0.01, 2.0, n).astype(np.float32)
    near = np.stack([base * (1 + rng.integers(-4, 5, n) * 2.0 ** -23) for _ in range(nb)])
    counts = rng.integers(0, 65536, (nb, n))
    return np.concatenate([mixed, refl, near, counts], axis=1).astype(np.float32)


def special_bands(nb, zeros):
    combos = list(itertools.product(SPECIAL, repeat=nb)) + list(zeros)
    return np.array(combos, np.float64).T.astype(np.float32)


def main():
    ms = ref_loader.load("multispectral")
    fns = {k: getattr(ms, "_%s_cpu" % k) for k in KERNELS}
    rng = np.random.default_rng(20261018)
    cases = []   # (kernel, label, [(kind, value)], bands)

    for k, (nb, zeros) in KERNELS.items():
        sp = special_bands(nb, zeros)
        rb = random_bands(rng, nb)
        if k == "savi":
            for L in (1.0, 0.5):
                cases.append((k, "special", [("float", L)], sp))
            for L in SOIL_VALUES:
                cases.append((k, "random", [("float", L)], rb))
        elif k == "evi":
            d = [("float", 6.0), ("float", 7.5), ("float", 1.0), ("float", 2.5)]
            cases.append((k, "special", d, sp))
            cases.append((k, "random", d, rb))
        else:
            cases.append((k, "special", [], sp))
            cases.append((k, "random", [], rb))

    typed = np.concatenate([random_bands(rng, 2, 256), special_bands(2, KERNELS["savi"][1])], axis=1)
    for kind, values in SAVI_TYPES.items():
        for v in values:
            cases.append(("savi", "savi_type", [(kind, v)], typed))
    typed = np.concatenate([random_bands(rng, 3, 256), special_bands(3, KERNELS["evi"][1])], axis=1)
    for sc in EVI_TYPED:
        cases.append(("evi", "evi_type", list(sc), typed))

    kernel, label, kinds, values, off, bands, outs = [], [], [], [], [0], [], []
    with np.errstate(all="ignore"):
        for k, lab, sc, b in cases:
            args = [x.reshape(1, -1).copy() for x in b]
            out = fns[k](*args, *[scalar(t, v) for t, v in sc]).ravel()
            assert out.dtype == np.float32
            kernel.append(k)
            label.append(lab)
            kinds.append(",".join(t for t, _ in sc))
            values.append([float(v) for _, v in sc] + [np.nan] * (4 - len(sc)))
            full = np.zeros((3, b.shape[1]), np.float32)
            full[:len(b)] = b
            bands.append(full)
            outs.append(out)
            off.append(off[-1] + b.shape[1])
    g = dict(kernel=np.array(kernel), label=np.array(label), scalar_kinds=np.array(kinds),
             scalar_values=np.array(values, np.float64), off=np.array(off, np.int64),
             bands=np.concatenate(bands, axis=1), out=np.concatenate(outs))
    write_npz(os.path.join(OUT_DIR, "multispectral_edges.npz"), g)
    print("%d cases, %d cells" % (len(cases), off[-1]))


def write_npz(path, arrays):
    """np.savez_compressed with fixed member timestamps, so equal arrays give equal bytes."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            z.writestr(info, buf.getvalue())


if __name__ == "__main__":
    main()
