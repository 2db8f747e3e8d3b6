"""Sources, option sets and the CPU restatement behind the scaled-IDCT tests (tests/test_idct_scaling.py),
tools/make_golden.py --idct-scaling and tools/gen_idct_scaled.py.

The restatement: jidctint.c's scaled IDCTs of block sizes 3, 5, 6, 7 and 9 .. 16 (jpeg_idct_3x3 .. jpeg_idct_16x16,
8-bit: CONST_BITS 13, PASS1_BITS 2, JLONG intermediates, plain products), one pass at a time.  For N < 8 pass 1 takes
coefficient rows 0 .. N-1 of columns 0 .. N-1 and pass 2 the N workspace values of a row; for N > 8 pass 1 takes the
eight rows of each of the eight columns into N workspace rows and pass 2 the eight values of each of them.  Each 1-D
function below is written once for both passes: `P` supplies what the reference writes differently in each, the DC
term with its rounding, the final descale (pass 1: to an int workspace entry; pass 2: the sample before the range
limit), and the sizes whose middle outputs pass 1 descales early and adds unscaled (6, 10 and 14).

The reference's decode of a gray (1 x 1) source at scale k/8 is exactly its k x k IDCT output, so the restatement is
checked against every recorded gray case without a GPU.

Every operation of a pass before its final descale is an exact integer sum of products, and an early descale only ever
adds a multiple of the descale unit, so each output of a pass is (sum_j m[o][j] * in[j] + 2^(s-1)) >> s for one
integer matrix m.  pass_matrix() finds m by running the 1-D function on linear forms; tools/gen_idct_scaled.py writes
the matrices as the device functions the kernels evaluate (mozjpeg_b200/csrc/idct_scaled.inc), and the tests hold the
matrices to the restatement on random and extreme inputs."""
import json
import os
from fractions import Fraction

import numpy as np

import decompress_options_cases as O
import recompress_cases as R

ROOT = R.ROOT
GOLDEN = os.path.join(ROOT, "tests", "golden", "idct_scaling_golden.json")

CONST_BITS, PASS1_BITS = 13, 2
NEW_SIZES = (3, 5, 6, 7, 9, 10, 11, 12, 13, 14, 15, 16)


def FIX(x):
    return int(x * (1 << CONST_BITS) + 0.5)


def _i32(x):
    """the (int) cast of a workspace store: modulo 2^32"""
    if isinstance(x, np.ndarray):
        return x.astype(np.int64).astype(np.int32).astype(np.int64)
    return x


class _Pass:
    """what the two passes of one function write differently"""

    def __init__(self, n):
        self.n = n
        self.shift = CONST_BITS - PASS1_BITS if n == 1 else CONST_BITS + PASS1_BITS + 3

    def dc(self, x):
        """the DC input scaled to CONST_BITS, with the pass's rounding folded in"""
        if self.n == 1:
            return (x << CONST_BITS) + (1 << (CONST_BITS - PASS1_BITS - 1))
        return (x + (1 << (PASS1_BITS + 2))) << CONST_BITS

    def out(self, x):
        return _i32(x >> self.shift) if self.n == 1 else x >> self.shift

    def mid(self, x, y):
        """a middle output: x (with the DC rounding) plus y, which both passes compute unscaled.  Pass 1 descales x
        on its own and adds y << PASS1_BITS; pass 2 adds y << CONST_BITS before its descale."""
        if self.n == 1:
            return _i32((x >> (CONST_BITS - PASS1_BITS)) + (y << PASS1_BITS))
        return (x + (y << CONST_BITS)) >> self.shift


def _idct3(d, P):                     # jidctint.c:812-890
    t0 = P.dc(d[0])
    t12 = d[2] * FIX(0.707106781)
    t10 = t0 + t12
    t2 = t0 - t12 - t12
    t0 = d[1] * FIX(1.224744871)
    return [P.out(t10 + t0), P.out(t2), P.out(t10 - t0)]


def _idct5(d, P):                     # jidctint.c:697-800
    t12 = P.dc(d[0])
    z1 = (d[2] + d[4]) * FIX(0.790569415)
    z2 = (d[2] - d[4]) * FIX(0.353553391)
    z3 = t12 + z2
    t10, t11 = z3 + z1, z3 - z1
    t12 = t12 - (z2 << 2)
    z1 = (d[1] + d[3]) * FIX(0.831253876)
    t0 = z1 + d[1] * FIX(0.513743148)
    t1 = z1 - d[3] * FIX(2.176250899)
    return [P.out(t10 + t0), P.out(t11 + t1), P.out(t12), P.out(t11 - t1), P.out(t10 - t0)]


def _idct6(d, P):                     # jidctint.c:576-690
    t0 = P.dc(d[0])
    t10 = d[4] * FIX(0.707106781)
    t1 = t0 + t10
    t11 = t0 - t10 - t10                       # the middle pair's even part
    t0 = d[2] * FIX(1.224744871)
    t10, t12 = t1 + t0, t1 - t0
    z1, z2, z3 = d[1], d[3], d[5]
    t1 = (z1 + z3) * FIX(0.366025404)
    t0 = t1 + ((z1 + z2) << CONST_BITS)
    t2 = t1 + ((z3 - z2) << CONST_BITS)
    t1 = z1 - z2 - z3                          # the middle pair's odd part, unscaled
    return [P.out(t10 + t0), P.mid(t11, t1), P.out(t12 + t2), P.out(t12 - t2), P.mid(t11, -t1), P.out(t10 - t0)]


def _idct7(d, P):                     # jidctint.c:427-570
    t13 = P.dc(d[0])
    z1, z2, z3 = d[2], d[4], d[6]
    t10 = (z2 - z3) * FIX(0.881747734)
    t12 = (z1 - z2) * FIX(0.314692123)
    t11 = t10 + t12 + t13 - z2 * FIX(1.841218003)
    t0 = z1 + z3
    z2 = z2 - t0
    t0 = t0 * FIX(1.274162392) + t13
    t10 = t10 + t0 - z3 * FIX(0.077722536)
    t12 = t12 + t0 - z1 * FIX(2.470602249)
    t13 = t13 + z2 * FIX(1.414213562)
    z1, z2, z3 = d[1], d[3], d[5]
    t1 = (z1 + z2) * FIX(0.935414347)
    t2 = (z1 - z2) * FIX(0.170262339)
    t0 = t1 - t2
    t1 = t1 + t2
    t2 = (z2 + z3) * -FIX(1.378756276)
    t1 = t1 + t2
    z2 = (z1 + z3) * FIX(0.613604268)
    t0 = t0 + z2
    t2 = t2 + z2 + z3 * FIX(1.870828693)
    return [P.out(t10 + t0), P.out(t11 + t1), P.out(t12 + t2), P.out(t13), P.out(t12 - t2), P.out(t11 - t1), P.out(t10 - t0)]


def _idct9(d, P):                     # jidctint.c:902-1066
    t0 = P.dc(d[0])
    z1, z2, z3 = d[2], d[4], d[6]
    t3 = z3 * FIX(0.707106781)
    t1 = t0 + t3
    t2 = t0 - t3 - t3
    t0 = (z1 - z2) * FIX(0.707106781)
    t11 = t2 + t0
    t14 = t2 - t0 - t0
    t0 = (z1 + z2) * FIX(1.328926049)
    t2 = z1 * FIX(1.083350441)
    t3 = z2 * FIX(0.245575608)
    t10 = t1 + t0 - t3
    t12 = t1 - t0 + t2
    t13 = t1 - t2 + t3
    z1, z2, z3, z4 = d[1], d[3], d[5], d[7]
    z2 = z2 * -FIX(1.224744871)
    t2 = (z1 + z3) * FIX(0.909038955)
    t3 = (z1 + z4) * FIX(0.483689525)
    t0 = t2 + t3 - z2
    t1 = (z3 - z4) * FIX(1.392728481)
    t2 = t2 + z2 - t1
    t3 = t3 + z2 + t1
    t1 = (z1 - z3 - z4) * FIX(1.224744871)
    e, o = [t10, t11, t12, t13], [t0, t1, t2, t3]
    return [P.out(e[i] + o[i]) for i in range(4)] + [P.out(t14)] + [P.out(e[i] - o[i]) for i in (3, 2, 1, 0)]


def _idct10(d, P):                    # jidctint.c:1073-1260
    z3 = P.dc(d[0])
    z1 = d[4] * FIX(1.144122806)
    z2 = d[4] * FIX(0.437016024)
    t10, t11 = z3 + z1, z3 - z2
    t22 = z3 - ((z1 - z2) << 1)                # the middle pair's even part
    z2, z3 = d[2], d[6]
    z1 = (z2 + z3) * FIX(0.831253876)
    t12 = z1 + z2 * FIX(0.513743148)
    t13 = z1 - z3 * FIX(2.176250899)
    t20, t24, t21, t23 = t10 + t12, t10 - t12, t11 + t13, t11 - t13
    z1, z2, z3, z4 = d[1], d[3], d[5], d[7]
    t11, t13 = z2 + z4, z2 - z4
    t12 = t13 * FIX(0.309016994)
    z5 = z3 << CONST_BITS
    z2 = t11 * FIX(0.951056516)
    z4 = z5 + t12
    t10 = z1 * FIX(1.396802247) + z2 + z4
    t14 = z1 * FIX(0.221231742) - z2 + z4
    z2 = t11 * FIX(0.587785252)
    z4 = z5 - t12 - (t13 << (CONST_BITS - 1))
    t12 = z1 - t13 - z3                        # the middle pair's odd part, unscaled
    t11 = z1 * FIX(1.260073511) - z2 - z4
    t13 = z1 * FIX(0.642039522) - z2 + z4
    return [P.out(t20 + t10), P.out(t21 + t11), P.mid(t22, t12), P.out(t23 + t13), P.out(t24 + t14),
            P.out(t24 - t14), P.out(t23 - t13), P.mid(t22, -t12), P.out(t21 - t11), P.out(t20 - t10)]


def _idct11(d, P):                    # jidctint.c:1268-1450
    t10 = P.dc(d[0])
    z1, z2, z3 = d[2], d[4], d[6]
    t20 = (z2 - z3) * FIX(2.546640132)
    t23 = (z2 - z1) * FIX(0.430815045)
    z4 = z1 + z3
    t24 = z4 * -FIX(1.155664402)
    z4 = z4 - z2
    t25 = t10 + z4 * FIX(1.356927976)
    t21 = t20 + t23 + t25 - z2 * FIX(1.821790775)
    t20 = t20 + t25 + z3 * FIX(2.115825087)
    t23 = t23 + t25 - z1 * FIX(1.513598477)
    t24 = t24 + t25
    t22 = t24 - z3 * FIX(0.788749120)
    t24 = t24 + z2 * FIX(1.944413522) - z1 * FIX(1.390975730)
    t25 = t10 - z4 * FIX(1.414213562)
    z1, z2, z3, z4 = d[1], d[3], d[5], d[7]
    t11 = z1 + z2
    t14 = (t11 + z3 + z4) * FIX(0.398430003)
    t11 = t11 * FIX(0.887983902)
    t12 = (z1 + z3) * FIX(0.670361295)
    t13 = t14 + (z1 + z4) * FIX(0.366151574)
    t10 = t11 + t12 + t13 - z1 * FIX(0.923107866)
    z1 = t14 - (z2 + z3) * FIX(1.163011579)
    t11 = t11 + z1 + z2 * FIX(2.073276588)
    t12 = t12 + z1 - z3 * FIX(1.192193623)
    z1 = (z2 + z4) * -FIX(1.798248910)
    t11 = t11 + z1
    t13 = t13 + z1 + z4 * FIX(2.102458632)
    t14 = t14 + z2 * -FIX(1.467221301) + z3 * FIX(1.001388905) - z4 * FIX(1.684843907)
    e, o = [t20, t21, t22, t23, t24], [t10, t11, t12, t13, t14]
    return [P.out(e[i] + o[i]) for i in range(5)] + [P.out(t25)] + [P.out(e[i] - o[i]) for i in (4, 3, 2, 1, 0)]


def _idct12(d, P):                    # jidctint.c:1462-1670
    z3 = P.dc(d[0])
    z4 = d[4] * FIX(1.224744871)
    t10, t11 = z3 + z4, z3 - z4
    z1 = d[2]
    z4 = z1 * FIX(1.366025404)
    z1 = z1 << CONST_BITS
    z2 = d[6] << CONST_BITS
    t12 = z1 - z2
    t21, t24 = z3 + t12, z3 - t12
    t12 = z4 + z2
    t20, t25 = t10 + t12, t10 - t12
    t12 = z4 - z1 - z2
    t22, t23 = t11 + t12, t11 - t12
    z1, z2, z3, z4 = d[1], d[3], d[5], d[7]
    t11 = z2 * FIX(1.306562965)
    t14 = z2 * -FIX(0.541196100)
    t10 = z1 + z3
    t15 = (t10 + z4) * FIX(0.860918669)
    t12 = t15 + t10 * FIX(0.261052384)
    t10 = t12 + t11 + z1 * FIX(0.280143716)
    t13 = (z3 + z4) * -FIX(1.045510580)
    t12 = t12 + t13 + t14 - z3 * FIX(1.478575242)
    t13 = t13 + t15 - t11 + z4 * FIX(1.586706681)
    t15 = t15 + t14 - z1 * FIX(0.676326758) - z4 * FIX(1.982889723)
    z1, z2 = z1 - z4, z2 - z3
    z3 = (z1 + z2) * FIX(0.541196100)
    t11 = z3 + z1 * FIX(0.765366865)
    t14 = z3 - z2 * FIX(1.847759065)
    e, o = [t20, t21, t22, t23, t24, t25], [t10, t11, t12, t13, t14, t15]
    return [P.out(e[i] + o[i]) for i in range(6)] + [P.out(e[i] - o[i]) for i in (5, 4, 3, 2, 1, 0)]


def _idct13(d, P):                    # jidctint.c:1678-1898
    z1 = P.dc(d[0])
    z2, z3, z4 = d[2], d[4], d[6]
    t10, t11 = z3 + z4, z3 - z4
    t12 = t10 * FIX(1.155388986)
    t13 = t11 * FIX(0.096834934) + z1
    t20 = z2 * FIX(1.373119086) + t12 + t13
    t22 = z2 * FIX(0.501487041) - t12 + t13
    t12 = t10 * FIX(0.316450131)
    t13 = t11 * FIX(0.486914739) + z1
    t21 = z2 * FIX(1.058554052) - t12 + t13
    t25 = z2 * -FIX(1.252223920) + t12 + t13
    t12 = t10 * FIX(0.435816023)
    t13 = t11 * FIX(0.937303064) - z1
    t23 = z2 * -FIX(0.170464608) - t12 - t13
    t24 = z2 * -FIX(0.803364869) + t12 - t13
    t26 = (t11 - z2) * FIX(1.414213562) + z1
    z1, z2, z3, z4 = d[1], d[3], d[5], d[7]
    t11 = (z1 + z2) * FIX(1.322312651)
    t12 = (z1 + z3) * FIX(1.163874945)
    t15 = z1 + z4
    t13 = t15 * FIX(0.937797057)
    t10 = t11 + t12 + t13 - z1 * FIX(2.020082300)
    t14 = (z2 + z3) * -FIX(0.338443458)
    t11 = t11 + t14 + z2 * FIX(0.837223564)
    t12 = t12 + t14 - z3 * FIX(1.572116027)
    t14 = (z2 + z4) * -FIX(1.163874945)
    t11 = t11 + t14
    t13 = t13 + t14 + z4 * FIX(2.205608352)
    t14 = (z3 + z4) * -FIX(0.657217813)
    t12 = t12 + t14
    t13 = t13 + t14
    t15 = t15 * FIX(0.338443458)
    t14 = t15 + z1 * FIX(0.318774355) - z2 * FIX(0.466105296)
    z1 = (z3 - z2) * FIX(0.937797057)
    t14 = t14 + z1
    t15 = t15 + z1 + z3 * FIX(0.384515595) - z4 * FIX(1.742345811)
    e, o = [t20, t21, t22, t23, t24, t25], [t10, t11, t12, t13, t14, t15]
    return [P.out(e[i] + o[i]) for i in range(6)] + [P.out(t26)] + [P.out(e[i] - o[i]) for i in (5, 4, 3, 2, 1, 0)]


def _idct14(d, P):                    # jidctint.c:1906-2124
    z1 = P.dc(d[0])
    z4 = d[4]
    z2 = z4 * FIX(1.274162392)
    z3 = z4 * FIX(0.314692123)
    z4 = z4 * FIX(0.881747734)
    t10, t11, t12 = z1 + z2, z1 + z3, z1 - z4
    t23 = z1 - ((z2 + z3 - z4) << 1)           # the middle pair's even part
    z1, z2 = d[2], d[6]
    z3 = (z1 + z2) * FIX(1.105676686)
    t13 = z3 + z1 * FIX(0.273079590)
    t14 = z3 - z2 * FIX(1.719280954)
    t15 = z1 * FIX(0.613604268) - z2 * FIX(1.378756276)
    t20, t26, t21, t25, t22, t24 = t10 + t13, t10 - t13, t11 + t14, t11 - t14, t12 + t15, t12 - t15
    z1, z2, z3, z4 = d[1], d[3], d[5], d[7]
    z4s = z4 << CONST_BITS
    t14 = z1 + z3
    t11 = (z1 + z2) * FIX(1.334852607)
    t12 = t14 * FIX(1.197448846)
    t10 = t11 + t12 + z4s - z1 * FIX(1.126980169)
    t14 = t14 * FIX(0.752406978)
    t16 = t14 - z1 * FIX(1.061150426)
    z1 = z1 - z2
    t15 = z1 * FIX(0.467085129) - z4s
    t16 = t16 + t15
    t13 = (z2 + z3) * -FIX(0.158341681) - z4s
    t11 = t11 + t13 - z2 * FIX(0.424103948)
    t12 = t12 + t13 - z3 * FIX(2.373959773)
    t13 = (z3 - z2) * FIX(1.405321284)
    t14 = t14 + t13 + z4s - z3 * FIX(1.6906431334)
    t15 = t15 + t13 + z2 * FIX(0.674957567)
    t13 = z1 + z4 - z3                         # the middle pair's odd part, unscaled
    e, o = [t20, t21, t22, None, t24, t25, t26], [t10, t11, t12, None, t14, t15, t16]
    return ([P.out(e[i] + o[i]) for i in range(3)] + [P.mid(t23, t13)] + [P.out(e[i] + o[i]) for i in range(4, 7)] +
            [P.out(e[i] - o[i]) for i in (6, 5, 4)] + [P.mid(t23, -t13)] + [P.out(e[i] - o[i]) for i in (2, 1, 0)])


def _idct15(d, P):                    # jidctint.c:2132-2366
    z1 = P.dc(d[0])
    z2, z3, z4 = d[2], d[4], d[6]
    t10 = z4 * FIX(0.437016024)
    t11 = z4 * FIX(1.144122806)
    t12, t13 = z1 - t10, z1 + t11
    z1 = z1 - ((t11 - t10) << 1)
    z4 = z2 - z3
    z3 = z3 + z2
    t10 = z3 * FIX(1.337628990)
    t11 = z4 * FIX(0.045680613)
    z2 = z2 * FIX(1.439773946)
    t20 = t13 + t10 + t11
    t23 = t12 - t10 + t11 + z2
    t10 = z3 * FIX(0.547059574)
    t11 = z4 * FIX(0.399234004)
    t25 = t13 - t10 - t11
    t26 = t12 + t10 - t11 - z2
    t10 = z3 * FIX(0.790569415)
    t11 = z4 * FIX(0.353553391)
    t21 = t12 + t10 + t11
    t24 = t13 - t10 + t11
    t11 = t11 + t11
    t22 = z1 + t11
    t27 = z1 - t11 - t11
    z1, z2 = d[1], d[3]
    z3 = d[5] * FIX(1.224744871)
    z4 = d[7]
    t13 = z2 - z4
    t15 = (z1 + t13) * FIX(0.831253876)
    t11 = t15 + z1 * FIX(0.513743148)
    t14 = t15 - t13 * FIX(2.176250899)
    t13 = z2 * -FIX(0.831253876)
    t15 = z2 * -FIX(1.344997024)
    z2 = z1 - z4
    t12 = z3 + z2 * FIX(1.406466353)
    t10 = t12 + z4 * FIX(2.457431844) - t15
    t16 = t12 - z1 * FIX(1.112434820) + t13
    t12 = z2 * FIX(1.224744871) - z3
    z2 = (z1 + z4) * FIX(0.575212477)
    t13 = t13 + z2 + z1 * FIX(0.475753014) - z3
    t15 = t15 + z2 - z4 * FIX(0.869244010) + z3
    e, o = [t20, t21, t22, t23, t24, t25, t26], [t10, t11, t12, t13, t14, t15, t16]
    return [P.out(e[i] + o[i]) for i in range(7)] + [P.out(t27)] + [P.out(e[i] - o[i]) for i in (6, 5, 4, 3, 2, 1, 0)]


def _idct16(d, P):                    # jidctint.c:2374-2625
    t0 = P.dc(d[0])
    t1 = d[4] * FIX(1.306562965)
    t2 = d[4] * FIX(0.541196100)
    t10, t11, t12, t13 = t0 + t1, t0 - t1, t0 + t2, t0 - t2
    z1, z2 = d[2], d[6]
    z3 = z1 - z2
    z4 = z3 * FIX(0.275899379)
    z3 = z3 * FIX(1.387039845)
    t0 = z3 + z2 * FIX(2.562915447)
    t1 = z4 + z1 * FIX(0.899976223)
    t2 = z3 - z1 * FIX(0.601344887)
    t3 = z4 - z2 * FIX(0.509795579)
    t20, t27, t21, t26 = t10 + t0, t10 - t0, t12 + t1, t12 - t1
    t22, t25, t23, t24 = t13 + t2, t13 - t2, t11 + t3, t11 - t3
    z1, z2, z3, z4 = d[1], d[3], d[5], d[7]
    t11 = z1 + z3
    t1 = (z1 + z2) * FIX(1.353318001)
    t2 = t11 * FIX(1.247225013)
    t3 = (z1 + z4) * FIX(1.093201867)
    t10 = (z1 - z4) * FIX(0.897167586)
    t11 = t11 * FIX(0.666655658)
    t12 = (z1 - z2) * FIX(0.410524528)
    t0 = t1 + t2 + t3 - z1 * FIX(2.286341144)
    t13 = t10 + t11 + t12 - z1 * FIX(1.835730603)
    z1 = (z2 + z3) * FIX(0.138617169)
    t1 = t1 + z1 + z2 * FIX(0.071888074)
    t2 = t2 + z1 - z3 * FIX(1.125726048)
    z1 = (z3 - z2) * FIX(1.407403738)
    t11 = t11 + z1 - z3 * FIX(0.766367282)
    t12 = t12 + z1 + z2 * FIX(1.971951411)
    z2 = z2 + z4
    z1 = z2 * -FIX(0.666655658)
    t1 = t1 + z1
    t3 = t3 + z1 + z4 * FIX(1.065388962)
    z2 = z2 * -FIX(1.247225013)
    t10 = t10 + z2 + z4 * FIX(3.141271809)
    t12 = t12 + z2
    z2 = (z3 + z4) * -FIX(1.353318001)
    t2 = t2 + z2
    t3 = t3 + z2
    z2 = (z4 - z3) * FIX(0.410524528)
    t10 = t10 + z2
    t11 = t11 + z2
    e, o = [t20, t21, t22, t23, t24, t25, t26, t27], [t0, t1, t2, t3, t10, t11, t12, t13]
    return [P.out(e[i] + o[i]) for i in range(8)] + [P.out(e[i] - o[i]) for i in range(7, -1, -1)]


IDCT_1D = {3: _idct3, 5: _idct5, 6: _idct6, 7: _idct7, 9: _idct9, 10: _idct10, 11: _idct11, 12: _idct12, 13: _idct13,
           14: _idct14, 15: _idct15, 16: _idct16}


def n_in(n):
    """inputs of each 1-D pass of size n: N below 8, 8 above"""
    return n if n < 8 else 8


def idct_scaled(coef, q, n):
    """jpeg_idct_NxN on blocks: coef [B, 64] natural-order int16 coefficients, q [64] or [B, 64] table entries (taken as
    unsigned 16-bit values, as ISLOW_MULT_TYPE int dequantizes them) -> [B, n, n] uint8 samples"""
    coef = np.asarray(coef, np.int64).reshape(-1, 8, 8)
    q = np.broadcast_to(np.asarray(q, np.int64).reshape(-1, 8, 8) & 0xFFFF, coef.shape)
    dq = coef * q                                             # DEQUANTIZE: an int product, which cannot overflow here
    m = n_in(n)
    f = IDCT_1D[n]
    ws = [f([dq[:, r, c] for r in range(m)], _Pass(1)) for c in range(m)]        # ws[col][row]
    out = np.empty((coef.shape[0], n, n), np.uint8)
    lim = R._range_limit_table()
    for r in range(n):
        row = f([ws[c][r] for c in range(m)], _Pass(2))
        for x in range(n):
            out[:, r, x] = lim[row[x] & 1023]
    return out


class _Lin:
    """a linear form sum_j c[j] * in[j] + k with rational coefficients: >> divides, << multiplies"""

    def __init__(self, c, k=Fraction(0)):
        self.c, self.k = c, k

    def _lin(self, o):
        return o if isinstance(o, _Lin) else _Lin({}, Fraction(o))

    def __add__(self, o):
        o = self._lin(o)
        c = dict(self.c)
        for j, v in o.c.items():
            c[j] = c.get(j, 0) + v
        return _Lin(c, self.k + o.k)

    __radd__ = __add__

    def __neg__(self):
        return _Lin({j: -v for j, v in self.c.items()}, -self.k)

    def __sub__(self, o):
        return self + -self._lin(o)

    def __rsub__(self, o):
        return self._lin(o) - self

    def __mul__(self, s):
        assert isinstance(s, int)
        return _Lin({j: v * s for j, v in self.c.items()}, self.k * s)

    __rmul__ = __mul__

    def __lshift__(self, s):
        return self * (1 << s)

    def __rshift__(self, s):
        return _Lin({j: v / (1 << s) for j, v in self.c.items()}, self.k / (1 << s))


def pass_matrix(n, p):
    """pass p (1 or 2) of size n as (m, s): output o = (sum_j m[o][j] * in[j] + 2^(s-1)) >> s"""
    P = _Pass(p)
    outs = IDCT_1D[n]([_Lin({j: Fraction(1)}) for j in range(n_in(n))], P)
    m = []
    for f in outs:
        k = f.k * (1 << P.shift)
        assert k == 1 << (P.shift - 1), (n, p, k)
        row = [f.c.get(j, Fraction(0)) * (1 << P.shift) for j in range(n_in(n))]
        assert all(v.denominator == 1 for v in row), (n, p, row)
        m.append([int(v) for v in row])
    return m, P.shift


def idct_by_matrix(coef, q, n):
    """idct_scaled through pass_matrix, the form the kernels evaluate: pass 1 in 64 bits to an int workspace, pass 2
    modulo 2^32"""
    coef = np.asarray(coef, np.int64).reshape(-1, 8, 8)
    q = np.broadcast_to(np.asarray(q, np.int64).reshape(-1, 8, 8) & 0xFFFF, coef.shape)
    dq = coef * q
    m = n_in(n)
    m1, s1 = pass_matrix(n, 1)
    m2, s2 = pass_matrix(n, 2)
    m1, m2 = np.array(m1, np.int64), np.array(m2, np.int64)
    # ws[b, c, r]: column c's output r
    ws = (np.einsum("rj,bjc->bcr", m1, dq[:, :m, :m]) + (1 << (s1 - 1))) >> s1
    ws = ws.astype(np.int32).astype(np.int64)
    # pass 2: row r of the block takes ws[:, 0..m-1, r]
    acc = np.einsum("xj,bjr->brx", m2, ws).astype(np.uint64).astype(np.uint32).astype(np.int64)
    acc = (acc + (1 << (s2 - 1))) & 0xFFFFFFFF
    return R._range_limit_table()[(acc >> s2) & 1023].astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------- cases
LAYOUT_IDS = [c[0] for c in O.LAYOUTS]                           # gray, 4:4:4, 4:2:2, 4:4:0, 4:2:0, RGB
CONTENT = ("q5", "q100", "q100_noise", "sof1_dqt16", "idct_q1", "idct_q255", "idct_q32767", "restart_1", "multi_scan")
LADDER = [(1, 1), (3, 4), (3, 8)]


def cases():
    """[(id, source id, (num, denom), dct, fancy, colorspace name or None)], ids as decompress_options_cases.case_id"""
    out = []

    def add(sid, scale, dct="int", fancy=True, cs=None):
        cid = O.case_id(sid, scale, dct, fancy, cs)
        if cid not in {c[0] for c in out}:
            out.append((cid, sid, scale, dct, fancy, cs))
    # every block size for every layout, fancy on and off; the three methods, which the new sizes never use
    for sid in LAYOUT_IDS:
        for k in range(1, 17):
            for fancy in (True, False):
                add(sid, (k, 8), "int", fancy)
        for k in NEW_SIZES:
            for dct in ("fast", "float"):
                add(sid, (k, 8), dct, True)
    # output colour spaces at new sizes
    for cs in ("gray", "rgb", "bgrx", "xbgr", "ycbcr"):
        add("o_420", (3, 4), "int", True, cs)
        add("o_422", (5, 4), "int", False, cs)
    for cs in ("rgb", "argb"):
        add("o_gray", (7, 8), "int", True, cs)
    # content: coefficient and table limits, restarts, several scans, at every new size
    for sid in CONTENT:
        for k in NEW_SIZES:
            add(sid, (k, 8), "int", True)
    # fractions the reference buckets into other sizes, and the 4K frame
    add("o_420", (5, 12)); add("o_422", (7, 16), "fast"); add("o_444", (11, 16)); add("o_420", (3, 2), "float", False)
    add("o_440", (9, 7)); add("o_rgb", (13, 9))
    add("o_4k", (3, 4)); add("o_4k", (3, 8), "int", False); add("o_4k", (2, 1))
    return out


# TurboJPEG scaling factors whose block sizes are new, and the layouts of yuv_decode_cases
TJ_NEW = [(2, 1), (15, 8), (7, 4), (13, 8), (3, 2), (11, 8), (5, 4), (9, 8), (7, 8), (3, 4), (5, 8), (3, 8)]
YUV_SOURCES = ("y_gray", "y_444", "y_422", "y_420", "y_440", "y_411", "y_441")
# (source, factor, dct): every new factor for every layout with JDCT_ISLOW, and TJPARAM_FASTDCT at a few, where the new
# sizes still read the islow-style table (4:2:0 chroma included: TurboJPEG runs luma's IDCT on it)
YUV_CASES = [(s, f, "int") for s in YUV_SOURCES for f in TJ_NEW] + \
            [("y_420", f, "fast") for f in ((3, 8), (3, 4), (5, 4), (2, 1))] + [("y_422", (7, 8), "fast"), ("y_gray", (15, 8), "fast")]


def golden():
    return json.load(open(GOLDEN))

