"""GPU: the DiffNet sampler (the step kernel k_hp_step, the fp32 SIMT path and the sampling loops around them) at the
edges of every configuration dsx_load_diffnet accepts, against diffnet_oracle in float64 on the CPU.

Each case builds dsx.DiffNet from a seeded state dict and runs the public DsxSampler.  Single evaluations run a batch
with a different t per utterance (0, 37, 99 of a 100-step schedule).  The edges:

  * T 1, 8, 9 (below and at the 8-frame halo), 63 / 64 / 65, 127 / 128 / 129 and 136 / 137 at dilation cycle 4: halo
    rows wholly outside the utterance, a 64-frame tile without a real frame (T <= 64 pads to 128), a last tile of 1 or 8
    frames;
  * (L, cycle) (1, 1), (1, 4), (2, 4), (3, 4), (5, 3), (7, 2), (31, 4) and (20, 1..4): odd L, L below the cycle, L not
    a multiple of the cycle;
  * B 1 (no partner utterance), 2 and 3 (one utterance without a partner); x and cond as transposed views;
  * the residency boundaries of the stack form, derived from DSX_INFO_SM_COUNT and DSX_INFO_CLUSTER_OCCUPANCY at
    T = 64 (128 padded frames): the last B that the automatic choice keeps at 64-frame tiles, one more (128-frame
    tiles), the last B with a 128-frame CTA per tile (utterances paired), one more (no pairing; CTA 0 walks a second
    tile);
  * DDPM and PLMS loops with every number of steps that changes what the fused head does (PLMS modes 0-4, the warm-up's
    second evaluation at table row n), and dsx_infer with K_step = 1 from a shallow and from a gaussian start;
  * the fp32 SIMT path at M > 2 C (the head's output projection is wider than a layer's GEMM rows), M = 16, M = 768
    (the largest it takes), dilation cycle 24, L = 1.

Every case runs in each form it can take (FORMS): the stack form of fp16, fp16x2 and fp16s at 64- and at 128-frame
tiles, fp16x2 in the hi / lo form (DSX_OPT_STACK_KERNEL = 0) and with one launch per layer (DSX_OPT_STACK_MODE = 0),
fp16x2 with the exact gate (DSX_OPT_GATE_APPROX = 0; the stack form's default is 1), fp16x3 (the two-stage ring without
the window) and fp32 SIMT.

Bounds.  Every bound is max(4 x sim, floor), where sim is the max error of diffnet_oracle's operand-format simulation
(fmt=) against float64 on the same case; fp16s takes the worst of three CPU draws of the stochastic weight sets (the
GPU's come from k_pack_wsr's own seed).  The floors hold the rounding the simulation leaves out (fp32 accumulation, the
tanh.approx gate): fp16 / fp16s 2e-4, fp16x2 1e-4, fp16x3 2e-5, fp32 1e-5.  fp32's sim is the fp32 oracle against
float64.  Single evaluations are max |eps| errors; loops are max |x| errors over max(1, max |x_ref|), the relative
bound test_plms_golden uses where the untrained PLMS state grows; dsx_infer is in the denormalised mel domain.  A
residency boundary takes the bound of the T = 64 case.  SIM holds the simulated errors; the bounds, per case and
format (fp16 / fp16x2 / fp16x3 / fp16s, then fp32), are:

    T1                           1.1e-03 / 5.5e-04 / 2.0e-05 / 1.0e-03  1.0e-05
    T8                           1.7e-03 / 8.7e-04 / 2.0e-05 / 1.5e-03  1.0e-05
    T9                           1.8e-03 / 8.7e-04 / 2.0e-05 / 1.5e-03  1.0e-05
    T63                          2.1e-03 / 1.0e-03 / 2.0e-05 / 2.0e-03  1.0e-05
    T64                          2.0e-03 / 1.1e-03 / 2.0e-05 / 2.0e-03  1.0e-05
    T65                          2.0e-03 / 1.1e-03 / 2.0e-05 / 2.2e-03  1.0e-05
    T127                         2.7e-03 / 1.2e-03 / 2.0e-05 / 2.0e-03  1.0e-05
    T128                         2.0e-03 / 1.1e-03 / 2.0e-05 / 2.2e-03  1.0e-05
    T129                         2.2e-03 / 1.4e-03 / 2.0e-05 / 2.2e-03  1.0e-05
    T136                         2.1e-03 / 1.1e-03 / 2.0e-05 / 2.3e-03  1.0e-05
    T137                         2.2e-03 / 1.2e-03 / 2.0e-05 / 2.2e-03  1.0e-05
    L1_cycle1                    2.4e-03 / 1.0e-03 / 2.0e-05 / 2.0e-03  1.0e-05
    L1_cycle4                    2.5e-03 / 1.0e-03 / 2.0e-05 / 2.1e-03  1.0e-05
    L2_cycle4                    2.2e-03 / 1.4e-03 / 2.0e-05 / 1.8e-03  1.0e-05
    L3_cycle4                    2.8e-03 / 1.0e-03 / 2.0e-05 / 2.2e-03  1.0e-05
    L5_cycle3                    2.2e-03 / 1.0e-03 / 2.0e-05 / 1.9e-03  1.0e-05
    L7_cycle2                    2.4e-03 / 1.2e-03 / 2.0e-05 / 2.2e-03  1.0e-05
    L31_cycle4                   2.2e-03 / 1.2e-03 / 2.0e-05 / 2.5e-03  1.0e-05
    L20_cycle1                   2.3e-03 / 1.2e-03 / 2.0e-05 / 2.5e-03  1.0e-05
    L20_cycle2                   2.2e-03 / 1.1e-03 / 2.0e-05 / 2.1e-03  1.0e-05
    L20_cycle3                   2.2e-03 / 1.2e-03 / 2.0e-05 / 2.3e-03  1.0e-05
    L20_cycle4                   2.3e-03 / 1.2e-03 / 2.0e-05 / 2.0e-03  1.0e-05
    B1                           2.2e-03 / 1.1e-03 / 2.0e-05 / 2.2e-03  1.0e-05
    B2                           2.1e-03 / 1.1e-03 / 2.0e-05 / 2.3e-03  1.0e-05
    strided_T1                   1.2e-03 / 5.5e-04 / 2.0e-05 / 1.2e-03  1.0e-05
    strided_T129                 2.0e-03 / 1.1e-03 / 2.0e-05 / 2.3e-03  1.0e-05
    L3_T129_ddpm_1_1             2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_ddpm_8_8             3.2e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_ddpm_100_3           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_plms_25_40           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_plms_41_40           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_plms_81_40           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_plms_121_40          2.2e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_plms_97_20           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_plms_6_1             2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_infer_shallow        2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L3_T129_infer_gaussian       2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_ddpm_1_1             2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_ddpm_8_8             3.4e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_ddpm_100_3           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_plms_25_40           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_plms_41_40           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_plms_81_40           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_plms_121_40          2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_plms_97_20           2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_plms_6_1             2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_infer_shallow        2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    L20_T65_infer_gaussian       2.0e-04 / 1.0e-04 / 2.0e-05 / 2.0e-04  1.0e-05
    M80_C16_H16                  1.0e-05
    M80_C32_H48                  1.0e-05
    M128_C48_H16                 1.0e-05
    M16_C16_H16                  1.0e-05
    M128_C64_H256                1.0e-05
    M768_C32_H16                 1.0e-05
    cycle24_L24_T300             1.0e-05
    L1                           1.0e-05

Exact properties, bit for bit in every form: an utterance's eps in a batch of mixed t equals its eps in a batch where
every t is its own; permuting the utterances permutes eps; a repeated call returns the same; an utterance at a
residency boundary gives what it gives alone.  dsx_load_diffnet refuses, with DsxError naming the limit, the
tensor-core precisions at M 128, C 128 or cycle 5 and the fp32 path at M 784 or C 2464.
Run on an H100: python -m pytest tests -m gpu -k diffnet_edges"""
import collections
import functools

import pytest
import torch

from conftest import rs_normal
from oracle import diffnet_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
T_UTT = (0, 37, 99)
FLOOR = {"fp16": 2e-4, "fp16x2": 1e-4, "fp16x3": 2e-5, "fp16s": 2e-4, "fp32": 1e-5}
FMTS = ("fp16", "fp16x2", "fp16x3", "fp16s")
SR_DRAWS = (0, 1000, 2000)


def bound(sim, fmt):
    return max(FLOOR[fmt], float(f"{4 * sim:.1e}"))


# ---- cases --------------------------------------------------------------------------------------------------------
def fwd_cases():
    c = {}
    for T in (1, 8, 9, 63, 64, 65, 127, 128, 129, 136, 137):
        c[f"T{T}"] = dict(L=20, cycle=4, B=3, T=T)
    for L, cyc in ((1, 1), (1, 4), (2, 4), (3, 4), (5, 3), (7, 2), (31, 4), (20, 1), (20, 2), (20, 3), (20, 4)):
        c[f"L{L}_cycle{cyc}"] = dict(L=L, cycle=cyc, B=3, T=100)
    for B in (1, 2):
        c[f"B{B}"] = dict(L=20, cycle=4, B=B, T=100)
    for T in (1, 129):
        c[f"strided_T{T}"] = dict(L=20, cycle=4, B=3, T=T, strided=True)
    return c


FWD = fwd_cases()
LOOP_SHAPES = {"L3_T129": (3, 129), "L20_T65": (20, 65)}
# DDPM (t_start, n_steps): one step; eight, the last at t = 0 (sigma 0, clamp); three from the top of the schedule.
# PLMS (t_start, interval): 1, 2, 3 and 4 steps; t_start not a multiple of the interval; six steps of 1.
LOOPS = {"ddpm_1_1": ("ddpm", 1, 1), "ddpm_8_8": ("ddpm", 8, 8), "ddpm_100_3": ("ddpm", 100, 3),
         "plms_25_40": ("plms", 25, 40), "plms_41_40": ("plms", 41, 40), "plms_81_40": ("plms", 81, 40),
         "plms_121_40": ("plms", 121, 40), "plms_97_20": ("plms", 97, 20), "plms_6_1": ("plms", 6, 1),
         "infer_shallow": ("infer", 1, 0), "infer_gaussian": ("infer", 1, 0)}
LOOP_CASES = {f"{s}_{lp}": (s, lp) for s in LOOP_SHAPES for lp in LOOPS}
# fp32 SIMT: (M, C, H, L, cycle, T)
SIMT = {"M80_C16_H16": (80, 16, 16, 3, 1, 100), "M80_C32_H48": (80, 32, 48, 3, 2, 100),
        "M128_C48_H16": (128, 48, 16, 3, 4, 100), "M16_C16_H16": (16, 16, 16, 3, 1, 100),
        "M128_C64_H256": (128, 64, 256, 3, 1, 100), "M768_C32_H16": (768, 32, 16, 2, 1, 40),
        "cycle24_L24_T300": (80, 64, 64, 24, 24, 300), "L1": (80, 64, 64, 1, 1, 100)}

# form -> (precision, options, simulated format)
FORMS = {
    "fp16_stack64": ("fp16", (("OPT_STACK_ROWS", 64),), "fp16"),
    "fp16_stack128": ("fp16", (("OPT_STACK_ROWS", 128),), "fp16"),
    "fp16x2_stack64": ("fp16x2", (("OPT_STACK_ROWS", 64),), "fp16x2"),
    "fp16x2_stack128": ("fp16x2", (("OPT_STACK_ROWS", 128),), "fp16x2"),
    "fp16s_stack64": ("fp16s", (("OPT_STACK_ROWS", 64),), "fp16s"),
    "fp16s_stack128": ("fp16s", (("OPT_STACK_ROWS", 128),), "fp16s"),
    "fp16x2_hilo": ("fp16x2", (("OPT_STACK_KERNEL", 0),), "fp16x2"),
    "fp16x2_per_layer": ("fp16x2", (("OPT_STACK_MODE", 0),), "fp16x2"),
    "fp16x2_gate_exact": ("fp16x2", (("OPT_GATE_APPROX", 0),), "fp16x2"),
    "fp16x3": ("fp16x3", (), "fp16x3"),
    "fp32": ("fp32", (), "fp32"),
}
# the automatic tile height, for the residency boundaries only
AUTO_FORMS = {"fp16x2_auto": ("fp16x2", (), "fp16x2"), "fp16s_auto": ("fp16s", (), "fp16s")}

# Simulated max errors against float64 (python -m oracle.diffnet_edge_sensitivity --sim prints them): per case,
# fp16 / fp16x2 / fp16x3 / fp16s (worst of SR_DRAWS) / fp32
SIM = {
    "T1": (2.83e-04, 1.38e-04, 5.08e-07, 2.53e-04, 4.50e-07),
    "T8": (4.15e-04, 2.17e-04, 6.99e-07, 3.84e-04, 4.83e-07),
    "T9": (4.44e-04, 2.18e-04, 5.85e-07, 3.83e-04, 5.14e-07),
    "T63": (5.28e-04, 2.49e-04, 8.06e-07, 5.06e-04, 5.54e-07),
    "T64": (4.99e-04, 2.64e-04, 9.48e-07, 4.90e-04, 5.47e-07),
    "T65": (5.09e-04, 2.67e-04, 7.88e-07, 5.54e-04, 6.08e-07),
    "T127": (6.76e-04, 3.02e-04, 8.73e-07, 4.99e-04, 5.52e-07),
    "T128": (5.00e-04, 2.87e-04, 7.86e-07, 5.43e-04, 7.02e-07),
    "T129": (5.50e-04, 3.51e-04, 8.55e-07, 5.59e-04, 5.93e-07),
    "T136": (5.26e-04, 2.73e-04, 9.61e-07, 5.71e-04, 7.10e-07),
    "T137": (5.62e-04, 3.11e-04, 8.21e-07, 5.57e-04, 5.76e-07),
    "L1_cycle1": (6.09e-04, 2.57e-04, 9.54e-07, 4.96e-04, 6.33e-07),
    "L1_cycle4": (6.29e-04, 2.52e-04, 8.35e-07, 5.22e-04, 5.36e-07),
    "L2_cycle4": (5.60e-04, 3.43e-04, 9.26e-07, 4.57e-04, 5.67e-07),
    "L3_cycle4": (6.94e-04, 2.56e-04, 7.90e-07, 5.46e-04, 6.65e-07),
    "L5_cycle3": (5.50e-04, 2.52e-04, 9.80e-07, 4.86e-04, 5.64e-07),
    "L7_cycle2": (5.96e-04, 3.03e-04, 7.93e-07, 5.49e-04, 5.54e-07),
    "L31_cycle4": (5.55e-04, 3.08e-04, 8.00e-07, 6.13e-04, 5.82e-07),
    "L20_cycle1": (5.87e-04, 2.88e-04, 8.15e-07, 6.29e-04, 7.43e-07),
    "L20_cycle2": (5.40e-04, 2.68e-04, 9.06e-07, 5.29e-04, 7.36e-07),
    "L20_cycle3": (5.62e-04, 3.04e-04, 7.64e-07, 5.84e-04, 5.83e-07),
    "L20_cycle4": (5.72e-04, 2.88e-04, 7.47e-07, 5.01e-04, 5.75e-07),
    "B1": (5.51e-04, 2.65e-04, 7.79e-07, 5.43e-04, 5.37e-07),
    "B2": (5.31e-04, 2.67e-04, 8.11e-07, 5.65e-04, 5.63e-07),
    "strided_T1": (2.90e-04, 1.37e-04, 4.85e-07, 2.91e-04, 3.48e-07),
    "strided_T129": (5.05e-04, 2.67e-04, 9.25e-07, 5.80e-04, 6.09e-07),
    "L3_T129_ddpm_1_1": (5.41e-06, 2.64e-06, 8.40e-09, 5.57e-06, 6.08e-08),
    "L3_T129_ddpm_8_8": (8.09e-05, 2.00e-05, 1.64e-07, 3.55e-05, 3.42e-07),
    "L3_T129_ddpm_100_3": (1.94e-05, 6.64e-06, 4.62e-08, 1.33e-05, 1.46e-07),
    "L3_T129_plms_25_40": (1.07e-06, 3.99e-07, 2.08e-09, 8.14e-07, 2.64e-08),
    "L3_T129_plms_41_40": (1.71e-05, 6.53e-06, 3.20e-08, 1.32e-05, 8.54e-08),
    "L3_T129_plms_81_40": (3.18e-05, 1.18e-05, 5.06e-08, 2.55e-05, 8.03e-08),
    "L3_T129_plms_121_40": (5.60e-05, 1.50e-05, 8.94e-08, 2.89e-05, 9.87e-08),
    "L3_T129_plms_97_20": (3.99e-05, 1.28e-05, 5.49e-08, 2.42e-05, 1.34e-07),
    "L3_T129_plms_6_1": (4.51e-06, 1.97e-06, 6.42e-09, 4.21e-06, 1.32e-07),
    "L3_T129_infer_shallow": (2.77e-06, 1.18e-06, 4.16e-09, 2.55e-06, 1.57e-07),
    "L3_T129_infer_gaussian": (2.78e-06, 1.66e-06, 5.07e-09, 2.65e-06, 1.02e-07),
    "L20_T65_ddpm_1_1": (5.41e-06, 2.84e-06, 7.55e-09, 5.43e-06, 5.96e-08),
    "L20_T65_ddpm_8_8": (8.61e-05, 2.26e-05, 1.65e-07, 4.45e-05, 3.48e-07),
    "L20_T65_ddpm_100_3": (2.25e-05, 7.02e-06, 3.17e-08, 1.06e-05, 1.36e-07),
    "L20_T65_plms_25_40": (1.18e-06, 4.93e-07, 2.01e-09, 9.85e-07, 2.91e-08),
    "L20_T65_plms_41_40": (1.44e-05, 5.90e-06, 2.73e-08, 1.08e-05, 5.74e-08),
    "L20_T65_plms_81_40": (3.84e-05, 1.41e-05, 5.62e-08, 2.58e-05, 1.00e-07),
    "L20_T65_plms_121_40": (3.95e-05, 1.44e-05, 7.52e-08, 3.30e-05, 1.23e-07),
    "L20_T65_plms_97_20": (3.65e-05, 1.33e-05, 5.83e-08, 2.49e-05, 1.19e-07),
    "L20_T65_plms_6_1": (4.37e-06, 2.02e-06, 5.86e-09, 3.43e-06, 1.24e-07),
    "L20_T65_infer_shallow": (2.64e-06, 1.47e-06, 4.06e-09, 2.57e-06, 1.90e-07),
    "L20_T65_infer_gaussian": (3.10e-06, 1.52e-06, 4.15e-09, 3.29e-06, 1.11e-07),
    "M80_C16_H16": (0, 0, 0, 0, 1.25e-07),
    "M80_C32_H48": (0, 0, 0, 0, 1.37e-07),
    "M128_C48_H16": (0, 0, 0, 0, 2.14e-07),
    "M16_C16_H16": (0, 0, 0, 0, 7.28e-08),
    "M128_C64_H256": (0, 0, 0, 0, 2.17e-07),
    "M768_C32_H16": (0, 0, 0, 0, 1.39e-07),
    "cycle24_L24_T300": (0, 0, 0, 0, 1.74e-07),
    "L1": (0, 0, 0, 0, 2.00e-07),
}


@functools.lru_cache(maxsize=None)
def state_dict(L, cycle, M=80, C=256, H=256):
    return O.build_state_dict(0, M, C, H, L, cycle)


def f64(sd):
    return {k: v.double() for k, v in sd.items()}


def fwd_inputs(name):
    c = FWD[name]
    B, T = c["B"], c["T"]
    seed = 100 + list(FWD).index(name)
    if c.get("strided"):
        spec = rs_normal(seed, (B, T, 80)).transpose(1, 2)[:, None]
        cond = rs_normal(seed + 50, (B, T, 256)).transpose(1, 2)
    else:
        spec, cond = rs_normal(seed, (B, 1, 80, T)), rs_normal(seed + 50, (B, 256, T))
    t = torch.tensor(T_UTT[:B] if B > 1 else (37,))
    return spec, t, cond


def schedule(n):
    return O.make_schedule(O.linear_beta_schedule(100, 0.06) if n == 100 else O.linear_beta_schedule(1000, 0.02))


def loop_inputs(name):
    shape, loop = LOOP_CASES[name]
    L, T = LOOP_SHAPES[shape]
    kind, a, b = LOOPS[loop]
    seed = 300 + list(LOOP_CASES).index(name)
    B, M = 2, 80
    inp = dict(L=L, T=T, kind=kind, a=a, b=b, xT=rs_normal(seed, (B, 1, M, T)), cond=rs_normal(seed + 1, (B, 256, T)))
    if kind == "ddpm":
        inp["noise"] = rs_normal(seed + 2, (b, B, 1, M, T))
    if kind == "infer":
        inp["smin"], inp["smax"] = torch.full((M,), -5.0), torch.full((M,), 0.5)
        inp["fs2_mel"] = rs_normal(seed + 3, (B, T, M)) - 2.0
        inp["start_noise"], inp["step_noise"] = rs_normal(seed + 4, (B, 1, M, T)), rs_normal(seed + 5, (1, B, 1, M, T))
        m2p = torch.arange(1, T + 1).repeat(B, 1)
        m2p[0, T // 3:T // 2] = 0                   # frames without a phoneme: masked to 0
        m2p[1, T - 7:] = 0
        inp["mel2ph"] = m2p
        inp["gaussian"] = loop == "infer_gaussian"
    return inp


def run_oracle_loop(sd, inp, fmt=None):
    """the float64 (fmt None) or simulated loop of case `inp`; sd in the dtype the computation runs in"""
    S = schedule(1000 if inp["kind"] == "plms" else 100)
    S = {k: v.to(next(iter(sd.values())).dtype) for k, v in S.items()}
    dt = S["betas"].dtype
    xT, cond = inp["xT"].to(dt), inp["cond"].to(dt)
    with torch.no_grad():
        if inp["kind"] == "ddpm":
            return O.sample_ddpm(sd, S, xT, cond, inp["a"], inp["noise"].to(dt), 4, fmt=fmt, n_steps=inp["b"])
        if inp["kind"] == "plms":
            return O.sample_plms(sd, S, xT, cond, inp["a"], inp["b"], 4, fmt=fmt)
        kw = dict(x_start=xT) if inp["gaussian"] else dict(fs2_mel=inp["fs2_mel"].to(dt),
                                                          start_noise=inp["start_noise"].to(dt))
        return O.infer_loop(sd, S, cond, 1, inp["smin"].to(dt)[None, None], inp["smax"].to(dt)[None, None],
                            step_noise=inp["step_noise"].to(dt), mel2ph=inp["mel2ph"], dilation_cycle_length=4,
                            fmt=fmt, **kw)


def loop_error(out, ref):
    ref = ref.double()
    return ((out.double() - ref).abs().max() / max(1.0, ref.abs().max().item())).item()


def simt_inputs(name):
    M, C, H, L, cyc, T = SIMT[name]
    seed = 500 + list(SIMT).index(name)
    return rs_normal(seed, (3, 1, M, T)), torch.tensor(T_UTT), rs_normal(seed + 1, (3, H, T))


# ---- float64 references, once per case --------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def fwd_ref(name):
    c = FWD[name]
    spec, t, cond = fwd_inputs(name)
    with torch.no_grad():
        return O.diffnet_forward(f64(state_dict(c["L"], c["cycle"])), spec.double(), t, cond.double(), c["cycle"])


@functools.lru_cache(maxsize=None)
def loop_ref(name):
    inp = loop_inputs(name)
    return run_oracle_loop(f64(state_dict(inp["L"], 4)), inp)


@functools.lru_cache(maxsize=None)
def simt_ref(name):
    M, C, H, L, cyc, T = SIMT[name]
    spec, t, cond = simt_inputs(name)
    with torch.no_grad():
        return O.diffnet_forward(f64(state_dict(L, cyc, M, C, H)), spec.double(), t, cond.double(), cyc)


# ---- samplers -----------------------------------------------------------------------------------------------------
_SAMPLERS = collections.OrderedDict()


def sampler(form, L, cycle, M=80, C=256, H=256):
    """a DsxSampler of `form` on the seeded model; the few most recent stay loaded"""
    import diffsinger_b200 as dsx
    from diffsinger_b200 import _capi
    key = (form, L, cycle, M, C, H)
    if key in _SAMPLERS:
        _SAMPLERS.move_to_end(key)
        return _SAMPLERS[key]
    while len(_SAMPLERS) >= 3:
        _SAMPLERS.popitem(last=False)[1].close()
    prec, opts, _ = {**FORMS, **AUTO_FORMS}[form]
    net = dsx.DiffNet(M, hparams=dict(hidden_size=H, residual_layers=L, residual_channels=C, dilation_cycle_length=cycle))
    net.load_state_dict(state_dict(L, cycle, M, C, H))
    s = dsx.DsxSampler(net.to(DEV).eval(), prec, cycle)
    s.ensure_weights(DEV)
    for k, v in opts:
        s.set_option(getattr(_capi, k), v)
    _SAMPLERS[key] = s
    return s


@pytest.fixture(scope="module", autouse=True)
def _close_samplers(lib_built):
    yield
    while _SAMPLERS:
        _SAMPLERS.popitem()[1].close()


def eps_of(s, spec, t, cond):
    return s.diffnet_forward(spec.to(DEV), t.to(DEV), cond.to(DEV)).cpu()


def check(err, sim, fmt, what):
    b = bound(sim, fmt)
    print(f"{what}: err {err:.2e} sim {sim:.2e} bound {b:.1e}")
    assert err <= b, (what, err, sim, b)


# ---- single evaluations -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("case", list(FWD))
def test_forward(case, form):
    c = FWD[case]
    s = sampler(form, c["L"], c["cycle"])
    spec, t, cond = fwd_inputs(case)
    eps = eps_of(s, spec, t, cond)
    assert torch.isfinite(eps).all()
    fmt = FORMS[form][2]
    check((eps.double() - fwd_ref(case)).abs().max().item(), SIM[case][FMTS.index(fmt) if fmt != "fp32" else 4],
          fmt, f"forward {case} {form}")


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("case", ["T129", "T1", "L31_cycle4"])
def test_forward_exact(case, form):
    """mixed t against one t per batch, permutation, repetition: bit for bit"""
    c = FWD[case]
    s = sampler(form, c["L"], c["cycle"])
    spec, t, cond = fwd_inputs(case)
    eps = eps_of(s, spec, t, cond)
    assert torch.equal(eps, eps_of(s, spec, t, cond))
    for b in range(c["B"]):
        same = eps_of(s, spec, torch.full_like(t, int(t[b])), cond)
        assert torch.equal(eps[b], same[b]), b
    perm = torch.tensor([2, 0, 1])
    assert torch.equal(eps_of(s, spec[perm], t[perm], cond[perm]), eps[perm])


# ---- residency boundaries -----------------------------------------------------------------------------------------
def boundaries(s):
    """B at each boundary of the stack form at T = 64 (128 padded frames: two 64-frame tiles or one 128-frame tile per
    utterance), with the rows the automatic choice must take"""
    from diffsinger_b200 import _capi
    sms = s.info(_capi.INFO_SM_COUNT)
    s.set_option(_capi.OPT_STACK_ROWS, 128)        # a 128-frame launch fills DSX_INFO_CLUSTER_OCCUPANCY
    x = torch.zeros(1, 1, 80, 64, device=DEV)
    s.diffnet_forward(x, torch.zeros(1, dtype=torch.long, device=DEV), torch.zeros(1, 256, 64, device=DEV))
    s.set_option(_capi.OPT_STACK_ROWS, 0)
    cap128 = s.info(_capi.INFO_CLUSTER_OCCUPANCY)
    cap64 = sms        # k_hp_step<1, 3> takes 162 KB of shared memory: one CTA per SM
    assert cap128 > 0 and cap128 % sms == 0
    return {"last_64_frame": (cap64 // 2, 64), "first_128_frame": (cap64 // 2 + 1, 128),
            "last_paired": (cap128, 128), "first_unpaired": (cap128 + 1, 128), "B9": (9, 64), "B17": (17, 64)}


def residency_ref(sd, spec, t, cond, b):
    with torch.no_grad():
        return O.diffnet_forward(sd, spec[b:b + 1].double(), t[b:b + 1], cond[b:b + 1].double(), 4)


@pytest.mark.parametrize("form", list(AUTO_FORMS))
def test_residency_boundaries(form):
    from diffsinger_b200 import _capi
    prec = AUTO_FORMS[form][0]
    s = sampler(form, 20, 4)
    sd = f64(state_dict(20, 4))
    points = boundaries(s)
    for name, (B, rows) in points.items():
        spec, cond = rs_normal(700 + B, (B, 1, 80, 64)), rs_normal(701 + B, (B, 256, 64))
        t = torch.tensor([T_UTT[b % 3] for b in range(B)])
        eps = eps_of(s, spec, t, cond)
        assert s.info(_capi.INFO_STACK_ROWS) == rows, (name, B, rows)
        print(f"residency {form} {name}: B {B}, INFO_STACK_ROWS {rows}")
        for b in sorted({0, 1, B - 2, B - 1}):
            alone = eps_of(s, spec[b:b + 1], t[b:b + 1], cond[b:b + 1])
            assert torch.equal(eps[b:b + 1], alone), (name, b)
            err = (eps[b:b + 1].double() - residency_ref(sd, spec, t, cond, b)).abs().max().item()
            check(err, SIM["T64"][FMTS.index(prec)], prec, f"residency {form} {name} utterance {b}")


# ---- sampling loops -----------------------------------------------------------------------------------------------
def run_loop(s, inp):
    x, cond = inp["xT"].to(DEV), inp["cond"].to(DEV)
    if inp["kind"] == "ddpm":
        s.set_schedule(schedule(100))
        return s.sample_ddpm(x, cond, inp["a"], inp["b"], noise=inp["noise"].to(DEV)).cpu()
    if inp["kind"] == "plms":
        s.set_schedule(schedule(1000))
        return s.sample_plms(x, cond, inp["a"], inp["b"]).cpu()
    s.set_schedule(schedule(100))
    kw = dict(x_start=x) if inp["gaussian"] else dict(fs2_mel=inp["fs2_mel"].to(DEV),
                                                     start_noise=inp["start_noise"].to(DEV))
    return s.infer(cond, 1, inp["smin"].to(DEV), inp["smax"].to(DEV), step_noise=inp["step_noise"].to(DEV),
                   mel2ph=inp["mel2ph"].to(DEV), **kw).cpu()


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("case", list(LOOP_CASES))
def test_loop(case, form):
    inp = loop_inputs(case)
    s = sampler(form, inp["L"], 4)
    out = run_loop(s, inp)
    assert torch.isfinite(out).all()
    if inp["kind"] == "infer":
        masked = inp["mel2ph"] == 0
        assert (out[masked] == 0).all()
    fmt = FORMS[form][2]
    check(loop_error(out, loop_ref(case)), SIM[case][FMTS.index(fmt) if fmt != "fp32" else 4], fmt,
          f"loop {case} {form}")


# ---- fp32 SIMT ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(SIMT))
def test_simt(case):
    M, C, H, L, cyc, T = SIMT[case]
    s = sampler("fp32", L, cyc, M, C, H)
    spec, t, cond = simt_inputs(case)
    eps = eps_of(s, spec, t, cond)
    assert torch.isfinite(eps).all()
    check((eps.double() - simt_ref(case)).abs().max().item(), SIM[case][4], "fp32", f"simt {case}")
    perm = torch.tensor([1, 2, 0])
    assert torch.equal(eps_of(s, spec[perm], t[perm], cond[perm]), eps[perm])


# ---- refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec,M,C,H,cycle,match", [
    ("fp16x2", 128, 256, 256, 1, "mel bins == 80"), ("fp16", 80, 128, 256, 1, "residual_channels"),
    ("fp16s", 80, 256, 256, 5, "dilation_cycle_length <= 4"), ("fp16x3", 80, 256, 128, 1, "hidden_size"),
    ("fp32", 784, 16, 16, 1, "mel bins must be <= 768"), ("fp32", 80, 2464, 16, 1, "residual channels <= 2448")])
def test_load_refuses(prec, M, C, H, cycle, match):
    import diffsinger_b200 as dsx
    L = 1 if C > 256 else 2
    net = dsx.DiffNet(M, hparams=dict(hidden_size=H, residual_layers=L, residual_channels=C, dilation_cycle_length=cycle))
    s = dsx.DsxSampler(net.to(DEV).eval(), prec, cycle)
    with pytest.raises(dsx.DsxError, match=match):
        s.ensure_weights(DEV)
    s.close()
