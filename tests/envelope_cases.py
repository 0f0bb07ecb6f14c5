"""The networks of the stage tests, shared by the CPU tests (reference anchor, composed stage references, routing) and
the GPU tests (every stage of the engine against fp64 at its own inputs): `cfg_of(kind, pad, act_fun)` builds the
oracle's SkipConfig of a named network (NETS) or of a row of the envelope table.

The envelope table: skip networks at the edges of what build_plan (csrc/engine.cu) and models.skip accept.  Each row is
data; a planner change that widens or moves the accepted range adds a row here and the tests pick it up.

Row fields: L (scales), in / out channels, per-scale down / up / skip widths, per-scale upsampling, downsample mode,
H x W, need_sigmoid, and which extra GPU paths run on it: `zero_pad` (again with pad='zero'), `input_grad` (dz),
`module` (through models.skip at precision 'fp32').  The comment above each row names what only that row reaches.
"""
from collections import namedtuple

from oracle import dip_oracle as O

Row = namedtuple("Row", "id L in_ch out_ch down up skips modes downsample H W sigmoid zero_pad input_grad module")

ROWS = [
    # one scale (level 0 is the deepest level); stored input depth 8 (5 real channels); BN width 24 (VL 6) and concat 28
    # (VL 7: non-power-of-two reductions); skinny head with 2 outputs; a 5 x 7 deepest level; W % 4 = 2 (the runner's
    # separate k_noise -> zbuf -> k_input_pad path).  Regression: this row caught the skinny 1x1 conv (k_skinny_fwd, narrow
    # path) folding a pixel's C/4 lanes with xor shuffles as if C/4 were a power of two: at C = 24 (the head over U here)
    # and every other width whose C/4 is not (the 4-channel skip convs over 40, 48, 104, ... channels in L2, L3avg, L4,
    # L7) the lanes of neighbouring pixels were summed together and the output was wrong
    Row("L1", 1, 5, 2, [24], [24], [4], ["bilinear"], "stride", 10, 14, True, True, False, False),
    # down != up widths: concat 76 (VL 19) and 40 (VL 10); fprop N = 40, 56, 72 (a half-valid last 32-row chunk);
    # stored input depth 4 from a 1-channel input; skinny head with 4 outputs; per-scale upsampling; skip 0 at level 0
    Row("L2", 2, 1, 4, [40, 72], [56, 40], [0, 4], ["nearest", "bilinear"], "stride", 12, 20, True, True, False, True),
    # avg pooling at three scales; stored input depth 64 (33 real channels); BN VL 12 / 20 / 28; concat 84 and 116
    # (dgrad / wgrad columns 96 and 128); fprop N = 48, 80, 112
    Row("L3avg", 3, 33, 3, [48, 80, 112], [48, 80, 112], [4, 4, 4], ["bilinear"] * 3, "avg", 16, 24, True, False, False, False),
    # stored input depth 128 (100 real channels: k_input_grad writes 100 of 128); logits with one output; BN VL 22 / 24 /
    # 26 / 30; concat 88, 92, 108, 120; fprop N = 96 unsplit and 104; skip 4 / 0 alternating.  This row caught L0.dPin
    # registered at the stored depth: the input-gradient conv writes the 100 real channels only, so the registered view
    # exposed 28 channels that nothing writes or reads (L0.dPin is now registered at the real depth)
    Row("L4", 4, 100, 1, [96, 104, 120, 88], [96, 104, 120, 88], [4, 0, 4, 0], ["bilinear", "nearest", "nearest", "bilinear"],
        "stride", 32, 48, False, True, True, True),
    # widths reversed between the down and the up path: down convs 128, 64, 32, 16, 8; the up convs of levels 4..0 read
    # concats 12 (VL 3), 132, 68, 36, 20 and write 128, 64, 32, 16, 8; skinny head over an 8-wide U
    Row("rev5", 5, 3, 3, [128, 64, 32, 16, 8], [8, 16, 32, 64, 128], [4] * 5, ["bilinear"] * 5, "stride", 64, 96, True, False,
        False, True),
    # six scales of the 128-wide skip=128 network: a 2 x 3 deepest level, fused head, parameter slots of L = 6
    Row("L6w", 6, 32, 3, [128] * 6, [128] * 6, [128] * 6, ["nearest"] * 6, "stride", 128, 192, True, False, False, False),
    # seven scales, widths 8..56: every BN VL 2..14, concat 12, 20, 28, 36, 44, 52, 60; 2 x 2 deepest level
    Row("L7", 7, 32, 3, [8, 16, 24, 32, 40, 48, 56], [8, 16, 24, 32, 40, 48, 56], [4] * 7, ["nearest"] * 7, "stride", 256, 256,
        True, True, False, False),
    # eight scales (the most build_plan accepts): bilinear-mask bits up to 7, 2 x 2 deepest level below 8 stride-2 convs,
    # concat 132 at two levels, skinny head over a 16-wide U
    Row("L8", 8, 32, 3, [16, 16, 32, 32, 64, 64, 128, 128], [16, 16, 32, 32, 64, 64, 128, 128], [4] * 8,
        ["bilinear", "nearest"] * 4, "stride", 512, 512, True, False, False, False),
]
BY_ID = {r.id: r for r in ROWS}


MODES5 = ["bilinear", "nearest", "bilinear", "nearest", "nearest"]
NETS = {
    "cs4": lambda: O.SkipConfig(skip_channels=4, upsample_mode="bilinear"),
    "cs128": lambda: O.SkipConfig(skip_channels=128, upsample_mode="nearest"),
    "cs0": lambda: O.SkipConfig(skip_channels=0, upsample_mode="bilinear"),
    "snail": lambda: O.SkipConfig(in_channels=3, channels=[8, 16, 32, 64, 128], skip_channels=[0, 0, 0, 4, 4]),
    "kate": lambda: O.SkipConfig(in_channels=3, channels=[16, 32, 64, 128, 128], skip_channels=0),   # + 'avg'
    "modes": lambda: O.SkipConfig(in_channels=3, skip_channels=4, upsample_mode=MODES5),
    "ingrad": lambda: O.SkipConfig(skip_channels=4, out_channels=1, need_sigmoid=False),
    # per-scale upsampling, logits as the output, one output channel (run with dL/d(input))
    "modes_ingrad": lambda: O.SkipConfig(in_channels=3, out_channels=1, skip_channels=4, need_sigmoid=False,
                                         upsample_mode=MODES5),
    "per_scale128": lambda: O.SkipConfig(channels=[128] * 5, skip_channels=[4] * 5),
    "avg128": lambda: O.SkipConfig(skip_channels=4),   # + 'avg'
    # models.skip(32, 3)'s widths, skips and upsampling (its own default padding is 'zero': pass pad='zero')
    "skipdefault": lambda: O.SkipConfig(upsample_mode="nearest", channels=[16, 32, 64, 128, 128], skip_channels=[4] * 5),
}
AVG = ("kate", "avg128")


def cfg_of(kind, pad="reflection", act_fun="LeakyReLU"):
    """the oracle's SkipConfig of a network of NETS or a row id of the envelope table (per-scale widths, channels_up set
    explicitly), with the given padding and activation"""
    if kind in BY_ID:
        row = BY_ID[kind]
        cfg = O.SkipConfig(in_channels=row.in_ch, out_channels=row.out_ch, num_scales=row.L, channels=list(row.down),
                           skip_channels=list(row.skips), upsample_mode=list(row.modes), need_sigmoid=row.sigmoid)
        cfg.channels_up = list(row.up)
        cfg.downsample_mode = row.downsample
    else:
        cfg = NETS[kind]()
        if kind in AVG:
            cfg.downsample_mode = "avg"
    cfg.pad, cfg.act_fun = pad, act_fun
    return cfg


def skip_kwargs(row, pad="reflection"):
    """models.skip(...) keyword arguments of a row (the reference's signature)"""
    return dict(num_input_channels=row.in_ch, num_output_channels=row.out_ch, num_channels_down=list(row.down),
                num_channels_up=list(row.up), num_channels_skip=list(row.skips), upsample_mode=list(row.modes),
                downsample_mode=row.downsample, need_sigmoid=row.sigmoid, need_bias=True, pad=pad)


def pads_of(row):
    return ["reflection", "zero"] if row.zero_pad else ["reflection"]
