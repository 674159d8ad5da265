"""numpy restatements of the RPN background plan (numpy only, so tools can use them without the test stack):
  strip_flags      b2s_rpn_strip_plan's flags: strips with a pixel whose receptive field holds data
  strip_bands      b2s_rpn_strip_bands' bands, per layer
  tail_tiles       b2s_rpn_strip_bands' computed tiles of the fused tail (8 x 16 pixels)"""
import numpy as np


def _dilate(mask):
    H, W = mask.shape[1:]
    pad = np.pad(mask, ((0, 0), (1, 1), (1, 1)))
    out = np.zeros_like(mask)
    for dy in range(3):
        for dx in range(3):
            out |= pad[:, dy:dy + H, dx:dx + W]
    return out


def strip_flags(occ, num_layers, rows, width=8):
    """per layer: [B, ceil(H/rows), ceil(W/width)] booleans, the data mask dilated by one pixel per layer."""
    B, H, W = occ.shape
    sh, sw = -(-H // rows), -(-W // width)
    cur, flags = occ.astype(bool), []
    for _ in range(num_layers):
        cur = _dilate(cur)
        pad = np.pad(cur, ((0, 0), (0, sh * rows - H), (0, sw * width - W)))
        flags.append(pad.reshape(B, sh, rows, sw, width).any(axis=(2, 4)))
    return flags


def tail_tiles(last, rows):
    """[B, ceil(H/8), ceil(W/16)]: a tail tile (8 / rows strip rows x 2 strip columns) is computed iff one of its
    strips is computed by the last layer (`last`, [B, strips_h, strips_w])."""
    B, sh, sw = last.shape
    per = 8 // rows
    th, tw = -(-sh // per), -(-sw // 2)
    pad = np.pad(last.astype(bool), ((0, 0), (0, th * per - sh), (0, tw * 2 - sw)))
    return pad.reshape(B, th, per, tw, 2).any(axis=(2, 4))


def strip_bands(flags, rows):
    """per layer: the strips the layer does not compute that a later launch reads, as [B, strips_h, strips_w]
    booleans.  Layer l < last: a strip of layer l + 1 lies in the 3x3 strip neighbourhood (itself included); the last
    layer: the strip lies in a computed tail tile."""
    out = []
    for cur, nxt in zip(flags[:-1], flags[1:]):
        out.append(_dilate(nxt.astype(bool)) & ~cur.astype(bool))
    last = flags[-1].astype(bool)
    per = 8 // rows
    tiles = tail_tiles(last, rows).repeat(per, axis=1).repeat(2, axis=2)[:, :last.shape[1], :last.shape[2]]
    out.append(tiles & ~last)
    return out
