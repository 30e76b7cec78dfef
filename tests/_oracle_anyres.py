"""The CPU oracle at any patch-multiple image size: TokenOracle's vision path on an H x W image with a given position table
([T, h], T = (H/P)(W/P) + 1, CLS row first), the rows the *_hw entry points return.  A subclass, so the pinned oracle and
TokenOracle stay exactly as they are."""
import numpy as np

import oracle as orc
from _oracle_tokens import TokenOracle


class AnyresOracle(TokenOracle):
    def _embed_hw(self, img, pos):
        P, hid = self.patch, self.v_hidden
        H, W = img.shape[:2]
        gh, gw = H // P, W // P
        assert img.shape == (gh * P, gw * P, 3) and pos.shape == (gh * gw + 1, hid)
        planar = np.ascontiguousarray(img.transpose(2, 0, 1), np.float32)
        patches = np.ascontiguousarray(planar.reshape(3, gh, P, gw, P).transpose(1, 3, 0, 2, 4).reshape(gh * gw, 3 * P * P))
        pw = self.t("v.patch_embd.weight")
        assert pw.type == orc.F16
        y = np.empty((gh * gw, hid), np.float32)
        buf = np.frombuffer(pw.data, np.uint8)
        assert orc.lib().orc_mul_mat(orc.F16, buf.ctypes.data, hid, 3 * P * P, orc._fp(patches), gh * gw, orc._fp(y), self.nt) == 0
        x = np.zeros((gh * gw + 1, hid), np.float32)
        x[0] = self.f32("v.class_embd")
        x[1:] = y
        x = x + np.asarray(pos, np.float32)
        return self.ln(x, "v.pre_ln.weight", "v.pre_ln.bias", self.v_eps), gh * gw + 1

    def image_tokens_hw(self, img: np.ndarray, pos: np.ndarray, layer: int = -1, post_ln: bool = False) -> np.ndarray:
        """img [H, W, 3], pos [T, h] -> [T, v_hidden]: the residual rows after `layer` blocks (post_ln on every row if asked)"""
        x, T = self._embed_hw(img, pos)
        x = self._blocks("v", x, self._blocks_for(layer, self.v_layers), self.v_heads, self.v_eps, T, False)
        return self.ln(x, "v.post_ln.weight", "v.post_ln.bias", self.v_eps) if post_ln else x

    def encode_image_hw(self, img: np.ndarray, pos: np.ndarray, normalize: bool = True) -> np.ndarray:
        """encode_image's pooled tail on the CLS row of image_tokens_hw"""
        x = self.image_tokens_hw(img, pos, -1)
        e = self.mul_mat("visual_projection.weight", self.ln(x[0:1], "v.post_ln.weight", "v.post_ln.bias", self.v_eps))[0]
        return self._normalize(e) if normalize else e

    def position_table_hw(self, gh: int, gw: int, resample) -> np.ndarray:
        """the model's table with its patch rows resampled to gh x gw by resample(table, g, gh, gw); the CLS row as it is"""
        pos = self.f32("v.position_embd.weight")
        g = self.image_size // self.patch
        return np.concatenate([pos[:1], resample(pos[1:], g, gh, gw)]).astype(np.float32)
