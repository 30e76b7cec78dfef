"""Per-token hidden states on the CPU oracle: the rows clip_b200_image_tokens / clip_b200_text_tokens return, computed with the
oracle's own arithmetic.  A subclass, so that the pinned OracleModel and its encode_image / encode_text stay exactly as they are.

Layer numbering follows HF hidden_states: 0 is the input of block 0, i the output of block i, negative values count from the end."""
import numpy as np

import oracle as orc


class TokenOracle(orc.OracleModel):
    def _blocks_for(self, layer, n_layers):
        assert -(n_layers + 1) <= layer <= n_layers, layer
        return layer + n_layers + 1 if layer < 0 else layer

    def image_tokens(self, img: np.ndarray, layer: int = -1, post_ln: bool = False) -> np.ndarray:
        """img [S, S, 3] -> [T, v_hidden]: the residual rows after `layer` blocks (post_ln applied to every row if asked)"""
        S, P, hid = self.image_size, self.patch, self.v_hidden
        assert img.shape == (S, S, 3)
        n = S // P
        # the embedding of encode_image, step for step
        planar = np.ascontiguousarray(img.transpose(2, 0, 1), np.float32)
        patches = np.ascontiguousarray(planar.reshape(3, n, P, n, P).transpose(1, 3, 0, 2, 4).reshape(n * n, 3 * P * P))
        pw = self.t("v.patch_embd.weight")
        assert pw.type == orc.F16
        y = np.empty((n * n, hid), np.float32)
        buf = np.frombuffer(pw.data, np.uint8)
        assert orc.lib().orc_mul_mat(orc.F16, buf.ctypes.data, hid, 3 * P * P, orc._fp(patches), n * n, orc._fp(y), self.nt) == 0
        x = np.zeros((n * n + 1, hid), np.float32)
        x[0] = self.f32("v.class_embd")
        x[1:] = y
        x = x + self.f32("v.position_embd.weight")
        x = self.ln(x, "v.pre_ln.weight", "v.pre_ln.bias", self.v_eps)
        x = self._blocks("v", x, self._blocks_for(layer, self.v_layers), self.v_heads, self.v_eps, n * n + 1, False)
        return self.ln(x, "v.post_ln.weight", "v.post_ln.bias", self.v_eps) if post_ln else x

    def text_tokens(self, ids, layer: int = -1, post_ln: bool = False) -> np.ndarray:
        """ids [N] -> [N, t_hidden], causal: row j depends on ids[:j + 1] only"""
        ids = np.asarray(ids, np.int64)
        N = ids.size
        x = self.f32("t.position_embd.weight")[:N] + self.f32("t.token_embd.weight")[ids]
        x = self._blocks("t", x, self._blocks_for(layer, self.t_layers), self.t_heads, self.t_eps, N, True)
        return self.ln(x, "t.post_ln.weight", "t.post_ln.bias", self.t_eps) if post_ln else x

    def project_image(self, rows, normalize=True):
        e = self.mul_mat("visual_projection.weight", rows)
        return np.stack([self._normalize(r) for r in e]) if normalize else e

    def project_text(self, rows, normalize=True):
        e = self.mul_mat("text_projection.weight", rows)
        return np.stack([self._normalize(r) for r in e]) if normalize else e
