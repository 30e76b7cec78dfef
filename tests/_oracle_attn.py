"""Attention probabilities on the CPU oracle: what an ATTENTION entry of the *_tokens calls returns, from the oracle's own hidden states.
The l-th block's attention is the softmax of its scores: the oracle's hidden states after block l - 1, LN1, Q (scaled) and K through
the oracle's mul_mat, then the softmax in fp64 per head (causal for text).  A subclass, so TokenOracle stays as it is."""
import numpy as np

from _oracle_anyres import AnyresOracle


class AttnOracle(AnyresOracle):
    def _attention(self, p, x, block, heads, eps, causal):
        """x [T, hid]: the input of block `block` -> [heads, T, T] fp64"""
        T, hid = x.shape
        dh = hid // heads
        b = "%s.blk.%d." % (p, block)
        cur = self.ln(x, b + "ln1.weight", b + "ln1.bias", eps)
        scale = np.float32(1.0) / np.float32(np.sqrt(np.float32(dh)))
        q = (self.f32(b + "attn_q.bias") + self.mul_mat(b + "attn_q.weight", cur)) * scale
        k = self.f32(b + "attn_k.bias") + self.mul_mat(b + "attn_k.weight", cur)
        q = q.astype(np.float64).reshape(T, heads, dh).transpose(1, 0, 2)
        k = k.astype(np.float64).reshape(T, heads, dh).transpose(1, 0, 2)
        s = q @ k.transpose(0, 2, 1)
        if causal:
            s = np.where(np.tril(np.ones((T, T), bool))[None], s, -np.inf)
        w = np.exp(s - s.max(-1, keepdims=True))
        return w / w.sum(-1, keepdims=True)

    def _block_of(self, layer, n_layers):
        assert layer != 0 and layer != -(n_layers + 1), layer
        return self._blocks_for(layer, n_layers) - 1

    def image_attention(self, img, layer, pos=None):
        """img [S, S, 3] (or [H, W, 3] with its position table pos) -> [v_heads, T, T]: the attention of the layer-th block"""
        blk = self._block_of(layer, self.v_layers)
        x = self.image_tokens(img, blk) if pos is None else self.image_tokens_hw(img, pos, blk)
        return self._attention("v", x, blk, self.v_heads, self.v_eps, False)

    def text_attention(self, ids, layer):
        """ids [N] -> [t_heads, N, N], causal"""
        blk = self._block_of(layer, self.t_layers)
        return self._attention("t", self.text_tokens(ids, blk), blk, self.t_heads, self.t_eps, True)
