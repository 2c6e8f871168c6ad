"""Dense-grid SDF / colour query of the mesher on the fused query kernel (SURVEY.md section 8 row f3).

`Mesher.query_points` keeps the reference's signature and return values (utils/mesher.py:40-164 of
PRBonn/PIN_SLAM): the per-batch `query_feature -> Decoder.sdf -> IDW sum` chain is ONE launch of K1 in
global-map, no-gradient mode per chunk.  Marching cubes / mesh IO stay with the reference (CPU, skimage/open3d);
this class only replaces the grid query that feeds them.
"""
import numpy as np
import torch


class Mesher:
    # queries per launch: large enough to fill the GPU many times over, small enough to bound the output buffers
    CHUNK = 1 << 22

    def __init__(self, config, neural_points, decoders: dict):
        self.config = config
        self.silence = config.silence
        self.neural_points = neural_points
        self.sdf_mlp = decoders["sdf"]
        self.sem_mlp = decoders.get("semantic")
        self.color_mlp = decoders.get("color")
        self.device = config.device
        self.cur_device = self.device
        self.dtype = config.dtype
        self.global_transform = np.eye(4)

    def query_points(self, coord, bs, query_sdf=True, query_sem=False, query_color=False, query_mask=True,
                     query_locally=False, mask_min_nn_count: int = 4, out_torch: bool = False):
        """Returns (sdf_pred, sem_pred, color_pred, mc_mask) like the reference; `bs` is accepted for
        compatibility (it only sets a lower bound on the chunk size, the kernel takes millions of points per
        launch)."""
        if query_sem:
            raise NotImplementedError("semantic head is outside the CUDA hot path")
        n = coord.shape[0]
        dev = self.neural_points.neural_points.device
        chunk = max(int(bs), self.CHUNK)
        sdf_pred = torch.zeros(n, device=dev) if query_sdf else None
        color_pred = torch.zeros((n, self.config.color_channel), device=dev) if query_color else None
        mc_mask = torch.zeros(n, dtype=torch.bool, device=dev) if query_mask else None
        work = {}
        for head in range(0, n, chunk):
            tail = min(head + chunk, n)
            q = coord[head:tail].to(device=dev, dtype=torch.float32).contiguous()
            o = self.neural_points.query_sdf(q, self.sdf_mlp, query_locally=query_locally, need_grad=False,
                                             color_decoder=self.color_mlp if query_color else None, out=work)
            if query_sdf:
                # rows without any neighbour are never decoded by the reference: they keep sdf 0 (mesher.py:118-131)
                sdf_pred[head:tail] = torch.where(o["nn_count"] >= 1, o["sdf"], torch.zeros_like(o["sdf"]))
            if query_color:
                color_pred[head:tail] = o["color"]
            if query_mask:
                mc_mask[head:tail] = o["nn_count"] >= mask_min_nn_count
        if out_torch:
            return sdf_pred, None, color_pred, mc_mask
        return (None if sdf_pred is None else sdf_pred.cpu().numpy().astype(np.float64), None,
                None if color_pred is None else color_pred.cpu().numpy().astype(np.float64),
                None if mc_mask is None else mc_mask.cpu().numpy().astype(np.float64))


def patch_reference_mesher(mesher_cls) -> None:
    """Route the reference's own `utils.mesher.Mesher` (marching cubes, mesh IO untouched) through the fused
    grid query:  `from utils.mesher import Mesher; patch_reference_mesher(Mesher)`."""
    mesher_cls.query_points = Mesher.query_points
    if not hasattr(mesher_cls, "CHUNK"):
        mesher_cls.CHUNK = Mesher.CHUNK
