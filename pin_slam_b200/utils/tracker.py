"""Point-to-implicit odometry on the fused kernels.

API-compatible with the reference `Tracker` (utils/tracker.py:20 of PRBonn/PIN_SLAM: same
constructor, `tracking(...)` arguments and 4-tuple result, `query_source_points(...)` 8-tuple,
`registration_step(...)` 7-tuple) but one Gauss-Newton iteration is three launches and ONE small
device->host read instead of ~470 ATen ops and ~29 host syncs:

    K1  pinb200_query_sdf   transform by the current pose + kNN + IDW + decoder + d sdf/dx
    K4  pinb200_gn_step     validity mask, robust weights, 6x6 normal equations, fp64 solve,
                            T <- dT @ T on the device
    D2H 32 doubles          (valid count, residual, dT) for the host-side convergence logic
"""
import math

import numpy as np
import torch

from .. import ops


def _angle_deg(rot: np.ndarray) -> float:
    c = (np.trace(rot) - 1.0) / 2.0
    return math.degrees(math.acos(min(1.0, max(-1.0, c))))


class Tracker:
    def __init__(self, config, neural_points, decoders: dict):
        self.config = config
        self.silence = config.silence
        self.neural_points = neural_points
        self.sdf_mlp = decoders["sdf"]
        self.sem_mlp = decoders.get("semantic")
        self.color_mlp = decoders.get("color")
        self.device = config.device
        self.dtype = config.dtype
        self.reg_local_map = True
        self.sdf_scale = config.logistic_gaussian_ratio * config.sigma_sigmoid_m
        self._sums = None
        self._result = None
        self._out = {}

    # ------------------------------------------------------------------ queries
    def query_source_points(self, coord, bs, query_sdf=True, query_sdf_grad=True, query_color=False,
                            query_color_grad=False, query_sem=False, query_mask=True, query_certainty=True,
                            query_locally=True, mask_min_nn_count: int = 4):
        """Same outputs as the reference (utils/tracker.py:227-365); `bs` is accepted for compatibility,
        the fused kernel takes the whole batch in one launch."""
        if query_sem:
            raise NotImplementedError("semantic head is outside the CUDA hot path")
        color_dec = self.color_mlp if query_color else None
        o = self.neural_points.query_sdf(coord.contiguous(), self.sdf_mlp, query_locally=query_locally,
                                         need_grad=query_sdf_grad or query_color_grad, color_decoder=color_dec,
                                         color_grad=query_color_grad)
        mask = (o["nn_count"] >= mask_min_nn_count) if query_mask else None
        return (o["sdf"] if query_sdf else None, o.get("grad") if query_sdf_grad else None, o.get("color"),
                o.get("color_grad"), None, mask, o["certainty"] if query_certainty else None,
                o["sdf_std"] if query_sdf else None)

    def _color_setup(self, source_colors):
        """(colour decoder, need colour gradient, K4 colour mode) for this call (tracker.py:385-386, 493-514)."""
        cfg = self.config
        if source_colors is None or not cfg.color_on or self.color_mlp is None:
            return None, False, 0
        if cfg.photometric_loss_on:
            return self.color_mlp, True, 2
        return self.color_mlp, False, (1 if cfg.consist_wieght_on else 0)

    def _gn(self, xyz, o, source_normals, source_sdf, min_grad_norm, max_grad_norm, gm_dist, gm_grad, lm_lambda,
            t_dev, source_colors=None, color_mode=0):
        if self._sums is None:
            self._sums = torch.empty(64, dtype=torch.float64, device=xyz.device)
            self._result = torch.empty(32, dtype=torch.float64, device=xyz.device)
        cfg = self.config
        return ops.gn_step(xyz, o["sdf"], o["grad"], o["sdf_std"], o["nn_count"],
                           min_nn=cfg.track_mask_query_nn_k, min_grad_norm=min_grad_norm,
                           max_grad_norm=max_grad_norm, max_sdf_std=cfg.surface_sample_range_m * cfg.max_sdf_std_ratio,
                           gm_dist=gm_dist, gm_grad=gm_grad, lm_lambda=lm_lambda, sdf_label=source_sdf,
                           normals=source_normals, t_inout=t_dev, sums=self._sums, result=self._result,
                           color_obs=None if not color_mode else source_colors[:, : cfg.color_channel].contiguous(),
                           color_pred=o.get("color") if color_mode else None,
                           color_grad=o.get("color_grad") if color_mode == 2 else None, color_mode=color_mode,
                           w_photo=cfg.photometric_loss_weight)

    def _iterate(self, src, t_dev, n_iter, source_normals, source_sdf, source_colors, cdec, cgrad, cmode):
        """n_iter x (K1 + K4) on the device pose `t_dev` from one host call (pinb200_track_iterations)."""
        cfg, npm = self.config, self.neural_points
        if self._sums is None or self._sums.device != src.device:
            self._sums = torch.empty(64, dtype=torch.float64, device=src.device)
            self._result = torch.empty(32, dtype=torch.float64, device=src.device)
        o = ops.track_iterations(
            npm.map_handle(self.reg_local_map), self.sdf_mlp.handle(), src, t_dev, n_iter, nn_k=cfg.query_nn_k,
            weighted_first=cfg.weighted_first, min_nn=cfg.track_mask_query_nn_k, min_grad_norm=cfg.reg_min_grad_norm,
            max_grad_norm=cfg.reg_max_grad_norm, max_sdf_std=cfg.surface_sample_range_m * cfg.max_sdf_std_ratio,
            gm_dist=cfg.reg_GM_dist_m if cfg.reg_GM_dist_m > 0 else None,
            gm_grad=cfg.reg_GM_grad if cfg.reg_GM_grad > 0 else None, lm_lambda=cfg.reg_lm_lambda, sums=self._sums,
            result=self._result, sdf_label=source_sdf, normals=source_normals,
            color_dec=None if cdec is None else cdec.handle(sigmoid_out=True), color_grad=cgrad,
            color_obs=None if not cmode else source_colors[:, : cfg.color_channel].contiguous(), color_mode=cmode,
            w_photo=cfg.photometric_loss_weight, out=self._out)
        return o, self._result, self._sums

    def registration_step(self, points, normals, sdf_labels, colors, min_grad_norm, max_grad_norm, GM_dist=None,
                          GM_grad=None, lm_lambda=0.0, vis_weight_pc=False):
        """One GN/LM step on already transformed points (reference: utils/tracker.py:367-611).
        Returns (T, cov_mat, eigenvalues, weight_point_cloud, valid_points, sdf_residual_mean_cm,
        color_residual_mean)."""
        cdec, cgrad, cmode = self._color_setup(colors)
        o = self.neural_points.query_sdf(points.contiguous(), self.sdf_mlp, query_locally=self.reg_local_map,
                                         need_grad=True, color_decoder=cdec, color_grad=cgrad, out=self._out)
        res, sums = self._gn(points.contiguous(), o, normals, sdf_labels, min_grad_norm, max_grad_norm, GM_dist,
                             GM_grad, lm_lambda, None, colors, cmode)
        r = res.cpu().numpy()
        T = torch.tensor(r[:16].reshape(4, 4), dtype=torch.float64, device=points.device)
        gnorm = o["grad"].norm(dim=-1)
        valid = ((o["nn_count"] >= self.config.track_mask_query_nn_k) & (gnorm < max_grad_norm) &
                 (gnorm > min_grad_norm) &
                 (o["sdf_std"] < self.config.surface_sample_range_m * self.config.max_sdf_std_ratio))
        cov, eig = None, None
        if vis_weight_pc and r[16] >= 10:
            cov, eig = self._cov_eig(sums, r)
        return T, cov, eig, None, points[valid], float(r[17]), (float(r[28]) if cmode == 2 else None)

    @staticmethod
    def _cov_eig(sums, r):
        s = sums.cpu().numpy()
        sc = r[16] / (2.0 * s[42])
        n_raw = (s[:36].reshape(6, 6) * sc).astype(np.float32).astype(np.float64)
        cov = torch.tensor(np.linalg.inv(n_raw) * r[21])
        eig = torch.tensor(r[18:21].copy())
        return cov, eig

    # ------------------------------------------------------------------ tracking loop
    def tracking(self, source_points, init_pose=None, source_colors=None, source_normals=None, source_semantics=None,
                 source_sdf=None, cur_ts=None, loop_reg: bool = False, vis_result: bool = False):
        """Reference: utils/tracker.py:43-225.  Returns (T [4,4] f64, cov_mat, weight_point_cloud, valid_flag)."""
        cfg = self.config
        dev = source_points.device
        cdec, cgrad, cmode = self._color_setup(source_colors)
        T_dev = (torch.eye(4, dtype=torch.float64, device=dev) if init_pose is None
                 else init_pose.to(device=dev, dtype=torch.float64).clone().contiguous())
        gm_dist = cfg.reg_GM_dist_m if cfg.reg_GM_dist_m > 0 else None
        gm_grad = cfg.reg_GM_grad if cfg.reg_GM_grad > 0 else None
        iter_n = cfg.reg_iter_n
        max_final_res_cm = cfg.surface_sample_range_m * cfg.final_residual_ratio_thre * 100.0
        min_valid_ratio = 0.15 if loop_reg else 0.2
        min_valid_points = 30
        converged, valid_flag = False, True
        last_res_cm = 1e5
        n_src = source_points.shape[0]
        src = source_points.contiguous()
        cov_mat, eigenvalues = None, None
        res_cm, n_valid, i = 0.0, 0, 0
        for i in range(iter_n):
            _, res, sums = self._iterate(src, T_dev, 1, source_normals, source_sdf, source_colors, cdec, cgrad, cmode)
            r = res.cpu().numpy()  # the one host sync of the iteration
            n_valid, res_cm = int(r[16]), float(r[17])
            dT = r[:16].reshape(4, 4)
            if vis_result and converged and n_valid >= 10:
                cov_mat, eigenvalues = self._cov_eig(sums, r)
            if (res_cm - last_res_cm) / last_res_cm > 1.1:
                valid_flag = False  # residual must not grow (tracker.py:150-159)
            else:
                last_res_cm = res_cm
            if n_valid < min_valid_points or n_valid / n_src < min_valid_ratio:
                valid_flag = False
            if not valid_flag or converged:
                break
            if (_angle_deg(dT[:3, :3]) < cfg.reg_term_thre_deg and float(np.linalg.norm(dT[:3, 3])) < cfg.reg_term_thre_m) \
                    or i == iter_n - 2:
                converged = True
        if res_cm > max_final_res_cm:
            valid_flag = False
        if eigenvalues is not None and cfg.eigenvalue_check:
            if float(eigenvalues.min()) < n_valid * cfg.eigenvalue_ratio_thre:
                valid_flag = False
        if cov_mat is not None:
            cov_mat = cov_mat.numpy()
        T = T_dev
        if not valid_flag and i < 10:
            T = init_pose
            cov_mat = None
        return T, cov_mat, None, valid_flag

    def track_fixed(self, source_points, init_pose, n_iter: int, source_normals=None, source_sdf=None,
                    source_colors=None):
        """Exactly `n_iter` GN iterations with NO host synchronisation at all (benchmark configuration
        "tracker GN (3 iters)"): the pose stays on the device and K4 updates it in place."""
        cfg = self.config
        T_dev = init_pose.to(dtype=torch.float64).clone().contiguous()
        src = source_points.contiguous()
        cdec, cgrad, cmode = self._color_setup(source_colors)
        self._iterate(src, T_dev, n_iter, source_normals, source_sdf, source_colors, cdec, cgrad, cmode)
        return T_dev, self._result
