"""GenericTrainer (inference subset: mode='val' and mode='export_mesh') on the o2345 kernels.

Mirror of reference reconstruction/models/trainer_generic.py: constructor :18-125, forward dispatch
:1052-1103, val_step :359-545, export_mesh_step :827-979, obtain_pyramid_feature_maps :1104-1125,
validate_colored_mesh :1309-1380.  Training (`train_step`, losses) stays with the reference.

With num_lods = 2 (the lod-1 refinement: a second, twice as fine volume built from the pruned lod-0 SDF) export_mesh
writes and returns only the lod-1 coloured mesh.  The reference also builds the lod-0 coloured mesh first and writes it
to the same <exp>/mesh.ply, which the lod-1 mesh then overwrites; that mesh is skipped here.
"""
from __future__ import annotations

import os
import time

import numpy as np
import torch
import torch.nn as nn

from .featurenet import obtain_pyramid_feature_maps
from .sparse_neus_renderer import SparseNeuSRenderer


from .mesh_io import merge_vertices, write_ply  # noqa: E402,F401  (write_ply re-exported: tests and tools import it from here)


class GenericTrainer(nn.Module):
    def __init__(self, rendering_network_outside, pyramid_feature_network_lod0, pyramid_feature_network_lod1,
                 sdf_network_lod0, sdf_network_lod1, variance_network_lod0, variance_network_lod1,
                 rendering_network_lod0, rendering_network_lod1, n_samples_lod0, n_importance_lod0, n_samples_lod1,
                 n_importance_lod1, n_outside, perturb, alpha_type='div', conf=None, timestamp="", mode='train',
                 base_exp_dir=None):
        super().__init__()
        self.conf, self.timestamp, self.base_exp_dir = conf, timestamp, base_exp_dir
        self.rendering_network_outside = rendering_network_outside
        self.pyramid_feature_network_geometry_lod0 = pyramid_feature_network_lod0
        self.pyramid_feature_network_geometry_lod1 = pyramid_feature_network_lod1
        self.sdf_network_lod0, self.sdf_network_lod1 = sdf_network_lod0, sdf_network_lod1
        self.variance_network_lod0, self.variance_network_lod1 = variance_network_lod0, variance_network_lod1
        self.rendering_network_lod0, self.rendering_network_lod1 = rendering_network_lod0, rendering_network_lod1
        self.n_samples_lod0, self.n_importance_lod0 = n_samples_lod0, n_importance_lod0
        self.n_samples_lod1, self.n_importance_lod1 = n_samples_lod1, n_importance_lod1
        self.n_outside, self.perturb, self.alpha_type = n_outside, perturb, alpha_type
        self.num_lods = conf.get_int('model.num_lods')
        if self.num_lods not in (1, 2):
            raise NotImplementedError(f"num_lods={self.num_lods}: 1 or 2 levels are on the accelerated path")
        self.prune_depth_filter = conf.get_bool('model.prune_depth_filter', default=False)
        if self.prune_depth_filter:
            raise NotImplementedError("model.prune_depth_filter (depth-map filtered pruning) is not on the accelerated path")
        self.sdf_renderer_lod0 = SparseNeuSRenderer(rendering_network_outside, sdf_network_lod0, variance_network_lod0,
                                                    rendering_network_lod0, n_samples_lod0, n_importance_lod0,
                                                    n_outside, perturb, alpha_type='div', conf=conf)
        self.sdf_renderer_lod1 = None
        if self.num_lods > 1:
            missing = [n for n, m in (("pyramid_feature_network_lod1", pyramid_feature_network_lod1),
                                      ("sdf_network_lod1", sdf_network_lod1), ("variance_network_lod1", variance_network_lod1),
                                      ("rendering_network_lod1", rendering_network_lod1)) if m is None]
            if missing:
                raise ValueError(f"num_lods = 2 needs {', '.join(missing)}")
            self.sdf_renderer_lod1 = SparseNeuSRenderer(rendering_network_outside, sdf_network_lod1, variance_network_lod1,
                                                        rendering_network_lod1, n_samples_lod1, n_importance_lod1,
                                                        n_outside, perturb, alpha_type='div', conf=conf)
        self.val_mesh_freq = 1

    def obtain_pyramid_feature_maps(self, imgs, lod=0):
        extractor = self.pyramid_feature_network_geometry_lod0 if lod == 0 else self.pyramid_feature_network_geometry_lod1
        return obtain_pyramid_feature_maps(extractor, imgs)

    def forward(self, sample, perturb_overwrite=-1, background_rgb=None, alpha_inter_ratio_lod0=0.0,
                alpha_inter_ratio_lod1=0.0, iter_step=0, mode='train', save_vis=False, resolution=360, target_faces=None,
                texture_size=None, normal_map=False, atlas="faces", project_view=None, min_component=None,
                ambient_occlusion=False, remesh=False):
        if mode == 'val':
            return self.val_step(sample, perturb_overwrite=perturb_overwrite, background_rgb=background_rgb,
                                 alpha_inter_ratio_lod0=alpha_inter_ratio_lod0, alpha_inter_ratio_lod1=alpha_inter_ratio_lod1,
                                 iter_step=iter_step, save_vis=save_vis)
        if mode == 'export_mesh':
            return self.export_mesh_step(sample, iter_step=iter_step, save_vis=save_vis, resolution=resolution,
                                         target_faces=target_faces, texture_size=texture_size, normal_map=normal_map,
                                         atlas=atlas, **({} if project_view is None else {"project_view": project_view}),
                                         **({} if min_component is None else {"min_component": min_component}),
                                         **({"ambient_occlusion": True} if ambient_occlusion else {}),
                                         **({"remesh": True} if remesh else {}))
        raise NotImplementedError(f"mode={mode!r}: only 'val' and 'export_mesh' run on the o2345 path")

    # ------------------------------------------------------------------ shared front end
    @torch.no_grad()
    def _conditional_features(self, sample):
        sizeW, sizeH = int(sample['img_wh'][0][0]), int(sample['img_wh'][0][1])
        imgs = sample['images'][0]
        fmaps = self.obtain_pyramid_feature_maps(imgs, lod=0)
        cond = self.sdf_network_lod0.get_conditional_volume(
            feature_maps=fmaps[None], partial_vol_origin=sample['partial_vol_origin'],
            proj_mats=sample['affine_mats'], sizeH=sizeH, sizeW=sizeW, lod=0)
        return imgs, fmaps, cond, sizeW, sizeH

    @torch.no_grad()
    def _lod1_volume(self, sample, imgs, cond, sizeW, sizeH):
        """lod-0 SDF volume -> pruned lod-0 voxels -> lod-1 conditional volume (reference :897-932); also returns the
        lod-1 feature maps."""
        origin = sample['partial_vol_origin']
        vol0, occ0, coords0 = cond['dense_volume_scale0'], cond['valid_mask_volume_scale0'], cond['coords_scale0']
        sdf0 = self.sdf_network_lod0.get_sdf_volume(vol0, occ0, coords0, origin)
        fmaps1 = self.obtain_pyramid_feature_maps(imgs, lod=1)
        pre_coords, pre_feats = self.sdf_renderer_lod0.get_valid_sparse_coords_by_sdf(sdf0[0], coords0[0], occ0[0], vol0[0])
        pre_coords[:, 1:] = pre_coords[:, 1:] * 2
        cond1 = self.sdf_network_lod1.get_conditional_volume(
            feature_maps=fmaps1[None], partial_vol_origin=origin, proj_mats=sample['affine_mats'], sizeH=sizeH, sizeW=sizeW,
            pre_coords=pre_coords, pre_feats=pre_feats)
        return fmaps1, cond1

    # ------------------------------------------------------------------ mode='val'
    @torch.no_grad()
    def val_step(self, sample, perturb_overwrite=-1, background_rgb=None, alpha_inter_ratio_lod0=0.0,
                 alpha_inter_ratio_lod1=0.0, iter_step=0, chunk_size=512, save_vis=False):
        """Renders the query view.  Returns dict(color [H*W,3], depth [H*W,1], normal [H*W,3]) as numpy,
        like the per-chunk host copies of the reference (:526-543) but with one copy at the end.
        `chunk_size` rays are marched per launch group (the reference uses 512; larger is faster)."""
        imgs, fmaps, cond, sizeW, sizeH = self._conditional_features(sample)
        levels = [("", self.sdf_renderer_lod0, self.sdf_network_lod0, self.rendering_network_lod0, alpha_inter_ratio_lod0,
                   cond['dense_volume_scale0'], cond['valid_mask_volume_scale0'], fmaps)]
        if self.num_lods > 1:
            fmaps1, cond1 = self._lod1_volume(sample, imgs, cond, sizeW, sizeH)
            levels.append(("_lod1", self.sdf_renderer_lod1, self.sdf_network_lod1, self.rendering_network_lod1,
                           alpha_inter_ratio_lod1, cond1['dense_volume_scale1'], cond1['valid_mask_volume_scale1'], fmaps1))
        near, far = sample['query_near_far'][0, :1], sample['query_near_far'][0, 1:]
        rays_o = sample['rays']['rays_o'][0].reshape(-1, 3)
        rays_d = sample['rays']['rays_v'][0].reshape(-1, 3)
        result = {}
        # every chunk of lod 0, then every chunk of lod 1 (reference :503-589): the host generator's draws follow that order
        for lod, (suffix, renderer, sdf_net, rnet, ratio, vol, occ, fm) in enumerate(levels):
            colors, depths, normals = [], [], []
            for ro, rd in zip(rays_o.split(chunk_size), rays_d.split(chunk_size)):
                out = renderer.render(
                    ro, rd, near, far, sdf_net, rnet, perturb_overwrite=perturb_overwrite, background_rgb=background_rgb,
                    alpha_inter_ratio=ratio, lod=lod, conditional_volume=vol, conditional_valid_mask_volume=occ,
                    feature_maps=fm, color_maps=imgs, w2cs=sample['w2cs'][0], intrinsics=sample['intrinsics'][0],
                    img_wh=[sizeW, sizeH], query_c2w=sample['query_c2w'], if_render_with_grad=False)
                colors.append(out['color_fine'])
                depths.append(out['depth'])
                normals.append((out['gradients'] * out['weights'][:, :, None] * out['inside_sphere'][..., None]).sum(dim=1))
            result.update({"color" + suffix: torch.cat(colors).cpu().numpy(), "depth" + suffix: torch.cat(depths).cpu().numpy(),
                           "normal" + suffix: torch.cat(normals).cpu().numpy()})
        return result

    # ------------------------------------------------------------------ any camera
    @torch.no_grad()
    def render_cameras(self, sample, c2ws, intrinsics, near_far, img_wh=None, chunk_size=65536, background_rgb=None,
                       alpha_inter_ratio=0.0):
        """Volume-renders the scene of `sample` from C cameras of its normalised frame (synthetic.normalise_cameras):
        c2ws [C,4,4] OpenCV c2w, intrinsics [C,3,3] (or one [3,3]), near_far [C,2].  The feature maps and the conditional
        volume are built once; the rays of every camera (pixel centres as the query view's, row-major) are concatenated
        and marched in launch groups of `chunk_size` rays that may mix cameras.  With num_lods = 2 the lod-1 level (the
        one export_mesh meshes) is rendered.  No jitter and no draws from the host generator: camera c gets the bits of
        val_step(perturb_overwrite=0) for a sample whose query camera is c.
        Returns device tensors: color [C,H,W,3], depth [C,H,W], normal [C,H,W,3] (val_step's formula) and weights_sum
        [C,H,W] (the opacity, for RGBA frames)."""
        from .synthetic import query_rays
        as_np = lambda x: (x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)).astype(np.float32)
        c2ws = as_np(c2ws).reshape(-1, 4, 4)
        n_cam = len(c2ws)
        if chunk_size < 1 or n_cam == 0:
            raise ValueError(f"chunk_size must be >= 1 and at least one camera is needed (got {chunk_size}, {n_cam})")
        intrinsics = np.broadcast_to(as_np(intrinsics).reshape(-1, 3, 3), (n_cam, 3, 3))
        near_far = as_np(near_far).reshape(n_cam, 2)
        imgs, fmaps, cond, sizeW, sizeH = self._conditional_features(sample)
        renderer, sdf_net, rnet, vol, occ, fm = (self.sdf_renderer_lod0, self.sdf_network_lod0, self.rendering_network_lod0,
                                                 cond['dense_volume_scale0'], cond['valid_mask_volume_scale0'], fmaps)
        if self.num_lods > 1:
            fmaps1, cond1 = self._lod1_volume(sample, imgs, cond, sizeW, sizeH)
            renderer, sdf_net, rnet, vol, occ, fm = (self.sdf_renderer_lod1, self.sdf_network_lod1, self.rendering_network_lod1,
                                                     cond1['dense_volume_scale1'], cond1['valid_mask_volume_scale1'], fmaps1)
        W, H = (sizeW, sizeH) if img_wh is None else (int(img_wh[0]), int(img_wh[1]))
        dev = vol.device
        HW = H * W
        rays = [query_rays(k, c, H, W) for k, c in zip(intrinsics, c2ws)]
        rays_o = torch.from_numpy(np.concatenate([o for o, _ in rays])).to(dev)
        rays_d = torch.from_numpy(np.concatenate([v for _, v in rays])).to(dev)
        nf = torch.from_numpy(np.repeat(near_far, HW, axis=0)).to(dev)
        # val_step marches 512-ray chunks and sums the normals per chunk; torch's reduction order depends on the tensor
        # shape, so the normals are summed over the same per-camera 512-ray units.  A launch group is whole units.
        unit = min(512, chunk_size)
        units = [(c * HW + a, c * HW + min(a + unit, HW)) for c in range(n_cam) for a in range(0, HW, unit)]
        groups, start = [], 0
        for i in range(1, len(units) + 1):
            if i == len(units) or units[i][1] - units[start][0] > max(chunk_size, unit):
                groups.append(units[start:i])
                start = i
        color = torch.empty(n_cam * HW, 3, device=dev)
        depth, opacity = torch.empty(n_cam * HW, 1, device=dev), torch.empty(n_cam * HW, 1, device=dev)
        normal = torch.empty(n_cam * HW, 3, device=dev)
        for g in groups:
            a, b = g[0][0], g[-1][1]
            out = renderer.render_views(rays_o[a:b], rays_d[a:b], nf[a:b, 0], nf[a:b, 1], sdf_net, rnet, vol, occ, fm, imgs,
                                        sample['w2cs'][0], sample['intrinsics'][0], [sizeW, sizeH],
                                        background_rgb=background_rgb, alpha_inter_ratio=alpha_inter_ratio)
            color[a:b], depth[a:b], opacity[a:b] = out["color"], out["depth"], out["weights_sum"]
            terms = out['gradients'] * out['weights'][:, :, None] * out['inside_sphere'][..., None]    # elementwise: any shape
            for u0, u1 in g:
                torch.sum(terms[u0 - a:u1 - a], dim=1, out=normal[u0:u1])
        return {"color": color.view(n_cam, H, W, 3), "depth": depth.view(n_cam, H, W), "normal": normal.view(n_cam, H, W, 3),
                "weights_sum": opacity.view(n_cam, H, W)}

    # ------------------------------------------------------------------ mode='export_mesh'
    @torch.no_grad()
    def export_mesh_step(self, sample, iter_step=0, chunk_size=512, resolution=360, save_vis=False, target_faces=None,
                         texture_size=None, normal_map=False, atlas="faces", project_view=None, min_component=None,
                         ambient_occlusion=False, remesh=False):
        """The coloured marching-cubes mesh; with target_faces it is simplified to that many faces (o2345/mesh_simplify.py)
        after the vertex merge and before mesh.ply is written.  With texture_size N the final mesh's colours are also baked
        into an N x N texture (o2345/mesh_texture.py): the result gains uv [F,3,2] and texture uint8 [N,N,3]; mesh.ply is
        written as without it.  normal_map (needs texture_size) also bakes the SDF gradient into a tangent-space normal
        map in the same uv: the result gains normal_texture uint8 [N,N,3].  atlas selects mesh_texture.bake's atlas
        ("faces" or "charts").  project_view: dict(photo uint8 [H,W,3] on white, alpha uint8 [H,W] or None), the input
        view (view 0) at any resolution: it is projected onto the final mesh from the query camera (sample['query_w2c'] and
        the shared intrinsics, rescaled from img_wh to the photo's size by mesh_texture.rescale_intrinsics), into the
        vertex colours and the baked texture (validate_colored_mesh).  min_component F: the components smaller than F times
        the largest one's area, or enclosed by it, are dropped after the vertex merge (o2345/mesh_clean.py), before
        target_faces, the projection and the bake; the result gains clean (its counts).  ambient_occlusion (needs
        texture_size) also bakes an occlusion map (validate_colored_mesh): the result gains occlusion_texture.  remesh
        (needs target_faces) replaces the simplification by an isotropic remesh (validate_colored_mesh)."""
        imgs, fmaps, cond, sizeW, sizeH = self._conditional_features(sample)
        kw = {} if min_component is None else {"min_component": min_component}
        kw = dict(kw, ambient_occlusion=True) if ambient_occlusion else kw
        kw = dict(kw, remesh=True) if remesh else kw
        if project_view is not None:
            from .mesh_texture import rescale_intrinsics
            K = sample['intrinsics'][0][0].cpu().numpy()           # every view of a scene shares K (synthetic.scene_cameras)
            H, W = np.shape(project_view["photo"])[:2]
            kw["project_view"] = dict(project_view, w2c=sample['query_w2c'][0][:3, :4],
                                      intr=rescale_intrinsics((K[0, 0], K[1, 1], K[0, 2], K[1, 2]), (sizeW, sizeH), (W, H)))
        if self.num_lods > 1:
            # the lod-1 mesh is coloured with the lod-0 feature maps, as in the reference (:959-978)
            _, cond1 = self._lod1_volume(sample, imgs, cond, sizeW, sizeH)
            return self.validate_colored_mesh(
                density_or_sdf_network=self.sdf_network_lod1,
                func_extract_geometry=self.sdf_renderer_lod1.extract_geometry, resolution=resolution,
                conditional_volume=cond1['dense_volume_scale1'],
                conditional_valid_mask_volume=cond1['valid_mask_volume_scale1'], feature_maps=fmaps, color_maps=imgs,
                w2cs=sample['w2cs'][0], intrinsics=sample['intrinsics'][0],
                rendering_network=self.rendering_network_lod1, lod=1, threshold=0, query_c2w=sample['query_c2w'],
                scale_mat=sample['scale_mat'], trans_mat=sample['trans_mat'], img_wh=[sizeW, sizeH], target_faces=target_faces,
                texture_size=texture_size, normal_map=normal_map, atlas=atlas, **kw)
        return self.validate_colored_mesh(
            density_or_sdf_network=self.sdf_network_lod0,
            func_extract_geometry=self.sdf_renderer_lod0.extract_geometry, resolution=resolution,
            conditional_volume=cond['dense_volume_scale0'],
            conditional_valid_mask_volume=cond['valid_mask_volume_scale0'], feature_maps=fmaps, color_maps=imgs,
            w2cs=sample['w2cs'][0], intrinsics=sample['intrinsics'][0],
            rendering_network=self.rendering_network_lod0, lod=0, threshold=0, query_c2w=sample['query_c2w'],
            scale_mat=sample['scale_mat'], trans_mat=sample['trans_mat'], img_wh=[sizeW, sizeH], target_faces=target_faces,
            texture_size=texture_size, normal_map=normal_map, atlas=atlas, **kw)

    @torch.no_grad()
    def validate_colored_mesh(self, density_or_sdf_network, func_extract_geometry, world_space=True, resolution=360,
                              threshold=0.0, mode='val', conditional_volume=None, conditional_valid_mask_volume=None,
                              feature_maps=None, color_maps=None, w2cs=None, target_candidate_w2cs=None,
                              intrinsics=None, rendering_network=None, rendering_projector=None, query_c2w=None,
                              lod=None, occupancy_mask=None, bound_min=[-1, -1, -1], bound_max=[1, 1, 1], meta='',
                              iter_step=0, scale_mat=None, trans_mat=None, img_wh=(256, 256), target_faces=None,
                              texture_size=None, colour_chunk=1 << 20, normal_map=False, atlas="faces", project_view=None,
                              min_component=None, ambient_occlusion=False, remesh=False):
        """project_view: dict(photo, alpha, w2c, intr) of a camera in the normalised frame (mesh_texture.prepare_view): the
        photo is blended into the final mesh's vertex colours (its vertex normals) and baked texture (its face normals),
        with one depth buffer of that mesh; the result gains project_weight [n] (the vertices' weights of the photo).
        min_component: 0 < F <= 1, the welded mesh is cleaned (o2345/mesh_clean.py) before everything that follows; the
        result gains clean, the counts of mesh_clean.clean.  ambient_occlusion (needs texture_size): the AO of every
        vertex of the welded (and cleaned) full mesh, before target_faces, is transferred onto the final mesh's texels
        (mesh_texture.ao_transfer_fn) and baked into occlusion_texture uint8 [N,N]; mesh.ply and the colours are as
        without it.  remesh (needs target_faces): the welded (and cleaned) mesh in the normalised frame is remeshed
        isotropically to about target_faces faces (o2345/mesh_remesh.py) instead of simplified; its vertices go to the
        world frame by the same scale_mat / trans_mat formula, its colours are colour() at its own vertices (quantised as
        above), and the projection and the bake read its arrays; the result gains remesh (mesh_remesh.remesh's stats)."""
        if remesh and target_faces is None:
            raise ValueError("remesh needs target_faces")
        if normal_map and texture_size is None:
            raise ValueError("normal_map needs texture_size")
        if ambient_occlusion and texture_size is None:
            raise ValueError("ambient_occlusion needs texture_size")
        bmin = torch.tensor(bound_min, dtype=torch.float32)
        bmax = torch.tensor(bound_max, dtype=torch.float32)
        vertices, triangles, fields = func_extract_geometry(
            density_or_sdf_network, bmin, bmax, resolution=resolution, threshold=threshold,
            device=conditional_volume.device, conditional_volume=conditional_volume, lod=lod,
            occupancy_mask=occupancy_mask)
        renderer = self.sdf_renderer_lod1 if lod == 1 else self.sdf_renderer_lod0
        vt = torch.tensor(vertices).to(conditional_volume)

        def colour(points):
            return renderer.blend_points(points, density_or_sdf_network, rendering_network, conditional_volume,
                                         conditional_valid_mask_volume, feature_maps, color_maps, w2cs, intrinsics, img_wh)[0]
        rgb = colour(vt)
        normalised = vertices

        def to_world(vertices):
            if scale_mat is not None:
                sm = scale_mat.cpu().numpy()
                vertices = vertices * sm[0][0, 0] + sm[0][:3, 3][None]
            if trans_mat is not None:
                tm = trans_mat.cpu().numpy().reshape(-1, 4, 4)[0]
                vh = np.concatenate([vertices, np.ones_like(vertices[:, :1])], axis=1)
                vertices = (vh @ tm.T)[:, :3]
            return vertices
        vertices = to_world(vertices)
        colors = (rgb.cpu() * 255).numpy().astype(np.uint8)
        # trimesh.Trimesh(vertices, triangles, vertex_colors=...) with its default process=True merges coincident vertices
        # before the export (reference :1374-1380).  Marching-cubes vertices can only coincide on lattice points: the renderer
        # listed the vertices that sit on one (on the device), and only those are compared.
        # each kept vertex's index into the extraction's arrays rides along with the colours (merge and simplify gather)
        vertices, triangles, kept = merge_vertices(vertices, triangles, np.arange(len(colors)),
                                                   candidates=getattr(renderer, "mc_lattice_candidates", None))
        cleaned = None
        if min_component is not None:
            # floating fragments and inner shells go before they take faces, texels or colours from the object
            from .mesh_clean import clean
            vertices, triangles, kept, cleaned = clean(vertices, triangles, kept, min_component, conditional_volume.device)
        ao_fn = None
        if ambient_occlusion:
            # the full surface's own cavities, in the normalised frame, before simplification takes them out
            from .mesh_texture import ao_transfer_fn
            ao_fn = ao_transfer_fn(normalised[kept], triangles, texture_size, conditional_volume.device)
        remeshed = None
        if remesh:
            # new vertices on the full surface: their own positions, world positions and colours
            from .mesh_remesh import remesh as remesh_mesh
            norm_k, triangles, remeshed = remesh_mesh(normalised[kept], triangles, None, target_faces,
                                                      conditional_volume.device)
            vertices = to_world(norm_k)
            rgb_k0 = colour(torch.tensor(norm_k).to(conditional_volume)) if len(norm_k) else rgb[:0]
            colors = (rgb_k0.cpu() * 255).numpy().astype(np.uint8)
        elif target_faces is not None:
            from .mesh_simplify import simplify
            vertices, triangles, kept, _ = simplify(vertices, triangles, kept, target_faces, conditional_volume.device)
        if not remesh:
            norm_k = normalised[kept]
        weight = None
        if project_view is None:
            colors = colors if remesh else colors[kept]
        else:
            # the final mesh in the normalised frame, where the query camera is
            from .mesh_texture import prepare_view, project_vertex_colors, quantise
            dev = conditional_volume.device
            vk = torch.from_numpy(np.ascontiguousarray(norm_k, np.float32)).to(dev)
            fk = torch.from_numpy(np.ascontiguousarray(triangles, np.int32)).to(dev)
            project_view = prepare_view(vk, fk, project_view)
            base = rgb_k0 if remesh else rgb[torch.from_numpy(np.asarray(kept)).long().to(dev)]
            rgb_k, weight = project_vertex_colors(vk, fk, base, project_view)
            colors = quantise(rgb_k)
        if self.base_exp_dir is not None:
            os.makedirs(self.base_exp_dir, exist_ok=True)
            write_ply(os.path.join(self.base_exp_dir, 'mesh.ply'), vertices, triangles, colors)
        out = {"vertices": vertices, "triangles": triangles, "colors": colors, "fields": fields}
        if cleaned is not None:
            out["clean"] = cleaned
        if remeshed is not None:
            out["remesh"] = remeshed
        if weight is not None:
            out["project_weight"] = weight.cpu().numpy()           # each vertex's weight of the photo
        if texture_size is not None:
            # baked in the normalised frame, where blend_points evaluates (the charts only scale with scale_mat)
            from .mesh_texture import bake
            chunked = lambda p: torch.cat([colour(c) for c in p.split(colour_chunk)]) if len(p) else p
            # the normal map's source is the SDF gradient at the texel points: the reconstruction's own surface normal
            gradient = lambda p: (torch.cat([density_or_sdf_network.gradient(c, conditional_volume, lod)[:, 0]
                                             for c in p.split(colour_chunk)]) if len(p) else p)
            baked = bake(norm_k, triangles, texture_size, chunked, conditional_volume.device,
                         **({"normal_fn": gradient} if normal_map else {}), **({} if atlas == "faces" else {"atlas": atlas}),
                         **({} if project_view is None else {"view": project_view}),
                         **({} if ao_fn is None else {"ao_fn": ao_fn}))
            out["uv"], out["texture"] = baked[:2]
            if normal_map:
                out["normal_texture"] = baked[2]
            if ao_fn is not None:
                out["occlusion_texture"] = baked[-1]
        return out
