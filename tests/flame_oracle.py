"""Torch restatement of FlameHead.forward + lbs (flame_model/flame.py:485-558, flame_model/lbs.py:25-304) in the
reference's op order, for tests and measurements only.  Runs in float32 (the reference's own arithmetic) or float64
(the yardstick both are measured against).  tests/golden/make_golden_flame.py pins it against the real reference."""
import torch

POSED = ("expr", "rotation", "neck_pose", "jaw_pose", "eyes_pose", "translation")


def batch_rodrigues(rot_vecs):   # lbs.py:25-57, as written (no small-angle guard)
    B, dtype, device = rot_vecs.shape[0], rot_vecs.dtype, rot_vecs.device
    angle = torch.norm(rot_vecs + 1e-8, dim=1, keepdim=True)
    rot_dir = rot_vecs / angle
    cos = torch.unsqueeze(torch.cos(angle), dim=1)
    sin = torch.unsqueeze(torch.sin(angle), dim=1)
    rx, ry, rz = torch.split(rot_dir, 1, dim=1)
    zeros = torch.zeros((B, 1), dtype=dtype, device=device)
    K = torch.cat([zeros, -rz, ry, rz, zeros, -rx, -ry, rx, zeros], dim=1).view((B, 3, 3))
    ident = torch.eye(3, dtype=dtype, device=device).unsqueeze(dim=0)
    return ident + sin * K + (1 - cos) * torch.bmm(K, K)


def batch_rigid_transform(rot_mats, joints, parents):   # lbs.py:254-304
    joints = torch.unsqueeze(joints, dim=-1)
    rel_joints = joints.clone()
    rel_joints[:, 1:] = rel_joints[:, 1:] - joints[:, parents[1:]]
    R = rot_mats.reshape(-1, 3, 3)
    t = rel_joints.reshape(-1, 3, 1)
    transforms_mat = torch.cat([torch.nn.functional.pad(R, [0, 0, 0, 1]),
                                torch.nn.functional.pad(t, [0, 0, 0, 1], value=1)], dim=2)
    transforms_mat = transforms_mat.view(-1, joints.shape[1], 4, 4)
    chain = [transforms_mat[:, 0]]
    for i in range(1, len(parents)):
        chain.append(torch.matmul(chain[parents[i]], transforms_mat[:, i]))
    transforms = torch.stack(chain, dim=1)
    posed_joints = transforms[:, :, :3, 3]
    joints_homogen = torch.nn.functional.pad(joints, [0, 0, 0, 1])
    rel_transforms = transforms - torch.nn.functional.pad(torch.matmul(transforms, joints_homogen), [3, 0, 0, 0, 0, 0, 0, 0])
    return posed_joints, rel_transforms


def flame_forward(assets, shape, expr, rotation, neck, jaw, eyes, translation, static_offset=None):
    """One batch of FlameHead.forward(zero_centered_at_root_node=False, return_landmarks=False,
    return_verts_cano=True): (verts, verts_cano, posed joints), each with a leading batch dimension.  `assets` holds
    v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights in the arithmetic's dtype."""
    a = assets
    B = shape.shape[0]
    dtype = a["v_template"].dtype
    betas = torch.cat([shape, expr], dim=1)
    full_pose = torch.cat([rotation, neck, jaw, eyes], dim=1)
    v_shaped = a["v_template"].unsqueeze(0).expand(B, -1, -1) + torch.einsum("bl,mkl->bmk", [betas, a["shapedirs"]])
    if static_offset is not None:
        v_shaped = v_shaped + static_offset
    J = torch.einsum("bik,ji->bjk", [v_shaped, a["J_regressor"]])
    ident = torch.eye(3, dtype=dtype, device=v_shaped.device)
    rot_mats = batch_rodrigues(full_pose.view(-1, 3)).view([B, -1, 3, 3])
    pose_feature = (rot_mats[:, 1:, :, :] - ident).view([B, -1])
    pose_offsets = torch.matmul(pose_feature, a["posedirs"]).view(B, -1, 3)
    v_posed = pose_offsets + v_shaped
    J_transformed, A = batch_rigid_transform(rot_mats, J, list(a["parents"]))
    W = a["lbs_weights"].unsqueeze(dim=0).expand([B, -1, -1])
    nj = a["J_regressor"].shape[0]
    T = torch.matmul(W, A.view(B, nj, 16)).view(B, -1, 4, 4)
    homogen = torch.ones([B, v_posed.shape[1], 1], dtype=dtype, device=v_posed.device)
    v_homo = torch.matmul(T, torch.unsqueeze(torch.cat([v_posed, homogen], dim=2), dim=-1))
    verts = v_homo[:, :, :3, 0] + translation[:, None, :]
    return verts, v_shaped, J_transformed + translation[:, None, :]


def select_mesh_by_timestep(assets, flame_param, t):
    """scene/flame_gaussian_model.py:121-134 on the dict's tensors (dtype of the assets): (verts, verts_cano, joints)."""
    dt = assets["v_template"].dtype
    fp = {k: v.to(dt) if v.dtype != dt else v for k, v in flame_param.items() if v is not None}
    return flame_forward(assets, fp["shape"][None, ...], fp["expr"][[t]], fp["rotation"][[t]], fp["neck_pose"][[t]],
                         fp["jaw_pose"][[t]], fp["eyes_pose"][[t]], fp["translation"][[t]], fp.get("static_offset"))


def assets_as(assets, dtype, device=None):
    return {k: (v.to(dtype=dtype, device=device) if isinstance(v, torch.Tensor) and v.is_floating_point() else v)
            for k, v in assets.items()}
