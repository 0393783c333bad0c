"""Wavefront OBJ I/O of the drop-in package on the H100 kernels (csrc/mesh_ops.cu).

Reference: SoftRas/functional/save_obj.py:9-33 (`create_texture_image`: face textures -> atlas image through
cuda/create_texture_image), :36-90 (`save_obj`), :96-104 (`save_voxel`), functional/load_obj.py:9-101 (`load_mtl`,
`load_textures`: atlas image -> face textures through cuda/load_textures), :104-167 (`load_obj`).  Image files are read /
written with PIL (the reference uses skimage, which is not a dependency here); everything between the file and the tensors
follows the reference.
"""
import os

import numpy as np
import torch

from ... import ops


def create_texture_image(textures, texture_res=16):
    """textures [F, R*R, 3] (cuda) -> (image [H,W,3] float32 numpy, flipped like the reference, vertices_textures [F,3,2])."""
    num_faces = textures.shape[0]
    tile_width = int((num_faces - 1.) ** 0.5) + 1
    tile_height = int((num_faces - 1.) / tile_width) + 1
    dev = textures.device
    image = torch.ones(tile_height * texture_res, tile_width * texture_res, 3, dtype=torch.float32, device=dev)
    vertices = torch.zeros((num_faces, 3, 2), dtype=torch.float32, device=dev)  # [:, :, UV]
    face_nums = torch.arange(num_faces, device=dev)
    column = (face_nums % tile_width).float()
    row = torch.div(face_nums, tile_width, rounding_mode="floor").float()  # (torch-1.1 integer division, save_obj.py:17)
    vertices[:, 0, 0] = column * texture_res + texture_res / 2
    vertices[:, 0, 1] = row * texture_res + 1
    vertices[:, 1, 0] = column * texture_res + 1
    vertices[:, 1, 1] = (row + 1) * texture_res - 1 - 1
    vertices[:, 2, 0] = (column + 1) * texture_res - 1 - 1
    vertices[:, 2, 1] = (row + 1) * texture_res - 1 - 1
    image = ops.create_texture_image(vertices, textures.detach().contiguous().float(), image, 1e-5)
    vertices[:, :, 0] /= (image.shape[1] - 1)
    vertices[:, :, 1] /= (image.shape[0] - 1)
    image = image.detach().cpu().numpy()[::-1, ::1]
    return image, vertices.detach().cpu().numpy()


def save_obj(filename, vertices, faces, textures=None, texture_res=16, texture_type="surface"):
    """functional/save_obj.py:36-90: geometry, and for surface textures an atlas PNG + .mtl."""
    assert vertices.ndimension() == 2 and faces.ndimension() == 2
    assert texture_type in ("surface", "vertex") and texture_res >= 2
    filename_mtl = filename[:-4] + ".mtl"
    filename_texture = filename[:-4] + ".png"
    material_name = "material_1"
    vertices_textures = None
    if textures is not None and texture_type == "surface":
        from PIL import Image
        texture_image, vertices_textures = create_texture_image(textures, texture_res)
        texture_image = (texture_image.clip(0, 1) * 255).astype("uint8")
        Image.fromarray(np.ascontiguousarray(texture_image)).save(filename_texture)
    faces = faces.detach().cpu().numpy()
    verts = vertices.detach().cpu().numpy()
    with open(filename, "w") as f:
        f.write("# %s\n#\n\n" % os.path.basename(filename))
        if textures is not None:
            f.write("mtllib %s\n\n" % os.path.basename(filename_mtl))
        if textures is not None and texture_type == "vertex":
            for v, c in zip(verts, textures.detach().cpu().numpy()):
                f.write("v %.8f %.8f %.8f %.8f %.8f %.8f\n" % (v[0], v[1], v[2], c[0], c[1], c[2]))
        else:
            for v in verts:
                f.write("v %.8f %.8f %.8f\n" % (v[0], v[1], v[2]))
        f.write("\n")
        if textures is not None and texture_type == "surface":
            for vt in vertices_textures.reshape((-1, 2)):
                f.write("vt %.8f %.8f\n" % (vt[0], vt[1]))
            f.write("\nusemtl %s\n" % material_name)
            for i, face in enumerate(faces):
                f.write("f %d/%d %d/%d %d/%d\n" % (face[0] + 1, 3 * i + 1, face[1] + 1, 3 * i + 2, face[2] + 1, 3 * i + 3))
            f.write("\n")
        else:
            for face in faces:
                f.write("f %d %d %d\n" % (face[0] + 1, face[1] + 1, face[2] + 1))
    if textures is not None and texture_type == "surface":
        with open(filename_mtl, "w") as f:
            f.write("newmtl %s\nmap_Kd %s\n" % (material_name, os.path.basename(filename_texture)))


def load_mtl(filename_mtl):
    """functional/load_obj.py:9-25: colours (Kd) and texture file names per material."""
    texture_filenames, colors, material_name = {}, {}, ""
    with open(filename_mtl) as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "newmtl":
                material_name = tok[1]
            if tok[0] == "map_Kd":
                texture_filenames[material_name] = tok[1]
            if tok[0] == "Kd":
                colors[material_name] = np.array(list(map(float, tok[1:4])))
    return colors, texture_filenames


def _vt_index(tok):
    return int(tok.split("/")[1]) if ("/" in tok and "//" not in tok) else 0


def load_textures(filename_obj, filename_mtl, texture_res, device="cuda"):
    """functional/load_obj.py:28-101: per-face surface textures [F, texture_res^2, 3] from the material's Kd / map_Kd."""
    with open(filename_obj) as f:
        lines = f.readlines()
    vts = np.vstack([[float(v) for v in ln.split()[1:3]] for ln in lines if ln.split() and ln.split()[0] == "vt"]).astype(np.float32)
    faces, material_names, material_name = [], [], ""
    for ln in lines:
        tok = ln.split()
        if not tok:
            continue
        if tok[0] == "f":
            vs = tok[1:]
            v0 = _vt_index(vs[0])
            for i in range(len(vs) - 2):
                faces.append((v0, _vt_index(vs[i + 1]), _vt_index(vs[i + 2])))
                material_names.append(material_name)
        if tok[0] == "usemtl":
            material_name = tok[1]
    faces = np.vstack(faces).astype(np.int32) - 1
    faces = torch.from_numpy(vts[faces]).to(device)
    faces[1 < faces] = faces[1 < faces] % 1
    colors, texture_filenames = load_mtl(filename_mtl)
    textures = torch.ones(faces.shape[0], texture_res ** 2, 3, dtype=torch.float32, device=device)
    names = np.array(material_names)
    for mname, color in colors.items():
        sel = torch.from_numpy(names == mname).to(device)
        textures[sel] = torch.from_numpy(color.astype(np.float32)).to(device)[None, None, :]
    for mname, fn in texture_filenames.items():
        from PIL import Image
        image = np.asarray(Image.open(os.path.join(os.path.dirname(filename_obj), fn))).astype(np.float32) / 255.
        if image.ndim == 2:
            image = np.stack((image,) * 3, -1)
        if image.shape[2] == 4:
            image = image[:, :, :3]
        image = torch.from_numpy(image[::-1, :, :].copy()).to(device)
        is_update = torch.from_numpy((names == mname).astype(np.int32)).to(device)
        textures = ops.load_textures(image, faces, textures, is_update)
    return textures


def load_obj(filename_obj, normalization=False, load_texture=False, texture_res=4, texture_type="surface"):
    """functional/load_obj.py:104-167: vertices [V,3] float32 and faces [F,3] int32 (polygons fan-triangulated) on the
    GPU, plus the textures with `load_texture` (surface: [F, texture_res^2, 3] from the .mtl; vertex: the colours of the
    `v` lines).  `normalization` centres and scales the vertices into [-1, 1]."""
    if texture_type not in ("surface", "vertex"):
        raise ValueError("texture type not applicable")
    verts, faces = [], []
    with open(filename_obj) as fh:
        for line in fh:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "f":
                ids = [int(x.split("/")[0]) - 1 for x in tok[1:]]
                faces.extend([ids[0], ids[k], ids[k + 1]] for k in range(1, len(ids) - 1))  # fan triangulation
    v = torch.tensor(verts, dtype=torch.float32).cuda()
    f = torch.tensor(faces, dtype=torch.int32).cuda()
    if normalization:  # centre and scale into [-1, 1]
        v = v - v.min(0)[0][None, :]
        v = v / torch.abs(v).max()
        v = v * 2
        v = v - v.max(0)[0][None, :] / 2
    if not load_texture:
        return v, f
    if texture_type == "surface":  # :139-146
        with open(filename_obj) as fh:
            mtl = [ln.split()[1] for ln in fh if ln.startswith("mtllib")]
        if not mtl:
            raise Exception("Failed to load textures.")
        textures = load_textures(filename_obj, os.path.join(os.path.dirname(filename_obj), mtl[-1]), texture_res)
    else:  # :147-154: colours ride on the `v` lines
        with open(filename_obj) as fh:
            cols = [[float(x) for x in ln.split()[4:7]] for ln in fh if ln.split() and ln.split()[0] == "v"]
        textures = torch.tensor(cols, dtype=torch.float32).cuda()
    return v, f, textures


def save_voxel(filename, voxel):
    """save_obj.py:96-104: one OBJ vertex (i/n0, j/n1, k/n2) per voxel equal to 1, in i, j, k order, and no faces.  (The
    reference hands its own `save_obj` a 1-D empty face tensor, which that function's assertion rejects; this writes the
    file it means to write, in `save_obj`'s format.)"""
    vox = voxel.detach().cpu().numpy() if torch.is_tensor(voxel) else np.asarray(voxel)
    idx = np.argwhere(vox == 1)  # row-major: the reference's i, j, k loop order
    verts = (idx / np.asarray(vox.shape, dtype=np.float64)).astype(np.float32)  # torch.tensor(list of floats): float32
    with open(filename, "w") as f:
        f.write("# %s\n#\n\n" % os.path.basename(filename))
        for v in verts:
            f.write("v %.8f %.8f %.8f\n" % (v[0], v[1], v[2]))
        f.write("\n")
