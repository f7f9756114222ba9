"""Import shim: with `<repo>/gaussianavatars_b200/compat` first on sys.path, the reference's `import nvdiffrast.torch
as dr` (mesh_renderer/__init__.py:10) resolves to this library's mesh kernels (nvdiffrast/torch.py)."""
