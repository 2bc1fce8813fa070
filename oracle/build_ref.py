"""Build the reference's OWN native Vox-Fusion code as bit-level oracles (test infrastructure).

  oracle/_ref/svo.so    third_party/sparse_octree (CPU C++, TorchScript class svo.Octree)
  oracle/_ref/grid.so   third_party/sparse_voxels (CUDA ext `grid`: svo_intersect,
                        inverse_cdf_sampling, ...) cross-compiled for sm_90a

Sources are compiled where they lie under /root/reference (never copied); outputs go only to
oracle/_ref/ (git-ignored, NOT gpurun-ignored: the .so files travel to the GPU box, where
/root/reference does not exist).  The reference's own build system is not used: two direct
torch.utils.cpp_extension.load calls.  Eigen is absent from the image; the one type the octree
needs comes from oracle/shim/eigen3/Eigen/Dense.

Run:  python oracle/build_ref.py      (no-op when /root/reference is missing or up to date)
"""
import glob
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('XRDSLAM_REFERENCE', '/root/reference')
OUT = os.path.join(HERE, '_ref')


def _build(name, sources, includes, cuda):
    target = os.path.join(OUT, name + '.so')
    if os.path.exists(target) and all(
            os.path.getmtime(target) >= os.path.getmtime(s) for s in sources):
        return target
    from torch.utils.cpp_extension import load
    os.environ.setdefault('TORCH_CUDA_ARCH_LIST', '9.0a')
    bdir = os.path.join(OUT, 'build_' + name)
    os.makedirs(bdir, exist_ok=True)
    load(name=name, sources=sources, extra_include_paths=includes,
         extra_cflags=['-O2', '-Wno-narrowing'], with_cuda=cuda, build_directory=bdir,
         is_python_module=False, verbose=False)
    shutil.copy(os.path.join(bdir, name + '.so'), target)
    return target


def main():
    if not os.path.isdir(os.path.join(REF, 'third_party')):
        print('build_ref: reference not present, nothing to do')
        return
    os.makedirs(OUT, exist_ok=True)
    oct_dir = os.path.join(REF, 'third_party', 'sparse_octree')
    _build('svo', [os.path.join(oct_dir, 'src', 'octree.cpp'),
                   os.path.join(oct_dir, 'src', 'bindings.cpp')],
           [os.path.join(oct_dir, 'include'), os.path.join(HERE, 'shim')], cuda=False)
    vox_dir = os.path.join(REF, 'third_party', 'sparse_voxels')
    srcs = sorted(glob.glob(os.path.join(vox_dir, 'src', '*.cpp')) +
                  glob.glob(os.path.join(vox_dir, 'src', '*.cu')))
    _build('grid', srcs, [os.path.join(vox_dir, 'include')], cuda=True)
    print('build_ref: ok ->', sorted(os.listdir(OUT)))


if __name__ == '__main__':
    main()
