"""The drop-in boundary is a C ABI: a plain-C client (examples/c_abi_minimal.c) compiles against include/prisma_b200.h,
links libprisma_b200.so and runs without Python or torch in the process.  On a machine without an H100 it also shows
that engine creation fails loudly (negative code + message) instead of falling back."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_plain_c_client_links_and_runs(tmp_path):
    lib_dir = os.path.join(ROOT, "prisma_b200")
    exe = str(tmp_path / "c_abi_minimal")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", os.path.join(ROOT, "examples", "c_abi_minimal.c"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + lib_dir, "-lprisma_b200", "-Wl,-rpath," + lib_dir, "-o", exe])
    env = dict(os.environ)
    # libcudart comes with the CUDA toolkit / the pip nvidia-cuda-runtime wheel; let the loader find whichever is present
    import glob
    import sysconfig
    cands = glob.glob(os.path.join(sysconfig.get_paths()["purelib"], "nvidia", "cuda_runtime", "lib")) + ["/usr/local/cuda/lib64"]
    env["LD_LIBRARY_PATH"] = os.pathsep.join(cands + [env.get("LD_LIBRARY_PATH", "")])
    out = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "prisma_b200" in out.stdout and "depth_anything         1920x1080 -> 924x518" in out.stdout
    assert "mask_mmdet             1920x1080 -> 1333x750" in out.stdout
    assert "expected error: unknown band" in out.stdout
