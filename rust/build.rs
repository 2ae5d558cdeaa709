// build.rs of the reference (build.rs:1-2: the capnpc stanza, unchanged) + the link stanza for the CUDA library.
//
//   DPLONK_ROOT=/path/to/this/repo cargo build --release --bin worker_gpu
//
// libdplonk.so is produced by `python -m distributed_plonk_b200.build`
// (nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared; the CUDA runtime is linked statically into it,
// so the Rust side needs no CUDA toolkit).  NCCL is only needed by worker_gpu's optional `nccl` feature (the
// fused peer-memory exchange of dp_peer_* needs nothing but the library).
fn main() {
    ::capnpc::CompilerCommand::new().file("src/hello_world.capnp").run().unwrap();

    let root = std::env::var("DPLONK_ROOT").expect("set DPLONK_ROOT to the distributed_plonk_b200 repository");
    println!("cargo:rustc-link-search=native={}/distributed_plonk_b200/_build", root);
    println!("cargo:rustc-link-lib=dylib=dplonk");
    println!("cargo:rustc-link-arg=-Wl,-rpath,{}/distributed_plonk_b200/_build", root);
    println!("cargo:rerun-if-env-changed=DPLONK_ROOT");
    println!("cargo:rerun-if-changed={}/include/dplonk.h", root);
    if std::env::var("CARGO_FEATURE_NCCL").is_ok() {
        println!("cargo:rustc-link-lib=dylib=nccl");
    }
}
