// libb200pde.so is built by `python -m rustpde_mpi_b200.build` (nvcc, sm_90a); point B200PDE_LIB_DIR at its directory.
fn main() {
    let dir = std::env::var("B200PDE_LIB_DIR").unwrap_or_else(|_| "../../rustpde_mpi_b200".to_string());
    println!("cargo:rustc-link-search=native={}", dir);
    println!("cargo:rustc-link-lib=dylib=b200pde");
    println!("cargo:rerun-if-env-changed=B200PDE_LIB_DIR");
}
