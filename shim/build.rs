// build.rs — link the H100 engine.  DFGPU_LIB_DIR = directory holding libdfgpu.so
// (built by `make -C datafusion_archive_b200/csrc`).
fn main() {
    if let Ok(dir) = std::env::var("DFGPU_LIB_DIR") {
        println!("cargo:rustc-link-search=native={}", dir);
    }
    println!("cargo:rustc-link-lib=dylib=dfgpu");
    println!("cargo:rerun-if-env-changed=DFGPU_LIB_DIR");
}
