// splat_cuda_module.cpp — torch binding that re-exports the C ABI (include/gsr_b200.h) under the
// reference's module surface: the 14 callables of src/bindings.cpp:118-159 with the same names,
// argument order, in-place-output convention and error behaviour (TORCH_CHECK -> RuntimeError;
// checks mirror src/checks.cuh:5-14 and the per-op shape checks), plus the fused entry points
// used by gaussian_splatting_b200.rasterize.  Tensors are only unwrapped to raw pointers here;
// all arithmetic is behind the C ABI.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <tuple>

#include "../../include/gsr_b200.h"

namespace {

#define CHECK_VALID_INPUT(x)                                        \
    TORCH_CHECK((x).is_cuda(), #x " is not a CUDA tensor");         \
    TORCH_CHECK((x).is_contiguous(), #x " is not a contiguous tensor")
#define CHECK_FLOAT_TENSOR(x) TORCH_CHECK((x).dtype() == torch::kFloat32, #x " is not a float tensor")
#define CHECK_DOUBLE_TENSOR(x) TORCH_CHECK((x).dtype() == torch::kFloat64, #x " is not a double tensor")
#define CHECK_INT_TENSOR(x) TORCH_CHECK((x).dtype() == torch::kInt32, #x " is not an int tensor")

inline void* cur_stream() { return (void*)at::cuda::getCurrentCUDAStream().stream(); }

inline void check_rc(int rc, const char* what) {
    TORCH_CHECK(rc == 0, what, " failed with status ", rc,
                rc > 0 ? std::string(" (") + cudaGetErrorString((cudaError_t)rc) + ")" : std::string());
}

// dtype of `lead`; every tensor in `rest` must match (reference: CHECK_FLOAT_TENSOR / CHECK_DOUBLE_TENSOR)
inline int common_dtype(const torch::Tensor& lead, std::initializer_list<const torch::Tensor*> rest) {
    if (lead.dtype() == torch::kFloat32) {
        for (auto* t : rest) TORCH_CHECK(t->dtype() == torch::kFloat32, "tensor is not a float tensor");
        return GSR_F32;
    }
    if (lead.dtype() == torch::kFloat64) {
        for (auto* t : rest) TORCH_CHECK(t->dtype() == torch::kFloat64, "tensor is not a double tensor");
        return GSR_F64;
    }
    AT_ERROR("Inputs must be float32 or float64");
}

// ---------------------------------------------------------------------------------------------
// per-Gaussian operators
// ---------------------------------------------------------------------------------------------
void camera_projection_cuda(torch::Tensor xyz, torch::Tensor K, torch::Tensor uv) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(K); CHECK_VALID_INPUT(uv);
    const int N = xyz.size(0);
    TORCH_CHECK(xyz.size(1) == 3, "xyz must have shape Nx3");
    TORCH_CHECK(K.size(0) == 3 && K.size(1) == 3, "K must have shape 3x3");
    TORCH_CHECK(uv.size(0) == N && uv.size(1) == 2, "uv must have shape Nx2");
    const int dt = common_dtype(xyz, {&K, &uv});
    c10::cuda::CUDAGuard guard(xyz.device());
    check_rc(gsr_camera_projection(dt, N, xyz.data_ptr(), K.data_ptr(), uv.data_ptr(), cur_stream()),
             "camera_projection_cuda");
}

void camera_projection_backward_cuda(torch::Tensor xyz, torch::Tensor K, torch::Tensor uv_grad_out,
                                     torch::Tensor xyz_grad_in) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(K); CHECK_VALID_INPUT(uv_grad_out); CHECK_VALID_INPUT(xyz_grad_in);
    const int N = xyz.size(0);
    TORCH_CHECK(xyz.size(1) == 3, "xyz must be of shape Nx3");
    TORCH_CHECK(K.size(0) == 3 && K.size(1) == 3, "K must be of shape 3x3");
    TORCH_CHECK(uv_grad_out.size(0) == N && uv_grad_out.size(1) == 2, "uv_grad_out must be of shape Nx2");
    TORCH_CHECK(xyz_grad_in.size(0) == N && xyz_grad_in.size(1) == 3, "xyz_grad_in must be of shape Nx3");
    const int dt = common_dtype(xyz, {&K, &uv_grad_out, &xyz_grad_in});
    c10::cuda::CUDAGuard guard(xyz.device());
    check_rc(gsr_camera_projection_backward(dt, N, xyz.data_ptr(), K.data_ptr(), uv_grad_out.data_ptr(),
                                            xyz_grad_in.data_ptr(), cur_stream()),
             "camera_projection_backward_cuda");
}

void compute_sigma_world_cuda(torch::Tensor quaternion, torch::Tensor scale, torch::Tensor sigma_world) {
    CHECK_VALID_INPUT(quaternion); CHECK_VALID_INPUT(scale); CHECK_VALID_INPUT(sigma_world);
    const int N = quaternion.size(0);
    TORCH_CHECK(quaternion.size(1) == 4, "quaternion must have shape Nx4");
    TORCH_CHECK(scale.size(0) == N, "scale must have shape Nx3");
    TORCH_CHECK(sigma_world.size(0) == N && sigma_world.size(1) == 3 && sigma_world.size(2) == 3,
                "sigma_world must have shape Nx3x3");
    const int dt = common_dtype(quaternion, {&scale, &sigma_world});
    c10::cuda::CUDAGuard guard(quaternion.device());
    check_rc(gsr_compute_sigma_world(dt, N, quaternion.data_ptr(), scale.data_ptr(), sigma_world.data_ptr(),
                                     cur_stream()),
             "compute_sigma_world_cuda");
}

void compute_sigma_world_backward_cuda(torch::Tensor quaternion, torch::Tensor scale,
                                       torch::Tensor sigma_world_grad_out, torch::Tensor quaternion_grad_in,
                                       torch::Tensor scale_grad_in) {
    CHECK_VALID_INPUT(quaternion); CHECK_VALID_INPUT(scale); CHECK_VALID_INPUT(sigma_world_grad_out);
    CHECK_VALID_INPUT(quaternion_grad_in); CHECK_VALID_INPUT(scale_grad_in);
    const int N = quaternion.size(0);
    TORCH_CHECK(quaternion.size(1) == 4, "quaternion must have shape Nx4");
    TORCH_CHECK(scale.size(0) == N && scale.size(1) == 3, "scale must have shape Nx3");
    TORCH_CHECK(sigma_world_grad_out.size(0) == N && sigma_world_grad_out.size(1) == 3 &&
                    sigma_world_grad_out.size(2) == 3,
                "sigma_world_grad_out must have shape Nx3x3");
    TORCH_CHECK(quaternion_grad_in.size(0) == N && quaternion_grad_in.size(1) == 4,
                "quaternion_grad_in must have shape Nx4");
    TORCH_CHECK(scale_grad_in.size(0) == N && scale_grad_in.size(1) == 3, "scale_grad_in must have shape Nx3");
    const int dt = common_dtype(quaternion, {&scale, &sigma_world_grad_out, &quaternion_grad_in, &scale_grad_in});
    c10::cuda::CUDAGuard guard(quaternion.device());
    check_rc(gsr_compute_sigma_world_backward(dt, N, quaternion.data_ptr(), scale.data_ptr(),
                                              sigma_world_grad_out.data_ptr(), quaternion_grad_in.data_ptr(),
                                              scale_grad_in.data_ptr(), cur_stream()),
             "compute_sigma_world_backward_cuda");
}

void compute_projection_jacobian_cuda(torch::Tensor xyz, torch::Tensor K, torch::Tensor J) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(K); CHECK_VALID_INPUT(J);
    const int N = xyz.size(0);
    TORCH_CHECK(xyz.size(1) == 3, "xyz must have shape Nx3");
    TORCH_CHECK(K.size(0) == 3 && K.size(1) == 3, "K must have shape 3x3");
    TORCH_CHECK(J.size(0) == N && J.size(1) == 2 && J.size(2) == 3, "J must have shape Nx2x3");
    const int dt = common_dtype(xyz, {&K, &J});
    c10::cuda::CUDAGuard guard(xyz.device());
    check_rc(gsr_compute_projection_jacobian(dt, N, xyz.data_ptr(), K.data_ptr(), J.data_ptr(), cur_stream()),
             "compute_projection_jacobian_cuda");
}

void compute_projection_jacobian_backward_cuda(torch::Tensor xyz, torch::Tensor K, torch::Tensor jac_grad_out,
                                               torch::Tensor xyz_grad_in) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(K); CHECK_VALID_INPUT(jac_grad_out); CHECK_VALID_INPUT(xyz_grad_in);
    const int N = xyz.size(0);
    TORCH_CHECK(xyz.size(1) == 3, "xyz must have shape Nx3");
    TORCH_CHECK(K.size(0) == 3 && K.size(1) == 3, "K must have shape 3x3");
    TORCH_CHECK(jac_grad_out.size(0) == N && jac_grad_out.size(1) == 2 && jac_grad_out.size(2) == 3,
                "jac_grad_out must have shape Nx2x3");
    TORCH_CHECK(xyz_grad_in.size(0) == N && xyz_grad_in.size(1) == 3, "xyz_grad_in must have shape Nx3");
    const int dt = common_dtype(xyz, {&K, &jac_grad_out, &xyz_grad_in});
    c10::cuda::CUDAGuard guard(xyz.device());
    check_rc(gsr_compute_projection_jacobian_backward(dt, N, xyz.data_ptr(), K.data_ptr(),
                                                      jac_grad_out.data_ptr(), xyz_grad_in.data_ptr(),
                                                      cur_stream()),
             "compute_projection_jacobian_backward_cuda");
}

void compute_conic_cuda(torch::Tensor sigma_world, torch::Tensor J, torch::Tensor camera_T_world,
                        torch::Tensor conic) {
    CHECK_VALID_INPUT(sigma_world); CHECK_VALID_INPUT(J); CHECK_VALID_INPUT(camera_T_world); CHECK_VALID_INPUT(conic);
    const int N = sigma_world.size(0);
    TORCH_CHECK(sigma_world.size(1) == 3 && sigma_world.size(2) == 3, "sigma_world must have shape Nx3x3");
    TORCH_CHECK(J.size(0) == N && J.size(1) == 2 && J.size(2) == 3, "J must have shape Nx2x3");
    TORCH_CHECK(camera_T_world.size(0) == 4 && camera_T_world.size(1) == 4, "camera_T_world must have shape 4x4");
    TORCH_CHECK(conic.size(0) == N && conic.size(1) == 3, "conic must have shape Nx3");
    const int dt = common_dtype(sigma_world, {&J, &camera_T_world, &conic});
    c10::cuda::CUDAGuard guard(sigma_world.device());
    check_rc(gsr_compute_conic(dt, N, sigma_world.data_ptr(), J.data_ptr(), camera_T_world.data_ptr(),
                               conic.data_ptr(), cur_stream()),
             "compute_conic_cuda");
}

void compute_conic_backward_cuda(torch::Tensor sigma_world, torch::Tensor J, torch::Tensor camera_T_world,
                                 torch::Tensor conic_grad_out, torch::Tensor sigma_world_grad_in,
                                 torch::Tensor J_grad_in) {
    CHECK_VALID_INPUT(sigma_world); CHECK_VALID_INPUT(J); CHECK_VALID_INPUT(camera_T_world);
    CHECK_VALID_INPUT(conic_grad_out); CHECK_VALID_INPUT(sigma_world_grad_in); CHECK_VALID_INPUT(J_grad_in);
    const int N = sigma_world.size(0);
    TORCH_CHECK(sigma_world.size(1) == 3 && sigma_world.size(2) == 3, "sigma_world must have shape Nx3x3");
    TORCH_CHECK(J.size(0) == N && J.size(1) == 2 && J.size(2) == 3, "J must have shape Nx2x3");
    TORCH_CHECK(camera_T_world.size(0) == 4 && camera_T_world.size(1) == 4, "camera_T_world must have shape 4x4");
    TORCH_CHECK(conic_grad_out.size(0) == N && conic_grad_out.size(1) == 3, "conic_grad_out must have shape Nx3");
    TORCH_CHECK(sigma_world_grad_in.size(0) == N && sigma_world_grad_in.size(1) == 3 &&
                    sigma_world_grad_in.size(2) == 3,
                "sigma_world_grad_in must have shape Nx3x3");
    TORCH_CHECK(J_grad_in.size(0) == N && J_grad_in.size(1) == 2 && J_grad_in.size(2) == 3,
                "J_grad_in must have shape Nx2x3");
    const int dt =
        common_dtype(sigma_world, {&J, &camera_T_world, &conic_grad_out, &sigma_world_grad_in, &J_grad_in});
    c10::cuda::CUDAGuard guard(sigma_world.device());
    check_rc(gsr_compute_conic_backward(dt, N, sigma_world.data_ptr(), J.data_ptr(), camera_T_world.data_ptr(),
                                        conic_grad_out.data_ptr(), sigma_world_grad_in.data_ptr(),
                                        J_grad_in.data_ptr(), cur_stream()),
             "compute_conic_backward_cuda");
}

void precompute_rgb_from_sh_cuda(const torch::Tensor xyz, const torch::Tensor sh_coeff,
                                 const torch::Tensor camera_T_world, torch::Tensor rgb) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(sh_coeff); CHECK_VALID_INPUT(camera_T_world); CHECK_VALID_INPUT(rgb);
    const int N = xyz.size(0);
    TORCH_CHECK(xyz.size(1) == 3, "Input xyz should have 3 channels");
    TORCH_CHECK(sh_coeff.size(0) == N, "N xyz and sh_coeff should match");
    TORCH_CHECK(sh_coeff.size(1) == 3, "SH coefficients should have 3 channels");
    const int n_sh = sh_coeff.dim() == 3 ? (int)sh_coeff.size(2) : 1;
    TORCH_CHECK(camera_T_world.size(0) == 4 && camera_T_world.size(1) == 4,
                "camera_T_world should be 4x4 transformation matrix");
    TORCH_CHECK(rgb.size(0) == N && rgb.size(1) == 3, "Output rgb should be Nx3");
    TORCH_CHECK(n_sh == 1 || n_sh == 4 || n_sh == 9 || n_sh == 16, "Invalid number of SH coefficients");
    const int dt = common_dtype(xyz, {&sh_coeff, &camera_T_world, &rgb});
    c10::cuda::CUDAGuard guard(xyz.device());
    check_rc(gsr_precompute_rgb_from_sh(dt, N, n_sh, xyz.data_ptr(), sh_coeff.data_ptr(),
                                        camera_T_world.data_ptr(), rgb.data_ptr(), cur_stream()),
             "precompute_rgb_from_sh_cuda");
}

void precompute_rgb_from_sh_backward_cuda(const torch::Tensor xyz, const torch::Tensor camera_T_world,
                                          const torch::Tensor grad_rgb, torch::Tensor grad_sh) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(camera_T_world); CHECK_VALID_INPUT(grad_rgb); CHECK_VALID_INPUT(grad_sh);
    const int N = xyz.size(0);
    TORCH_CHECK(xyz.size(1) == 3, "Input xyz should have 3 channels");
    TORCH_CHECK(camera_T_world.size(0) == 4 && camera_T_world.size(1) == 4,
                "camera_T_world should be 4x4 transformation matrix");
    TORCH_CHECK(grad_rgb.size(0) == N && grad_rgb.size(1) == 3, "grad_rgb should be Nx3");
    TORCH_CHECK(grad_sh.size(0) == N && grad_sh.size(1) == 3, "grad_sh should be Nx3(xK)");
    const int n_sh = grad_sh.dim() == 3 ? (int)grad_sh.size(2) : 1;
    TORCH_CHECK(n_sh == 1 || n_sh == 4 || n_sh == 9 || n_sh == 16, "Invalid number of SH coefficients");
    const int dt = common_dtype(xyz, {&camera_T_world, &grad_rgb, &grad_sh});
    c10::cuda::CUDAGuard guard(xyz.device());
    check_rc(gsr_precompute_rgb_from_sh_backward(dt, N, n_sh, xyz.data_ptr(), camera_T_world.data_ptr(),
                                                 grad_rgb.data_ptr(), grad_sh.data_ptr(), cur_stream()),
             "precompute_rgb_from_sh_backward_cuda");
}

// ---------------------------------------------------------------------------------------------
// tile binning
// ---------------------------------------------------------------------------------------------
std::tuple<torch::Tensor, torch::Tensor> get_sorted_gaussian_list(const int max_tiles_per_gaussian,
                                                                  torch::Tensor uvs,
                                                                  torch::Tensor xyz_camera_frame,
                                                                  torch::Tensor conic, const int n_tiles_x,
                                                                  const int n_tiles_y, const float mh_dist) {
    (void)max_tiles_per_gaussian;  // ignored by the reference as well (SURVEY.md Q11)
    CHECK_VALID_INPUT(uvs); CHECK_VALID_INPUT(xyz_camera_frame); CHECK_VALID_INPUT(conic);
    CHECK_FLOAT_TENSOR(uvs); CHECK_FLOAT_TENSOR(xyz_camera_frame); CHECK_FLOAT_TENSOR(conic);
    const int N = uvs.size(0);
    TORCH_CHECK(xyz_camera_frame.size(0) == N && conic.size(0) == N, "uvs, xyz_camera_frame, conic must have N rows");
    c10::cuda::CUDAGuard guard(uvs.device());
    auto i32 = torch::dtype(torch::kInt32).device(uvs.device());
    auto u8 = torch::dtype(torch::kUInt8).device(uvs.device());
    torch::Tensor offsets = torch::empty({N + 1}, i32);
    const size_t tb = gsr_binning_count_temp_bytes(N);
    torch::Tensor temp = torch::empty({(int64_t)tb}, u8);
    check_rc(gsr_binning_count(N, uvs.data_ptr<float>(), conic.data_ptr<float>(), n_tiles_x, n_tiles_y, mh_dist,
                               offsets.data_ptr<int>(), temp.data_ptr(), tb, cur_stream()),
             "gsr_binning_count");
    const int P = offsets[N].item<int>();  // the one host sync of this operator (reference: three)
    torch::Tensor sorted = torch::empty({P}, i32);
    torch::Tensor ranges = torch::empty({n_tiles_x * n_tiles_y + 1}, i32);
    const size_t sb = gsr_binning_sort_temp_bytes(P);
    torch::Tensor temp2 = torch::empty({(int64_t)sb}, u8);
    check_rc(gsr_binning_emit_sort(N, P, uvs.data_ptr<float>(), xyz_camera_frame.data_ptr<float>(),
                                   conic.data_ptr<float>(), n_tiles_x, n_tiles_y, mh_dist,
                                   offsets.data_ptr<int>(), sorted.data_ptr<int>(), ranges.data_ptr<int>(),
                                   temp2.data_ptr(), sb, cur_stream()),
             "gsr_binning_emit_sort");
    return std::make_tuple(sorted, ranges);
}

// ---------------------------------------------------------------------------------------------
// tile renderers
// ---------------------------------------------------------------------------------------------
struct RenderShapes {
    int N, H, W, n_sh;
};

RenderShapes check_render_inputs(const torch::Tensor& uvs, const torch::Tensor& opacity, const torch::Tensor& rgb,
                                 const torch::Tensor& conic, const torch::Tensor& view_dir_by_pixel,
                                 const torch::Tensor& ranges, const torch::Tensor& idx,
                                 const torch::Tensor& background_rgb, const torch::Tensor& image_like) {
    RenderShapes s;
    s.N = uvs.size(0);
    TORCH_CHECK(uvs.size(1) == 2, "uvs must be Nx2 (u, v)");
    TORCH_CHECK(opacity.size(0) == s.N, "Opacity must have the same number of elements as uvs");
    TORCH_CHECK(opacity.size(1) == 1, "Opacity must be Nx1");
    TORCH_CHECK(rgb.size(0) == s.N, "RGB must have the same number of elements as uvs");
    TORCH_CHECK(rgb.size(1) == 3, "RGB must be Nx3");
    TORCH_CHECK(conic.size(0) == s.N, "Conic must have the same number of elements as uvs");
    TORCH_CHECK(conic.size(1) == 3, "Conic must be Nx3");
    TORCH_CHECK(image_like.size(2) == 3, "Image must be HxWx3");
    TORCH_CHECK(background_rgb.dim() == 1, "Background RGB must be 1D");
    TORCH_CHECK(background_rgb.size(0) == 3, "Background RGB must have 3 elements");
    s.H = image_like.size(0);
    s.W = image_like.size(1);
    s.n_sh = rgb.dim() == 3 ? (int)rgb.size(2) : 1;
    TORCH_CHECK(s.n_sh == 1 || s.n_sh == 4 || s.n_sh == 9 || s.n_sh == 16, "Invalid number of SH coefficients");
    if (s.n_sh > 1) {
        TORCH_CHECK(view_dir_by_pixel.size(0) == s.H && view_dir_by_pixel.size(1) == s.W,
                    "view_dir_by_pixel must have the same size as the image");
        TORCH_CHECK(view_dir_by_pixel.size(2) == 3, "view_dir_by_pixel must have 3 channels");
    }
    CHECK_INT_TENSOR(ranges);
    CHECK_INT_TENSOR(idx);
    const int n_tiles = ((s.W + 15) / 16) * ((s.H + 15) / 16);
    TORCH_CHECK(ranges.numel() == n_tiles + 1, "splat_start_end_idx_by_tile_idx must have n_tiles + 1 entries");
    return s;
}

void render_tiles_cuda(torch::Tensor uvs, torch::Tensor opacity, torch::Tensor rgb, torch::Tensor conic,
                       torch::Tensor view_dir_by_pixel, torch::Tensor splat_start_end_idx_by_tile_idx,
                       torch::Tensor gaussian_idx_by_splat_idx, torch::Tensor background_rgb,
                       torch::Tensor num_splats_per_pixel, torch::Tensor final_weight_per_pixel,
                       torch::Tensor rendered_image) {
    CHECK_VALID_INPUT(uvs); CHECK_VALID_INPUT(opacity); CHECK_VALID_INPUT(rgb); CHECK_VALID_INPUT(conic);
    CHECK_VALID_INPUT(view_dir_by_pixel); CHECK_VALID_INPUT(splat_start_end_idx_by_tile_idx);
    CHECK_VALID_INPUT(gaussian_idx_by_splat_idx); CHECK_VALID_INPUT(background_rgb);
    CHECK_VALID_INPUT(num_splats_per_pixel); CHECK_VALID_INPUT(final_weight_per_pixel);
    CHECK_VALID_INPUT(rendered_image);
    const RenderShapes s = check_render_inputs(uvs, opacity, rgb, conic, view_dir_by_pixel,
                                               splat_start_end_idx_by_tile_idx, gaussian_idx_by_splat_idx,
                                               background_rgb, rendered_image);
    CHECK_INT_TENSOR(num_splats_per_pixel);
    const int dt = common_dtype(uvs, {&opacity, &rgb, &conic, &view_dir_by_pixel, &background_rgb,
                                      &final_weight_per_pixel, &rendered_image});
    c10::cuda::CUDAGuard guard(uvs.device());
    const int P = gaussian_idx_by_splat_idx.numel();
    if (dt == GSR_F32 && s.n_sh == 1) {
        torch::Tensor records = torch::empty({std::max(P, 1), GSR_REC_FLOATS}, uvs.options());
        check_rc(gsr_pack_records(P, gaussian_idx_by_splat_idx.data_ptr<int>(), uvs.data_ptr<float>(),
                                  opacity.data_ptr<float>(), rgb.data_ptr<float>(), conic.data_ptr<float>(),
                                  records.data_ptr<float>(), cur_stream()),
                 "gsr_pack_records");
        check_rc(gsr_render_forward(records.data_ptr<float>(), splat_start_end_idx_by_tile_idx.data_ptr<int>(),
                                    background_rgb.data_ptr<float>(), s.H, s.W,
                                    num_splats_per_pixel.data_ptr<int>(), final_weight_per_pixel.data_ptr<float>(),
                                    rendered_image.data_ptr<float>(), nullptr, cur_stream()),
                 "gsr_render_forward");
    } else {
        check_rc(gsr_render_forward_generic(
                     dt, s.N, s.n_sh, uvs.data_ptr(), opacity.data_ptr(), rgb.data_ptr(), conic.data_ptr(),
                     view_dir_by_pixel.data_ptr(), splat_start_end_idx_by_tile_idx.data_ptr<int>(),
                     gaussian_idx_by_splat_idx.data_ptr<int>(), background_rgb.data_ptr(), s.H, s.W,
                     num_splats_per_pixel.data_ptr<int>(), final_weight_per_pixel.data_ptr(),
                     rendered_image.data_ptr(), cur_stream()),
                 "gsr_render_forward_generic");
    }
}

void render_tiles_backward_cuda(torch::Tensor uvs, torch::Tensor opacity, torch::Tensor rgb, torch::Tensor conic,
                                torch::Tensor view_dir_by_pixel, torch::Tensor splat_start_end_idx_by_tile_idx,
                                torch::Tensor gaussian_idx_by_splat_idx, torch::Tensor background_rgb,
                                torch::Tensor num_splats_per_pixel, torch::Tensor final_weight_per_pixel,
                                torch::Tensor grad_image, torch::Tensor grad_rgb, torch::Tensor grad_opacity,
                                torch::Tensor grad_uvs, torch::Tensor grad_conic) {
    CHECK_VALID_INPUT(uvs); CHECK_VALID_INPUT(opacity); CHECK_VALID_INPUT(rgb); CHECK_VALID_INPUT(conic);
    CHECK_VALID_INPUT(view_dir_by_pixel); CHECK_VALID_INPUT(splat_start_end_idx_by_tile_idx);
    CHECK_VALID_INPUT(gaussian_idx_by_splat_idx); CHECK_VALID_INPUT(background_rgb);
    CHECK_VALID_INPUT(num_splats_per_pixel); CHECK_VALID_INPUT(final_weight_per_pixel);
    CHECK_VALID_INPUT(grad_image); CHECK_VALID_INPUT(grad_rgb); CHECK_VALID_INPUT(grad_opacity);
    CHECK_VALID_INPUT(grad_uvs); CHECK_VALID_INPUT(grad_conic);
    const RenderShapes s = check_render_inputs(uvs, opacity, rgb, conic, view_dir_by_pixel,
                                               splat_start_end_idx_by_tile_idx, gaussian_idx_by_splat_idx,
                                               background_rgb, grad_image);
    CHECK_INT_TENSOR(num_splats_per_pixel);
    TORCH_CHECK(grad_rgb.sizes() == rgb.sizes(), "grad_rgb must have the shape of rgb");
    TORCH_CHECK(grad_opacity.size(0) == s.N, "grad_opacity must be Nx1");
    TORCH_CHECK(grad_uvs.size(0) == s.N && grad_uvs.size(1) == 2, "grad_uvs must be Nx2");
    TORCH_CHECK(grad_conic.size(0) == s.N && grad_conic.size(1) == 3, "grad_conic must be Nx3");
    const int dt = common_dtype(uvs, {&opacity, &rgb, &conic, &view_dir_by_pixel, &background_rgb,
                                      &final_weight_per_pixel, &grad_image, &grad_rgb, &grad_opacity, &grad_uvs,
                                      &grad_conic});
    c10::cuda::CUDAGuard guard(uvs.device());
    const int P = gaussian_idx_by_splat_idx.numel();
    if (dt == GSR_F32 && s.n_sh == 1) {
        torch::Tensor records = torch::empty({std::max(P, 1), GSR_REC_FLOATS}, uvs.options());
        check_rc(gsr_pack_records(P, gaussian_idx_by_splat_idx.data_ptr<int>(), uvs.data_ptr<float>(),
                                  opacity.data_ptr<float>(), rgb.data_ptr<float>(), conic.data_ptr<float>(),
                                  records.data_ptr<float>(), cur_stream()),
                 "gsr_pack_records");
        check_rc(gsr_render_backward(records.data_ptr<float>(), gaussian_idx_by_splat_idx.data_ptr<int>(),
                                     splat_start_end_idx_by_tile_idx.data_ptr<int>(),
                                     background_rgb.data_ptr<float>(), s.H, s.W,
                                     num_splats_per_pixel.data_ptr<int>(), final_weight_per_pixel.data_ptr<float>(),
                                     grad_image.data_ptr<float>(), grad_rgb.data_ptr<float>(),
                                     grad_opacity.data_ptr<float>(), grad_uvs.data_ptr<float>(),
                                     grad_conic.data_ptr<float>(), nullptr, cur_stream()),
                 "gsr_render_backward");
    } else {
        check_rc(gsr_render_backward_generic(
                     dt, s.N, s.n_sh, uvs.data_ptr(), opacity.data_ptr(), rgb.data_ptr(), conic.data_ptr(),
                     view_dir_by_pixel.data_ptr(), splat_start_end_idx_by_tile_idx.data_ptr<int>(),
                     gaussian_idx_by_splat_idx.data_ptr<int>(), background_rgb.data_ptr(), s.H, s.W,
                     num_splats_per_pixel.data_ptr<int>(), final_weight_per_pixel.data_ptr(),
                     grad_image.data_ptr(), grad_rgb.data_ptr(), grad_opacity.data_ptr(), grad_uvs.data_ptr(),
                     grad_conic.data_ptr(), cur_stream()),
                 "gsr_render_backward_generic");
    }
}

void render_depth_cuda(torch::Tensor xyz_camera_frame, torch::Tensor uvs, torch::Tensor opacity,
                       torch::Tensor conic, torch::Tensor splat_start_end_idx_by_tile_idx,
                       torch::Tensor gaussian_idx_by_splat_idx, const float alpha_threshold,
                       torch::Tensor depth_image) {
    CHECK_VALID_INPUT(xyz_camera_frame); CHECK_VALID_INPUT(uvs); CHECK_VALID_INPUT(opacity); CHECK_VALID_INPUT(conic);
    CHECK_VALID_INPUT(splat_start_end_idx_by_tile_idx); CHECK_VALID_INPUT(gaussian_idx_by_splat_idx);
    CHECK_VALID_INPUT(depth_image);
    CHECK_FLOAT_TENSOR(xyz_camera_frame); CHECK_FLOAT_TENSOR(uvs); CHECK_FLOAT_TENSOR(opacity);
    CHECK_FLOAT_TENSOR(conic); CHECK_FLOAT_TENSOR(depth_image);
    CHECK_INT_TENSOR(splat_start_end_idx_by_tile_idx); CHECK_INT_TENSOR(gaussian_idx_by_splat_idx);
    const int N = uvs.size(0);
    TORCH_CHECK(uvs.size(1) == 2, "uvs must be Nx2 (u, v)");
    TORCH_CHECK(xyz_camera_frame.size(0) == N && xyz_camera_frame.size(1) == 3, "xyz_camera_frame must be Nx3");
    TORCH_CHECK(opacity.size(0) == N, "Opacity must have the same number of elements as uvs");
    TORCH_CHECK(conic.size(0) == N && conic.size(1) == 3, "Conic must be Nx3");
    const int H = depth_image.size(0), W = depth_image.size(1);
    c10::cuda::CUDAGuard guard(uvs.device());
    check_rc(gsr_render_depth(N, xyz_camera_frame.data_ptr<float>(), uvs.data_ptr<float>(),
                              opacity.data_ptr<float>(), conic.data_ptr<float>(),
                              splat_start_end_idx_by_tile_idx.data_ptr<int>(),
                              gaussian_idx_by_splat_idx.data_ptr<int>(), alpha_threshold, H, W,
                              depth_image.data_ptr<float>(), cur_stream()),
             "render_depth_cuda");
}

// ---------------------------------------------------------------------------------------------
// fused path (used by gaussian_splatting_b200.rasterize): thin pointer plumbing, no arithmetic
// ---------------------------------------------------------------------------------------------
#define F32PTR(t) ((t).data_ptr<float>())

// returns (records[N,12], depth_key[N] i32-viewed u32, visible[N] u8, scan[N] i64-viewed u64)
// returns (records, depth_key, visible, scan, tile_mask, tile_win); the last two are empty unless with_tiles
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
fused_preprocess_forward_impl(
    torch::Tensor xyz, c10::optional<torch::Tensor> xyz_camera_frame, torch::Tensor quaternion, torch::Tensor scale,
    torch::Tensor opacity_logit, torch::Tensor rgb_dc, c10::optional<torch::Tensor> sh_rest,
    torch::Tensor camera_T_world, torch::Tensor K, c10::optional<torch::Tensor> camera_centre, int64_t H, int64_t W,
    double near_thresh, double far_thresh, double cull_mask_padding, double mh_dist, int64_t depth_base,
    bool with_tiles) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(quaternion); CHECK_VALID_INPUT(scale); CHECK_VALID_INPUT(opacity_logit);
    CHECK_VALID_INPUT(rgb_dc); CHECK_VALID_INPUT(camera_T_world); CHECK_VALID_INPUT(K);
    CHECK_FLOAT_TENSOR(xyz); CHECK_FLOAT_TENSOR(quaternion); CHECK_FLOAT_TENSOR(scale);
    CHECK_FLOAT_TENSOR(opacity_logit); CHECK_FLOAT_TENSOR(rgb_dc); CHECK_FLOAT_TENSOR(camera_T_world);
    CHECK_FLOAT_TENSOR(K);
    const int N = xyz.size(0);
    TORCH_CHECK(xyz.dim() == 2 && xyz.size(1) == 3, "xyz must have shape Nx3");
    TORCH_CHECK(quaternion.size(0) == N && quaternion.size(1) == 4, "quaternion must have shape Nx4");
    TORCH_CHECK(scale.size(0) == N && scale.size(1) == 3, "scale must have shape Nx3");
    TORCH_CHECK(opacity_logit.numel() == N, "opacity must have shape Nx1");
    TORCH_CHECK(rgb_dc.size(0) == N && rgb_dc.size(1) == 3, "rgb must have shape Nx3");
    TORCH_CHECK(camera_T_world.numel() == 16 && K.numel() == 9, "camera_T_world must be 4x4 and K 3x3");
    const float* cam_ptr = nullptr;
    int cam_first = 0;
    if (xyz_camera_frame.has_value()) {  // positions of the LAST xyz_camera_frame.size(0) gaussians
        const torch::Tensor& pc = *xyz_camera_frame;
        CHECK_VALID_INPUT(pc); CHECK_FLOAT_TENSOR(pc);
        TORCH_CHECK(pc.dim() == 2 && pc.size(0) <= N && pc.size(1) == 3, "xyz_camera_frame must have shape Rx3, R <= N");
        cam_ptr = pc.data_ptr<float>();
        cam_first = N - (int)pc.size(0);
    }
    const float* centre_ptr = nullptr;
    if (camera_centre.has_value()) {
        CHECK_VALID_INPUT((*camera_centre)); CHECK_FLOAT_TENSOR((*camera_centre));
        TORCH_CHECK(camera_centre->numel() == 3, "camera_centre must have 3 elements");
        centre_ptr = camera_centre->data_ptr<float>();
    }
    int n_rest = 0;
    const float* sh_ptr = nullptr;
    if (sh_rest.has_value()) {
        const torch::Tensor& sh = *sh_rest;
        CHECK_VALID_INPUT(sh); CHECK_FLOAT_TENSOR(sh);
        TORCH_CHECK(sh.dim() == 3 && sh.size(0) == N && sh.size(1) == 3, "sh must have shape Nx3xK");
        n_rest = sh.size(2);
        TORCH_CHECK(n_rest == 3 || n_rest == 8 || n_rest == 15, "sh must hold 3, 8 or 15 coefficients per channel");
        sh_ptr = sh.data_ptr<float>();
    }
    c10::cuda::CUDAGuard guard(xyz.device());
    auto opt = xyz.options();
    torch::Tensor records = torch::empty({N, GSR_REC_FLOATS}, opt);
    torch::Tensor zkey = torch::empty({N}, opt.dtype(torch::kInt32));
    torch::Tensor visible = torch::empty({N}, opt.dtype(torch::kUInt8));
    torch::Tensor scan = torch::empty({N}, opt.dtype(torch::kInt64));
    torch::Tensor tile_mask = torch::empty({with_tiles ? N : 0}, opt.dtype(torch::kInt64));
    torch::Tensor tile_win = torch::empty({with_tiles ? N : 0}, opt.dtype(torch::kInt32));
    const size_t tb = gsr_preprocess_temp_bytes(N);
    torch::Tensor temp = torch::empty({(int64_t)tb}, opt.dtype(torch::kUInt8));
    check_rc(gsr_preprocess_forward(N, n_rest, F32PTR(xyz), cam_ptr, cam_first, F32PTR(quaternion), F32PTR(scale),
                                    F32PTR(opacity_logit), F32PTR(rgb_dc), sh_ptr, F32PTR(camera_T_world),
                                    F32PTR(K), centre_ptr, (int)H, (int)W, (float)near_thresh, (float)far_thresh,
                                    (float)cull_mask_padding, (float)mh_dist, (uint32_t)depth_base, F32PTR(records),
                                    (uint32_t*)zkey.data_ptr<int>(), visible.data_ptr<uint8_t>(),
                                    (uint64_t*)scan.data_ptr<int64_t>(),
                                    with_tiles && N > 0 ? (uint64_t*)tile_mask.data_ptr<int64_t>() : nullptr,
                                    with_tiles && N > 0 ? (uint32_t*)tile_win.data_ptr<int>() : nullptr, temp.data_ptr(), tb,
                                    cur_stream()),
             "gsr_preprocess_forward");
    return std::make_tuple(records, zkey, visible, scan, tile_mask, tile_win);
}

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> fused_preprocess_forward(
    torch::Tensor xyz, c10::optional<torch::Tensor> xyz_camera_frame, torch::Tensor quaternion, torch::Tensor scale,
    torch::Tensor opacity_logit, torch::Tensor rgb_dc, c10::optional<torch::Tensor> sh_rest,
    torch::Tensor camera_T_world, torch::Tensor K, c10::optional<torch::Tensor> camera_centre, int64_t H, int64_t W,
    double near_thresh, double far_thresh, double cull_mask_padding, double mh_dist, int64_t depth_base) {
    auto r = fused_preprocess_forward_impl(xyz, xyz_camera_frame, quaternion, scale, opacity_logit, rgb_dc, sh_rest,
                                           camera_T_world, K, camera_centre, H, W, near_thresh, far_thresh,
                                           cull_mask_padding, mh_dist, depth_base, false);
    return std::make_tuple(std::get<0>(r), std::get<1>(r), std::get<2>(r), std::get<3>(r));
}

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
fused_preprocess_forward_tiles(
    torch::Tensor xyz, c10::optional<torch::Tensor> xyz_camera_frame, torch::Tensor quaternion, torch::Tensor scale,
    torch::Tensor opacity_logit, torch::Tensor rgb_dc, c10::optional<torch::Tensor> sh_rest,
    torch::Tensor camera_T_world, torch::Tensor K, c10::optional<torch::Tensor> camera_centre, int64_t H, int64_t W,
    double near_thresh, double far_thresh, double cull_mask_padding, double mh_dist, int64_t depth_base) {
    return fused_preprocess_forward_impl(xyz, xyz_camera_frame, quaternion, scale, opacity_logit, rgb_dc, sh_rest,
                                         camera_T_world, K, camera_centre, H, W, near_thresh, far_thresh,
                                         cull_mask_padding, mh_dist, depth_base, true);
}

// (M, P known) -> sorted gaussian ids [P] i32, tile ranges [n_tiles+1] i32, sorted record stream [P,12],
//                 vis_idx [M] i32, uv [M,2]
// speculative = true: M and P are CAPACITIES (the host has not read the real counts yet): buffers are sized by
// them, the pair buffer is padded behind the real pairs (gsr_emit_*'s `capacity`), and every tensor is returned at
// full capacity — the caller narrows them once it knows M and P, and redoes the call if P exceeded the capacity.
// no_stream = true: the tile kernels will fetch records through the sorted pair list themselves
// (gsr_render_*_gather): no record stream is produced; returns the sorted keys (and id_bits) instead.
// returns (ids_sorted, ranges, stream_rec, vis_idx, uv, keys_sorted, id_bits)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, int64_t> fused_bin(
    torch::Tensor records, torch::Tensor zkey, torch::Tensor visible, torch::Tensor scan, int64_t M, int64_t P,
    int64_t H, int64_t W, double mh_dist, int64_t depth_bits, bool speculative, bool no_stream,
    c10::optional<torch::Tensor> tile_mask, c10::optional<torch::Tensor> tile_win) {
    const bool tiles = tile_mask.has_value() && tile_win.has_value() && tile_mask->numel() == records.size(0) &&
                       tile_win->numel() == records.size(0) && records.size(0) > 0;
    const uint64_t* tmask = tiles ? (const uint64_t*)tile_mask->data_ptr<int64_t>() : nullptr;
    const uint32_t* twin = tiles ? (const uint32_t*)tile_win->data_ptr<int>() : nullptr;
    const int N = records.size(0);
    const int ntx = (W + 15) / 16, nty = (H + 15) / 16, n_tiles = ntx * nty;
    c10::cuda::CUDAGuard guard(records.device());
    auto opt = records.options();
    auto i32 = opt.dtype(torch::kInt32);
    const int64_t Pa = std::max<int64_t>(P, 1);
    torch::Tensor keys = torch::empty({2 * Pa}, opt.dtype(torch::kInt64));
    const int id_bits_probe = gsr_packed_id_bits(N, n_tiles, (int)depth_bits);
    // with the id in the key and no stream, nobody needs the separate id array
    torch::Tensor ids_sorted = torch::empty({(no_stream && id_bits_probe > 0) ? 0 : Pa}, i32);
    torch::Tensor vis_idx = torch::empty({M}, i32);
    torch::Tensor uv = torch::empty({M, 2}, opt);
    torch::Tensor ranges = torch::empty({n_tiles + 1}, i32);
    torch::Tensor stream_rec = torch::empty({no_stream ? 0 : Pa, GSR_REC_FLOATS}, opt);
    uint64_t* keys_a = (uint64_t*)keys.data_ptr<int64_t>();
    uint64_t* keys_b = keys_a + Pa;
    const int id_bits = gsr_packed_id_bits(N, n_tiles, (int)depth_bits);
    if (id_bits > 0) {  // (tile | depth | id) keys, keys-only radix sort
        check_rc(gsr_emit_keys(N, F32PTR(records), (const uint32_t*)zkey.data_ptr<int>(), visible.data_ptr<uint8_t>(),
                               (const uint64_t*)scan.data_ptr<int64_t>(), ntx, nty, (float)mh_dist, (int)depth_bits,
                               id_bits, keys_a, vis_idx.data_ptr<int>(), F32PTR(uv), speculative ? P : 0, tmask, twin,
                               cur_stream()),
                 "gsr_emit_keys");
        const size_t sb = gsr_sort_keys_temp_bytes((int)P);
        torch::Tensor temp = torch::empty({(int64_t)sb}, opt.dtype(torch::kUInt8));
        check_rc(gsr_sort_keys((int)P, n_tiles, (int)depth_bits, id_bits, keys_a, keys_b, temp.data_ptr(), sb,
                               cur_stream()),
                 "gsr_sort_keys");
        check_rc(gsr_tile_ranges((int)P, n_tiles, (int)depth_bits + id_bits, keys_b, ranges.data_ptr<int>(),
                                 cur_stream()),
                 "gsr_tile_ranges");
        if (!no_stream)
            check_rc(gsr_gather_records_keys((int)P, id_bits, keys_b, F32PTR(records), F32PTR(stream_rec),
                                             ids_sorted.data_ptr<int>(), nullptr, cur_stream()),
                     "gsr_gather_records_keys");
    } else {
        torch::Tensor ids = torch::empty({Pa}, i32);
        check_rc(gsr_emit_pairs(N, F32PTR(records), (const uint32_t*)zkey.data_ptr<int>(),
                                visible.data_ptr<uint8_t>(), (const uint64_t*)scan.data_ptr<int64_t>(), ntx, nty,
                                (float)mh_dist, (int)depth_bits, keys_a, (uint32_t*)ids.data_ptr<int>(),
                                vis_idx.data_ptr<int>(), F32PTR(uv), speculative ? P : 0, tmask, twin, cur_stream()),
                 "gsr_emit_pairs");
        const size_t sb = gsr_sort_pairs_temp_bytes((int)P);
        torch::Tensor temp = torch::empty({(int64_t)sb}, opt.dtype(torch::kUInt8));
        check_rc(gsr_sort_pairs((int)P, n_tiles, (int)depth_bits, keys_a, (const uint32_t*)ids.data_ptr<int>(), keys_b,
                                (uint32_t*)ids_sorted.data_ptr<int>(), temp.data_ptr(), sb, cur_stream()),
                 "gsr_sort_pairs");
        check_rc(gsr_tile_ranges((int)P, n_tiles, (int)depth_bits, keys_b, ranges.data_ptr<int>(), cur_stream()),
                 "gsr_tile_ranges");
        if (!no_stream)
            check_rc(gsr_gather_records((int)P, (const uint32_t*)ids_sorted.data_ptr<int>(), F32PTR(records),
                                        F32PTR(stream_rec), nullptr, nullptr, cur_stream()),
                     "gsr_gather_records");
    }
    torch::Tensor keys_sorted = (no_stream && id_bits > 0) ? keys.narrow(0, Pa, Pa) : torch::empty({0}, opt.dtype(torch::kInt64));
    return std::make_tuple(ids_sorted.numel() > 0 ? ids_sorted.narrow(0, 0, P) : ids_sorted, ranges, stream_rec, vis_idx,
                           uv, keys_sorted, (int64_t)id_bits);
}

// image [H,W,3], n [H,W] i32, wlast [H,W], contribution masks (i32 words; empty when record_masks is false)
// records: the record stream [P,12] — or, when keys_sorted / ids_sorted name the sorted pair list (gather mode), the
// per-gaussian record array [N,12]
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor> fused_render_forward(
    torch::Tensor stream_rec, torch::Tensor ranges, torch::Tensor background, int64_t H, int64_t W, int64_t P,
    bool record_masks, c10::optional<torch::Tensor> keys_sorted, c10::optional<torch::Tensor> ids_sorted,
    int64_t id_bits, bool gather) {
    CHECK_VALID_INPUT(background); CHECK_FLOAT_TENSOR(background);
    TORCH_CHECK(background.numel() == 3, "Background RGB must have 3 elements");
    c10::cuda::CUDAGuard guard(stream_rec.device());
    auto opt = stream_rec.options();
    torch::Tensor image = torch::empty({H, W, 3}, opt);
    torch::Tensor n = torch::empty({H, W}, opt.dtype(torch::kInt32));
    torch::Tensor w = torch::empty({H, W}, opt);
    torch::Tensor masks = record_masks
                              ? torch::zeros({(int64_t)gsr_contribution_mask_words(P, (int)H, (int)W)}, opt.dtype(torch::kInt32))
                              : torch::empty({0}, opt.dtype(torch::kInt32));
    uint32_t* mptr = record_masks ? (uint32_t*)masks.data_ptr<int>() : nullptr;
    if (gather) {
        const bool by_key = keys_sorted.has_value() && keys_sorted->numel() > 0;
        TORCH_CHECK(by_key || (ids_sorted.has_value() && ids_sorted->numel() > 0) || P == 0, "gather mode needs the sorted pair list");
        check_rc(gsr_render_forward_gather(F32PTR(stream_rec),
                                           by_key ? (const uint64_t*)keys_sorted->data_ptr<int64_t>() : nullptr, (int)id_bits,
                                           (!by_key && ids_sorted.has_value() && ids_sorted->numel() > 0) ? ids_sorted->data_ptr<int>() : nullptr,
                                           ranges.data_ptr<int>(), F32PTR(background), (int)H, (int)W, n.data_ptr<int>(),
                                           F32PTR(w), F32PTR(image), mptr, cur_stream()),
                 "gsr_render_forward_gather");
    } else {
        check_rc(gsr_render_forward(F32PTR(stream_rec), ranges.data_ptr<int>(), F32PTR(background), (int)H, (int)W,
                                    n.data_ptr<int>(), F32PTR(w), F32PTR(image), mptr, cur_stream()),
                 "gsr_render_forward");
    }
    return std::make_tuple(image, n, w, masks);
}

// per-gaussian gradient slab, flat [9N]: rgb [N,3] | opacity [N] | uv [N,2] | conic [N,3], rows indexed by
// gaussian; zero-filled, then accumulated into by the render backward
torch::Tensor fused_render_backward(torch::Tensor grad_image, int64_t N, torch::Tensor stream_rec,
                                    torch::Tensor ids_sorted, torch::Tensor ranges, torch::Tensor background,
                                    torch::Tensor n, torch::Tensor w, torch::Tensor masks,
                                    c10::optional<torch::Tensor> keys_sorted, int64_t id_bits, bool gather) {
    CHECK_VALID_INPUT(grad_image); CHECK_FLOAT_TENSOR(grad_image);
    const int H = n.size(0), W = n.size(1);
    TORCH_CHECK(grad_image.dim() == 3 && grad_image.size(0) == H && grad_image.size(1) == W &&
                    grad_image.size(2) == 3,
                "grad_image must be HxWx3");
    c10::cuda::CUDAGuard guard(grad_image.device());
    // gather mode: interleaved rows [N,12] (vector reductions); stream mode: planar [9N]
    torch::Tensor slab = torch::zeros({N * (gather ? (int64_t)GSR_GRAD_ROW_FLOATS : 9)}, grad_image.options());
    float* g_rgb = slab.data_ptr<float>();
    float* g_opa = g_rgb + (size_t)N * 3;
    float* g_uv = g_opa + (size_t)N;
    float* g_conic = g_uv + (size_t)N * 2;
    const uint32_t* mptr = masks.numel() > 0 ? (const uint32_t*)masks.data_ptr<int>() : nullptr;
    if (gather) {
        const bool by_key = keys_sorted.has_value() && keys_sorted->numel() > 0;
        check_rc(gsr_render_backward_gather(F32PTR(stream_rec),
                                            by_key ? (const uint64_t*)keys_sorted->data_ptr<int64_t>() : nullptr, (int)id_bits,
                                            (!by_key && ids_sorted.numel() > 0) ? ids_sorted.data_ptr<int>() : nullptr,
                                            ranges.data_ptr<int>(), F32PTR(background), H, W, n.data_ptr<int>(), F32PTR(w),
                                            F32PTR(grad_image), nullptr, nullptr, nullptr, nullptr, g_rgb, mptr,
                                            cur_stream()),
                 "gsr_render_backward_gather");
    } else {
        check_rc(gsr_render_backward(F32PTR(stream_rec), ids_sorted.data_ptr<int>(), ranges.data_ptr<int>(),
                                     F32PTR(background), H, W, n.data_ptr<int>(), F32PTR(w), F32PTR(grad_image),
                                     g_rgb, g_opa, g_uv, g_conic, mptr, cur_stream()),
                 "gsr_render_backward");
    }
    return slab;
}

// grads of (xyz, quaternion, scale, opacity_logit, rgb_dc[, sh_rest]) from the slab [9N] (rows by gaussian).
// grad_uv_compact [M,2] (optional): gradient on the compact uv, added to — or, with use_slab_uv false, replacing —
// the slab's uv section.
std::vector<torch::Tensor> fused_preprocess_backward(torch::Tensor slab, torch::Tensor xyz,
                                                     torch::Tensor quaternion, torch::Tensor scale,
                                                     torch::Tensor opacity_logit,
                                                     c10::optional<torch::Tensor> sh_rest,
                                                     torch::Tensor camera_T_world, torch::Tensor K,
                                                     c10::optional<torch::Tensor> camera_centre,
                                                     torch::Tensor visible,
                                                     c10::optional<torch::Tensor> out_flat,
                                                     c10::optional<torch::Tensor> grad_uv_compact,
                                                     c10::optional<torch::Tensor> scan, bool use_slab_uv) {
    CHECK_VALID_INPUT(slab); CHECK_FLOAT_TENSOR(slab);
    const int64_t N = xyz.size(0);
    const bool rows = slab.numel() == N * (int64_t)GSR_GRAD_ROW_FLOATS && N > 0;  // interleaved [N,12] (else planar [9N])
    TORCH_CHECK(rows || slab.numel() == N * 9, "gradient slab must hold 9 (planar) or 12 (rows) floats per gaussian");
    c10::cuda::CUDAGuard guard(xyz.device());
    auto opt = xyz.options();
    const float* g_rgb = slab.data_ptr<float>();
    const float* g_opa = g_rgb + (size_t)N * 3;
    const float* g_uv = use_slab_uv ? g_opa + (size_t)N : nullptr;
    const float* g_conic = g_opa + (size_t)N * 3;
    const int n_rest = sh_rest.has_value() ? (int)sh_rest->size(2) : 0;
    const float* g_uv_compact = nullptr;
    const uint64_t* scan_ptr = nullptr;
    if (grad_uv_compact.has_value() && grad_uv_compact->numel() > 0) {
        CHECK_VALID_INPUT((*grad_uv_compact)); CHECK_FLOAT_TENSOR((*grad_uv_compact));
        TORCH_CHECK(scan.has_value() && scan->numel() == N && scan->scalar_type() == torch::kInt64,
                    "grad_uv_compact needs the packed scan of the forward pass");
        TORCH_CHECK(grad_uv_compact->dim() == 2 && grad_uv_compact->size(1) == 2, "grad_uv_compact must be Mx2");
        g_uv_compact = grad_uv_compact->data_ptr<float>();
        scan_ptr = (const uint64_t*)scan->data_ptr<int64_t>();
    }
    // All parameter gradients of a view live in ONE allocation, [xyz 3N | quaternion 4N | scale 3N |
    // opacity N | rgb 3N | sh 3*n_rest*N], every section starting on a 16-byte boundary (TMA bulk stores):
    // a trainer that sums gradients over views / ranks reduces that one buffer (view_parallel.py).
    const int64_t widths[6] = {3, 4, 3, 1, 3, 3 * (int64_t)n_rest};
    int64_t offs[7];
    offs[0] = 0;
    for (int i = 0; i < 6; ++i) offs[i + 1] = (offs[i] + N * widths[i] + 3) & ~(int64_t)3;
    // out_flat: a caller-owned buffer of the same layout (e.g. symmetric memory peers can read, view_parallel.py)
    torch::Tensor flat;
    if (out_flat.has_value()) {
        flat = *out_flat;
        CHECK_VALID_INPUT(flat); CHECK_FLOAT_TENSOR(flat);
        TORCH_CHECK(flat.numel() == offs[6], "out_flat must hold ", offs[6], " floats");
        TORCH_CHECK((reinterpret_cast<uintptr_t>(flat.data_ptr()) & 15u) == 0, "out_flat must be 16-byte aligned");
    } else {
        flat = torch::empty({offs[6]}, opt);
    }
    for (int i = 0; i < 6; ++i)  // padding between sections (only when N is not a multiple of 4)
        if (offs[i + 1] > offs[i] + N * widths[i]) flat.narrow(0, offs[i] + N * widths[i], offs[i + 1] - offs[i] - N * widths[i]).zero_();
    auto section = [&](int i, std::vector<int64_t> shape) {
        return flat.narrow(0, offs[i], N * widths[i]).view(shape);
    };
    torch::Tensor o_xyz = section(0, {N, 3}), o_q = section(1, {N, 4}), o_s = section(2, {N, 3}),
                  o_o = section(3, {N}), o_dc = section(4, {N, 3});
    torch::Tensor g_sh;
    if (n_rest) g_sh = section(5, {N, 3, (int64_t)n_rest});
    check_rc(gsr_preprocess_backward((int)N, n_rest, F32PTR(xyz), F32PTR(quaternion), F32PTR(scale),
                                     F32PTR(opacity_logit), F32PTR(camera_T_world), F32PTR(K),
                                     camera_centre.has_value() ? camera_centre->data_ptr<float>() : nullptr,
                                     visible.data_ptr<uint8_t>(), g_rgb, g_opa, g_uv, g_conic,
                                     rows ? slab.data_ptr<float>() : nullptr, use_slab_uv ? 1 : 0, g_uv_compact,
                                     scan_ptr, F32PTR(o_xyz),
                                     F32PTR(o_q), F32PTR(o_s), F32PTR(o_o), F32PTR(o_dc),
                                     n_rest ? F32PTR(g_sh) : nullptr, cur_stream()),
             "gsr_preprocess_backward");
    std::vector<torch::Tensor> out = {o_xyz, o_q, o_s, o_o, o_dc};
    if (n_rest) out.push_back(g_sh);
    out.push_back(flat);  // last: the allocation all the others are views of
    return out;
}

// sizes of the flat parameter / gradient layout: exclusive end of each section, in elements
std::vector<int64_t> flat_section_ends(int64_t N, int64_t n_sh_rest) {
    const int64_t widths[6] = {3, 4, 3, 1, 3, 3 * n_sh_rest};
    std::vector<int64_t> ends;
    int64_t off = 0;
    for (int i = 0; i < 6; ++i) {
        off = (off + N * widths[i] + 3) & ~(int64_t)3;
        if (widths[i] > 0) ends.push_back(off);
    }
    return ends;
}

void adam_step_flat(torch::Tensor p, torch::Tensor g, torch::Tensor m, torch::Tensor v,
                    std::vector<int64_t> section_end, std::vector<double> section_lr, double beta1, double beta2,
                    double eps, int64_t step) {
    CHECK_VALID_INPUT(p); CHECK_VALID_INPUT(g); CHECK_VALID_INPUT(m); CHECK_VALID_INPUT(v);
    CHECK_FLOAT_TENSOR(p); CHECK_FLOAT_TENSOR(g); CHECK_FLOAT_TENSOR(m); CHECK_FLOAT_TENSOR(v);
    const int64_t n = p.numel();
    TORCH_CHECK(g.numel() == n && m.numel() == n && v.numel() == n, "p, g, m, v must have the same length");
    TORCH_CHECK(section_end.size() == section_lr.size() && !section_end.empty() && section_end.back() == n,
                "sections must cover the buffer");
    c10::cuda::CUDAGuard guard(p.device());
    check_rc(gsr_adam_step(n, F32PTR(p), F32PTR(g), F32PTR(m), F32PTR(v), (int)section_end.size(),
                           section_end.data(), section_lr.data(), beta1, beta2, eps, (int)step, cur_stream()),
             "gsr_adam_step");
}

void adam_step_sharded(int64_t lo, int64_t hi, std::vector<int64_t> peer_grad_ptrs,
                       std::vector<int64_t> peer_param_ptrs, int64_t self_rank, torch::Tensor m_shard,
                       torch::Tensor v_shard, std::vector<int64_t> section_end, std::vector<double> section_lr,
                       double beta1, double beta2, double eps, int64_t step) {
    CHECK_VALID_INPUT(m_shard); CHECK_VALID_INPUT(v_shard); CHECK_FLOAT_TENSOR(m_shard); CHECK_FLOAT_TENSOR(v_shard);
    TORCH_CHECK(peer_grad_ptrs.size() == peer_param_ptrs.size() && !peer_grad_ptrs.empty(), "one pointer per rank");
    TORCH_CHECK(m_shard.numel() == hi - lo && v_shard.numel() == hi - lo, "state shards must hold hi - lo elements");
    TORCH_CHECK(section_end.size() == section_lr.size() && !section_end.empty(), "bad sections");
    std::vector<const float*> gp;
    std::vector<float*> pp;
    for (size_t q = 0; q < peer_grad_ptrs.size(); ++q) {
        gp.push_back(reinterpret_cast<const float*>(peer_grad_ptrs[q]));
        pp.push_back(reinterpret_cast<float*>(peer_param_ptrs[q]));
    }
    c10::cuda::CUDAGuard guard(m_shard.device());
    check_rc(gsr_adam_step_sharded(lo, hi, (int)gp.size(), gp.data(), pp.data(), (int)self_rank, F32PTR(m_shard),
                                   F32PTR(v_shard), (int)section_end.size(), section_end.data(), section_lr.data(),
                                   beta1, beta2, eps, (int)step, cur_stream()),
             "gsr_adam_step_sharded");
}

void densify_accumulate(torch::Tensor vis_idx, torch::Tensor uv_grad, torch::Tensor xyz_grad, torch::Tensor K,
                        torch::Tensor uv_grad_accum, torch::Tensor xyz_grad_accum, torch::Tensor grad_accum_count) {
    CHECK_VALID_INPUT(vis_idx); CHECK_VALID_INPUT(uv_grad); CHECK_VALID_INPUT(xyz_grad); CHECK_VALID_INPUT(K);
    CHECK_VALID_INPUT(uv_grad_accum); CHECK_VALID_INPUT(xyz_grad_accum); CHECK_VALID_INPUT(grad_accum_count);
    CHECK_FLOAT_TENSOR(uv_grad); CHECK_FLOAT_TENSOR(xyz_grad); CHECK_FLOAT_TENSOR(K);
    CHECK_FLOAT_TENSOR(uv_grad_accum); CHECK_FLOAT_TENSOR(xyz_grad_accum);
    TORCH_CHECK(vis_idx.scalar_type() == torch::kInt32 && grad_accum_count.scalar_type() == torch::kInt32,
                "vis_idx and grad_accum_count must be int32");
    const int64_t N = xyz_grad.size(0), M = vis_idx.numel();
    TORCH_CHECK(uv_grad.numel() == 2 * M && uv_grad_accum.numel() == 2 * N && xyz_grad_accum.numel() == 3 * N &&
                    grad_accum_count.numel() == N && K.numel() == 9,
                "shape mismatch");
    c10::cuda::CUDAGuard guard(xyz_grad.device());
    check_rc(gsr_densify_accumulate((int)N, (int)M, vis_idx.data_ptr<int>(), F32PTR(uv_grad), F32PTR(xyz_grad), F32PTR(K),
                                    F32PTR(uv_grad_accum), F32PTR(xyz_grad_accum), grad_accum_count.data_ptr<int>(),
                                    cur_stream()),
             "gsr_densify_accumulate");
}

// the plan of one adaptive-density-control pass applied to the flat parameter buffer and both Adam moments;
// returns (p_out, m_out, v_out) freshly allocated (m_out / v_out undefined tensors when no moments were given)
std::vector<torch::Tensor> densify_apply(torch::Tensor p_in, c10::optional<torch::Tensor> m_in,
                                         c10::optional<torch::Tensor> v_in, int64_t n_in, int64_t n_sh_rest,
                                         torch::Tensor src, c10::optional<torch::Tensor> clone_row,
                                         c10::optional<torch::Tensor> split_row, c10::optional<torch::Tensor> xyz_sub,
                                         c10::optional<torch::Tensor> xyz_add, c10::optional<torch::Tensor> q_set,
                                         c10::optional<torch::Tensor> scale_set,
                                         c10::optional<torch::Tensor> p_out_buf) {
    CHECK_VALID_INPUT(p_in); CHECK_FLOAT_TENSOR(p_in); CHECK_VALID_INPUT(src);
    TORCH_CHECK(src.scalar_type() == torch::kInt32, "src must be int32");
    TORCH_CHECK(p_in.numel() == gsr_flat_numel(n_in, (int)n_sh_rest), "p_in does not match the flat layout of n_in gaussians");
    const int64_t n_out = src.numel();
    const int64_t total = gsr_flat_numel(n_out, (int)n_sh_rest);
    const bool moments = m_in.has_value();
    TORCH_CHECK(moments == v_in.has_value(), "m_in and v_in go together");
    auto i32ptr = [&](const c10::optional<torch::Tensor>& t, const char* name) -> const int32_t* {
        if (!t.has_value()) return nullptr;
        CHECK_VALID_INPUT((*t));
        TORCH_CHECK(t->scalar_type() == torch::kInt32 && t->numel() == n_out, name, " must be int32 [n_out]");
        return t->data_ptr<int32_t>();
    };
    auto f32ptr = [&](const c10::optional<torch::Tensor>& t) -> const float* {
        if (!t.has_value() || t->numel() == 0) return nullptr;
        CHECK_VALID_INPUT((*t)); CHECK_FLOAT_TENSOR((*t));
        return t->data_ptr<float>();
    };
    const int32_t* cr = i32ptr(clone_row, "clone_row");
    const int32_t* sr = i32ptr(split_row, "split_row");
    // an index array without its value table means "no such rows": the kernel then must not see the index array
    const float* sub = f32ptr(xyz_sub);
    const float* add = f32ptr(xyz_add);
    const float* qs = f32ptr(q_set);
    const float* ss = f32ptr(scale_set);
    if (sub == nullptr) cr = nullptr;
    if (add == nullptr || qs == nullptr || ss == nullptr) sr = nullptr;
    c10::cuda::CUDAGuard guard(p_in.device());
    torch::Tensor p_out;
    if (p_out_buf.has_value()) {  // caller-owned destination (e.g. symmetric memory)
        p_out = *p_out_buf;
        CHECK_VALID_INPUT(p_out); CHECK_FLOAT_TENSOR(p_out);
        TORCH_CHECK(p_out.numel() == total && p_out.data_ptr() != p_in.data_ptr(), "bad p_out buffer");
    } else {
        p_out = torch::empty({total}, p_in.options());
    }
    torch::Tensor m_out, v_out;
    if (moments) {
        CHECK_VALID_INPUT((*m_in)); CHECK_VALID_INPUT((*v_in)); CHECK_FLOAT_TENSOR((*m_in)); CHECK_FLOAT_TENSOR((*v_in));
        TORCH_CHECK(m_in->numel() == p_in.numel() && v_in->numel() == p_in.numel(), "moments must match p_in");
        m_out = torch::empty({total}, p_in.options());
        v_out = torch::empty({total}, p_in.options());
    }
    check_rc(gsr_densify_apply((int)n_in, (int)n_out, (int)n_sh_rest, F32PTR(p_in), moments ? F32PTR((*m_in)) : nullptr,
                               moments ? F32PTR((*v_in)) : nullptr, src.data_ptr<int32_t>(), cr, sr, sub, add, qs, ss,
                               F32PTR(p_out), moments ? F32PTR(m_out) : nullptr, moments ? F32PTR(v_out) : nullptr,
                               cur_stream()),
             "gsr_densify_apply");
    if (moments) return {p_out, m_out, v_out};
    return {p_out};
}

// inverse(camera_T_world)[:3, 3] with torch's bits (gsr_camera_centre)
torch::Tensor camera_centre(torch::Tensor camera_T_world) {
    CHECK_VALID_INPUT(camera_T_world); CHECK_FLOAT_TENSOR(camera_T_world);
    TORCH_CHECK(camera_T_world.numel() == 16, "camera_T_world must be 4x4");
    c10::cuda::CUDAGuard guard(camera_T_world.device());
    torch::Tensor out = torch::empty({3}, camera_T_world.options());
    check_rc(gsr_camera_centre(F32PTR(camera_T_world), F32PTR(out), cur_stream()), "gsr_camera_centre");
    return out;
}

// ---------------------------------------------------------------------------------------------
// photometric loss (gsr_photometric_loss_*): [H,W,C] (the renderer's image, B = 1) or [B,C,H,W], any strides
// ---------------------------------------------------------------------------------------------
struct LossShape {
    int B, C, H, W;
    std::vector<int64_t> strides;  // (B, C, H, W) element strides
};

LossShape loss_shape(const torch::Tensor& t, const char* name) {
    TORCH_CHECK(t.is_cuda(), name, " is not a CUDA tensor");
    TORCH_CHECK(t.dim() == 3 || t.dim() == 4, name, " must be [H,W,C] or [B,C,H,W]");
    LossShape s;
    if (t.dim() == 3) {
        s.B = 1;
        s.H = t.size(0);
        s.W = t.size(1);
        s.C = t.size(2);
        s.strides = {t.size(0) * t.stride(0), t.stride(2), t.stride(0), t.stride(1)};
    } else {
        s.B = t.size(0);
        s.C = t.size(1);
        s.H = t.size(2);
        s.W = t.size(3);
        s.strides = {t.stride(0), t.stride(1), t.stride(2), t.stride(3)};
    }
    return s;
}

LossShape check_loss_inputs(const torch::Tensor& pred, const torch::Tensor& target, const std::vector<double>& window,
                            int* dt) {
    LossShape s = loss_shape(pred, "pred");
    LossShape ts = loss_shape(target, "target");
    TORCH_CHECK(pred.sizes() == target.sizes(), "pred and target must have the same shape");
    TORCH_CHECK(pred.device() == target.device(), "pred and target must be on the same device");
    TORCH_CHECK(window.size() == 11, "window must have 11 taps");
    TORCH_CHECK(s.H >= 11 && s.W >= 11, "H and W must be at least 11");
    *dt = common_dtype(pred, {&target});
    return s;
}

// returns out [3] = (loss, L1, SSIM) in pred's dtype
torch::Tensor photometric_loss_forward(torch::Tensor pred, torch::Tensor target, std::vector<double> window,
                                       double c1, double c2, double l1_weight, double ssim_weight) {
    int dt = 0;
    const LossShape s = check_loss_inputs(pred, target, window, &dt);
    const LossShape ts = loss_shape(target, "target");
    c10::cuda::CUDAGuard guard(pred.device());
    torch::Tensor out = torch::empty({3}, pred.options());
    const size_t tb = gsr_photometric_loss_temp_bytes(s.B, s.C, s.H, s.W);
    torch::Tensor temp = torch::empty({(int64_t)tb}, pred.options().dtype(torch::kUInt8));
    check_rc(gsr_photometric_loss_forward(dt, s.B, s.C, s.H, s.W, pred.data_ptr(), s.strides.data(),
                                          target.data_ptr(), ts.strides.data(), window.data(), c1, c2, l1_weight,
                                          ssim_weight, out.data_ptr(), temp.data_ptr(), tb, cur_stream()),
             "gsr_photometric_loss_forward");
    return out;
}

// returns grad_loss * d loss / d pred, allocated with empty_like(pred) (a permuted view keeps its strides)
torch::Tensor photometric_loss_backward(torch::Tensor pred, torch::Tensor target, std::vector<double> window,
                                        double c1, double c2, double l1_weight, double ssim_weight,
                                        torch::Tensor grad_loss) {
    int dt = 0;
    const LossShape s = check_loss_inputs(pred, target, window, &dt);
    const LossShape ts = loss_shape(target, "target");
    TORCH_CHECK(grad_loss.is_cuda() && grad_loss.device() == pred.device(), "grad_loss must be on pred's device");
    TORCH_CHECK(grad_loss.numel() == 1 && grad_loss.dtype() == pred.dtype(), "grad_loss must be a scalar of pred's dtype");
    c10::cuda::CUDAGuard guard(pred.device());
    torch::Tensor grad = torch::empty_like(pred);
    const LossShape gs = loss_shape(grad, "grad");
    check_rc(gsr_photometric_loss_backward(dt, s.B, s.C, s.H, s.W, pred.data_ptr(), s.strides.data(),
                                           target.data_ptr(), ts.strides.data(), window.data(), c1, c2, l1_weight,
                                           ssim_weight, grad_loss.data_ptr(), grad.data_ptr(), gs.strides.data(),
                                           cur_stream()),
             "gsr_photometric_loss_backward");
    return grad;
}

std::string version() { return gsr_version(); }

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    // the reference surface (src/bindings.cpp:118-159)
    m.def("render_tiles_cuda", &render_tiles_cuda, "Render tiles CUDA");
    m.def("render_tiles_backward_cuda", &render_tiles_backward_cuda, "Render tiles backward");
    m.def("camera_projection_cuda", &camera_projection_cuda, "project point into image CUDA");
    m.def("camera_projection_backward_cuda", &camera_projection_backward_cuda,
          "project point into image backward CUDA");
    m.def("compute_sigma_world_cuda", &compute_sigma_world_cuda, "compute sigma world CUDA");
    m.def("compute_sigma_world_backward_cuda", &compute_sigma_world_backward_cuda,
          "compute sigma world backward CUDA");
    m.def("compute_projection_jacobian_cuda", &compute_projection_jacobian_cuda,
          "compute projection jacobian CUDA");
    m.def("compute_projection_jacobian_backward_cuda", &compute_projection_jacobian_backward_cuda,
          "compute projection jacobian backward CUDA");
    m.def("compute_conic_cuda", &compute_conic_cuda, "compute conic CUDA");
    m.def("compute_conic_backward_cuda", &compute_conic_backward_cuda, "compute conic backward CUDA");
    m.def("get_sorted_gaussian_list", &get_sorted_gaussian_list, "get sorted gaussian list");
    m.def("precompute_rgb_from_sh_cuda", &precompute_rgb_from_sh_cuda, "precompute rgb from sh per gaussian");
    m.def("precompute_rgb_from_sh_backward_cuda", &precompute_rgb_from_sh_backward_cuda,
          "precompute rgb from sh per gaussian backward");
    m.def("render_depth_cuda", &render_depth_cuda, "Render depth CUDA");
    // fused path
    m.def("fused_preprocess_forward", &fused_preprocess_forward, "fused per-gaussian stage");
    m.def("fused_preprocess_forward_tiles", &fused_preprocess_forward_tiles,
          "fused per-gaussian stage, also returning every gaussian's tile-hit mask and window");
    m.def("fused_bin", &fused_bin, "pair emission + radix sort + tile ranges + record stream");
    m.def("fused_render_forward", &fused_render_forward, "tile renderer forward on a record stream");
    m.def("fused_render_backward", &fused_render_backward, "tile renderer backward -> per-gaussian gradient slab");
    m.def("fused_preprocess_backward", &fused_preprocess_backward, "fused per-gaussian backward");
    m.def("flat_section_ends", &flat_section_ends, "section ends of the flat parameter/gradient layout");
    m.def("adam_step_flat", &adam_step_flat, "Adam on the flat parameter buffer");
    m.def("adam_step_sharded", &adam_step_sharded, "reduce-scatter + Adam + all-gather over peer memory");
    m.def("densify_accumulate", &densify_accumulate, "per-step densification statistics");
    m.def("densify_apply", &densify_apply, "clone / split / delete applied to the flat parameter + Adam buffers");
    m.def("camera_centre", &camera_centre, "inverse(camera_T_world)[:3, 3] with torch's bits, one kernel");
    m.def("photometric_loss_forward", &photometric_loss_forward,
          "(1 - ssim_frac) * L1 + ssim_frac * (1 - SSIM) forward -> (loss, L1, SSIM)");
    m.def("photometric_loss_backward", &photometric_loss_backward, "photometric loss backward -> gradient on pred");
    m.def("version", &version, "library version string");
}
