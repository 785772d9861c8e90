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
#include "../../include/gsr_selective_adam.h"
#include "../../include/gsr_features.h"
#include "../../include/gsr_batch.h"
#include "../../include/gsr_fisheye.h"
#include "../../include/gsr_distortion.h"
#include "../../include/gsr_pose.h"
#include "../../include/gsr_calib.h"
#include "../../include/gsr_bilagrid.h"
#include "../../include/gsr_shutter.h"
#include "../../include/gsr_surfels.h"
#include "../../include/gsr_surfels_lens.h"
#include "../../include/gsr_surfels_features.h"
#include "../../include/gsr_surfels_median.h"

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

// The sorted pair list the tile renderers read record ids through: the keys when the id rides in them, else the
// sorted id array.  An empty view (P == 0) may have neither (the key/value fallback narrows its id array to nothing);
// the kernels still run, to write the background, and read no pair: any well-formed source will do.
struct PairSource {
    const uint64_t* keys;
    const int32_t* ids;
};
PairSource pair_source(const c10::optional<torch::Tensor>& keys_sorted, const c10::optional<torch::Tensor>& ids_sorted,
                       int64_t P) {
    static const int32_t no_pair = 0;
    if (keys_sorted.has_value() && keys_sorted->numel() > 0)
        return {(const uint64_t*)keys_sorted->data_ptr<int64_t>(), nullptr};
    if (ids_sorted.has_value() && ids_sorted->numel() > 0) return {nullptr, ids_sorted->data_ptr<int>()};
    TORCH_CHECK(P == 0, "the tile renderers need the sorted pair list");
    return {nullptr, &no_pair};
}

// fp32 per-gaussian arrays of the reference surface -> the renderers' per-gaussian records [N,12]
torch::Tensor pack_records(const torch::Tensor& uvs, const torch::Tensor& opacity, const torch::Tensor& rgb,
                           const torch::Tensor& conic, int N) {
    torch::Tensor records = torch::empty({std::max(N, 1), GSR_REC_FLOATS}, uvs.options());
    check_rc(gsr_pack_gaussian_records(N, uvs.data_ptr<float>(), opacity.data_ptr<float>(), rgb.data_ptr<float>(),
                                       conic.data_ptr<float>(), records.data_ptr<float>(), cur_stream()),
             "gsr_pack_gaussian_records");
    return records;
}

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
    if (dt == GSR_F32 && s.n_sh == 1) {
        const torch::Tensor records = pack_records(uvs, opacity, rgb, conic, s.N);
        const PairSource ps = pair_source(c10::nullopt, gaussian_idx_by_splat_idx, gaussian_idx_by_splat_idx.numel());
        check_rc(gsr_render_forward_gather(records.data_ptr<float>(), nullptr, 0, ps.ids, nullptr, 0, 0,
                                           splat_start_end_idx_by_tile_idx.data_ptr<int>(),
                                           background_rgb.data_ptr<float>(), s.H, s.W,
                                           num_splats_per_pixel.data_ptr<int>(),
                                           final_weight_per_pixel.data_ptr<float>(), rendered_image.data_ptr<float>(),
                                           nullptr, nullptr, nullptr, cur_stream()),
                 "gsr_render_forward_gather");
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
    if (dt == GSR_F32 && s.n_sh == 1) {
        const torch::Tensor records = pack_records(uvs, opacity, rgb, conic, s.N);
        const PairSource ps = pair_source(c10::nullopt, gaussian_idx_by_splat_idx, gaussian_idx_by_splat_idx.numel());
        // the caller's planar gradient arrays, accumulated into as the reference does
        check_rc(gsr_render_backward_gather(0, records.data_ptr<float>(), nullptr, 0, ps.ids, nullptr, 0, 0,
                                            splat_start_end_idx_by_tile_idx.data_ptr<int>(),
                                            background_rgb.data_ptr<float>(), s.H, s.W,
                                            num_splats_per_pixel.data_ptr<int>(),
                                            final_weight_per_pixel.data_ptr<float>(), grad_image.data_ptr<float>(),
                                            nullptr, nullptr, grad_rgb.data_ptr<float>(),
                                            grad_opacity.data_ptr<float>(), grad_uvs.data_ptr<float>(),
                                            grad_conic.data_ptr<float>(), nullptr, nullptr, cur_stream()),
                 "gsr_render_backward_gather");
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

// the 3-D filter [N] or [N,1] of the fused per-gaussian stages (GSR_MODE_FILTER3D), or NULL
static const float* filter3d_ptr(const c10::optional<torch::Tensor>& filter3d, int64_t N) {
    if (!filter3d.has_value()) return nullptr;
    const torch::Tensor& f = *filter3d;
    CHECK_VALID_INPUT(f); CHECK_FLOAT_TENSOR(f);
    TORCH_CHECK(f.numel() == N && (f.dim() == 1 || (f.dim() == 2 && f.size(1) == 1)), "filter3d must have shape [N] or [N,1]");
    return f.data_ptr<float>();
}

// The camera model of the per-gaussian stages, a GSR_LENS_* value (gsr_pose.h): the pinhole (libgsr_b200.so,
// libgsr_batch.so) or a lens whose per-view constants the lens library's entry points read: OPENCV_FISHEYE
// (libgsr_fisheye.so, {k1, k2, k3, k4, theta_max}) or OPENCV radial-tangential distortion (libgsr_distortion.so,
// {k1, k2, p1, p2, k3, r2_max}).  Returns the lens's constants per view (0 for the pinhole); the coefficients that
// get a gradient are all of them but the last, the cull limit.
static int64_t lens_consts_per_view(int64_t lens) {
    TORCH_CHECK(lens == GSR_LENS_PINHOLE || lens == GSR_LENS_FISHEYE || lens == GSR_LENS_DISTORTION,
                "lens must be 0 (pinhole), 1 (fisheye) or 2 (distortion)");
    return lens == GSR_LENS_FISHEYE ? GSR_FISHEYE_CONSTS : lens == GSR_LENS_DISTORTION ? GSR_DISTORTION_CONSTS : 0;
}

// the lens constants of C views (fp32 on xyz's device), or NULL for the pinhole
static const float* lens_ptr(int64_t lens, const c10::optional<torch::Tensor>& consts, int64_t C,
                             const torch::Tensor& xyz) {
    const int64_t per_view = lens_consts_per_view(lens);
    if (per_view == 0) {
        TORCH_CHECK(!consts.has_value(), "the pinhole takes no lens constants");
        return nullptr;
    }
    TORCH_CHECK(consts.has_value(), "a lens needs its constants");
    const torch::Tensor& f = *consts;
    const char* name = lens == GSR_LENS_FISHEYE ? "fisheye" : "distortion";
    CHECK_VALID_INPUT(f); CHECK_FLOAT_TENSOR(f);
    TORCH_CHECK(f.numel() == C * per_view, name, " constants must hold ", per_view, " floats per view");
    TORCH_CHECK(f.device() == xyz.device(), name, " constants must be on the gaussians' device");
    return f.data_ptr<float>();
}

// the number of views: 1 for a single view (camera_T_world [4,4], K [3,3]), else C (camera_T_world [C,4,4], K [C,3,3])
static int64_t check_views(bool batched, const torch::Tensor& camera_T_world, const torch::Tensor& K) {
    CHECK_VALID_INPUT(camera_T_world); CHECK_VALID_INPUT(K);
    CHECK_FLOAT_TENSOR(camera_T_world); CHECK_FLOAT_TENSOR(K);
    if (!batched) {
        TORCH_CHECK(camera_T_world.numel() == 16 && K.numel() == 9, "camera_T_world must be 4x4 and K 3x3");
        return 1;
    }
    const int64_t C = camera_T_world.size(0);
    TORCH_CHECK(camera_T_world.dim() == 3 && C >= 1 && camera_T_world.size(1) == 4 && camera_T_world.size(2) == 4,
                "camera_T_world must have shape Cx4x4, C >= 1");
    TORCH_CHECK(K.dim() == 3 && K.size(0) == C && K.size(1) == 3 && K.size(2) == 3, "K must have shape Cx3x3");
    return C;
}

// Rolling-shutter twists xi of C views (gsr_shutter.h): fp32 [6] for one view, [C,6] for C views, on xyz's device; or
// NULL (a global shutter)
static const float* shutter_ptr(const c10::optional<torch::Tensor>& xi, int64_t C, bool batched,
                                const torch::Tensor& xyz) {
    if (!xi.has_value()) return nullptr;
    const torch::Tensor& t = *xi;
    CHECK_VALID_INPUT(t); CHECK_FLOAT_TENSOR(t);
    TORCH_CHECK(batched ? (t.dim() == 2 && t.size(0) == C && t.size(1) == 6) : (t.dim() == 1 && t.size(0) == 6),
                batched ? "rolling_shutter must have shape Cx6" : "rolling_shutter must have shape 6");
    TORCH_CHECK(t.device() == xyz.device(), "rolling_shutter must be on the gaussians' device");
    return t.data_ptr<float>();
}

// The per-gaussian forward (gsr_preprocess_forward, or the lens's: lens a GSR_LENS_* value, lc its constants [C, n+1]).
// One view (batched false): returns [records [N,12], depth_key [N] i32-viewed u32, visible [N] u8, scan [N]
// i64-viewed u64] and, with_tiles, also [tile_mask [N] i64-viewed u64, tile_win [N] i32-viewed u32].  C views
// (batched, camera_T_world [C,4,4], K [C,3,3]): the single-view forward of every view into the same outputs with a
// leading view dimension, each view's own packed inclusive scan; xyz_camera_frame [C,R,3] holds the camera-frame
// positions of the LAST R gaussians of every view, camera_centre [C,3].  mode: GSR_MODE_* bits.  shutter: the views'
// rolling-shutter twists ([6] / [C,6], gsr_shutter_preprocess_forward with `readout`), or none.
static std::vector<torch::Tensor> preprocess_forward(
    bool batched, torch::Tensor xyz, c10::optional<torch::Tensor> xyz_camera_frame, torch::Tensor quaternion,
    torch::Tensor scale, torch::Tensor opacity_logit, torch::Tensor rgb_dc, c10::optional<torch::Tensor> sh_rest,
    torch::Tensor camera_T_world, torch::Tensor K, c10::optional<torch::Tensor> camera_centre, int64_t H, int64_t W,
    double near_thresh, double far_thresh, double cull_mask_padding, double mh_dist, int64_t depth_base,
    bool with_tiles, int64_t mode, c10::optional<torch::Tensor> filter3d, int64_t lens,
    c10::optional<torch::Tensor> lc, c10::optional<torch::Tensor> shutter, int64_t readout) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(quaternion); CHECK_VALID_INPUT(scale); CHECK_VALID_INPUT(opacity_logit);
    CHECK_VALID_INPUT(rgb_dc);
    CHECK_FLOAT_TENSOR(xyz); CHECK_FLOAT_TENSOR(quaternion); CHECK_FLOAT_TENSOR(scale);
    CHECK_FLOAT_TENSOR(opacity_logit); CHECK_FLOAT_TENSOR(rgb_dc);
    const int64_t C = check_views(batched, camera_T_world, K);
    const int N = xyz.size(0);
    TORCH_CHECK(xyz.dim() == 2 && xyz.size(1) == 3, "xyz must have shape Nx3");
    TORCH_CHECK(quaternion.size(0) == N && quaternion.size(1) == 4, "quaternion must have shape Nx4");
    TORCH_CHECK(scale.size(0) == N && scale.size(1) == 3, "scale must have shape Nx3");
    TORCH_CHECK(opacity_logit.numel() == N, "opacity must have shape Nx1");
    TORCH_CHECK(rgb_dc.size(0) == N && rgb_dc.size(1) == 3, "rgb must have shape Nx3");
    const float* cam_ptr = nullptr;
    int64_t R = 0;
    if (xyz_camera_frame.has_value()) {  // positions of the LAST R gaussians
        const torch::Tensor& pc = *xyz_camera_frame;
        CHECK_VALID_INPUT(pc); CHECK_FLOAT_TENSOR(pc);
        TORCH_CHECK(pc.dim() == (batched ? 3 : 2) && (!batched || pc.size(0) == C) && pc.size(-2) <= N &&
                        pc.size(-1) == 3,
                    batched ? "xyz_camera_frame must have shape CxRx3, R <= N"
                            : "xyz_camera_frame must have shape Rx3, R <= N");
        cam_ptr = pc.data_ptr<float>();
        R = pc.size(-2);
    }
    const float* centre_ptr = nullptr;
    if (camera_centre.has_value()) {
        CHECK_VALID_INPUT((*camera_centre)); CHECK_FLOAT_TENSOR((*camera_centre));
        TORCH_CHECK(camera_centre->numel() == 3 * C,
                    batched ? "camera_centre must have shape Cx3" : "camera_centre must have 3 elements");
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
    const float* f3d = filter3d_ptr(filter3d, N);
    const float* lens_consts = lens_ptr(lens, lc, C, xyz);
    const float* xi = shutter_ptr(shutter, C, batched, xyz);
    const int64_t lens_per_view = lens_consts_per_view(lens);
    c10::cuda::CUDAGuard guard(xyz.device());
    auto opt = xyz.options();
    // one view's outputs have no view dimension
    auto shape = [&](std::initializer_list<int64_t> s) {
        std::vector<int64_t> v(s);
        if (batched) v.insert(v.begin(), C);
        return v;
    };
    torch::Tensor records = torch::empty(shape({N, GSR_REC_FLOATS}), opt);
    torch::Tensor zkey = torch::empty(shape({N}), opt.dtype(torch::kInt32));
    torch::Tensor visible = torch::empty(shape({N}), opt.dtype(torch::kUInt8));
    torch::Tensor scan = torch::empty(shape({N}), opt.dtype(torch::kInt64));
    torch::Tensor tile_mask = torch::empty(shape({with_tiles ? N : 0}), opt.dtype(torch::kInt64));
    torch::Tensor tile_win = torch::empty(shape({with_tiles ? N : 0}), opt.dtype(torch::kInt32));
    const size_t tb = gsr_preprocess_temp_bytes(N);
    torch::Tensor temp = torch::empty({(int64_t)tb}, opt.dtype(torch::kUInt8));
    const bool tiles = with_tiles && N > 0;
    // one view calls its entry point also for an empty scene (which only checks the arguments)
    for (int64_t c = 0; c < C && (N > 0 || !batched); ++c) {
#define GSR_FWD_ARGS                                                                                                  \
    (int)mode, N, n_rest, F32PTR(xyz), cam_ptr ? cam_ptr + c * R * 3 : nullptr, N - (int)R, F32PTR(quaternion),       \
        F32PTR(scale), F32PTR(opacity_logit), f3d, F32PTR(rgb_dc), sh_ptr, F32PTR(camera_T_world) + 16 * c,            \
        F32PTR(K) + 9 * c, centre_ptr ? centre_ptr + 3 * c : nullptr, (int)H, (int)W, (float)near_thresh,              \
        (float)far_thresh, (float)cull_mask_padding, (float)mh_dist, (uint32_t)depth_base,                             \
        F32PTR(records) + c * N * GSR_REC_FLOATS, (uint32_t*)zkey.data_ptr<int>() + c * N,                             \
        visible.data_ptr<uint8_t>() + c * N, (uint64_t*)scan.data_ptr<int64_t>() + c * N,                              \
        tiles ? (uint64_t*)tile_mask.data_ptr<int64_t>() + c * N : nullptr,                                            \
        tiles ? (uint32_t*)tile_win.data_ptr<int>() + c * N : nullptr, temp.data_ptr(), tb
        if (xi != nullptr)
            check_rc(gsr_shutter_preprocess_forward((int)lens, GSR_FWD_ARGS,
                                                    lens_consts ? lens_consts + lens_per_view * c : nullptr,
                                                    xi + 6 * c, (int)readout, cur_stream()),
                     "gsr_shutter_preprocess_forward");
        else if (lens == GSR_LENS_FISHEYE)
            check_rc(gsr_fisheye_preprocess_forward(GSR_FWD_ARGS, lens_consts + GSR_FISHEYE_CONSTS * c, cur_stream()),
                     "gsr_fisheye_preprocess_forward");
        else if (lens == GSR_LENS_DISTORTION)
            check_rc(gsr_distortion_preprocess_forward(GSR_FWD_ARGS, lens_consts + GSR_DISTORTION_CONSTS * c,
                                                       cur_stream()),
                     "gsr_distortion_preprocess_forward");
        else
            check_rc(gsr_preprocess_forward(GSR_FWD_ARGS, cur_stream()), "gsr_preprocess_forward");
#undef GSR_FWD_ARGS
    }
    if (!with_tiles) return {records, zkey, visible, scan};
    return {records, zkey, visible, scan, tile_mask, tile_win};
}

std::vector<torch::Tensor> fused_preprocess_forward(
    torch::Tensor xyz, c10::optional<torch::Tensor> xyz_camera_frame, torch::Tensor quaternion, torch::Tensor scale,
    torch::Tensor opacity_logit, torch::Tensor rgb_dc, c10::optional<torch::Tensor> sh_rest,
    torch::Tensor camera_T_world, torch::Tensor K, c10::optional<torch::Tensor> camera_centre, int64_t H, int64_t W,
    double near_thresh, double far_thresh, double cull_mask_padding, double mh_dist, int64_t depth_base,
    bool with_tiles, int64_t mode, c10::optional<torch::Tensor> filter3d, int64_t lens,
    c10::optional<torch::Tensor> lens_consts, c10::optional<torch::Tensor> rolling_shutter, int64_t readout) {
    return preprocess_forward(false, xyz, xyz_camera_frame, quaternion, scale, opacity_logit, rgb_dc, sh_rest,
                              camera_T_world, K, camera_centre, H, W, near_thresh, far_thresh, cull_mask_padding,
                              mh_dist, depth_base, with_tiles, mode, filter3d, lens, lens_consts, rolling_shutter,
                              readout);
}

std::vector<torch::Tensor> batch_preprocess_forward(
    torch::Tensor xyz, c10::optional<torch::Tensor> xyz_camera_frame, torch::Tensor quaternion, torch::Tensor scale,
    torch::Tensor opacity_logit, torch::Tensor rgb_dc, c10::optional<torch::Tensor> sh_rest,
    torch::Tensor camera_T_world, torch::Tensor K, c10::optional<torch::Tensor> camera_centre, int64_t H, int64_t W,
    double near_thresh, double far_thresh, double cull_mask_padding, double mh_dist, int64_t depth_base, int64_t mode,
    c10::optional<torch::Tensor> filter3d, int64_t lens, c10::optional<torch::Tensor> lens_consts,
    c10::optional<torch::Tensor> rolling_shutter, int64_t readout) {
    return preprocess_forward(true, xyz, xyz_camera_frame, quaternion, scale, opacity_logit, rgb_dc, sh_rest,
                              camera_T_world, K, camera_centre, H, W, near_thresh, far_thresh, cull_mask_padding,
                              mh_dist, depth_base, true, mode, filter3d, lens, lens_consts, rolling_shutter, readout);
}

// (M, P known) -> the sorted pair list the tile renderers read records through, tile ranges [n_tiles+1] i32,
//                 vis_idx [M] i32, uv [M,2]
// speculative = true: M and P are CAPACITIES (the host has not read the real counts yet): buffers are sized by
// them, the pair buffer is padded behind the real pairs (gsr_emit_*'s `capacity`), and every tensor is returned at
// full capacity — the caller narrows them once it knows M and P, and redoes the call if P exceeded the capacity.
// The pair list is the sorted keys when the gaussian id rides in their low id_bits (ids_sorted is then empty), else
// the sorted gaussian ids [P] i32 (keys_sorted is then empty and id_bits 0).
// returns (ids_sorted, ranges, vis_idx, uv, keys_sorted, id_bits)
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, int64_t> fused_bin(
    torch::Tensor records, torch::Tensor zkey, torch::Tensor visible, torch::Tensor scan, int64_t M, int64_t P,
    int64_t H, int64_t W, double mh_dist, int64_t depth_bits, bool speculative,
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
    const int id_bits = gsr_packed_id_bits(N, n_tiles, (int)depth_bits);
    // with the id in the key, nobody needs the separate id array
    torch::Tensor ids_sorted = torch::empty({id_bits > 0 ? 0 : Pa}, i32);
    torch::Tensor vis_idx = torch::empty({M}, i32);
    torch::Tensor uv = torch::empty({M, 2}, opt);
    torch::Tensor ranges = torch::empty({n_tiles + 1}, i32);
    uint64_t* keys_a = (uint64_t*)keys.data_ptr<int64_t>();
    uint64_t* keys_b = keys_a + Pa;
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
    }
    torch::Tensor keys_sorted = id_bits > 0 ? keys.narrow(0, Pa, Pa) : torch::empty({0}, opt.dtype(torch::kInt64));
    return std::make_tuple(ids_sorted.numel() > 0 ? ids_sorted.narrow(0, 0, P) : ids_sorted, ranges, vis_idx, uv,
                           keys_sorted, (int64_t)id_bits);
}

// returns (image [H,W,3], n [H,W] i32, wlast [H,W], contribution masks (i32 words; empty when record_masks is false),
// depth [H,W,1], alpha [H,W,1]); depth and alpha are None unless depth_key (the per-gaussian depth keys of the forward,
// read when the pair list is a sorted id array) asks for the depth/alpha kernels.
// records: the per-gaussian record array [N,12], read through the sorted pair list keys_sorted / ids_sorted
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
fused_render_forward(torch::Tensor records, torch::Tensor ranges, torch::Tensor background, int64_t H, int64_t W,
                     int64_t P, bool record_masks, c10::optional<torch::Tensor> keys_sorted,
                     c10::optional<torch::Tensor> ids_sorted, int64_t id_bits,
                     c10::optional<torch::Tensor> depth_key, int64_t depth_base, int64_t depth_bits,
                     c10::optional<torch::Tensor> weight_sum, c10::optional<torch::Tensor> weight_max,
                     c10::optional<torch::Tensor> pixel_count, c10::optional<torch::Tensor> pair_total,
                     int64_t pair_capacity) {
    CHECK_VALID_INPUT(background); CHECK_FLOAT_TENSOR(background);
    TORCH_CHECK(background.numel() == 3, "Background RGB must have 3 elements");
    const int n_stats = weight_sum.has_value() + weight_max.has_value() + pixel_count.has_value();
    TORCH_CHECK(n_stats == 0 || n_stats == 3, "weight_sum, weight_max and pixel_count go together");
    if (n_stats == 3) {
        const int64_t N = records.size(0);
        for (const torch::Tensor* t : {&*weight_sum, &*weight_max, &*pixel_count}) {
            CHECK_VALID_INPUT((*t));
            TORCH_CHECK(t->device() == records.device(), "weight statistics must be on the records' device");
            TORCH_CHECK(t->dim() == 1 && t->size(0) == N, "weight statistics must have shape [N]");
        }
        TORCH_CHECK(weight_sum->scalar_type() == torch::kFloat32 && weight_max->scalar_type() == torch::kFloat32,
                    "weight_sum and weight_max must be float32");
        TORCH_CHECK(pixel_count->scalar_type() == torch::kInt32, "pixel_count must be int32");
    }
    if (pair_total.has_value()) {
        CHECK_VALID_INPUT((*pair_total));
        TORCH_CHECK(pair_total->scalar_type() == torch::kInt64 && pair_total->numel() >= 1,
                    "pair_total must be an int64 tensor (the pair scan; its last element is read)");
        TORCH_CHECK(pair_total->device() == records.device(), "pair_total must be on the records' device");
    }
    c10::cuda::CUDAGuard guard(records.device());
    auto opt = records.options();
    torch::Tensor image = torch::empty({H, W, 3}, opt);
    torch::Tensor n = torch::empty({H, W}, opt.dtype(torch::kInt32));
    torch::Tensor w = torch::empty({H, W}, opt);
    torch::Tensor depth, alpha;
    if (depth_key.has_value()) {
        depth = torch::empty({H, W, 1}, opt);
        alpha = torch::empty({H, W, 1}, opt);
    }
    torch::Tensor masks = record_masks
                              ? torch::zeros({(int64_t)gsr_contribution_mask_words(P, (int)H, (int)W)}, opt.dtype(torch::kInt32))
                              : torch::empty({0}, opt.dtype(torch::kInt32));
    uint32_t* mptr = record_masks ? (uint32_t*)masks.data_ptr<int>() : nullptr;
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    const bool stats = weight_sum.has_value();
    check_rc(gsr_render_forward_gather_stats(
                 F32PTR(records), ps.keys, (int)id_bits, ps.ids,
                 depth_key.has_value() ? (const uint32_t*)depth_key->data_ptr<int>() : nullptr,
                 (uint32_t)depth_base, (int)depth_bits, ranges.data_ptr<int>(), F32PTR(background), (int)H, (int)W,
                 n.data_ptr<int>(), F32PTR(w), F32PTR(image), depth.defined() ? F32PTR(depth) : nullptr,
                 alpha.defined() ? F32PTR(alpha) : nullptr, mptr, stats ? F32PTR((*weight_sum)) : nullptr,
                 stats ? F32PTR((*weight_max)) : nullptr, stats ? pixel_count->data_ptr<int>() : nullptr,
                 pair_total.has_value() ? (const uint64_t*)(pair_total->data_ptr<int64_t>() + pair_total->numel() - 1)
                                        : nullptr,
                 pair_capacity, cur_stream()),
             "gsr_render_forward_gather_stats");
    return std::make_tuple(image, n, w, masks, depth, alpha);
}

// per-gaussian gradient slab, rows indexed by gaussian; zero-filled, then accumulated into by the render backward:
// interleaved rows [N,12] rgb3 opacity | uv2 conic0 conic1 | conic2 pad3 (vector reductions); with
// grad_depth / grad_alpha [H,W,1] (the upstream gradients on the depth/alpha maps, with the forward's depth keys)
// conic2 z pad2, z the gradient on the camera-frame z.  mode: GSR_MODE_* bits, passed to gsr_render_backward_gather
// (GSR_MODE_ABSGRAD: conic2 z|0 |u| |v|, the per-pixel absolute uv gradients summed).
torch::Tensor fused_render_backward(torch::Tensor grad_image, int64_t N, int64_t P, torch::Tensor records,
                                    torch::Tensor ids_sorted, torch::Tensor ranges, torch::Tensor background,
                                    torch::Tensor n, torch::Tensor w, torch::Tensor masks,
                                    c10::optional<torch::Tensor> keys_sorted, int64_t id_bits,
                                    c10::optional<torch::Tensor> grad_depth, c10::optional<torch::Tensor> grad_alpha,
                                    c10::optional<torch::Tensor> depth_key, int64_t depth_base, int64_t depth_bits,
                                    int64_t mode) {
    CHECK_VALID_INPUT(grad_image); CHECK_FLOAT_TENSOR(grad_image);
    const int H = n.size(0), W = n.size(1);
    TORCH_CHECK(grad_image.dim() == 3 && grad_image.size(0) == H && grad_image.size(1) == W &&
                    grad_image.size(2) == 3,
                "grad_image must be HxWx3");
    const bool depth = grad_depth.has_value();
    if (depth) {
        TORCH_CHECK(grad_alpha.has_value() && depth_key.has_value(),
                    "the depth/alpha backward needs grad_alpha and depth_key");
        CHECK_VALID_INPUT((*grad_depth)); CHECK_FLOAT_TENSOR((*grad_depth));
        CHECK_VALID_INPUT((*grad_alpha)); CHECK_FLOAT_TENSOR((*grad_alpha));
        TORCH_CHECK(grad_depth->numel() == (int64_t)H * W && grad_alpha->numel() == (int64_t)H * W,
                    "grad_depth and grad_alpha must hold H*W values");
    }
    c10::cuda::CUDAGuard guard(grad_image.device());
    torch::Tensor slab = torch::zeros({N * (int64_t)GSR_GRAD_ROW_FLOATS}, grad_image.options());
    const uint32_t* mptr = masks.numel() > 0 ? (const uint32_t*)masks.data_ptr<int>() : nullptr;
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    check_rc(gsr_render_backward_gather(
                 (int)mode, F32PTR(records), ps.keys, (int)id_bits, ps.ids,
                 depth ? (const uint32_t*)depth_key->data_ptr<int>() : nullptr, (uint32_t)depth_base,
                 (int)depth_bits, ranges.data_ptr<int>(), F32PTR(background), H, W, n.data_ptr<int>(), F32PTR(w),
                 F32PTR(grad_image), depth ? F32PTR((*grad_depth)) : nullptr,
                 depth ? F32PTR((*grad_alpha)) : nullptr, nullptr, nullptr, nullptr, nullptr, F32PTR(slab), mptr,
                 cur_stream()),
             "gsr_render_backward_gather");
    return slab;
}

// feature_map [H,W,D]: features [N, stride] (stride = D rounded up to a multiple of 4, the padding columns 0) blended
// with the colour forward's weights over the same pair list (gsr_render_features_forward)
torch::Tensor fused_render_features_forward(torch::Tensor records, torch::Tensor ranges, int64_t H, int64_t W,
                                            int64_t P, c10::optional<torch::Tensor> keys_sorted,
                                            c10::optional<torch::Tensor> ids_sorted, int64_t id_bits,
                                            torch::Tensor features, int64_t D) {
    CHECK_VALID_INPUT(features); CHECK_FLOAT_TENSOR(features);
    TORCH_CHECK(features.dim() == 2 && features.size(0) == records.size(0), "features must be [N, stride]");
    TORCH_CHECK(features.device() == records.device(), "features must be on the records' device");
    c10::cuda::CUDAGuard guard(records.device());
    torch::Tensor fmap = torch::empty({H, W, D}, records.options());
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    check_rc(gsr_render_features_forward(F32PTR(records), ps.keys, (int)id_bits, ps.ids, ranges.data_ptr<int>(), (int)H,
                                         (int)W, F32PTR(features), (int)features.size(1), (int)D, F32PTR(fmap),
                                         cur_stream()),
             "gsr_render_features_forward");
    return fmap;
}

// the feature backward (gsr_render_features_backward): adds the feature loss's opacity / uv / conic part into the
// gradient slab of fused_render_backward and returns grad_features [N, stride]
torch::Tensor fused_render_features_backward(torch::Tensor grad_map, torch::Tensor slab, int64_t P,
                                             torch::Tensor records, torch::Tensor ids_sorted, torch::Tensor ranges,
                                             torch::Tensor n, torch::Tensor w, torch::Tensor masks,
                                             c10::optional<torch::Tensor> keys_sorted, int64_t id_bits,
                                             torch::Tensor features) {
    CHECK_VALID_INPUT(grad_map); CHECK_FLOAT_TENSOR(grad_map);
    CHECK_VALID_INPUT(slab); CHECK_FLOAT_TENSOR(slab);
    CHECK_VALID_INPUT(features); CHECK_FLOAT_TENSOR(features);
    const int64_t N = records.size(0);
    TORCH_CHECK(grad_map.dim() == 3 && grad_map.size(0) == n.size(0) && grad_map.size(1) == n.size(1),
                "grad_map must be [H, W, D]");
    TORCH_CHECK(features.dim() == 2 && features.size(0) == N, "features must be [N, stride]");
    TORCH_CHECK(slab.numel() == N * (int64_t)GSR_GRAD_ROW_FLOATS, "gradient slab must hold ", GSR_GRAD_ROW_FLOATS,
                " floats per gaussian");
    c10::cuda::CUDAGuard guard(grad_map.device());
    torch::Tensor grad_features = torch::zeros_like(features);
    const uint32_t* mptr = masks.numel() > 0 ? (const uint32_t*)masks.data_ptr<int>() : nullptr;
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    check_rc(gsr_render_features_backward(F32PTR(records), ps.keys, (int)id_bits, ps.ids, ranges.data_ptr<int>(),
                                          (int)n.size(0), (int)n.size(1), n.data_ptr<int>(), F32PTR(w),
                                          F32PTR(features), (int)features.size(1), (int)grad_map.size(2),
                                          F32PTR(grad_map), F32PTR(grad_features), F32PTR(slab), mptr, cur_stream()),
             "gsr_render_features_backward");
    return grad_features;
}

// The flat parameter / gradient layout: [xyz 3N | quaternion 4N | scale 3N | opacity N | rgb 3N | sh 3*n_sh_rest*N],
// every section starting on a 16-byte boundary (TMA bulk stores).  width: floats per gaussian of each section; off:
// each section's start, off[6] the total.
struct FlatLayout {
    int64_t width[6];
    int64_t off[7];
};
static FlatLayout flat_layout(int64_t N, int64_t n_sh_rest) {
    FlatLayout l = {{3, 4, 3, 1, 3, 3 * n_sh_rest}, {0}};
    for (int i = 0; i < 6; ++i) l.off[i + 1] = (l.off[i] + N * l.width[i] + 3) & ~(int64_t)3;
    return l;
}

// The per-gaussian backward: grads of (xyz, quaternion, scale, opacity_logit, rgb_dc[, sh_rest]) from the gradient
// rows of the render backward, interleaved [N,12] by gaussian.  One view (batched false): slab [N*12] of
// fused_render_backward, visible / scan [N] of fused_preprocess_forward (gsr_preprocess_backward, or the lens's).
// C views (batched): slab [C, N*12] of batch_render_backward, visible / scan [C,N] of batch_preprocess_forward,
// grad_uv_compact [sum M_c, 2], the gradient summed over the views in one pass (gsr_batch_preprocess_backward, or the
// lens's).  grad_uv_compact [M,2] (optional): gradient on the compact uv, added to — or, with use_slab_uv false,
// replacing — the slab's uv section.  mode: the GSR_MODE_* bits of the forward: GSR_MODE_DEPTH_ALPHA reads the z
// gradient of the depth/alpha rows, GSR_MODE_ANTIALIASED takes the rows' opacity slot as the gradient on the
// compensated opacity, GSR_MODE_FILTER3D needs the forward's filter3d.  lens, lc: the forward's.
// camera_grads: 0 none; 1 also d loss / d camera_T_world (gsr_pose_*, libgsr_pose.so); 2 also the intrinsics and
// lens-coefficient gradients (gsr_camera_*, libgsr_calib.so).  shutter, readout, H, W: the forward's rolling shutter
// (gsr_shutter_*, libgsr_shutter.so), where camera_grads 1 also gives the gradient on the twists and 2 is refused.
// Returns the gaussian gradients, then `flat` (the one allocation they are views of), then with camera_grads >= 1
// g_pose [4,4] / [C,4,4] (last row 0), then with camera_grads 2 d loss / d (fx, fy, cx, cy) [4] / [C,4] and d loss /
// d lens coefficients [n] / [C,n] (n = 0 for the pinhole); with a shutter and camera_grads 1: g_pose, then g_xi
// [6] / [C,6].
static std::vector<torch::Tensor> preprocess_backward(
    bool batched, torch::Tensor slab, torch::Tensor xyz, torch::Tensor quaternion, torch::Tensor scale,
    torch::Tensor opacity_logit, c10::optional<torch::Tensor> sh_rest, torch::Tensor camera_T_world, torch::Tensor K,
    c10::optional<torch::Tensor> camera_centre, torch::Tensor visible, c10::optional<torch::Tensor> out_flat,
    c10::optional<torch::Tensor> grad_uv_compact, c10::optional<torch::Tensor> scan, bool use_slab_uv, int64_t mode,
    c10::optional<torch::Tensor> filter3d, int64_t lens, c10::optional<torch::Tensor> lc, int64_t camera_grads,
    c10::optional<torch::Tensor> shutter, int64_t readout, int64_t H, int64_t W) {
    TORCH_CHECK(camera_grads >= 0 && camera_grads <= 2,
                "camera_grads must be 0 (none), 1 (pose) or 2 (pose, intrinsics and lens)");
    TORCH_CHECK(!(shutter.has_value() && camera_grads == 2),
                "intrinsics and lens-coefficient gradients are not available with a rolling shutter");
    CHECK_VALID_INPUT(slab); CHECK_FLOAT_TENSOR(slab);
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(quaternion); CHECK_VALID_INPUT(scale); CHECK_VALID_INPUT(opacity_logit);
    CHECK_VALID_INPUT(visible);
    const int64_t C = check_views(batched, camera_T_world, K);
    const int64_t N = xyz.size(0);
    TORCH_CHECK(slab.numel() == C * N * (int64_t)GSR_GRAD_ROW_FLOATS, "gradient slab must hold ",
                GSR_GRAD_ROW_FLOATS, " floats per gaussian and view");
    TORCH_CHECK(visible.numel() == C * N && visible.scalar_type() == torch::kUInt8,
                "visible must hold one uint8 per gaussian and view");
    const float* centre_ptr = nullptr;
    if (camera_centre.has_value()) {
        CHECK_VALID_INPUT((*camera_centre)); CHECK_FLOAT_TENSOR((*camera_centre));
        TORCH_CHECK(camera_centre->numel() == 3 * C, "camera_centre must hold 3 floats per view");
        centre_ptr = camera_centre->data_ptr<float>();
    }
    const int n_rest = sh_rest.has_value() ? (int)sh_rest->size(2) : 0;
    const float* g_uv_compact = nullptr;
    const uint64_t* scan_ptr = nullptr;
    if (grad_uv_compact.has_value() && grad_uv_compact->numel() > 0) {
        CHECK_VALID_INPUT((*grad_uv_compact)); CHECK_FLOAT_TENSOR((*grad_uv_compact));
        TORCH_CHECK(scan.has_value() && scan->numel() == C * N && scan->scalar_type() == torch::kInt64,
                    "grad_uv_compact needs the packed scan of the forward pass");
        CHECK_VALID_INPUT((*scan));
        TORCH_CHECK(grad_uv_compact->dim() == 2 && grad_uv_compact->size(1) == 2, "grad_uv_compact must be Mx2");
        g_uv_compact = grad_uv_compact->data_ptr<float>();
        scan_ptr = (const uint64_t*)scan->data_ptr<int64_t>();
    }
    const float* f3d = filter3d_ptr(filter3d, N);
    const float* lens_consts = lens_ptr(lens, lc, C, xyz);
    const float* xi = shutter_ptr(shutter, C, batched, xyz);
    c10::cuda::CUDAGuard guard(xyz.device());
    auto opt = xyz.options();
    // All parameter gradients live in ONE allocation of the flat layout: a trainer that sums gradients over views /
    // ranks reduces that one buffer (view_parallel.py).  out_flat: a caller-owned buffer of the same layout (e.g.
    // symmetric memory peers can read, view_parallel.py)
    const FlatLayout l = flat_layout(N, n_rest);
    torch::Tensor flat;
    if (out_flat.has_value()) {
        flat = *out_flat;
        CHECK_VALID_INPUT(flat); CHECK_FLOAT_TENSOR(flat);
        TORCH_CHECK(flat.numel() == l.off[6], "out_flat must hold ", l.off[6], " floats");
        TORCH_CHECK((reinterpret_cast<uintptr_t>(flat.data_ptr()) & 15u) == 0, "out_flat must be 16-byte aligned");
    } else {
        flat = torch::empty({l.off[6]}, opt);
    }
    for (int i = 0; i < 6; ++i)  // padding between sections (only when N is not a multiple of 4)
        if (l.off[i + 1] > l.off[i] + N * l.width[i])
            flat.narrow(0, l.off[i] + N * l.width[i], l.off[i + 1] - l.off[i] - N * l.width[i]).zero_();
    auto section = [&](int i, std::vector<int64_t> shape) {
        return flat.narrow(0, l.off[i], N * l.width[i]).view(shape);
    };
    torch::Tensor o_xyz = section(0, {N, 3}), o_q = section(1, {N, 4}), o_s = section(2, {N, 3}),
                  o_o = section(3, {N}), o_dc = section(4, {N, 3});
    torch::Tensor g_sh;
    if (n_rest) g_sh = section(5, {N, 3, (int64_t)n_rest});
    // the arguments after (mode[, C]) shared by every backward entry point
#define GSR_BWD_ARGS                                                                                                 \
    (int)N, n_rest, F32PTR(xyz), F32PTR(quaternion), F32PTR(scale), F32PTR(opacity_logit), f3d,                      \
        F32PTR(camera_T_world), F32PTR(K), centre_ptr, visible.data_ptr<uint8_t>(), F32PTR(slab),                    \
        use_slab_uv ? 1 : 0, g_uv_compact, scan_ptr, F32PTR(o_xyz), F32PTR(o_q), F32PTR(o_s), F32PTR(o_o),           \
        F32PTR(o_dc), n_rest ? F32PTR(g_sh) : nullptr
    const int md = (int)mode, nc = (int)C, ln = (int)lens;
    std::vector<torch::Tensor> out = {o_xyz, o_q, o_s, o_o, o_dc};
    if (n_rest) out.push_back(g_sh);
    out.push_back(flat);
    if (xi != nullptr) {
        torch::Tensor g_pose, g_xi, temp;
        if (camera_grads == 1) {
            g_pose = torch::empty(batched ? std::vector<int64_t>{C, 4, 4} : std::vector<int64_t>{4, 4}, opt);
            g_xi = torch::empty(batched ? std::vector<int64_t>{C, 6} : std::vector<int64_t>{6}, opt);
            temp = torch::empty({(int64_t)gsr_shutter_temp_bytes(nc, (int)N)}, opt.dtype(torch::kUInt8));
        }
        float* gp = camera_grads == 1 ? F32PTR(g_pose) : nullptr;
        float* gx = camera_grads == 1 ? F32PTR(g_xi) : nullptr;
        void* tp = camera_grads == 1 ? temp.data_ptr() : nullptr;
        const size_t tb = camera_grads == 1 ? (size_t)temp.numel() : 0;
        check_rc(batched ? gsr_shutter_batch_preprocess_backward(ln, md, nc, GSR_BWD_ARGS, lens_consts, xi, (int)readout,
                                                                 (int)H, (int)W, gp, gx, tp, tb, cur_stream())
                         : gsr_shutter_preprocess_backward(ln, md, GSR_BWD_ARGS, lens_consts, xi, (int)readout, (int)H,
                                                           (int)W, gp, gx, tp, tb, cur_stream()),
                 batched ? "gsr_shutter_batch_preprocess_backward" : "gsr_shutter_preprocess_backward");
        if (camera_grads == 1) {
            out.push_back(g_pose);
            out.push_back(g_xi);
        }
        return out;
    }
    if (camera_grads == 0) {
        if (lens == GSR_LENS_FISHEYE)
            check_rc(batched ? gsr_fisheye_batch_preprocess_backward(md, nc, GSR_BWD_ARGS, lens_consts, cur_stream())
                             : gsr_fisheye_preprocess_backward(md, GSR_BWD_ARGS, lens_consts, cur_stream()),
                     batched ? "gsr_fisheye_batch_preprocess_backward" : "gsr_fisheye_preprocess_backward");
        else if (lens == GSR_LENS_DISTORTION)
            check_rc(batched
                         ? gsr_distortion_batch_preprocess_backward(md, nc, GSR_BWD_ARGS, lens_consts, cur_stream())
                         : gsr_distortion_preprocess_backward(md, GSR_BWD_ARGS, lens_consts, cur_stream()),
                     batched ? "gsr_distortion_batch_preprocess_backward" : "gsr_distortion_preprocess_backward");
        else
            check_rc(batched ? gsr_batch_preprocess_backward(md, nc, GSR_BWD_ARGS, cur_stream())
                             : gsr_preprocess_backward(md, GSR_BWD_ARGS, cur_stream()),
                     batched ? "gsr_batch_preprocess_backward" : "gsr_preprocess_backward");
        return out;
    }
    // one view's camera gradients have no view dimension
    auto shape = [&](std::initializer_list<int64_t> s) {
        std::vector<int64_t> v(s);
        if (batched) v.insert(v.begin(), C);
        return v;
    };
    torch::Tensor g_pose = torch::empty(shape({4, 4}), opt);
    out.push_back(g_pose);
    if (camera_grads == 1) {
        torch::Tensor temp = torch::empty({(int64_t)gsr_pose_temp_bytes(nc, (int)N)}, opt.dtype(torch::kUInt8));
        void* tp = temp.data_ptr();
        const size_t tb = (size_t)temp.numel();
        check_rc(batched ? gsr_pose_batch_preprocess_backward(ln, md, nc, GSR_BWD_ARGS, lens_consts, F32PTR(g_pose), tp,
                                                              tb, cur_stream())
                         : gsr_pose_preprocess_backward(ln, md, GSR_BWD_ARGS, lens_consts, F32PTR(g_pose), tp, tb,
                                                        cur_stream()),
                 batched ? "gsr_pose_batch_preprocess_backward" : "gsr_pose_preprocess_backward");
        return out;
    }
    torch::Tensor g_intr = torch::empty(shape({4}), opt);
    const int64_t n_coeffs = std::max<int64_t>(lens_consts_per_view(lens) - 1, 0);
    torch::Tensor g_lens = torch::empty(shape({n_coeffs}), opt);
    torch::Tensor temp = torch::empty({(int64_t)gsr_camera_temp_bytes(ln, nc, (int)N)}, opt.dtype(torch::kUInt8));
    void* tp = temp.data_ptr();
    const size_t tb = (size_t)temp.numel();
    float* gl = g_lens.numel() ? F32PTR(g_lens) : nullptr;
    check_rc(batched ? gsr_camera_batch_preprocess_backward(ln, md, nc, GSR_BWD_ARGS, lens_consts, F32PTR(g_pose),
                                                            F32PTR(g_intr), gl, tp, tb, cur_stream())
                     : gsr_camera_preprocess_backward(ln, md, GSR_BWD_ARGS, lens_consts, F32PTR(g_pose),
                                                      F32PTR(g_intr), gl, tp, tb, cur_stream()),
             batched ? "gsr_camera_batch_preprocess_backward" : "gsr_camera_preprocess_backward");
#undef GSR_BWD_ARGS
    out.push_back(g_intr);
    out.push_back(g_lens);
    return out;
}

std::vector<torch::Tensor> fused_preprocess_backward(
    torch::Tensor slab, torch::Tensor xyz, torch::Tensor quaternion, torch::Tensor scale, torch::Tensor opacity_logit,
    c10::optional<torch::Tensor> sh_rest, torch::Tensor camera_T_world, torch::Tensor K,
    c10::optional<torch::Tensor> camera_centre, torch::Tensor visible, c10::optional<torch::Tensor> out_flat,
    c10::optional<torch::Tensor> grad_uv_compact, c10::optional<torch::Tensor> scan, bool use_slab_uv, int64_t mode,
    c10::optional<torch::Tensor> filter3d, int64_t lens, c10::optional<torch::Tensor> lens_consts,
    int64_t camera_grads, c10::optional<torch::Tensor> rolling_shutter, int64_t readout, int64_t H, int64_t W) {
    return preprocess_backward(false, slab, xyz, quaternion, scale, opacity_logit, sh_rest, camera_T_world, K,
                               camera_centre, visible, out_flat, grad_uv_compact, scan, use_slab_uv, mode, filter3d,
                               lens, lens_consts, camera_grads, rolling_shutter, readout, H, W);
}

std::vector<torch::Tensor> batch_preprocess_backward(
    torch::Tensor slab, torch::Tensor xyz, torch::Tensor quaternion, torch::Tensor scale, torch::Tensor opacity_logit,
    c10::optional<torch::Tensor> sh_rest, torch::Tensor camera_T_world, torch::Tensor K,
    c10::optional<torch::Tensor> camera_centre, torch::Tensor visible, c10::optional<torch::Tensor> out_flat,
    c10::optional<torch::Tensor> grad_uv_compact, c10::optional<torch::Tensor> scan, bool use_slab_uv, int64_t mode,
    c10::optional<torch::Tensor> filter3d, int64_t lens, c10::optional<torch::Tensor> lens_consts,
    int64_t camera_grads, c10::optional<torch::Tensor> rolling_shutter, int64_t readout, int64_t H, int64_t W) {
    return preprocess_backward(true, slab, xyz, quaternion, scale, opacity_logit, sh_rest, camera_T_world, K,
                               camera_centre, visible, out_flat, grad_uv_compact, scan, use_slab_uv, mode, filter3d,
                               lens, lens_consts, camera_grads, rolling_shutter, readout, H, W);
}

// ---------------------------------------------------------------------------------------------
// multi-view fused path (rasterize_batch): C views of one scene, per-view arrays stacked view-major
// ---------------------------------------------------------------------------------------------
// fused_render_backward of every view into one stacked slab [C, N*12]: grad_image [C,H,W,3], per view the forward's
// pair list (keys_sorted or ids_sorted, the other one empty), ranges, n, w and masks (empty: none); records [C,N,12],
// background [C,3]; with grad_depth / grad_alpha [C,H,W,1] also depth_key [C,N].
torch::Tensor batch_render_backward(torch::Tensor grad_image, int64_t N, std::vector<int64_t> P, torch::Tensor records,
                                    std::vector<torch::Tensor> ids_sorted, std::vector<torch::Tensor> keys_sorted,
                                    std::vector<int64_t> id_bits, std::vector<torch::Tensor> ranges,
                                    torch::Tensor background, std::vector<torch::Tensor> n,
                                    std::vector<torch::Tensor> w, std::vector<torch::Tensor> masks,
                                    c10::optional<torch::Tensor> grad_depth, c10::optional<torch::Tensor> grad_alpha,
                                    c10::optional<torch::Tensor> depth_key, int64_t depth_base, int64_t depth_bits,
                                    int64_t mode) {
    CHECK_VALID_INPUT(grad_image); CHECK_FLOAT_TENSOR(grad_image);
    CHECK_VALID_INPUT(records); CHECK_FLOAT_TENSOR(records);
    CHECK_VALID_INPUT(background); CHECK_FLOAT_TENSOR(background);
    const int64_t C = (int64_t)P.size();
    TORCH_CHECK(C >= 1 && (int64_t)ids_sorted.size() == C && (int64_t)keys_sorted.size() == C &&
                    (int64_t)id_bits.size() == C && (int64_t)ranges.size() == C && (int64_t)n.size() == C &&
                    (int64_t)w.size() == C && (int64_t)masks.size() == C,
                "every per-view list must hold C >= 1 entries");
    const int H = n[0].size(0), W = n[0].size(1);
    TORCH_CHECK(grad_image.dim() == 4 && grad_image.size(0) == C && grad_image.size(1) == H &&
                    grad_image.size(2) == W && grad_image.size(3) == 3,
                "grad_image must be CxHxWx3");
    TORCH_CHECK(records.numel() == C * N * (int64_t)GSR_REC_FLOATS, "records must have shape CxNx12");
    TORCH_CHECK(background.numel() == 3 * C, "background must have shape Cx3");
    const bool depth = grad_depth.has_value();
    if (depth) {
        TORCH_CHECK(grad_alpha.has_value() && depth_key.has_value(),
                    "the depth/alpha backward needs grad_alpha and depth_key");
        CHECK_VALID_INPUT((*grad_depth)); CHECK_FLOAT_TENSOR((*grad_depth));
        CHECK_VALID_INPUT((*grad_alpha)); CHECK_FLOAT_TENSOR((*grad_alpha));
        CHECK_VALID_INPUT((*depth_key));
        TORCH_CHECK(grad_depth->numel() == C * H * W && grad_alpha->numel() == C * H * W,
                    "grad_depth and grad_alpha must hold C*H*W values");
        TORCH_CHECK(depth_key->numel() == C * N, "depth_key must have shape CxN");
    }
    c10::cuda::CUDAGuard guard(grad_image.device());
    torch::Tensor slab = torch::zeros({C, N * (int64_t)GSR_GRAD_ROW_FLOATS}, grad_image.options());
    const int64_t HW = (int64_t)H * W;
    for (int64_t c = 0; c < C && N > 0; ++c) {
        TORCH_CHECK(n[c].size(0) == H && n[c].size(1) == W, "every view must have the same image size");
        const uint32_t* mptr = masks[c].numel() > 0 ? (const uint32_t*)masks[c].data_ptr<int>() : nullptr;
        const PairSource ps = pair_source(keys_sorted[c], ids_sorted[c], P[c]);
        check_rc(gsr_render_backward_gather(
                     (int)mode, F32PTR(records) + c * N * GSR_REC_FLOATS, ps.keys, (int)id_bits[c], ps.ids,
                     depth ? (const uint32_t*)depth_key->data_ptr<int>() + c * N : nullptr, (uint32_t)depth_base,
                     (int)depth_bits, ranges[c].data_ptr<int>(), F32PTR(background) + 3 * c, H, W,
                     n[c].data_ptr<int>(), F32PTR(w[c]), F32PTR(grad_image) + c * HW * 3,
                     depth ? F32PTR((*grad_depth)) + c * HW : nullptr, depth ? F32PTR((*grad_alpha)) + c * HW : nullptr,
                     nullptr, nullptr, nullptr, nullptr, F32PTR(slab[c]), mptr, cur_stream()),
                 "gsr_render_backward_gather");
    }
    return slab;
}

// gsr_fisheye_theta_max of 4 coefficients (host floats)
double fisheye_theta_max(std::vector<double> k) {
    TORCH_CHECK(k.size() == 4, "fisheye needs 4 coefficients k1 k2 k3 k4");
    const float kf[4] = {(float)k[0], (float)k[1], (float)k[2], (float)k[3]};
    return (double)gsr_fisheye_theta_max(kf);
}

// gsr_distortion_r2_max of 5 coefficients k1 k2 p1 p2 k3 (host floats)
double distortion_r2_max(std::vector<double> k) {
    TORCH_CHECK(k.size() == 5, "distortion needs 5 coefficients k1 k2 p1 p2 k3");
    const float kf[5] = {(float)k[0], (float)k[1], (float)k[2], (float)k[3], (float)k[4]};
    return (double)gsr_distortion_r2_max(kf);
}

// Mip-Splatting's 3-D filter size per gaussian (gsr_filter3d): xyz [N,3], camera_T_world [C,4,4], K [C,3,3],
// width / height int32 [C], all on xyz's device -> filter3d [N]
torch::Tensor filter3d(torch::Tensor xyz, torch::Tensor camera_T_world, torch::Tensor K, torch::Tensor width,
                       torch::Tensor height, double near, double margin, double variance) {
    CHECK_VALID_INPUT(xyz); CHECK_VALID_INPUT(camera_T_world); CHECK_VALID_INPUT(K); CHECK_VALID_INPUT(width);
    CHECK_VALID_INPUT(height);
    CHECK_FLOAT_TENSOR(xyz); CHECK_FLOAT_TENSOR(camera_T_world); CHECK_FLOAT_TENSOR(K);
    CHECK_INT_TENSOR(width); CHECK_INT_TENSOR(height);
    TORCH_CHECK(xyz.dim() == 2 && xyz.size(1) == 3, "xyz must have shape Nx3");
    const int64_t C = camera_T_world.size(0);
    TORCH_CHECK(camera_T_world.dim() == 3 && camera_T_world.size(1) == 4 && camera_T_world.size(2) == 4,
                "camera_T_world must have shape Cx4x4");
    TORCH_CHECK(K.dim() == 3 && K.size(0) == C && K.size(1) == 3 && K.size(2) == 3, "K must have shape Cx3x3");
    TORCH_CHECK(width.numel() == C && height.numel() == C, "width and height must hold C values");
    c10::cuda::CUDAGuard guard(xyz.device());
    torch::Tensor out = torch::empty({xyz.size(0)}, xyz.options());
    check_rc(gsr_filter3d((int)xyz.size(0), F32PTR(xyz), (int)C, F32PTR(camera_T_world), F32PTR(K),
                          width.data_ptr<int>(), height.data_ptr<int>(), (float)near, (float)margin, (float)variance,
                          F32PTR(out), cur_stream()),
             "gsr_filter3d");
    return out;
}

// sizes of the flat parameter / gradient layout: exclusive end of each section, in elements
std::vector<int64_t> flat_section_ends(int64_t N, int64_t n_sh_rest) {
    const FlatLayout l = flat_layout(N, n_sh_rest);
    std::vector<int64_t> ends;
    for (int i = 0; i < 6; ++i)
        if (l.width[i] > 0) ends.push_back(l.off[i + 1]);
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

// visible: CUDA bool / uint8 [N], nonzero = the row is updated (rasterize's state.visible); N = visible.numel()
void adam_step_selective(torch::Tensor p, torch::Tensor g, torch::Tensor m, torch::Tensor v, torch::Tensor visible,
                         int64_t n_sh_rest, std::vector<int64_t> section_end, std::vector<double> section_lr,
                         double beta1, double beta2, double eps, int64_t step) {
    CHECK_VALID_INPUT(p); CHECK_VALID_INPUT(g); CHECK_VALID_INPUT(m); CHECK_VALID_INPUT(v);
    CHECK_FLOAT_TENSOR(p); CHECK_FLOAT_TENSOR(g); CHECK_FLOAT_TENSOR(m); CHECK_FLOAT_TENSOR(v);
    CHECK_VALID_INPUT(visible);
    TORCH_CHECK(visible.dtype() == torch::kBool || visible.dtype() == torch::kUInt8, "visible must be bool or uint8");
    TORCH_CHECK(visible.device() == p.device() && g.device() == p.device() && m.device() == p.device() &&
                    v.device() == p.device(), "p, g, m, v and visible must be on one device");
    const int64_t n = p.numel();
    TORCH_CHECK(g.numel() == n && m.numel() == n && v.numel() == n, "p, g, m, v must have the same length");
    TORCH_CHECK(section_end.size() == section_lr.size() && !section_end.empty() && section_end.back() == n,
                "sections must cover the buffer");
    const int64_t rows = visible.numel();
    TORCH_CHECK(n_sh_rest >= 0 && flat_section_ends(rows, n_sh_rest) == section_end,
                "visible has ", rows, " rows, which do not match the flat layout of the buffer");
    c10::cuda::CUDAGuard guard(p.device());
    check_rc(gsr_adam_step_selective(rows, (int)n_sh_rest, F32PTR(p), F32PTR(g), F32PTR(m), F32PTR(v),
                                     reinterpret_cast<const uint8_t*>(visible.data_ptr()), (int)section_end.size(),
                                     section_end.data(), section_lr.data(), beta1, beta2, eps, (int)step,
                                     cur_stream()),
             "gsr_adam_step_selective");
}

void adam_step_selective_sharded(int64_t lo, int64_t hi, std::vector<int64_t> peer_grad_ptrs,
                                 std::vector<int64_t> peer_param_ptrs, std::vector<int64_t> peer_visible_ptrs,
                                 int64_t self_rank, torch::Tensor m_shard, torch::Tensor v_shard, int64_t n_rows,
                                 int64_t n_sh_rest, std::vector<int64_t> section_end, std::vector<double> section_lr,
                                 double beta1, double beta2, double eps, int64_t step) {
    CHECK_VALID_INPUT(m_shard); CHECK_VALID_INPUT(v_shard); CHECK_FLOAT_TENSOR(m_shard); CHECK_FLOAT_TENSOR(v_shard);
    TORCH_CHECK(peer_grad_ptrs.size() == peer_param_ptrs.size() && peer_grad_ptrs.size() == peer_visible_ptrs.size() &&
                    !peer_grad_ptrs.empty(), "one pointer per rank");
    TORCH_CHECK(m_shard.numel() == hi - lo && v_shard.numel() == hi - lo, "state shards must hold hi - lo elements");
    TORCH_CHECK(section_end.size() == section_lr.size() && !section_end.empty(), "bad sections");
    std::vector<const float*> gp;
    std::vector<float*> pp;
    std::vector<const uint8_t*> vp;
    for (size_t q = 0; q < peer_grad_ptrs.size(); ++q) {
        gp.push_back(reinterpret_cast<const float*>(peer_grad_ptrs[q]));
        pp.push_back(reinterpret_cast<float*>(peer_param_ptrs[q]));
        vp.push_back(reinterpret_cast<const uint8_t*>(peer_visible_ptrs[q]));
    }
    c10::cuda::CUDAGuard guard(m_shard.device());
    check_rc(gsr_adam_step_selective_sharded(lo, hi, (int)gp.size(), gp.data(), pp.data(), vp.data(), (int)self_rank,
                                             F32PTR(m_shard), F32PTR(v_shard), n_rows, (int)n_sh_rest,
                                             (int)section_end.size(), section_end.data(), section_lr.data(), beta1,
                                             beta2, eps, (int)step, cur_stream()),
             "gsr_adam_step_selective_sharded");
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

// 3DGS-MCMC relocation of n sampled rows -> (new_opacity [n], new_scale [n,3]) (gsr_mcmc_relocation)
std::vector<torch::Tensor> mcmc_relocation(torch::Tensor opacity, torch::Tensor scale, torch::Tensor ratio,
                                           int64_t n_max, double min_opacity) {
    CHECK_VALID_INPUT(opacity); CHECK_VALID_INPUT(scale); CHECK_VALID_INPUT(ratio);
    CHECK_FLOAT_TENSOR(opacity); CHECK_FLOAT_TENSOR(scale); CHECK_INT_TENSOR(ratio);
    const int64_t n = opacity.numel();
    TORCH_CHECK(scale.numel() == 3 * n && ratio.numel() == n, "opacity [n], scale [n,3] and ratio [n] must match");
    TORCH_CHECK(scale.device() == opacity.device() && ratio.device() == opacity.device(), "tensors on different devices");
    TORCH_CHECK(n_max >= 1, "n_max must be at least 1");
    c10::cuda::CUDAGuard guard(opacity.device());
    torch::Tensor new_opacity = torch::empty({n}, opacity.options());
    torch::Tensor new_scale = torch::empty({n, 3}, opacity.options());
    check_rc(gsr_mcmc_relocation((int)n, F32PTR(opacity), F32PTR(scale), ratio.data_ptr<int32_t>(), (int)n_max,
                                 (float)min_opacity, F32PTR(new_opacity), F32PTR(new_scale), cur_stream()),
             "gsr_mcmc_relocation");
    return {new_opacity, new_scale};
}

// a relocation / growth plan applied to the flat parameter buffer and both Adam moments (gsr_mcmc_apply); returns
// (p_out, m_out, v_out) freshly allocated (p_out: p_out_buf when given; only p_out without moments)
std::vector<torch::Tensor> mcmc_apply(torch::Tensor p_in, c10::optional<torch::Tensor> m_in,
                                      c10::optional<torch::Tensor> v_in, int64_t n_in, int64_t n_sh_rest,
                                      torch::Tensor src, c10::optional<torch::Tensor> set_row,
                                      c10::optional<torch::Tensor> new_opacity, c10::optional<torch::Tensor> new_scale,
                                      c10::optional<torch::Tensor> p_out_buf) {
    CHECK_VALID_INPUT(p_in); CHECK_FLOAT_TENSOR(p_in); CHECK_VALID_INPUT(src); CHECK_INT_TENSOR(src);
    TORCH_CHECK(n_in >= 0 && n_sh_rest >= 0, "n_in and n_sh_rest must be non-negative");
    TORCH_CHECK(p_in.numel() == gsr_flat_numel(n_in, (int)n_sh_rest), "p_in does not match the flat layout of n_in gaussians");
    const int64_t n_out = src.numel();
    TORCH_CHECK(n_out >= n_in, "mcmc_apply keeps every row: src must have at least n_in entries");
    const int64_t total = gsr_flat_numel(n_out, (int)n_sh_rest);
    const bool moments = m_in.has_value();
    TORCH_CHECK(moments == v_in.has_value(), "m_in and v_in go together");
    const bool sets = set_row.has_value();
    TORCH_CHECK(sets == new_opacity.has_value() && sets == new_scale.has_value(),
                "set_row, new_opacity and new_scale go together");
    TORCH_CHECK(src.device() == p_in.device(), "src must be on p_in's device");
    if (sets) {
        CHECK_VALID_INPUT((*set_row)); CHECK_INT_TENSOR((*set_row));
        CHECK_VALID_INPUT((*new_opacity)); CHECK_FLOAT_TENSOR((*new_opacity));
        CHECK_VALID_INPUT((*new_scale)); CHECK_FLOAT_TENSOR((*new_scale));
        TORCH_CHECK(set_row->numel() == n_out, "set_row must have one entry per output row");
        TORCH_CHECK(new_scale->numel() == 3 * new_opacity->numel(), "new_opacity [m] and new_scale [m,3] must match");
        for (auto* t : {&*set_row, &*new_opacity, &*new_scale})
            TORCH_CHECK(t->device() == p_in.device(), "plan tensors must be on p_in's device");
    }
    c10::cuda::CUDAGuard guard(p_in.device());
    torch::Tensor p_out;
    if (p_out_buf.has_value()) {  // caller-owned destination (e.g. symmetric memory)
        p_out = *p_out_buf;
        CHECK_VALID_INPUT(p_out); CHECK_FLOAT_TENSOR(p_out);
        TORCH_CHECK(p_out.numel() == total && p_out.device() == p_in.device(), "bad p_out buffer");
    } else {
        p_out = torch::empty({total}, p_in.options());
    }
    torch::Tensor m_out, v_out;
    if (moments) {
        CHECK_VALID_INPUT((*m_in)); CHECK_VALID_INPUT((*v_in)); CHECK_FLOAT_TENSOR((*m_in)); CHECK_FLOAT_TENSOR((*v_in));
        TORCH_CHECK(m_in->numel() == p_in.numel() && v_in->numel() == p_in.numel(), "moments must match p_in");
        TORCH_CHECK(m_in->device() == p_in.device() && v_in->device() == p_in.device(), "moments must be on p_in's device");
        m_out = torch::empty({total}, p_in.options());
        v_out = torch::empty({total}, p_in.options());
    }
    check_rc(gsr_mcmc_apply((int)n_in, (int)n_out, (int)n_sh_rest, F32PTR(p_in), moments ? F32PTR((*m_in)) : nullptr,
                            moments ? F32PTR((*v_in)) : nullptr, src.data_ptr<int32_t>(),
                            sets ? set_row->data_ptr<int32_t>() : nullptr, sets ? F32PTR((*new_opacity)) : nullptr,
                            sets ? F32PTR((*new_scale)) : nullptr, F32PTR(p_out), moments ? F32PTR(m_out) : nullptr,
                            moments ? F32PTR(v_out) : nullptr, cur_stream()),
             "gsr_mcmc_apply");
    if (moments) return {p_out, m_out, v_out};
    return {p_out};
}

// SGLD position noise in place on the flat parameter buffer of N gaussians (gsr_mcmc_noise)
void mcmc_noise(torch::Tensor p, int64_t N, int64_t n_sh_rest, double scaler, double k, double x0, int64_t seed,
                int64_t offset, c10::optional<torch::Tensor> eps_in, c10::optional<torch::Tensor> eps_out) {
    CHECK_VALID_INPUT(p); CHECK_FLOAT_TENSOR(p);
    TORCH_CHECK(N >= 0 && n_sh_rest >= 0, "N and n_sh_rest must be non-negative");
    TORCH_CHECK(p.numel() == gsr_flat_numel(N, (int)n_sh_rest), "p does not match the flat layout of N gaussians");
    TORCH_CHECK(offset >= 0, "offset must be non-negative");
    for (auto* t : {&eps_in, &eps_out}) {
        if (!t->has_value()) continue;
        CHECK_VALID_INPUT((**t)); CHECK_FLOAT_TENSOR((**t));
        TORCH_CHECK((*t)->numel() == 3 * N, "eps_in / eps_out must have shape [N,3]");
        TORCH_CHECK((*t)->device() == p.device(), "eps_in / eps_out must be on p's device");
    }
    c10::cuda::CUDAGuard guard(p.device());
    check_rc(gsr_mcmc_noise((int)N, (int)n_sh_rest, F32PTR(p), scaler, k, x0, (uint64_t)seed, (uint64_t)offset,
                            eps_in.has_value() ? F32PTR((*eps_in)) : nullptr,
                            eps_out.has_value() ? F32PTR((*eps_out)) : nullptr, cur_stream()),
             "gsr_mcmc_noise");
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

// ---------------------------------------------------------------------------------------------
// bilateral-grid appearance correction (gsr_bilagrid_*): rgb [C,H,W,3] any strides, grids [N,12,L,GY,GX] contiguous,
// ids [C] int32 on the device (range-checked by the caller)
// ---------------------------------------------------------------------------------------------
void check_bilagrid_grids(const torch::Tensor& grids) {
    CHECK_VALID_INPUT(grids);
    CHECK_FLOAT_TENSOR(grids);
    TORCH_CHECK(grids.dim() == 5 && grids.size(1) == 12, "grids must be [N,12,L,GY,GX]");
}

void check_bilagrid_slice(const torch::Tensor& rgb, const torch::Tensor& grids, const torch::Tensor& ids) {
    check_bilagrid_grids(grids);
    TORCH_CHECK(rgb.is_cuda() && rgb.device() == grids.device(), "rgb must be on the grids' device");
    CHECK_FLOAT_TENSOR(rgb);
    TORCH_CHECK(rgb.dim() == 4 && rgb.size(3) == 3, "rgb must be [C,H,W,3]");
    CHECK_VALID_INPUT(ids);
    CHECK_INT_TENSOR(ids);
    TORCH_CHECK(ids.device() == grids.device() && ids.dim() == 1 && ids.size(0) == rgb.size(0),
                "ids must be [C] on the grids' device");
}

torch::Tensor bilagrid_slice_forward(torch::Tensor rgb, torch::Tensor grids, torch::Tensor ids) {
    check_bilagrid_slice(rgb, grids, ids);
    c10::cuda::CUDAGuard guard(rgb.device());
    torch::Tensor out = torch::empty(rgb.sizes(), rgb.options().memory_format(torch::MemoryFormat::Contiguous));
    const int64_t rs[4] = {rgb.stride(0), rgb.stride(1), rgb.stride(2), rgb.stride(3)};
    check_rc(gsr_bilagrid_slice_forward((int)rgb.size(0), (int)rgb.size(1), (int)rgb.size(2), F32PTR(rgb), rs,
                                        F32PTR(grids), (int)grids.size(0), (int)grids.size(2), (int)grids.size(3),
                                        (int)grids.size(4), ids.data_ptr<int32_t>(), F32PTR(out), cur_stream()),
             "gsr_bilagrid_slice_forward");
    return out;
}

// returns (grad_rgb [C,H,W,3] contiguous or None, grad_grids [N,12,L,GY,GX] or None)
std::vector<torch::Tensor> bilagrid_slice_backward(torch::Tensor rgb, torch::Tensor grids, torch::Tensor ids,
                                                   torch::Tensor grad_out, bool need_rgb, bool need_grids) {
    check_bilagrid_slice(rgb, grids, ids);
    TORCH_CHECK(grad_out.is_cuda() && grad_out.device() == rgb.device(), "grad_out must be on rgb's device");
    CHECK_FLOAT_TENSOR(grad_out);
    TORCH_CHECK(grad_out.sizes() == rgb.sizes(), "grad_out must have rgb's shape");
    c10::cuda::CUDAGuard guard(rgb.device());
    const int C = rgb.size(0), H = rgb.size(1), W = rgb.size(2);
    const int L = grids.size(2), GY = grids.size(3), GX = grids.size(4);
    torch::Tensor grad_rgb, grad_grids, temp;
    if (need_rgb) grad_rgb = torch::empty(rgb.sizes(), rgb.options().memory_format(torch::MemoryFormat::Contiguous));
    size_t tb = 0;
    if (need_grids) {
        grad_grids = torch::empty_like(grids);
        tb = gsr_bilagrid_slice_backward_temp_bytes(C, H, L, GY, GX);
        temp = torch::empty({(int64_t)tb}, grids.options().dtype(torch::kUInt8));
    }
    const int64_t rs[4] = {rgb.stride(0), rgb.stride(1), rgb.stride(2), rgb.stride(3)};
    const int64_t gs[4] = {grad_out.stride(0), grad_out.stride(1), grad_out.stride(2), grad_out.stride(3)};
    check_rc(gsr_bilagrid_slice_backward(C, H, W, F32PTR(rgb), rs, F32PTR(grids), (int)grids.size(0), L, GY, GX,
                                         ids.data_ptr<int32_t>(), F32PTR(grad_out), gs,
                                         need_rgb ? F32PTR(grad_rgb) : nullptr,
                                         need_grids ? F32PTR(grad_grids) : nullptr,
                                         need_grids ? temp.data_ptr() : nullptr, tb, cur_stream()),
             "gsr_bilagrid_slice_backward");
    return {grad_rgb, grad_grids};
}

// returns tv(grids) as a 0-dim float tensor on the device
torch::Tensor bilagrid_tv_forward(torch::Tensor grids) {
    check_bilagrid_grids(grids);
    c10::cuda::CUDAGuard guard(grids.device());
    const int N = grids.size(0), L = grids.size(2), GY = grids.size(3), GX = grids.size(4);
    torch::Tensor out = torch::empty({}, grids.options());
    const size_t tb = gsr_bilagrid_tv_temp_bytes(N, L, GY, GX);
    torch::Tensor temp = torch::empty({(int64_t)tb}, grids.options().dtype(torch::kUInt8));
    check_rc(gsr_bilagrid_tv_forward(N, L, GY, GX, F32PTR(grids), F32PTR(out), temp.data_ptr(), tb, cur_stream()),
             "gsr_bilagrid_tv_forward");
    return out;
}

torch::Tensor bilagrid_tv_backward(torch::Tensor grids, torch::Tensor grad_tv) {
    check_bilagrid_grids(grids);
    TORCH_CHECK(grad_tv.is_cuda() && grad_tv.device() == grids.device(), "grad_tv must be on the grids' device");
    TORCH_CHECK(grad_tv.numel() == 1 && grad_tv.dtype() == torch::kFloat32, "grad_tv must be a float scalar");
    c10::cuda::CUDAGuard guard(grids.device());
    torch::Tensor grad = torch::empty_like(grids);
    check_rc(gsr_bilagrid_tv_backward((int)grids.size(0), (int)grids.size(2), (int)grids.size(3), (int)grids.size(4),
                                      F32PTR(grids), F32PTR(grad_tv), F32PTR(grad), cur_stream()),
             "gsr_bilagrid_tv_backward");
    return grad;
}

// ---- 2-D Gaussian surfels (libgsr_surfels.so) -------------------------------------------------------------------------
static const float* opt_f32(const c10::optional<torch::Tensor>& t) {
    if (!t.has_value()) return nullptr;
    CHECK_VALID_INPUT((*t)); CHECK_FLOAT_TENSOR((*t));
    return t->data_ptr<float>();
}

// returns (surfels [N,20], bin_records [N,12], depth_key, visible, scan, tile_mask, tile_win): the inputs of fused_bin
// (with bin_records as its records) and of the surfel tile kernels
// lens 0: the pinhole (gsr_surfel_preprocess_forward), else GSR_SURFEL_LENS_* with its constants lens_consts
std::vector<torch::Tensor> surfel_forward_any(int64_t lens, const c10::optional<torch::Tensor>& lens_consts,
                                              torch::Tensor xyz, c10::optional<torch::Tensor> xyz_cam,
                                              torch::Tensor quaternion, torch::Tensor scale,
                                              torch::Tensor opacity_logit, torch::Tensor rgb,
                                              c10::optional<torch::Tensor> sh_rest, torch::Tensor camera_T_world,
                                              torch::Tensor K, c10::optional<torch::Tensor> camera_centre, int64_t H,
                                              int64_t W, double near_thresh, double far_thresh, double pad,
                                              double mh_dist, int64_t depth_base) {
    for (const torch::Tensor* t : {&xyz, &quaternion, &scale, &opacity_logit, &rgb, &camera_T_world, &K}) {
        CHECK_VALID_INPUT((*t)); CHECK_FLOAT_TENSOR((*t));
    }
    const int64_t N = xyz.size(0);
    const int n_rest = sh_rest.has_value() ? (int)sh_rest->size(2) : 0;
    const float* cam = opt_f32(xyz_cam);
    const int cam_first = xyz_cam.has_value() ? (int)(N - xyz_cam->size(0)) : 0;
    c10::cuda::CUDAGuard guard(xyz.device());
    auto opt = xyz.options();
    torch::Tensor surfels = torch::empty({N, GSR_SURFEL_REC_FLOATS}, opt);
    torch::Tensor bins = torch::empty({N, GSR_REC_FLOATS}, opt);
    torch::Tensor zkey = torch::empty({N}, opt.dtype(torch::kInt32));
    torch::Tensor visible = torch::empty({N}, opt.dtype(torch::kUInt8));
    torch::Tensor scan = torch::empty({N}, opt.dtype(torch::kInt64));
    torch::Tensor tile_mask = torch::empty({N}, opt.dtype(torch::kInt64));
    torch::Tensor tile_win = torch::empty({N}, opt.dtype(torch::kInt32));
    torch::Tensor temp = torch::empty({(int64_t)gsr_surfel_temp_bytes((int)N)}, opt.dtype(torch::kUInt8));
    if (lens == 0) {
        check_rc(gsr_surfel_preprocess_forward(
                     (int)N, n_rest, F32PTR(xyz), cam, cam_first, F32PTR(quaternion), F32PTR(scale),
                     F32PTR(opacity_logit), F32PTR(rgb), opt_f32(sh_rest), F32PTR(camera_T_world), F32PTR(K),
                     opt_f32(camera_centre), (int)H, (int)W, (float)near_thresh, (float)far_thresh, (float)pad,
                     (float)mh_dist, (uint32_t)depth_base, F32PTR(surfels), F32PTR(bins),
                     (uint32_t*)zkey.data_ptr<int>(), visible.data_ptr<uint8_t>(), (uint64_t*)scan.data_ptr<int64_t>(),
                     (uint64_t*)tile_mask.data_ptr<int64_t>(), (uint32_t*)tile_win.data_ptr<int>(), temp.data_ptr(),
                     (size_t)temp.numel(), cur_stream()),
                 "gsr_surfel_preprocess_forward");
    } else {
        check_rc(gsr_surfel_lens_preprocess_forward(
                     (int)lens, (int)N, n_rest, F32PTR(xyz), cam, cam_first, F32PTR(quaternion), F32PTR(scale),
                     F32PTR(opacity_logit), F32PTR(rgb), opt_f32(sh_rest), F32PTR(camera_T_world), F32PTR(K),
                     opt_f32(camera_centre), (int)H, (int)W, (float)near_thresh, (float)far_thresh, (float)pad,
                     (float)mh_dist, (uint32_t)depth_base, F32PTR(surfels), F32PTR(bins),
                     (uint32_t*)zkey.data_ptr<int>(), visible.data_ptr<uint8_t>(), (uint64_t*)scan.data_ptr<int64_t>(),
                     (uint64_t*)tile_mask.data_ptr<int64_t>(), (uint32_t*)tile_win.data_ptr<int>(), temp.data_ptr(),
                     (size_t)temp.numel(), opt_f32(lens_consts), cur_stream()),
                 "gsr_surfel_lens_preprocess_forward");
    }
    return {surfels, bins, zkey, visible, scan, tile_mask, tile_win};
}

std::vector<torch::Tensor> surfel_forward(torch::Tensor xyz, c10::optional<torch::Tensor> xyz_cam,
                                          torch::Tensor quaternion, torch::Tensor scale, torch::Tensor opacity_logit,
                                          torch::Tensor rgb, c10::optional<torch::Tensor> sh_rest,
                                          torch::Tensor camera_T_world, torch::Tensor K,
                                          c10::optional<torch::Tensor> camera_centre, int64_t H, int64_t W,
                                          double near_thresh, double far_thresh, double pad, double mh_dist,
                                          int64_t depth_base) {
    return surfel_forward_any(0, c10::nullopt, xyz, xyz_cam, quaternion, scale, opacity_logit, rgb, sh_rest,
                              camera_T_world, K, camera_centre, H, W, near_thresh, far_thresh, pad, mh_dist,
                              depth_base);
}

std::vector<torch::Tensor> surfel_lens_forward(int64_t lens, torch::Tensor lens_consts, torch::Tensor xyz,
                                               c10::optional<torch::Tensor> xyz_cam, torch::Tensor quaternion,
                                               torch::Tensor scale, torch::Tensor opacity_logit, torch::Tensor rgb,
                                               c10::optional<torch::Tensor> sh_rest, torch::Tensor camera_T_world,
                                               torch::Tensor K, c10::optional<torch::Tensor> camera_centre, int64_t H,
                                               int64_t W, double near_thresh, double far_thresh, double pad,
                                               double mh_dist, int64_t depth_base) {
    TORCH_CHECK(lens == GSR_SURFEL_LENS_FISHEYE || lens == GSR_SURFEL_LENS_DISTORTION, "unknown surfel lens ", lens);
    return surfel_forward_any(lens, lens_consts, xyz, xyz_cam, quaternion, scale, opacity_logit, rgb, sh_rest,
                              camera_T_world, K, camera_centre, H, W, near_thresh, far_thresh, pad, mh_dist,
                              depth_base);
}

// the ray map [H, W, 3] of a lens (gsr_surfel_rays)
torch::Tensor surfel_rays(int64_t lens, torch::Tensor lens_consts, torch::Tensor K, int64_t H, int64_t W) {
    CHECK_VALID_INPUT(K); CHECK_FLOAT_TENSOR(K);
    CHECK_VALID_INPUT(lens_consts); CHECK_FLOAT_TENSOR(lens_consts);
    c10::cuda::CUDAGuard guard(K.device());
    torch::Tensor rays = torch::empty({H, W, 3}, K.options());
    check_rc(gsr_surfel_rays((int)lens, (int)H, (int)W, F32PTR(K), F32PTR(lens_consts), F32PTR(rays), cur_stream()),
             "gsr_surfel_rays");
    return rays;
}

// returns (image [H,W,3], depth [H,W,1], alpha [H,W,1], normal [H,W,3], distortion [H,W,1], last [H,W] i32,
// totals [H,W,3])
// rays: the lens's ray map (gsr_surfel_lens_render_forward), or none for the pinhole
std::vector<torch::Tensor> surfel_render_forward_any(const c10::optional<torch::Tensor>& rays, torch::Tensor surfels,
                                                     torch::Tensor ranges, torch::Tensor background, int64_t H,
                                                     int64_t W, int64_t P, c10::optional<torch::Tensor> keys_sorted,
                                                     c10::optional<torch::Tensor> ids_sorted, int64_t id_bits,
                                                     double near_thresh, double m_scale, double mh_dist) {
    CHECK_VALID_INPUT(surfels); CHECK_FLOAT_TENSOR(surfels);
    CHECK_VALID_INPUT(background); CHECK_FLOAT_TENSOR(background);
    TORCH_CHECK(background.numel() == 3, "Background RGB must have 3 elements");
    c10::cuda::CUDAGuard guard(surfels.device());
    auto opt = surfels.options();
    torch::Tensor image = torch::empty({H, W, 3}, opt), depth = torch::empty({H, W, 1}, opt),
                  alpha = torch::empty({H, W, 1}, opt), normal = torch::empty({H, W, 3}, opt),
                  dist = torch::empty({H, W, 1}, opt), last = torch::empty({H, W}, opt.dtype(torch::kInt32)),
                  totals = torch::empty({H, W, 3}, opt);
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    const bool keys = ps.keys != nullptr;  // else ids (with P == 0 a placeholder the kernels never read)
    if (!rays.has_value()) {
        check_rc(gsr_surfel_render_forward(F32PTR(surfels), ps.keys, keys ? (int)id_bits : 0, keys ? nullptr : ps.ids,
                                           ranges.data_ptr<int>(), F32PTR(background), (int)H, (int)W,
                                           (float)near_thresh, (float)m_scale, (float)mh_dist, F32PTR(image),
                                           F32PTR(depth), F32PTR(alpha), F32PTR(normal), F32PTR(dist),
                                           last.data_ptr<int>(), F32PTR(totals), cur_stream()),
                 "gsr_surfel_render_forward");
    } else {
        TORCH_CHECK(rays->numel() == H * W * 3, "rays must be [H, W, 3]");
        check_rc(gsr_surfel_lens_render_forward(F32PTR(surfels), ps.keys, keys ? (int)id_bits : 0,
                                                keys ? nullptr : ps.ids, ranges.data_ptr<int>(), F32PTR(background),
                                                (int)H, (int)W, (float)near_thresh, (float)m_scale, (float)mh_dist,
                                                opt_f32(rays), F32PTR(image), F32PTR(depth), F32PTR(alpha),
                                                F32PTR(normal), F32PTR(dist), last.data_ptr<int>(), F32PTR(totals),
                                                cur_stream()),
                 "gsr_surfel_lens_render_forward");
    }
    return {image, depth, alpha, normal, dist, last, totals};
}

std::vector<torch::Tensor> surfel_render_forward(torch::Tensor surfels, torch::Tensor ranges, torch::Tensor background,
                                                 int64_t H, int64_t W, int64_t P,
                                                 c10::optional<torch::Tensor> keys_sorted,
                                                 c10::optional<torch::Tensor> ids_sorted, int64_t id_bits,
                                                 double near_thresh, double m_scale, double mh_dist) {
    return surfel_render_forward_any(c10::nullopt, surfels, ranges, background, H, W, P, keys_sorted, ids_sorted,
                                     id_bits, near_thresh, m_scale, mh_dist);
}

std::vector<torch::Tensor> surfel_lens_render_forward(torch::Tensor rays, torch::Tensor surfels, torch::Tensor ranges,
                                                      torch::Tensor background, int64_t H, int64_t W, int64_t P,
                                                      c10::optional<torch::Tensor> keys_sorted,
                                                      c10::optional<torch::Tensor> ids_sorted, int64_t id_bits,
                                                      double near_thresh, double m_scale, double mh_dist) {
    return surfel_render_forward_any(rays, surfels, ranges, background, H, W, P, keys_sorted, ids_sorted, id_bits,
                                     near_thresh, m_scale, mh_dist);
}

// the surfel gradient rows [N, 20] (zero-filled, accumulated by the tile backward)
torch::Tensor surfel_render_backward_any(const c10::optional<torch::Tensor>& rays, int64_t N, torch::Tensor surfels,
                                         torch::Tensor ranges, torch::Tensor background, int64_t H, int64_t W,
                                         int64_t P, c10::optional<torch::Tensor> keys_sorted,
                                         c10::optional<torch::Tensor> ids_sorted, int64_t id_bits,
                                         double near_thresh, double m_scale, double mh_dist, torch::Tensor alpha,
                                         torch::Tensor last, torch::Tensor totals, torch::Tensor g_image,
                                         torch::Tensor g_depth, torch::Tensor g_alpha, torch::Tensor g_normal,
                                         torch::Tensor g_distortion) {
    for (const torch::Tensor* t : {&surfels, &background, &alpha, &totals, &g_image, &g_depth, &g_alpha, &g_normal,
                                   &g_distortion}) {
        CHECK_VALID_INPUT((*t)); CHECK_FLOAT_TENSOR((*t));
    }
    TORCH_CHECK(g_image.numel() == H * W * 3 && g_normal.numel() == H * W * 3 && g_depth.numel() == H * W &&
                    g_alpha.numel() == H * W && g_distortion.numel() == H * W,
                "upstream gradients must match the maps' shapes");
    c10::cuda::CUDAGuard guard(surfels.device());
    torch::Tensor rows = torch::zeros({N, GSR_SURFEL_GRAD_FLOATS}, surfels.options());
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    const bool keys = ps.keys != nullptr;
    if (!rays.has_value()) {
        check_rc(gsr_surfel_render_backward(F32PTR(surfels), ps.keys, keys ? (int)id_bits : 0,
                                            keys ? nullptr : ps.ids, ranges.data_ptr<int>(), F32PTR(background),
                                            (int)H, (int)W, (float)near_thresh, (float)m_scale, (float)mh_dist,
                                            F32PTR(alpha), last.data_ptr<int>(), F32PTR(totals), F32PTR(g_image),
                                            F32PTR(g_depth), F32PTR(g_alpha), F32PTR(g_normal), F32PTR(g_distortion),
                                            F32PTR(rows), cur_stream()),
                 "gsr_surfel_render_backward");
    } else {
        TORCH_CHECK(rays->numel() == H * W * 3, "rays must be [H, W, 3]");
        check_rc(gsr_surfel_lens_render_backward(F32PTR(surfels), ps.keys, keys ? (int)id_bits : 0,
                                                 keys ? nullptr : ps.ids, ranges.data_ptr<int>(), F32PTR(background),
                                                 (int)H, (int)W, (float)near_thresh, (float)m_scale, (float)mh_dist,
                                                 opt_f32(rays), F32PTR(alpha), last.data_ptr<int>(), F32PTR(totals),
                                                 F32PTR(g_image), F32PTR(g_depth), F32PTR(g_alpha), F32PTR(g_normal),
                                                 F32PTR(g_distortion), F32PTR(rows), cur_stream()),
                 "gsr_surfel_lens_render_backward");
    }
    return rows;
}

torch::Tensor surfel_render_backward(int64_t N, torch::Tensor surfels, torch::Tensor ranges, torch::Tensor background,
                                     int64_t H, int64_t W, int64_t P, c10::optional<torch::Tensor> keys_sorted,
                                     c10::optional<torch::Tensor> ids_sorted, int64_t id_bits, double near_thresh,
                                     double m_scale, double mh_dist, torch::Tensor alpha, torch::Tensor last,
                                     torch::Tensor totals, torch::Tensor g_image, torch::Tensor g_depth,
                                     torch::Tensor g_alpha, torch::Tensor g_normal, torch::Tensor g_distortion) {
    return surfel_render_backward_any(c10::nullopt, N, surfels, ranges, background, H, W, P, keys_sorted, ids_sorted,
                                      id_bits, near_thresh, m_scale, mh_dist, alpha, last, totals, g_image, g_depth,
                                      g_alpha, g_normal, g_distortion);
}

torch::Tensor surfel_lens_render_backward(torch::Tensor rays, int64_t N, torch::Tensor surfels, torch::Tensor ranges,
                                          torch::Tensor background, int64_t H, int64_t W, int64_t P,
                                          c10::optional<torch::Tensor> keys_sorted,
                                          c10::optional<torch::Tensor> ids_sorted, int64_t id_bits,
                                          double near_thresh, double m_scale, double mh_dist, torch::Tensor alpha,
                                          torch::Tensor last, torch::Tensor totals, torch::Tensor g_image,
                                          torch::Tensor g_depth, torch::Tensor g_alpha, torch::Tensor g_normal,
                                          torch::Tensor g_distortion) {
    return surfel_render_backward_any(rays, N, surfels, ranges, background, H, W, P, keys_sorted, ids_sorted, id_bits,
                                      near_thresh, m_scale, mh_dist, alpha, last, totals, g_image, g_depth, g_alpha,
                                      g_normal, g_distortion);
}

// the feature kernels' common checks: features [N, stride] (stride = D rounded up to a multiple of 4, the padding
// columns 0) next to the surfel records, and the ray map of a lens
static void check_surfel_features(const torch::Tensor& surfels, const torch::Tensor& features, int64_t D,
                                  const c10::optional<torch::Tensor>& rays, int64_t H, int64_t W) {
    CHECK_VALID_INPUT(surfels); CHECK_FLOAT_TENSOR(surfels);
    CHECK_VALID_INPUT(features); CHECK_FLOAT_TENSOR(features);
    TORCH_CHECK(features.dim() == 2 && features.size(0) == surfels.size(0), "features must be [N, stride]");
    TORCH_CHECK(features.device() == surfels.device(), "features must be on the surfels' device");
    TORCH_CHECK(D >= 1 && features.size(1) >= D, "features must hold D >= 1 columns");
    if (rays.has_value()) {
        CHECK_VALID_INPUT((*rays)); CHECK_FLOAT_TENSOR((*rays));
        TORCH_CHECK(rays->numel() == H * W * 3, "rays must be [H, W, 3]");
    }
}

// feature_map [H,W,D]: features blended with the surfel colour forward's weights, up to its `last` contributor
// (gsr_surfel_render_features_forward); rays: the lens's ray map, or none for the pinhole
torch::Tensor surfel_features_forward(const c10::optional<torch::Tensor>& rays, torch::Tensor surfels,
                                      torch::Tensor ranges, int64_t H, int64_t W, int64_t P,
                                      c10::optional<torch::Tensor> keys_sorted, c10::optional<torch::Tensor> ids_sorted,
                                      int64_t id_bits, double mh_dist, torch::Tensor last, torch::Tensor features,
                                      int64_t D) {
    check_surfel_features(surfels, features, D, rays, H, W);
    CHECK_VALID_INPUT(last); CHECK_INT_TENSOR(last);
    TORCH_CHECK(last.numel() == H * W, "last must be [H, W]");
    c10::cuda::CUDAGuard guard(surfels.device());
    torch::Tensor fmap = torch::empty({H, W, D}, surfels.options());
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    const bool keys = ps.keys != nullptr;
    check_rc(gsr_surfel_render_features_forward(F32PTR(surfels), ps.keys, keys ? (int)id_bits : 0,
                                                keys ? nullptr : ps.ids, ranges.data_ptr<int>(), (int)H, (int)W,
                                                (float)mh_dist, opt_f32(rays), last.data_ptr<int>(), F32PTR(features),
                                                (int)features.size(1), (int)D, F32PTR(fmap), cur_stream()),
             "gsr_surfel_render_features_forward");
    return fmap;
}

// the feature backward (gsr_surfel_render_features_backward): adds the feature loss's part of d alpha into the surfel
// gradient rows [N, 20] of surfel_render_backward (in place) and returns grad_features [N, stride]
torch::Tensor surfel_features_backward(const c10::optional<torch::Tensor>& rays, torch::Tensor surfels,
                                       torch::Tensor ranges, int64_t H, int64_t W, int64_t P,
                                       c10::optional<torch::Tensor> keys_sorted,
                                       c10::optional<torch::Tensor> ids_sorted, int64_t id_bits, double mh_dist,
                                       torch::Tensor last, torch::Tensor totals, torch::Tensor features, int64_t D,
                                       torch::Tensor grad_map, torch::Tensor rows) {
    check_surfel_features(surfels, features, D, rays, H, W);
    CHECK_VALID_INPUT(last); CHECK_INT_TENSOR(last);
    CHECK_VALID_INPUT(totals); CHECK_FLOAT_TENSOR(totals);
    CHECK_VALID_INPUT(grad_map); CHECK_FLOAT_TENSOR(grad_map);
    CHECK_VALID_INPUT(rows); CHECK_FLOAT_TENSOR(rows);
    TORCH_CHECK(last.numel() == H * W && totals.numel() == H * W * 3, "last and totals must be [H, W] and [H, W, 3]");
    TORCH_CHECK(grad_map.numel() == H * W * D, "grad_map must be [H, W, D]");
    TORCH_CHECK(rows.numel() == surfels.size(0) * (int64_t)GSR_SURFEL_GRAD_FLOATS, "rows must hold ",
                GSR_SURFEL_GRAD_FLOATS, " floats per gaussian");
    c10::cuda::CUDAGuard guard(surfels.device());
    torch::Tensor grad_features = torch::zeros_like(features);
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    const bool keys = ps.keys != nullptr;
    check_rc(gsr_surfel_render_features_backward(
                 F32PTR(surfels), ps.keys, keys ? (int)id_bits : 0, keys ? nullptr : ps.ids, ranges.data_ptr<int>(),
                 (int)H, (int)W, (float)mh_dist, opt_f32(rays), last.data_ptr<int>(), F32PTR(totals),
                 F32PTR(features), (int)features.size(1), (int)D, F32PTR(grad_map), F32PTR(grad_features),
                 F32PTR(rows), cur_stream()),
             "gsr_surfel_render_features_backward");
    return grad_features;
}

// (median [H,W,1], median_id [H,W] int32): each pixel's median contributor of the surfel colour forward, up to its
// `last` (gsr_surfel_render_median_forward); rays: the lens's ray map, or none for the pinhole
std::vector<torch::Tensor> surfel_median_forward(const c10::optional<torch::Tensor>& rays, torch::Tensor surfels,
                                                 torch::Tensor ranges, int64_t H, int64_t W, int64_t P,
                                                 c10::optional<torch::Tensor> keys_sorted,
                                                 c10::optional<torch::Tensor> ids_sorted, int64_t id_bits,
                                                 double mh_dist, torch::Tensor last) {
    CHECK_VALID_INPUT(surfels); CHECK_FLOAT_TENSOR(surfels);
    CHECK_VALID_INPUT(ranges); CHECK_INT_TENSOR(ranges);
    CHECK_VALID_INPUT(last); CHECK_INT_TENSOR(last);
    TORCH_CHECK(last.numel() == H * W, "last must be [H, W]");
    if (rays.has_value()) {
        CHECK_VALID_INPUT((*rays)); CHECK_FLOAT_TENSOR((*rays));
        TORCH_CHECK(rays->numel() == H * W * 3, "rays must be [H, W, 3]");
    }
    c10::cuda::CUDAGuard guard(surfels.device());
    torch::Tensor median = torch::empty({H, W, 1}, surfels.options());
    torch::Tensor median_id = torch::empty({H, W}, last.options());
    const PairSource ps = pair_source(keys_sorted, ids_sorted, P);
    const bool keys = ps.keys != nullptr;
    check_rc(gsr_surfel_render_median_forward(F32PTR(surfels), ps.keys, keys ? (int)id_bits : 0,
                                              keys ? nullptr : ps.ids, ranges.data_ptr<int>(), (int)H, (int)W,
                                              (float)mh_dist, opt_f32(rays), last.data_ptr<int>(), F32PTR(median),
                                              median_id.data_ptr<int>(), cur_stream()),
             "gsr_surfel_render_median_forward");
    return {median, median_id};
}

// the median backward (gsr_surfel_render_median_backward): adds d loss / d median through each pixel's median surfel's
// z into the surfel gradient rows [N, 20] of surfel_render_backward, in place
void surfel_median_backward(const c10::optional<torch::Tensor>& rays, torch::Tensor surfels, int64_t H, int64_t W,
                            double mh_dist, torch::Tensor median_id, torch::Tensor grad_median, torch::Tensor rows) {
    CHECK_VALID_INPUT(surfels); CHECK_FLOAT_TENSOR(surfels);
    CHECK_VALID_INPUT(median_id); CHECK_INT_TENSOR(median_id);
    CHECK_VALID_INPUT(grad_median); CHECK_FLOAT_TENSOR(grad_median);
    CHECK_VALID_INPUT(rows); CHECK_FLOAT_TENSOR(rows);
    TORCH_CHECK(median_id.numel() == H * W && grad_median.numel() == H * W, "median_id and grad_median must be [H, W]");
    TORCH_CHECK(rows.numel() == surfels.size(0) * (int64_t)GSR_SURFEL_GRAD_FLOATS, "rows must hold ",
                GSR_SURFEL_GRAD_FLOATS, " floats per gaussian");
    if (rays.has_value()) {
        CHECK_VALID_INPUT((*rays)); CHECK_FLOAT_TENSOR((*rays));
        TORCH_CHECK(rays->numel() == H * W * 3, "rays must be [H, W, 3]");
    }
    c10::cuda::CUDAGuard guard(surfels.device());
    check_rc(gsr_surfel_render_median_backward(F32PTR(surfels), (int)H, (int)W, (float)mh_dist, opt_f32(rays),
                                               median_id.data_ptr<int>(), F32PTR(grad_median), F32PTR(rows),
                                               cur_stream()),
             "gsr_surfel_render_median_backward");
}

// uv.grad [M,2] of the visible gaussians vis_idx from the gradient rows
torch::Tensor surfel_uv_grad(torch::Tensor vis_idx, torch::Tensor surfels, torch::Tensor rows) {
    CHECK_VALID_INPUT(vis_idx); CHECK_INT_TENSOR(vis_idx);
    CHECK_VALID_INPUT(surfels); CHECK_VALID_INPUT(rows);
    c10::cuda::CUDAGuard guard(surfels.device());
    const int64_t M = vis_idx.numel();
    torch::Tensor out = torch::empty({M, 2}, surfels.options());
    check_rc(gsr_surfel_uv_grad((int)M, vis_idx.data_ptr<int>(), F32PTR(surfels), F32PTR(rows), F32PTR(out),
                                cur_stream()),
             "gsr_surfel_uv_grad");
    return out;
}

// uv.grad [M,2] of a lens surfel view (gsr_surfel_lens_uv_grad)
torch::Tensor surfel_lens_uv_grad(int64_t lens, torch::Tensor lens_consts, torch::Tensor K, torch::Tensor vis_idx,
                                  torch::Tensor surfels, torch::Tensor rows) {
    CHECK_VALID_INPUT(vis_idx); CHECK_INT_TENSOR(vis_idx);
    CHECK_VALID_INPUT(surfels); CHECK_VALID_INPUT(rows); CHECK_VALID_INPUT(K); CHECK_VALID_INPUT(lens_consts);
    c10::cuda::CUDAGuard guard(surfels.device());
    const int64_t M = vis_idx.numel();
    torch::Tensor out = torch::empty({M, 2}, surfels.options());
    check_rc(gsr_surfel_lens_uv_grad((int)lens, (int)M, vis_idx.data_ptr<int>(), F32PTR(surfels), F32PTR(rows),
                                     F32PTR(K), F32PTR(lens_consts), F32PTR(out), cur_stream()),
             "gsr_surfel_lens_uv_grad");
    return out;
}

// the per-gaussian backward into the flat layout of fused_preprocess_backward (out_flat: a caller-owned buffer of it);
// returns the gaussian gradients (xyz, quaternion, scale, opacity, rgb[, sh]) and then `flat`
std::vector<torch::Tensor> surfel_backward_any(int64_t lens, const c10::optional<torch::Tensor>& lens_consts,
                                               torch::Tensor rows, torch::Tensor xyz, torch::Tensor quaternion,
                                               torch::Tensor scale, torch::Tensor opacity_logit,
                                               c10::optional<torch::Tensor> sh_rest, torch::Tensor camera_T_world,
                                               torch::Tensor K, c10::optional<torch::Tensor> camera_centre,
                                               torch::Tensor visible, torch::Tensor surfels,
                                               c10::optional<torch::Tensor> out_flat,
                                               c10::optional<torch::Tensor> grad_uv_compact,
                                               c10::optional<torch::Tensor> scan, bool uv_grad_emitted) {
    for (const torch::Tensor* t : {&rows, &xyz, &quaternion, &scale, &opacity_logit, &camera_T_world, &K, &surfels}) {
        CHECK_VALID_INPUT((*t)); CHECK_FLOAT_TENSOR((*t));
    }
    CHECK_VALID_INPUT(visible);
    const int64_t N = xyz.size(0);
    TORCH_CHECK(rows.numel() == N * GSR_SURFEL_GRAD_FLOATS && surfels.numel() == N * GSR_SURFEL_REC_FLOATS &&
                    visible.numel() == N,
                "surfel rows, records and visible must hold one entry per gaussian");
    const int n_rest = sh_rest.has_value() ? (int)sh_rest->size(2) : 0;
    const float* guv = nullptr;
    const uint64_t* scan_ptr = nullptr;
    if (grad_uv_compact.has_value() && grad_uv_compact->numel() > 0) {
        guv = opt_f32(grad_uv_compact);
        TORCH_CHECK(scan.has_value() && scan->numel() == N, "grad_uv_compact needs the forward's scan");
        scan_ptr = (const uint64_t*)scan->data_ptr<int64_t>();
    }
    c10::cuda::CUDAGuard guard(xyz.device());
    const FlatLayout l = flat_layout(N, n_rest);
    torch::Tensor flat;
    if (out_flat.has_value()) {
        flat = *out_flat;
        CHECK_VALID_INPUT(flat); CHECK_FLOAT_TENSOR(flat);
        TORCH_CHECK(flat.numel() == l.off[6], "out_flat must hold ", l.off[6], " floats");
    } else {
        flat = torch::empty({l.off[6]}, xyz.options());
    }
    for (int i = 0; i < 6; ++i)
        if (l.off[i + 1] > l.off[i] + N * l.width[i])
            flat.narrow(0, l.off[i] + N * l.width[i], l.off[i + 1] - l.off[i] - N * l.width[i]).zero_();
    auto section = [&](int i, std::vector<int64_t> shape) { return flat.narrow(0, l.off[i], N * l.width[i]).view(shape); };
    std::vector<torch::Tensor> out = {section(0, {N, 3}), section(1, {N, 4}), section(2, {N, 3}), section(3, {N}),
                                      section(4, {N, 3})};
    if (n_rest) out.push_back(section(5, {N, 3, (int64_t)n_rest}));
    if (lens == 0) {
        check_rc(gsr_surfel_preprocess_backward((int)N, n_rest, F32PTR(xyz), F32PTR(quaternion), F32PTR(scale),
                                                F32PTR(opacity_logit), F32PTR(camera_T_world), F32PTR(K),
                                                opt_f32(camera_centre), visible.data_ptr<uint8_t>(), F32PTR(surfels),
                                                F32PTR(rows), guv, scan_ptr, uv_grad_emitted ? 1 : 0, F32PTR(out[0]),
                                                F32PTR(out[1]), F32PTR(out[2]), F32PTR(out[3]), F32PTR(out[4]),
                                                n_rest ? F32PTR(out[5]) : nullptr, cur_stream()),
                 "gsr_surfel_preprocess_backward");
    } else {
        check_rc(gsr_surfel_lens_preprocess_backward(
                     (int)lens, (int)N, n_rest, F32PTR(xyz), F32PTR(quaternion), F32PTR(scale), F32PTR(opacity_logit),
                     F32PTR(camera_T_world), F32PTR(K), opt_f32(camera_centre), visible.data_ptr<uint8_t>(),
                     F32PTR(surfels), F32PTR(rows), guv, scan_ptr, uv_grad_emitted ? 1 : 0, F32PTR(out[0]),
                     F32PTR(out[1]), F32PTR(out[2]), F32PTR(out[3]), F32PTR(out[4]), n_rest ? F32PTR(out[5]) : nullptr,
                     opt_f32(lens_consts), cur_stream()),
                 "gsr_surfel_lens_preprocess_backward");
    }
    out.push_back(flat);
    return out;
}

std::vector<torch::Tensor> surfel_backward(torch::Tensor rows, torch::Tensor xyz, torch::Tensor quaternion,
                                           torch::Tensor scale, torch::Tensor opacity_logit,
                                           c10::optional<torch::Tensor> sh_rest, torch::Tensor camera_T_world,
                                           torch::Tensor K, c10::optional<torch::Tensor> camera_centre,
                                           torch::Tensor visible, torch::Tensor surfels,
                                           c10::optional<torch::Tensor> out_flat,
                                           c10::optional<torch::Tensor> grad_uv_compact,
                                           c10::optional<torch::Tensor> scan, bool uv_grad_emitted) {
    return surfel_backward_any(0, c10::nullopt, rows, xyz, quaternion, scale, opacity_logit, sh_rest, camera_T_world,
                               K, camera_centre, visible, surfels, out_flat, grad_uv_compact, scan, uv_grad_emitted);
}

std::vector<torch::Tensor> surfel_lens_backward(int64_t lens, torch::Tensor lens_consts, torch::Tensor rows,
                                                torch::Tensor xyz, torch::Tensor quaternion, torch::Tensor scale,
                                                torch::Tensor opacity_logit, c10::optional<torch::Tensor> sh_rest,
                                                torch::Tensor camera_T_world, torch::Tensor K,
                                                c10::optional<torch::Tensor> camera_centre, torch::Tensor visible,
                                                torch::Tensor surfels, c10::optional<torch::Tensor> out_flat,
                                                c10::optional<torch::Tensor> grad_uv_compact,
                                                c10::optional<torch::Tensor> scan, bool uv_grad_emitted) {
    TORCH_CHECK(lens == GSR_SURFEL_LENS_FISHEYE || lens == GSR_SURFEL_LENS_DISTORTION, "unknown surfel lens ", lens);
    return surfel_backward_any(lens, lens_consts, rows, xyz, quaternion, scale, opacity_logit, sh_rest,
                               camera_T_world, K, camera_centre, visible, surfels, out_flat, grad_uv_compact, scan,
                               uv_grad_emitted);
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
    m.def("fused_preprocess_forward", &fused_preprocess_forward,
          "fused per-gaussian stage (with_tiles: also every gaussian's tile-hit mask and window; mode: MODE_* bits; "
          "lens: LENS_*, lens_consts its [n+1] constants)",
          py::arg("xyz"), py::arg("xyz_camera_frame"), py::arg("quaternion"), py::arg("scale"),
          py::arg("opacity_logit"), py::arg("rgb_dc"), py::arg("sh_rest"), py::arg("camera_T_world"), py::arg("K"),
          py::arg("camera_centre"), py::arg("H"), py::arg("W"), py::arg("near_thresh"), py::arg("far_thresh"),
          py::arg("cull_mask_padding"), py::arg("mh_dist"), py::arg("depth_base"), py::arg("with_tiles") = false,
          py::arg("mode") = 0, py::arg("filter3d") = py::none(), py::arg("lens") = GSR_LENS_PINHOLE,
          py::arg("lens_consts") = py::none(),
          py::arg("rolling_shutter") = py::none(), py::arg("readout") = GSR_READOUT_TOP_TO_BOTTOM);
    m.def("fused_bin", &fused_bin, "pair emission + radix sort + tile ranges");
    m.def("fused_render_forward", &fused_render_forward,
          "tile renderer forward (with depth_key: also the depth and alpha maps; with weight_sum / weight_max / "
          "pixel_count: also accumulates the per-gaussian blend-weight statistics, skipped when the last element of "
          "pair_total exceeds pair_capacity)",
          py::arg("records"), py::arg("ranges"), py::arg("background"), py::arg("H"), py::arg("W"), py::arg("P"),
          py::arg("record_masks"), py::arg("keys_sorted"), py::arg("ids_sorted"), py::arg("id_bits"),
          py::arg("depth_key"), py::arg("depth_base"), py::arg("depth_bits"), py::arg("weight_sum") = py::none(),
          py::arg("weight_max") = py::none(), py::arg("pixel_count") = py::none(),
          py::arg("pair_total") = py::none(), py::arg("pair_capacity") = 0);
    m.def("fused_render_backward", &fused_render_backward,
          "tile renderer backward -> per-gaussian gradient slab (with grad_depth / grad_alpha: rows incl. z; "
          "mode: MODE_* bits, MODE_ABSGRAD: rows incl. the absolute uv gradients)",
          py::arg("grad_image"), py::arg("N"), py::arg("P"), py::arg("records"), py::arg("ids_sorted"),
          py::arg("ranges"), py::arg("background"), py::arg("n"), py::arg("w"), py::arg("masks"),
          py::arg("keys_sorted"), py::arg("id_bits"), py::arg("grad_depth"), py::arg("grad_alpha"),
          py::arg("depth_key"), py::arg("depth_base"), py::arg("depth_bits"), py::arg("mode") = 0);
    m.def("fused_render_features_forward", &fused_render_features_forward,
          "feature map [H,W,D] blended with the colour's weights (gsr_render_features_forward)");
    m.def("fused_render_features_backward", &fused_render_features_backward,
          "feature backward: grad_features [N, stride], and the geometry part added into the slab");
    m.def("fused_preprocess_backward", &fused_preprocess_backward,
          "fused per-gaussian backward (mode: MODE_* bits; filter3d, lens, lens_consts: the forward's; camera_grads: "
          "0 none, 1 also d loss / d camera_T_world [4,4], 2 also d loss / d (fx, fy, cx, cy) [4] and d loss / d lens "
          "coefficients [n])",
          py::arg("slab"), py::arg("xyz"), py::arg("quaternion"), py::arg("scale"), py::arg("opacity_logit"),
          py::arg("sh_rest"), py::arg("camera_T_world"), py::arg("K"), py::arg("camera_centre"), py::arg("visible"),
          py::arg("out_flat"), py::arg("grad_uv_compact"), py::arg("scan"), py::arg("use_slab_uv"), py::arg("mode"),
          py::arg("filter3d") = py::none(), py::arg("lens") = GSR_LENS_PINHOLE, py::arg("lens_consts") = py::none(),
          py::arg("camera_grads") = 0, py::arg("rolling_shutter") = py::none(),
          py::arg("readout") = GSR_READOUT_TOP_TO_BOTTOM, py::arg("height") = 0, py::arg("width") = 0);
    m.def("batch_preprocess_forward", &batch_preprocess_forward,
          "per-gaussian forward of C views into stacked records / keys / visibility / scans (rasterize_batch; "
          "lens_consts [C,n+1])",
          py::arg("xyz"), py::arg("xyz_camera_frame"), py::arg("quaternion"), py::arg("scale"),
          py::arg("opacity_logit"), py::arg("rgb_dc"), py::arg("sh_rest"), py::arg("camera_T_world"), py::arg("K"),
          py::arg("camera_centre"), py::arg("H"), py::arg("W"), py::arg("near_thresh"), py::arg("far_thresh"),
          py::arg("cull_mask_padding"), py::arg("mh_dist"), py::arg("depth_base"), py::arg("mode"),
          py::arg("filter3d") = py::none(), py::arg("lens") = GSR_LENS_PINHOLE, py::arg("lens_consts") = py::none(),
          py::arg("rolling_shutter") = py::none(), py::arg("readout") = GSR_READOUT_TOP_TO_BOTTOM);
    m.def("batch_render_backward", &batch_render_backward,
          "render backward of C views into one stacked gradient slab [C, N*12]");
    m.def("batch_preprocess_backward", &batch_preprocess_backward,
          "per-gaussian backward of C views in one pass: the gradient summed over the views; the camera gradients "
          "of fused_preprocess_backward per view, [C,4,4], [C,4] and [C,n]",
          py::arg("slab"), py::arg("xyz"), py::arg("quaternion"), py::arg("scale"), py::arg("opacity_logit"),
          py::arg("sh_rest"), py::arg("camera_T_world"), py::arg("K"), py::arg("camera_centre"), py::arg("visible"),
          py::arg("out_flat"), py::arg("grad_uv_compact"), py::arg("scan"), py::arg("use_slab_uv"), py::arg("mode"),
          py::arg("filter3d") = py::none(), py::arg("lens") = GSR_LENS_PINHOLE, py::arg("lens_consts") = py::none(),
          py::arg("camera_grads") = 0, py::arg("rolling_shutter") = py::none(),
          py::arg("readout") = GSR_READOUT_TOP_TO_BOTTOM, py::arg("height") = 0, py::arg("width") = 0);
    m.def("fisheye_theta_max", &fisheye_theta_max, "the fisheye cull limit of 4 coefficients (gsr_fisheye_theta_max)");
    m.def("distortion_r2_max", &distortion_r2_max,
          "the radial fold limit s = r^2 of 5 coefficients k1 k2 p1 p2 k3 (gsr_distortion_r2_max)");
    m.def("filter3d", &filter3d, "Mip-Splatting's 3-D filter size per gaussian from the training cameras (gsr_filter3d)",
          py::arg("xyz"), py::arg("camera_T_world"), py::arg("K"), py::arg("width"), py::arg("height"),
          py::arg("near"), py::arg("margin"), py::arg("variance"));
    m.attr("MODE_DEPTH_ALPHA") = GSR_MODE_DEPTH_ALPHA;
    m.attr("MODE_ANTIALIASED") = GSR_MODE_ANTIALIASED;
    m.attr("MODE_ABSGRAD") = GSR_MODE_ABSGRAD;
    m.attr("MODE_FILTER3D") = GSR_MODE_FILTER3D;
    m.attr("LENS_PINHOLE") = GSR_LENS_PINHOLE;
    m.attr("LENS_FISHEYE") = GSR_LENS_FISHEYE;
    m.attr("LENS_DISTORTION") = GSR_LENS_DISTORTION;
    m.attr("READOUT_TOP_TO_BOTTOM") = GSR_READOUT_TOP_TO_BOTTOM;
    m.attr("READOUT_BOTTOM_TO_TOP") = GSR_READOUT_BOTTOM_TO_TOP;
    m.attr("READOUT_LEFT_TO_RIGHT") = GSR_READOUT_LEFT_TO_RIGHT;
    m.attr("READOUT_RIGHT_TO_LEFT") = GSR_READOUT_RIGHT_TO_LEFT;
    m.def("flat_section_ends", &flat_section_ends, "section ends of the flat parameter/gradient layout");
    m.def("adam_step_flat", &adam_step_flat, "Adam on the flat parameter buffer");
    m.def("adam_step_sharded", &adam_step_sharded, "reduce-scatter + Adam + all-gather over peer memory");
    m.def("adam_step_selective", &adam_step_selective,
          "Adam on the flat parameter buffer, only the rows whose visible byte is nonzero (gsr_adam_step_selective)");
    m.def("adam_step_selective_sharded", &adam_step_selective_sharded,
          "reduce-scatter + Adam + all-gather of the rows any rank's view saw (gsr_adam_step_selective_sharded)");
    m.def("densify_accumulate", &densify_accumulate, "per-step densification statistics");
    m.def("densify_apply", &densify_apply, "clone / split / delete applied to the flat parameter + Adam buffers");
    m.def("mcmc_relocation", &mcmc_relocation, "3DGS-MCMC relocation: opacity and scale of N copies (fp64 sum)",
          py::arg("opacity"), py::arg("scale"), py::arg("ratio"), py::arg("n_max"), py::arg("min_opacity"));
    m.def("mcmc_apply", &mcmc_apply, "3DGS-MCMC relocation / growth plan applied to the flat parameter + Adam buffers",
          py::arg("p_in"), py::arg("m_in"), py::arg("v_in"), py::arg("n_in"), py::arg("n_sh_rest"), py::arg("src"),
          py::arg("set_row"), py::arg("new_opacity"), py::arg("new_scale"), py::arg("p_out") = py::none());
    m.def("mcmc_noise", &mcmc_noise, "3DGS-MCMC position noise, in place on the flat parameter buffer",
          py::arg("p"), py::arg("N"), py::arg("n_sh_rest"), py::arg("scaler"), py::arg("k"), py::arg("x0"),
          py::arg("seed"), py::arg("offset"), py::arg("eps_in") = py::none(), py::arg("eps_out") = py::none());
    m.def("camera_centre", &camera_centre, "inverse(camera_T_world)[:3, 3] with torch's bits, one kernel");
    m.def("photometric_loss_forward", &photometric_loss_forward,
          "(1 - ssim_frac) * L1 + ssim_frac * (1 - SSIM) forward -> (loss, L1, SSIM)");
    m.def("photometric_loss_backward", &photometric_loss_backward, "photometric loss backward -> gradient on pred");
    m.def("bilagrid_slice_forward", &bilagrid_slice_forward,
          "bilateral-grid slice: per-pixel affine colour transform from grids[ids[c]] (gsr_bilagrid_slice_forward)",
          py::arg("rgb"), py::arg("grids"), py::arg("ids"));
    m.def("bilagrid_slice_backward", &bilagrid_slice_backward,
          "bilateral-grid slice backward -> (grad_rgb or None, grad_grids or None) (gsr_bilagrid_slice_backward)",
          py::arg("rgb"), py::arg("grids"), py::arg("ids"), py::arg("grad_out"), py::arg("need_rgb"),
          py::arg("need_grids"));
    m.def("bilagrid_tv_forward", &bilagrid_tv_forward, "total variation of the grids, on the device");
    m.def("bilagrid_tv_backward", &bilagrid_tv_backward, "total variation backward -> gradient on the grids");
    m.def("surfel_forward", &surfel_forward, "2-D surfels: per-gaussian forward (gsr_surfel_preprocess_forward)");
    m.def("surfel_render_forward", &surfel_render_forward, "2-D surfels: tile forward (gsr_surfel_render_forward)");
    m.def("surfel_render_backward", &surfel_render_backward, "2-D surfels: tile backward (gsr_surfel_render_backward)");
    m.def("surfel_uv_grad", &surfel_uv_grad, "2-D surfels: uv.grad of the visible gaussians (gsr_surfel_uv_grad)");
    m.def("surfel_backward", &surfel_backward, "2-D surfels: per-gaussian backward (gsr_surfel_preprocess_backward)");
    m.attr("SURFEL_LENS_FISHEYE") = (int)GSR_SURFEL_LENS_FISHEYE;
    m.attr("SURFEL_LENS_DISTORTION") = (int)GSR_SURFEL_LENS_DISTORTION;
    m.def("surfel_rays", &surfel_rays, "2-D surfels through a lens: the ray map [H,W,3] (gsr_surfel_rays)");
    m.def("surfel_lens_forward", &surfel_lens_forward,
          "2-D surfels through a lens: per-gaussian forward (gsr_surfel_lens_preprocess_forward)");
    m.def("surfel_lens_render_forward", &surfel_lens_render_forward,
          "2-D surfels through a lens: tile forward along the ray map (gsr_surfel_lens_render_forward)");
    m.def("surfel_lens_render_backward", &surfel_lens_render_backward,
          "2-D surfels through a lens: tile backward along the ray map (gsr_surfel_lens_render_backward)");
    m.def("surfel_lens_uv_grad", &surfel_lens_uv_grad,
          "2-D surfels through a lens: uv.grad of the visible gaussians (gsr_surfel_lens_uv_grad)");
    m.def("surfel_lens_backward", &surfel_lens_backward,
          "2-D surfels through a lens: per-gaussian backward (gsr_surfel_lens_preprocess_backward)");
    m.def("surfel_features_forward", &surfel_features_forward,
          "2-D surfels: feature map [H,W,D] with the colour's weights (gsr_surfel_render_features_forward)");
    m.def("surfel_features_backward", &surfel_features_backward,
          "2-D surfels: feature backward into the gradient rows -> grad_features "
          "(gsr_surfel_render_features_backward)");
    m.def("surfel_median_forward", &surfel_median_forward,
          "2-D surfels: median depth [H,W,1] and median surfel [H,W] (gsr_surfel_render_median_forward)");
    m.def("surfel_median_backward", &surfel_median_backward,
          "2-D surfels: median backward into the gradient rows (gsr_surfel_render_median_backward)");
    m.def("version", &version, "library version string");
    m.def("contribution_mask_words",
          [](int64_t P, int64_t H, int64_t W) { return (int64_t)gsr_contribution_mask_words(P, (int)H, (int)W); },
          "32-bit words of the contribution masks of P pairs over an H x W image");
}
