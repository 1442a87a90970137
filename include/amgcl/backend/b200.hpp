#ifndef AMGCL_BACKEND_B200_HPP
#define AMGCL_BACKEND_B200_HPP

/**
 * \file   amgcl/backend/b200.hpp
 * \brief  H100-native solve-phase backend for AMGCL (drop-in for backend::cuda).
 *
 * Usage is identical to the reference CUDA backend
 * (tutorial/1.poisson3Db/poisson3Db_cuda.cu:51-87):
 *
 * \code
 *   typedef amgcl::backend::b200<double> Backend;
 *   typedef amgcl::make_solver<
 *       amgcl::amg<Backend, amgcl::coarsening::smoothed_aggregation,
 *                  amgcl::relaxation::damped_jacobi>,   // or spai0
 *       amgcl::solver::cg<Backend>                      // or bicgstab
 *       > Solver;
 *   Backend::params bprm;                 // default: library context on the current device
 *   Solver solve(std::tie(n, ptr, col, val), prm, bprm);
 *   auto f = Backend::copy_vector(rhs, bprm);
 *   auto x = Backend::create_vector(n, bprm);
 *   std::tie(iters, error) = solve(*f, *x);
 * \endcode
 *
 * The header owns no numerical code: every primitive forwards to the C ABI of
 * libamgcl_b200.so (include/amgcl_b200.h), whose kernels are hand-written
 * sm_90a CUDA.  It implements the concept amgcl/backend/cuda.hpp:472-807
 * satisfies: a backend struct plus partial specialisations of the *_impl
 * customisation points of amgcl/backend/interface.hpp:191-249.  In addition
 * relaxation::damped_jacobi and relaxation::spai0 are specialised for this
 * backend so a smoother sweep is ONE fused pass over A instead of
 * residual + vmul (damped_jacobi.hpp:108-109, spai0.hpp:91-92), and solver::cg /
 * solver::bicgstab are specialised so an iteration's vector updates and inner
 * products are fused passes with device-resident scalars (cg.hpp:180-198,
 * bicgstab.hpp:198-236; C ABI section "Krylov steps").
 */

#include <iostream>
#include <memory>
#include <string>
#include <vector>
#include <type_traits>

#include <amgcl/util.hpp>
#include <amgcl/backend/builtin.hpp>
#include <amgcl/backend/interface.hpp>
#include <amgcl/relaxation/damped_jacobi.hpp>
#include <amgcl/relaxation/spai0.hpp>
#include <amgcl/solver/cg.hpp>
#include <amgcl/solver/bicgstab.hpp>

#include <amgcl_b200.h>

namespace amgcl {
namespace backend {

namespace detail {
/// Turns a non-zero C ABI status into the reference's error convention
/// (precondition() -> std::runtime_error, util.hpp:89-99; cf. AMGCL_CALL_CUDA,
/// cuda.hpp:91-108).
inline void b200_check(int rc, const char *what) {
    if (rc != B200_OK) {
        std::string msg = std::string("b200 backend: ") + what + " failed (" +
            std::to_string(rc) + "): " + b200_last_error();
        precondition(false, msg);
    }
}
#define AMGCL_CALL_B200(call) ::amgcl::backend::detail::b200_check(call, #call)

inline b200_ctx_t b200_default_ctx() {
    b200_ctx_t ctx = 0;
    AMGCL_CALL_B200(b200_ctx_default(&ctx));
    return ctx;
}
} // namespace detail

/// Parameters of the b200 backend: the library context (device + stream).
/// Plays the role of cuda<>::params::cusparse_handle (cuda.hpp:490-507).
struct b200_params {
    b200_ctx_t ctx;
    b200_params(b200_ctx_t ctx = 0) : ctx(ctx) {}
    b200_ctx_t context() const { return ctx ? ctx : detail::b200_default_ctx(); }
};

namespace detail {
// element-type dispatch onto the typed C entry points
inline int b200_vec_new(b200_ctx_t c, size_t n, b200_vec_t *h, double*) { return b200_vec_create(c, n, h); }
inline int b200_vec_new(b200_ctx_t c, size_t n, b200_vec_t *h, float*)  { return b200_vec_create_f32(c, n, h); }
inline int b200_vec_put(b200_vec_t h, const double *p, size_t n) { return b200_vec_upload(h, p, n); }
inline int b200_vec_put(b200_vec_t h, const float  *p, size_t n) { return b200_vec_upload_f32(h, p, n); }
inline int b200_vec_get(b200_vec_t h, double *p, size_t n) { return b200_vec_download(h, p, n); }
inline int b200_vec_get(b200_vec_t h, float  *p, size_t n) { return b200_vec_download_f32(h, p, n); }
template <class T> struct b200_is_real : std::integral_constant<bool,
    std::is_same<T, double>::value || std::is_same<T, float>::value> {};
} // namespace detail

/// Device vector (replaces thrust::device_vector<real>, cuda.hpp:483).
template <typename real>
class b200_vector {
    static_assert(detail::b200_is_real<real>::value, "b200 vectors are FP64 or FP32");
    public:
        typedef real value_type;

        b200_vector() : ctx(0), h(0), n(0) {}

        b200_vector(size_t n, const b200_params &prm = b200_params())
            : ctx(prm.context()), h(0), n(n)
        {
            AMGCL_CALL_B200(detail::b200_vec_new(ctx, n, &h, (real*)0));
        }

        b200_vector(const real *host, size_t n, const b200_params &prm = b200_params())
            : ctx(prm.context()), h(0), n(n)
        {
            AMGCL_CALL_B200(detail::b200_vec_new(ctx, n, &h, (real*)0));
            AMGCL_CALL_B200(detail::b200_vec_put(h, host, n));
        }

        /// From a host container (std::vector / numa_vector of the same element type).
        template <class Vector>
        explicit b200_vector(const Vector &host, const b200_params &prm = b200_params(),
                typename std::enable_if<is_builtin_vector<Vector>::value, int>::type = 0)
            : ctx(prm.context()), h(0), n(host.size())
        {
            AMGCL_CALL_B200(detail::b200_vec_new(ctx, n, &h, (real*)0));
            AMGCL_CALL_B200(detail::b200_vec_put(h, host.data(), n));
        }

        b200_vector(const b200_vector&) = delete;
        b200_vector& operator=(const b200_vector&) = delete;

        b200_vector(b200_vector &&o) : ctx(o.ctx), h(o.h), n(o.n) { o.h = 0; o.n = 0; }

        ~b200_vector() { if (h) b200_vec_destroy(h); }

        size_t size() const { return n; }
        size_t bytes() const { return n * sizeof(real); }
        b200_vec_t handle() const { return h; }
        b200_ctx_t context() const { return ctx; }

        /// Copy to a host container (resized by the caller).
        void download(real *host) const { AMGCL_CALL_B200(detail::b200_vec_get(h, host, n)); }
        void upload(const real *host)   { AMGCL_CALL_B200(detail::b200_vec_put(h, host, n)); }
        /// Multi-GPU: only the rows this rank owns, into their place in the full-size host array.
        void download_local(double *host) const { AMGCL_CALL_B200(b200_vec_download_local(h, host, n)); }

    private:
        b200_ctx_t ctx;
        b200_vec_t h;
        size_t     n;
};

/// Device CSR matrix (replaces cuda_matrix<real>, cuda.hpp:219-333).
template <typename real>
class b200_matrix {
    static_assert(detail::b200_is_real<real>::value, "b200 matrices are FP64 or FP32");
    public:
        typedef real value_type;

        template <class Col, class Ptr>
        b200_matrix(const crs<real, Col, Ptr> &A, const b200_params &prm)
            : ctx(prm.context()), h(0), nrows(A.nrows), ncols(A.ncols), nnz(A.nnz)
        {
            create(A.nrows, A.ncols, A.ptr, A.col, A.val);
        }

        b200_matrix(const b200_matrix&) = delete;
        b200_matrix& operator=(const b200_matrix&) = delete;

        ~b200_matrix() { if (h) b200_csr_destroy(h); }

        size_t rows()     const { return nrows; }
        size_t cols()     const { return ncols; }
        size_t nonzeros() const { return nnz;   }
        size_t bytes()    const { size_t b = 0; b200_csr_bytes(h, &b); return b; }
        b200_csr_t handle()  const { return h; }
        b200_ctx_t context() const { return ctx; }

    private:
        b200_ctx_t ctx;
        b200_csr_t h;
        size_t nrows, ncols, nnz;

        void create(size_t n, size_t m, const int64_t *ptr, const int64_t *col, const double *val) {
            AMGCL_CALL_B200(b200_csr_create_i64(ctx, n, m, ptr, col, val, &h));
        }
        void create(size_t n, size_t m, const int32_t *ptr, const int32_t *col, const double *val) {
            AMGCL_CALL_B200(b200_csr_create_i32(ctx, n, m, ptr, col, val, &h));
        }
        void create(size_t n, size_t m, const int64_t *ptr, const int64_t *col, const float *val) {
            AMGCL_CALL_B200(b200_csr_create_i64_f32(ctx, n, m, ptr, col, val, &h));
        }
        void create(size_t n, size_t m, const int32_t *ptr, const int32_t *col, const float *val) {
            AMGCL_CALL_B200(b200_csr_create_i32_f32(ctx, n, m, ptr, col, val, &h));
        }
        // long / long long differ from int64_t on some ABIs: same width, reinterpret
        template <class I>
        typename std::enable_if<
            sizeof(I) == 8 && !std::is_same<I, int64_t>::value, void>::type
        create(size_t n, size_t m, const I *ptr, const I *col, const real *val) {
            create(n, m, reinterpret_cast<const int64_t*>(ptr),
                    reinterpret_cast<const int64_t*>(col), val);
        }
};

} // namespace backend

namespace solver {

/// Coarsest-level direct solver that stays on the device (replaces
/// solver::cuda_skyline_lu, cuda.hpp:61-84, which round-trips through the host
/// every cycle): dense inverse formed once, applied as a GEMV.
template <typename real>
class b200_dense_inverse {
    public:
        typedef real value_type;

        template <class Col, class Ptr>
        b200_dense_inverse(const backend::crs<real, Col, Ptr> &A, const backend::b200_params &prm)
            : ctx(prm.context()), h(0), n(A.nrows)
        {
            create(A.ptr, A.col, A.val);
        }

        b200_dense_inverse(const b200_dense_inverse&) = delete;
        b200_dense_inverse& operator=(const b200_dense_inverse&) = delete;
        ~b200_dense_inverse() { if (h) b200_coarse_destroy(h); }

        /// Same threshold as solver::skyline_lu (skyline_lu.hpp:93-95), so the
        /// hierarchy has exactly the levels the builtin backend would build.
        static size_t coarse_enough() { return 3000; }

        /// amg::cycle is a template over the vector types it is handed, so this call is
        /// instantiated for the outer solver's vectors as well (single-level hierarchies).
        template <typename V1, typename V2>
        void operator()(const backend::b200_vector<V1> &rhs, backend::b200_vector<V2> &x) const {
            AMGCL_CALL_B200(b200_coarse_solve(ctx, h, rhs.handle(), x.handle()));
        }

        size_t bytes() const { size_t b = 0; b200_coarse_bytes(h, &b); return b; }

    private:
        b200_ctx_t    ctx;
        b200_coarse_t h;
        size_t        n;

        void create(const int64_t *ptr, const int64_t *col, const double *val) {
            AMGCL_CALL_B200(b200_coarse_create_i64(ctx, n, ptr, col, val, &h));
        }
        void create(const int32_t *ptr, const int32_t *col, const double *val) {
            AMGCL_CALL_B200(b200_coarse_create_i32(ctx, n, ptr, col, val, &h));
        }
        void create(const int64_t *ptr, const int64_t *col, const float *val) {
            AMGCL_CALL_B200(b200_coarse_create_i64_f32(ctx, n, ptr, col, val, &h));
        }
        void create(const int32_t *ptr, const int32_t *col, const float *val) {
            AMGCL_CALL_B200(b200_coarse_create_i32_f32(ctx, n, ptr, col, val, &h));
        }
        template <class I>
        typename std::enable_if<
            sizeof(I) == 8 && !std::is_same<I, int64_t>::value, void>::type
        create(const I *ptr, const I *col, const real *val) {
            create(reinterpret_cast<const int64_t*>(ptr), reinterpret_cast<const int64_t*>(col), val);
        }
};

} // namespace solver

namespace backend {

/// H100 backend.
/**
 * Hand-written sm_90a kernels for every solve-phase primitive; the hierarchy
 * is built on the host by AMGCL's own coarsening and uploaded once.
 *
 * \param real        Value type (double).
 * \param ColumnType  Host column index type used during setup (ptrdiff_t as in
 *                    backend::cuda, cuda.hpp:480-481; int halves setup memory).
 */
template <
    typename real,
    typename ColumnType  = ptrdiff_t,
    typename PointerType = ColumnType,
    class DirectSolver   = solver::b200_dense_inverse<real>
    >
struct b200 {
    static_assert(detail::b200_is_real<real>::value,
            "Unsupported value type for b200 backend (double, or float for the hierarchy of a "
            "mixed-precision solver)");

    typedef real        value_type;
    typedef ColumnType  col_type;
    typedef PointerType ptr_type;

    typedef b200_matrix<real> matrix;
    typedef b200_vector<real> vector;
    typedef b200_vector<real> matrix_diagonal;
    typedef DirectSolver      direct_solver;

    struct provides_row_iterator : std::false_type {};

    typedef b200_params params;

    static std::string name() { return "b200"; }

    typedef typename builtin<real, col_type, ptr_type>::matrix host_matrix;

    /// Copy matrix from builtin backend (deep copy; cf. cuda.hpp:512-518).
    static std::shared_ptr<matrix>
    copy_matrix(std::shared_ptr<host_matrix> A, const params &prm)
    {
        return std::make_shared<matrix>(*A, prm);
    }

    /// Copy vector from builtin backend (cf. cuda.hpp:521-533).
    static std::shared_ptr<vector>
    copy_vector(const numa_vector<real> &x, const params &prm)
    {
        return std::make_shared<vector>(x.data(), x.size(), prm);
    }

    static std::shared_ptr<vector>
    copy_vector(const std::vector<real> &x, const params &prm)
    {
        return std::make_shared<vector>(x.data(), x.size(), prm);
    }

    static std::shared_ptr<vector>
    copy_vector(std::shared_ptr< numa_vector<real> > x, const params &prm)
    {
        return copy_vector(*x, prm);
    }

    /// Create vector of the specified size (zero filled; cf. cuda.hpp:536-540).
    static std::shared_ptr<vector>
    create_vector(size_t size, const params &prm)
    {
        return std::make_shared<vector>(size, prm);
    }

    /// Create direct solver for coarse level (cf. cuda.hpp:543-547).
    static std::shared_ptr<direct_solver>
    create_solver(std::shared_ptr<host_matrix> A, const params &prm)
    {
        return std::make_shared<direct_solver>(*A, prm);
    }

    /// dst[k] = src[I[k]] (cuda.hpp:548-564).
    struct gather {
        gather(size_t src_size, const std::vector<ptrdiff_t> &I, const params &prm)
            : idx(0), n(I.size())
        {
            std::vector<int64_t> I64(I.begin(), I.end());
            AMGCL_CALL_B200(b200_index_create_i64(prm.context(), I64.data(), n, src_size, &idx));
            ctx = prm.context();
        }
        gather(const gather&) = delete;
        gather& operator=(const gather&) = delete;
        ~gather() { if (idx) b200_index_destroy(idx); }

        void operator()(const vector &src, vector &dst) const {
            AMGCL_CALL_B200(b200_gather(ctx, idx, src.handle(), dst.handle()));
        }
        void operator()(const vector &vec, std::vector<value_type> &vals) const {
            AMGCL_CALL_B200(b200_gather_host(ctx, idx, vec.handle(), vals.data()));
        }

        b200_ctx_t ctx;
        b200_index_t idx;
        size_t n;
    };

    /// dst[I[k]] = src[k] (cuda.hpp:566-577).
    struct scatter {
        scatter(size_t size, const std::vector<ptrdiff_t> &I, const params &prm)
            : idx(0)
        {
            std::vector<int64_t> I64(I.begin(), I.end());
            AMGCL_CALL_B200(b200_index_create_i64(prm.context(), I64.data(), I.size(), size, &idx));
            ctx = prm.context();
        }
        scatter(const scatter&) = delete;
        scatter& operator=(const scatter&) = delete;
        ~scatter() { if (idx) b200_index_destroy(idx); }

        void operator()(const vector &src, vector &dst) const {
            AMGCL_CALL_B200(b200_scatter(ctx, idx, src.handle(), dst.handle()));
        }

        b200_ctx_t ctx;
        b200_index_t idx;
    };
};

/// An FP64 Krylov solver may drive an FP32 hierarchy (mixed precision, as
/// builtin<double> / builtin<float> allow: builtin.hpp:1014-1015,
/// tutorial/1.poisson3Db/poisson3Db.cpp:45-51).
template <typename V1, typename V2, typename C, typename P, class DS1, class DS2>
struct backends_compatible< b200<V1, C, P, DS1>, b200<V2, C, P, DS2> > : std::true_type {};

//---------------------------------------------------------------------------
// Backend interface implementation.  The C ABI dispatches on the element types of
// the handles, so every customisation point is a thin template over them.
//---------------------------------------------------------------------------
template <typename V>
struct bytes_impl< b200_vector<V> > {
    static size_t get(const b200_vector<V> &v) { return v.bytes(); }
};

template <typename Alpha, typename Beta, typename VM, typename V1, typename V2>
struct spmv_impl<Alpha, b200_matrix<VM>, b200_vector<V1>, Beta, b200_vector<V2> >
{
    static void apply(Alpha alpha, const b200_matrix<VM> &A, const b200_vector<V1> &x,
            Beta beta, b200_vector<V2> &y)
    {
        AMGCL_CALL_B200(b200_spmv(A.context(), static_cast<double>(alpha), A.handle(),
                    x.handle(), static_cast<double>(beta), y.handle()));
    }
};

template <typename VM, typename V1, typename V2, typename V3>
struct residual_impl<b200_matrix<VM>, b200_vector<V1>, b200_vector<V2>, b200_vector<V3> >
{
    static void apply(const b200_vector<V1> &rhs, const b200_matrix<VM> &A,
            const b200_vector<V2> &x, b200_vector<V3> &r)
    {
        AMGCL_CALL_B200(b200_residual(A.context(), rhs.handle(), A.handle(), x.handle(), r.handle()));
    }
};

template <typename V>
struct clear_impl< b200_vector<V> >
{
    static void apply(b200_vector<V> &x) {
        AMGCL_CALL_B200(b200_clear(x.context(), x.handle()));
    }
};

template <typename V1, typename V2>
struct copy_impl<b200_vector<V1>, b200_vector<V2> >
{
    static void apply(const b200_vector<V1> &x, b200_vector<V2> &y) {
        AMGCL_CALL_B200(b200_copy(x.context(), x.handle(), y.handle()));
    }
};

/// host -> device
template <class HostVec, typename V>
struct copy_impl<HostVec, b200_vector<V>,
    typename std::enable_if<is_builtin_vector<HostVec>::value>::type >
{
    static void apply(const HostVec &x, b200_vector<V> &y) {
        precondition(x.size() == y.size(), "b200 copy: size mismatch");
        y.upload(x.data());
    }
};

/// device -> host
template <typename V, class HostVec>
struct copy_impl<b200_vector<V>, HostVec,
    typename std::enable_if<is_builtin_vector<HostVec>::value>::type >
{
    static void apply(const b200_vector<V> &x, HostVec &y) {
        precondition(x.size() == y.size(), "b200 copy: size mismatch");
        x.download(y.data());
    }
};

template <typename V>
struct inner_product_impl<b200_vector<V>, b200_vector<V> >
{
    static V get(const b200_vector<V> &x, const b200_vector<V> &y) {
        double r = 0;
        AMGCL_CALL_B200(b200_dot(x.context(), x.handle(), y.handle(), &r));
        return static_cast<V>(r);
    }
};

template <typename A, typename B, typename V1, typename V2>
struct axpby_impl<A, b200_vector<V1>, B, b200_vector<V2> >
{
    static void apply(A a, const b200_vector<V1> &x, B b, b200_vector<V2> &y) {
        AMGCL_CALL_B200(b200_axpby(x.context(), static_cast<double>(a), x.handle(),
                    static_cast<double>(b), y.handle()));
    }
};

template <typename A, typename B, typename C, typename V1, typename V2, typename V3>
struct axpbypcz_impl<A, b200_vector<V1>, B, b200_vector<V2>, C, b200_vector<V3> >
{
    static void apply(A a, const b200_vector<V1> &x, B b, const b200_vector<V2> &y,
            C c, b200_vector<V3> &z)
    {
        AMGCL_CALL_B200(b200_axpbypcz(x.context(), static_cast<double>(a), x.handle(),
                    static_cast<double>(b), y.handle(), static_cast<double>(c), z.handle()));
    }
};

template <typename A, typename B, typename V1, typename V2, typename V3>
struct vmul_impl<A, b200_vector<V1>, b200_vector<V2>, B, b200_vector<V3> >
{
    static void apply(A a, const b200_vector<V1> &x, const b200_vector<V2> &y,
            B b, b200_vector<V3> &z)
    {
        AMGCL_CALL_B200(b200_vmul(x.context(), static_cast<double>(a), x.handle(), y.handle(),
                    static_cast<double>(b), z.handle()));
    }
};

} // namespace backend

//---------------------------------------------------------------------------
// Fused smoothers: same public API as the primary templates, one pass over A.
//---------------------------------------------------------------------------
namespace relaxation {

/// damped_jacobi for the b200 backend (primary: relaxation/damped_jacobi.hpp:54-138)
template <typename real, typename C, typename P, class DS>
struct damped_jacobi< backend::b200<real, C, P, DS> > {
    typedef backend::b200<real, C, P, DS>              Backend;
    typedef typename Backend::value_type               value_type;
    typedef typename math::scalar_of<value_type>::type scalar_type;

    /// Relaxation parameters (identical to the primary template's).
    struct params {
        scalar_type damping;
        params(scalar_type damping = 0.72) : damping(damping) {}

#ifndef AMGCL_NO_BOOST
        params(const boost::property_tree::ptree &p)
            : AMGCL_PARAMS_IMPORT_VALUE(p, damping)
        {
            check_params(p, {"damping"});
        }
        void get(boost::property_tree::ptree &p, const std::string &path) const {
            AMGCL_PARAMS_EXPORT_VALUE(p, path, damping);
        }
#endif
    } prm;

    std::shared_ptr<typename Backend::matrix_diagonal> dia;

    template <class Matrix>
    damped_jacobi(const Matrix &A, const params &prm,
            const typename Backend::params &backend_prm)
        : prm(prm), dia( Backend::copy_vector( diagonal(A, true), backend_prm ) )
    { }

    // x <- x + damping * D^-1 (rhs - A x), fused.  rhs / x may be FP64 vectors of the outer
    // solver while A, D^-1 and tmp are this (FP32) hierarchy's: mixed precision, finest level.
    template <typename VR, typename VX, typename VT>
    void apply_pre(const typename Backend::matrix &A, const backend::b200_vector<VR> &rhs,
            backend::b200_vector<VX> &x, backend::b200_vector<VT> &tmp) const
    {
        AMGCL_CALL_B200(b200_relax(A.context(), A.handle(), rhs.handle(), x.handle(),
                    tmp.handle(), dia->handle(), prm.damping));
    }

    template <typename VR, typename VX, typename VT>
    void apply_post(const typename Backend::matrix &A, const backend::b200_vector<VR> &rhs,
            backend::b200_vector<VX> &x, backend::b200_vector<VT> &tmp) const
    {
        apply_pre(A, rhs, x, tmp);
    }

    template <class Matrix, class VectorRHS, class VectorX>
    void apply(const Matrix&, const VectorRHS &rhs, VectorX &x) const
    {
        backend::vmul(math::identity<scalar_type>(), *dia, rhs, math::zero<scalar_type>(), x);
    }

    size_t bytes() const { return backend::bytes(*dia); }
};

/// spai0 for the b200 backend (primary: relaxation/spai0.hpp:50-117)
template <typename real, typename C, typename P, class DS>
struct spai0< backend::b200<real, C, P, DS> > {
    typedef backend::b200<real, C, P, DS>              Backend;
    typedef typename Backend::value_type               value_type;
    typedef typename Backend::matrix_diagonal          matrix_diagonal;
    typedef typename math::scalar_of<value_type>::type scalar_type;
    typedef amgcl::detail::empty_params params;

    /// SPAI-0 weights M_i = a_ii / sum_j a_ij^2 (same quantity the primary
    /// template computes at spai0.hpp:60-82), evaluated here straight off the
    /// raw CRS arrays of the host build matrix and uploaded once.
    template <class HostCol, class HostPtr>
    spai0(const backend::crs<value_type, HostCol, HostPtr> &A, const params &,
            const typename Backend::params &backend_prm)
    {
        const ptrdiff_t n = static_cast<ptrdiff_t>(A.nrows);
        std::vector<value_type> w(A.nrows);

#pragma omp parallel for
        for(ptrdiff_t row = 0; row < n; ++row) {
            scalar_type sum_sq = 0;
            value_type  on_diag = 0;
            for(HostPtr e = A.ptr[row], stop = A.ptr[row + 1]; e < stop; ++e) {
                const value_type a_ij = A.val[e];
                sum_sq += a_ij * a_ij;
                if (static_cast<ptrdiff_t>(A.col[e]) == row) on_diag += a_ij;
            }
            w[row] = (scalar_type(1) / sum_sq) * on_diag;
        }

        M = Backend::copy_vector(w, backend_prm);
    }

    // x <- x + M (rhs - A x), fused (vector element types as for damped_jacobi above)
    template <typename VR, typename VX, typename VT>
    void apply_pre(const typename Backend::matrix &A, const backend::b200_vector<VR> &rhs,
            backend::b200_vector<VX> &x, backend::b200_vector<VT> &tmp) const
    {
        AMGCL_CALL_B200(b200_relax(A.context(), A.handle(), rhs.handle(), x.handle(),
                    tmp.handle(), M->handle(), 1.0));
    }

    template <typename VR, typename VX, typename VT>
    void apply_post(const typename Backend::matrix &A, const backend::b200_vector<VR> &rhs,
            backend::b200_vector<VX> &x, backend::b200_vector<VT> &tmp) const
    {
        apply_pre(A, rhs, x, tmp);
    }

    template <class Matrix, class VectorRHS, class VectorX>
    void apply(const Matrix&, const VectorRHS &rhs, VectorX &x) const
    {
        backend::vmul(math::identity<scalar_type>(), *M, rhs, math::zero<scalar_type>(), x);
    }

    size_t bytes() const { return backend::bytes(*M); }

    std::shared_ptr<matrix_diagonal> M;
};

} // namespace relaxation

//---------------------------------------------------------------------------
// Krylov solvers: same public API as the primary templates, fused iteration body.
//---------------------------------------------------------------------------
namespace backend {

/// The same backend under a distinct type: selects the PRIMARY templates of solver::cg /
/// solver::bicgstab (the reference's call sequence on the b200 primitives).  The
/// specialisations below delegate to it for everything they do not fuse (left
/// preconditioning, a user-supplied system matrix of another type, option "fused_krylov" = 0).
template <typename real, typename C = ptrdiff_t, typename P = C,
          class DS = solver::b200_dense_inverse<real> >
struct b200_generic : b200<real, C, P, DS> {};

} // namespace backend

namespace solver {

namespace detail {
/// Owns the C-ABI workspace (device-resident scalars of one solver instance).
struct b200_krylov_handle {
    b200_ctx_t ctx;
    b200_krylov_t K;
    b200_krylov_handle(const backend::b200_params &bprm, size_t n) : ctx(bprm.context()), K(0) {
        int64_t fused = 1;
        b200_ctx_get_option(ctx, "fused_krylov", &fused);
        if (fused && b200_krylov_create(ctx, n, &K) != B200_OK) K = 0;   // -> generic path
    }
    ~b200_krylov_handle() { if (K) b200_krylov_destroy(K); }
    b200_krylov_handle(const b200_krylov_handle&) = delete;
    b200_krylov_handle& operator=(const b200_krylov_handle&) = delete;
    /// Fused steps are used unless the option was switched off after construction.
    bool active() const {
        if (!K) return false;
        int64_t fused = 1;
        b200_ctx_get_option(ctx, "fused_krylov", &fused);
        return fused != 0;
    }
};
} // namespace detail

/// Conjugate Gradient on the b200 backend (primary: solver/cg.hpp:62-263).
/**
 * Same parameters, same results (iteration count, residual) as the primary template; per
 * iteration it issues P.apply + two C-ABI steps (b200_cg_direction, b200_cg_step) and one
 * host synchronisation instead of 7 primitives and 3 synchronisations.
 */
template <typename C, typename P, class DS>
class cg< backend::b200<double, C, P, DS>, detail::default_inner_product > {
    public:
        typedef backend::b200<double, C, P, DS> Backend;
        typedef Backend backend_type;
        typedef typename Backend::vector     vector;
        typedef typename Backend::value_type value_type;
        typedef typename Backend::params     backend_params;
        typedef double scalar_type;
        typedef double coef_type;

        typedef cg< backend::b200_generic<double, C, P, DS>, detail::default_inner_product > generic_solver;
        /// Solver parameters: the primary template's (cg.hpp:80-124).
        typedef typename generic_solver::params params;

        cg(size_t n, const params &prm = params(),
           const backend_params &bprm = backend_params(),
           const detail::default_inner_product& = detail::default_inner_product())
            : prm(prm), n(n), bprm(bprm), kh(bprm, n),
              r(Backend::create_vector(n, bprm)), s(Backend::create_vector(n, bprm)),
              p(Backend::create_vector(n, bprm)), q(Backend::create_vector(n, bprm))
        { }

        /// Fused path: the system matrix and the vectors live on this backend.
        template <class VM, class Precond>
        std::tuple<size_t, scalar_type> operator()(
                const backend::b200_matrix<VM> &A, const Precond &Prec,
                const backend::b200_vector<double> &rhs, backend::b200_vector<double> &x) const
        {
            if (!kh.active()) return fallback()(A, Prec, rhs, x);

            ios_saver ss(std::cout);

            scalar_type norm_rhs = sqrt(fabs(backend::inner_product(rhs, rhs)));
            if (norm_rhs < amgcl::detail::eps<scalar_type>(1)) {
                if (prm.ns_search) {
                    norm_rhs = math::identity<scalar_type>();
                } else {
                    backend::clear(x);
                    return std::make_tuple(size_t(0), norm_rhs);
                }
            }
            scalar_type eps = std::max(prm.tol * norm_rhs, prm.abstol);

            double rr = 0;
            AMGCL_CALL_B200(b200_krylov_residual(kh.K, rhs.handle(), A.handle(), x.handle(), r->handle(), &rr));
            scalar_type res_norm = sqrt(fabs(rr));

            size_t iter = 0;
            for(; iter < prm.maxiter && res_norm > eps; ++iter) {
                Prec.apply(*r, *s);
                // rho = <r,s> (left behind by the last smoother sweep); p = s + (rho/rho_prev) p
                AMGCL_CALL_B200(b200_cg_direction(kh.K, r->handle(), s->handle(), p->handle()));
                // q = A p; alpha = rho/<q,p>; x += alpha p; r -= alpha q; <r,r>
                AMGCL_CALL_B200(b200_cg_step(kh.K, A.handle(), p->handle(), q->handle(),
                            x.handle(), r->handle(), &rr));
                res_norm = sqrt(fabs(rr));
                if (prm.verbose && iter % 5 == 0)
                    std::cout << iter << "\t" << std::scientific << res_norm / norm_rhs << std::endl;
            }
            return std::make_tuple(iter, res_norm / norm_rhs);
        }

        /// Anything else (foreign matrix / vector types): the reference's sequence.
        template <class Matrix, class Precond, class Vec1, class Vec2>
        std::tuple<size_t, scalar_type> operator()(
                const Matrix &A, const Precond &Prec, const Vec1 &rhs, Vec2 &&x) const
        {
            return fallback()(A, Prec, rhs, x);
        }

        template <class Precond, class Vec1, class Vec2>
        std::tuple<size_t, scalar_type> operator()(const Precond &Prec, const Vec1 &rhs, Vec2 &&x) const {
            return (*this)(Prec.system_matrix(), Prec, rhs, x);
        }

        size_t bytes() const {
            return backend::bytes(*r) + backend::bytes(*s) + backend::bytes(*p) + backend::bytes(*q)
                + (generic ? generic->bytes() : 0);
        }

        friend std::ostream& operator<<(std::ostream &os, const cg &s) {
            return os
                << "Type:             CG"
                << "\nUnknowns:         " << s.n
                << "\nMemory footprint: " << human_readable_memory(s.bytes())
                << std::endl;
        }

    public:
        params prm;

    private:
        size_t n;
        backend_params bprm;
        detail::b200_krylov_handle kh;
        std::shared_ptr<vector> r, s, p, q;
        mutable std::unique_ptr<generic_solver> generic;

        generic_solver& fallback() const {
            if (!generic) generic.reset(new generic_solver(n, prm, bprm));
            generic->prm = prm;
            return *generic;
        }
};

/// BiCGStab on the b200 backend (primary: solver/bicgstab.hpp:52-316).
/**
 * Right preconditioning (the default) runs as P.apply + b200_bicg_direction / _step_s /
 * _step_r with two host synchronisations per iteration (its two convergence tests) instead
 * of six; left preconditioning delegates to the primary template.
 */
template <typename C, typename P, class DS>
class bicgstab< backend::b200<double, C, P, DS>, detail::default_inner_product > {
    public:
        typedef backend::b200<double, C, P, DS> Backend;
        typedef Backend backend_type;
        typedef typename Backend::vector     vector;
        typedef typename Backend::value_type value_type;
        typedef typename Backend::params     backend_params;
        typedef double scalar_type;
        typedef double coef_type;

        typedef bicgstab< backend::b200_generic<double, C, P, DS>, detail::default_inner_product > generic_solver;
        /// Solver parameters: the primary template's (bicgstab.hpp:72-124).
        typedef typename generic_solver::params params;

        bicgstab(size_t n, const params &prm = params(),
                 const backend_params &bprm = backend_params(),
                 const detail::default_inner_product& = detail::default_inner_product())
            : prm(prm), n(n), bprm(bprm), kh(bprm, n),
              r (Backend::create_vector(n, bprm)), p (Backend::create_vector(n, bprm)),
              v (Backend::create_vector(n, bprm)), s (Backend::create_vector(n, bprm)),
              t (Backend::create_vector(n, bprm)), rh(Backend::create_vector(n, bprm)),
              T (Backend::create_vector(n, bprm))
        { }

        template <class VM, class Precond>
        std::tuple<size_t, scalar_type> operator()(
                const backend::b200_matrix<VM> &A, const Precond &Prec,
                const backend::b200_vector<double> &rhs, backend::b200_vector<double> &x) const
        {
            namespace side = preconditioner::side;
            if (!kh.active() || prm.pside != side::right) return fallback()(A, Prec, rhs, x);

            ios_saver ss(std::cout);

            scalar_type norm_rhs = sqrt(fabs(backend::inner_product(rhs, rhs)));
            if (norm_rhs < amgcl::detail::eps<scalar_type>(1)) {
                if (prm.ns_search) {
                    norm_rhs = math::identity<scalar_type>();
                } else {
                    backend::clear(x);
                    return std::make_tuple(size_t(0), norm_rhs);
                }
            }

            double rr = 0, ssq = 0, rho = 0, omega = 0;
            AMGCL_CALL_B200(b200_krylov_residual(kh.K, rhs.handle(), A.handle(), x.handle(), r->handle(), &rr));
            AMGCL_CALL_B200(b200_bicg_start(kh.K, r->handle(), rh->handle()));

            scalar_type eps = std::max(norm_rhs * prm.tol, prm.abstol);
            scalar_type res = prm.check_after ? 2 * eps : sqrt(fabs(rr));

            coef_type rho_prev = 0;
            size_t iter = 0;
            for(bool first = true; res > eps && iter < prm.maxiter; ++iter) {
                if (first) first = false;
                else precondition(!math::is_zero(rho_prev), "Zero rho in BiCGStab");

                // p = r + beta (p - omega v); p = r on the first iteration
                AMGCL_CALL_B200(b200_bicg_direction(kh.K, r->handle(), v->handle(), p->handle()));
                Prec.apply(*p, *T);
                // v = A T; alpha = rho/<rh,v>; x += alpha T; s = r - alpha v; <s,s>
                AMGCL_CALL_B200(b200_bicg_step_s(kh.K, A.handle(), rh->handle(), T->handle(), v->handle(),
                            r->handle(), s->handle(), x.handle(), &ssq, &rho));
                rho_prev = rho;

                if ((res = sqrt(fabs(ssq))) > eps) {
                    Prec.apply(*s, *T);
                    // t = A T; omega = <t,s>/<t,t>; x += omega T; r = s - omega t; <r,r>; next rho
                    AMGCL_CALL_B200(b200_bicg_step_r(kh.K, A.handle(), rh->handle(), T->handle(), t->handle(),
                                s->handle(), r->handle(), x.handle(), &rr, &omega));
                    precondition(!math::is_zero(omega), "Zero omega in BiCGStab");
                    res = sqrt(fabs(rr));
                }

                if (prm.verbose && iter % 5 == 0)
                    std::cout << iter << "\t" << std::scientific << res / norm_rhs << std::endl;
            }
            return std::make_tuple(iter, res / norm_rhs);
        }

        template <class Matrix, class Precond, class Vec1, class Vec2>
        std::tuple<size_t, scalar_type> operator()(
                const Matrix &A, const Precond &Prec, const Vec1 &rhs, Vec2 &&x) const
        {
            return fallback()(A, Prec, rhs, x);
        }

        template <class Precond, class Vec1, class Vec2>
        std::tuple<size_t, scalar_type> operator()(const Precond &Prec, const Vec1 &rhs, Vec2 &&x) const {
            return (*this)(Prec.system_matrix(), Prec, rhs, x);
        }

        size_t bytes() const {
            return backend::bytes(*r) + backend::bytes(*p) + backend::bytes(*v) + backend::bytes(*s)
                + backend::bytes(*t) + backend::bytes(*rh) + backend::bytes(*T)
                + (generic ? generic->bytes() : 0);
        }

        friend std::ostream& operator<<(std::ostream &os, const bicgstab &s) {
            return os
                << "Type:             BiCGStab"
                << "\nUnknowns:         " << s.n
                << "\nMemory footprint: " << human_readable_memory(s.bytes())
                << std::endl;
        }

    public:
        params prm;

    private:
        size_t n;
        backend_params bprm;
        detail::b200_krylov_handle kh;
        std::shared_ptr<vector> r, p, v, s, t, rh, T;
        mutable std::unique_ptr<generic_solver> generic;

        generic_solver& fallback() const {
            if (!generic) generic.reset(new generic_solver(n, prm, bprm));
            generic->prm = prm;
            return *generic;
        }
};

} // namespace solver

//---------------------------------------------------------------------------
// Whole-cycle CUDA graph (opt-in wrapper, SURVEY section 8(f) rank 1)
//---------------------------------------------------------------------------
namespace preconditioner {

/// Wraps a preconditioner that runs on backend::b200 (normally amgcl::amg<...>) and replays
/// its apply() as ONE CUDA graph launch:
///
/// \code
///   typedef amgcl::amg<Backend, coarsening::smoothed_aggregation, relaxation::damped_jacobi> AMG;
///   typedef amgcl::make_solver<amgcl::preconditioner::b200_cycle_graph<AMG>,
///                              amgcl::solver::cg<Backend>> Solver;
/// \endcode
///
/// amg::apply (amg.hpp:289-297) issues clear + cycle (amg.hpp:514-553) as a fixed sequence of
/// backend calls with no host-visible result, so the sequence is recorded once per distinct
/// (rhs, x, vector-state) combination through b200_graph_begin / _end and replayed afterwards.
/// The first application runs directly (it also performs one-off allocations); applications
/// the C library declines to replay (state mismatch, profiling, multi-GPU context) fall back
/// to recording another graph or to the direct path, so results are always those of P.apply.
template <class Precond>
class b200_cycle_graph {
    public:
        typedef typename Precond::backend_type backend_type;
        typedef typename backend_type::matrix  matrix;
        typedef typename backend_type::value_type value_type;
        typedef typename backend_type::col_type col_type;
        typedef typename backend_type::ptr_type ptr_type;
        typedef typename backend::builtin<value_type, col_type, ptr_type>::matrix build_matrix;
        typedef typename Precond::params params;
        typedef typename backend_type::params backend_params;

        template <class Matrix>
        b200_cycle_graph(const Matrix &M, const params &prm = params(),
                const backend_params &bprm = backend_params())
            : P(M, prm, bprm), ctx(bprm.context()), applied(0), enabled(true) {}

        b200_cycle_graph(std::shared_ptr<build_matrix> M, const params &prm = params(),
                const backend_params &bprm = backend_params())
            : P(M, prm, bprm), ctx(bprm.context()), applied(0), enabled(true) {}

        ~b200_cycle_graph() {
            for (size_t i = 0; i < graphs.size(); ++i) b200_graph_destroy(graphs[i].g);
        }

        template <class Vec1, class Vec2>
        void apply(const Vec1 &rhs, Vec2 &&x) const {
            if (!enabled) { P.apply(rhs, x); return; }

            // a graph replays the recorded calls on the recorded handles: only graphs recorded
            // for this very (rhs, x) pair are candidates (BiCGStab and GMRES apply the
            // preconditioner to several pairs)
            const b200_vec_t hr = rhs.handle(), hx = x.handle();
            for (size_t i = 0; i < graphs.size(); ++i) {
                if (graphs[i].rhs != hr || graphs[i].x != hx) continue;
                int launched = 0;
                AMGCL_CALL_B200(b200_graph_launch(ctx, graphs[i].g, &launched));
                if (launched) return;
            }

            // the first application always runs directly: lazily allocated scratch must exist
            // before anything is recorded
            if (applied++ == 0) { P.apply(rhs, x); return; }
            drop_stale();
            if (graphs.size() >= max_graphs) { P.apply(rhs, x); return; }

            int recording = 0;
            AMGCL_CALL_B200(b200_graph_begin(ctx, &recording));
            if (!recording) { P.apply(rhs, x); return; }
            try {
                P.apply(rhs, x);
            } catch (...) {
                // something in this preconditioner cannot be recorded (e.g. an inner product in
                // a nested Krylov solver): restore the state and use the direct path from now on
                b200_graph_abort(ctx);
                enabled = false;
                P.apply(rhs, x);
                return;
            }
            b200_graph_t g = 0;
            if (b200_graph_end(ctx, &g) != B200_OK) {     // state was rolled back
                enabled = false;
                P.apply(rhs, x);
                return;
            }
            entry e = {hr, hx, g};
            graphs.push_back(e);
        }

        const Precond& base() const { return P; }
        Precond&       base()       { return P; }

        std::shared_ptr<matrix> system_matrix_ptr() const { return P.system_matrix_ptr(); }
        const matrix& system_matrix() const { return P.system_matrix(); }
        size_t bytes() const { return backend::bytes(P); }

        /// Recorded graphs, kernels per replay of the first one, replays over all of them.
        void graph_stats(size_t &ngraphs, size_t &kernels, size_t &replays) const {
            ngraphs = graphs.size(); kernels = 0; replays = 0;
            for (size_t i = 0; i < graphs.size(); ++i) {
                int64_t k = 0, n = 0, r = 0; int stale = 0;
                b200_graph_info(graphs[i].g, &k, &n, &r, &stale);
                if (i == 0) kernels = (size_t)k;
                replays += (size_t)r;
            }
        }

    private:
        static const size_t max_graphs = 64;

        void drop_stale() const {
            size_t keep = 0;
            for (size_t i = 0; i < graphs.size(); ++i) {
                int stale = 0;
                b200_graph_info(graphs[i].g, 0, 0, 0, &stale);
                if (stale) b200_graph_destroy(graphs[i].g);
                else graphs[keep++] = graphs[i];
            }
            graphs.resize(keep);
        }

        Precond P;
        b200_ctx_t ctx;
        mutable size_t applied;
        mutable bool enabled;
        struct entry { b200_vec_t rhs, x; b200_graph_t g; };
        mutable std::vector<entry> graphs;

        friend std::ostream& operator<<(std::ostream &os, const b200_cycle_graph &p) {
            return os << p.P;
        }
};

} // namespace preconditioner
} // namespace amgcl

#endif
