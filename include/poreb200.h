/* poreb200.h -- C ABI of libporeb200.so: H100 (sm_90a) MPFA / MPSA / Biot
 * interaction-region assembly and CSR SpMV behind PorePy's discretization API.
 *
 * Plain pointers and sizes only; no torch / numpy types.  The Python host side
 * (porepy_b200/_lib.py) binds these with ctypes.  Every entry point names the
 * reference interface (pmgbergen/porepy v1.11.0) it replaces.
 *
 * Ownership: the caller owns every host buffer passed in or out.  The library
 * owns the device memory inside a plan handle.  Handles are not thread-safe;
 * use one host thread (one process under torchrun) per GPU.
 *
 * Return codes (all functions returning int):
 *   PB_OK 0
 *   PB_EINVAL 1     invalid argument
 *   PB_ESINGULAR 2  singular local system; the node id is in pb_last_error_node()
 *                   -> Python raises ValueError("Error in inversion of local linear
 *                   systems"), parity with numerics/linalg/matrix_operations.py:1487-1490
 *   PB_ECELLTYPE 3  a cell vertex does not have exactly nd faces of the cell meeting
 *                   in it (pyramids ...) -> AssertionError, parity with
 *                   numerics/fv/_fvutils.py:735 and mpsa.py:1569
 *   PB_ECUDA 4      CUDA runtime error (text in pb_last_error())
 *   PB_ENOTIMPL 5   feature of the reference not covered by this build
 */
#ifndef POREB200_H
#define POREB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB_OK 0
#define PB_EINVAL 1
#define PB_ESINGULAR 2
#define PB_ECELLTYPE 3
#define PB_ECUDA 4
#define PB_ENOTIMPL 5

/* boundary-condition codes per face (scalar) / per component and face (vector) */
#define PB_BC_INTERIOR 0
#define PB_BC_DIR 1
#define PB_BC_NEU 2
#define PB_BC_ROB 3

/* sparsity patterns shared by the output matrices (scalar "base" patterns) */
#define PB_PAT_FACE_CELL 0  /* nf x nc : flux, bound_pressure_cell; x nd columns: vector_source;
                               nd x nd blocks: stress, bound_displacement_cell; ...          */
#define PB_PAT_FACE_BFACE 1 /* nf x nf : bound_flux, bound_pressure_face, bound_stress, ...   */
#define PB_PAT_CELL_CELL 2  /* nc x nc : mpsa_consistency, displacement_divergence (x nd)     */
#define PB_PAT_CELL_BFACE 3 /* nc x nf : boundary_displacement_divergence (x nd)              */

typedef struct pb_plan pb_plan; /* opaque */
struct pb_csr;                  /* opaque device CSR matrix, see "CSR SpMV" below */

/* ---- library state ------------------------------------------------------------------ */
const char *pb_last_error(void);
int64_t pb_last_error_node(void);
/* number of CUDA devices visible, or -1 (no driver / no device).  Never falls back to CPU. */
int pb_device_count(void);
/* device allocations that missed the pooled blocks: {cudaMalloc calls, seconds, cudaFree calls, seconds} since load */
void pb_alloc_stats(double *out4);
/* cudaSetDevice for this process (one process per GPU). */
int pb_set_device(int device);
/* kernels launched by this library since load (bench.py's gpu_launches evidence). */
int64_t pb_launch_count(void);

/* Return the device blocks cached by the library's size-keyed pool (see csrc/plan.hpp: DevPool) to the driver. */
void pb_device_pool_trim(void);

/* FP64 peak of this device, measured by a dependency-free register loop: kind 0 = DMMA mma.sync.m8n8k4.f64,
 * 1 = scalar DFMA, 2 / 3 / 4 = DMMA mma.sync.m16n8k4 / m16n8k8 / m16n8k16 .f64.  TFLOP/s, best of 5 launches
 * (roofline denominator). */
int pb_fp64_peak(int kind, double *tflops);

/* Page-locked host buffers for the CSR value arrays the *_download calls fill (full PCIe rate;
 * pageable NumPy buffers go through the driver's staging copies).  The caller frees them. */
int pb_host_alloc(uint64_t bytes, void **out);
void pb_host_free(void *p);

/* ---- plan: sub-cell topology + output patterns --------------------------------------- */
/* Replaces _fvutils.SubcellTopology.__init__ (numerics/fv/_fvutils.py:51-172), the
 * sub-face pairing (:163-172, pair_over_subfaces :183-216), cell_node_blocks /
 * sub_cell_index of scalar_tensor_vector_prod (:697-762), Mpfa._block_diagonal_structure
 * (numerics/fv/mpfa.py:1357-1412) and the implicit sparsity patterns of the scipy SpGEMM
 * chains (mpfa.py:1080-1147, mpsa.py:735-781, biot.py:776-866).
 *   nd: grid dimension (2 or 3).  cell_faces: nf x nc CSC with +-1 data (pp.Grid.cell_faces),
 *   face_nodes: nn x nf CSC (pp.Grid.face_nodes).  Row indices need not be sorted. */
int pb_plan_create(int nd, int64_t nc, int64_t nf, int64_t nn,
                   const int32_t *cf_indptr, const int32_t *cf_indices, const int8_t *cf_data,
                   const int32_t *fn_indptr, const int32_t *fn_indices,
                   pb_plan **out);
void pb_plan_destroy(pb_plan *p);

/* sizes: sub-cells, unique sub-faces, sub-half-faces, largest local system (sub-faces at a node) */
int pb_plan_sizes(const pb_plan *p, int64_t *num_subcells, int64_t *num_subfaces,
                  int64_t *num_subhalffaces, int32_t *max_subfaces_per_node,
                  int32_t *max_subcells_per_node);
/* Nodes per local-solver class of the classes last built for kind 0 (MPFA, at pb_mpfa_upload) or 1 (MPSA / Biot, at
 * pb_mpsa_upload): counts[2 * cfg + g] for solver configuration cfg (0-6, see csrc/plan.hpp) with the local matrix
 * in shared memory (g = 0) or in a global-memory workspace (g = 1).  counts has 14 entries.  Read-only. */
int pb_plan_class_counts(const pb_plan *p, int kind, int64_t *counts);
/* Shards: cell e of this plan is cell cells[e] of a larger (global) grid of n_source_cells cells.  The cell tensors of
 * the following pb_mpfa_upload / pb_mpsa_upload (permeability, stiffness, coupling tensors) are then the GLOBAL arrays
 * ((3,3,n_source), (9,9,n_source)) and are restricted on the device; NULL removes the map. */
int pb_plan_set_cell_map(pb_plan *p, const int64_t *cells, int64_t n_source_cells);
/* Restrict the assembly to the interaction regions of the flagged nodes (mask: nn bytes, NULL = all nodes).
 * Used by the multi-GPU path: a shard assembles the regions of its OWN nodes only; the outer nodes of its halo
 * layer are incomplete there and their rows are discarded anyway (reference: the overlap removal of
 * numerics/fv/mpfa.py:301-304).  Rows of faces with an inactive node are incomplete. */
int pb_plan_set_active_nodes(pb_plan *p, const uint8_t *mask);
/* base pattern `which` (PB_PAT_*): nrows and nnz; then copy indptr (nrows+1) / indices (nnz). */
int pb_plan_pattern_size(const pb_plan *p, int which, int64_t *nrows, int64_t *nnz);
int pb_plan_pattern_get(const pb_plan *p, int which, int32_t *indptr, int32_t *indices);

/* Block expansion of base pattern `which` into br x bc blocks (row r*br+i, column c*bc+j), built
 * on the device and copied to the caller's buffers: indptr (nrows*br+1), indices (br*bc*nnz).
 * The value of block entry (i,j) of base entry q of base row r lives at
 * br*bc*indptr[r] + i*bc*len_r + (q-indptr[r])*bc + j -- the layout the kernels scatter into.
 * PB_ENOTIMPL when br*bc*nnz does not fit int32. */
int pb_plan_pattern_expanded(pb_plan *p, int which, int br, int bc, int32_t *indptr, int32_t *indices);

/* Geometry the path reads from pp.Grid (grids/grid.py:32): nodes (3 x nn), face_normals /
 * face_centers (3 x nf), cell_centers (3 x nc) row-major as numpy stores them; face_areas (nf),
 * cell_volumes (nc).  Copied to the device inside the plan. */
int pb_plan_set_geometry(pb_plan *p, const double *nodes, const double *face_normals,
                         const double *face_centers, const double *face_areas,
                         const double *cell_centers, const double *cell_volumes);

/* ---- MPFA ----------------------------------------------------------------------------- */
/* Replaces Mpfa._flux_discretization (numerics/fv/mpfa.py:592-1156) incl. _create_bound_rhs
 * (:1414-1578), _discretize_vector_source (:1158-1307), reconstruct_presssure (:1628-1690),
 * _fvutils.scalar_tensor_vector_prod / compute_dist_face_cell / ExcludeBoundaries and
 * matrix_operations.invert_diagonal_blocks (numerics/linalg/matrix_operations.py:1175).
 *   perm:  SecondOrderTensor.values, (3,3,nc) row-major (params/tensor.py:157)
 *   bc:    nf codes PB_BC_* (internal/fracture faces already mapped to PB_BC_NEU, mpfa.py:1452)
 *   robin_weight: nf doubles (may be NULL when no Robin face)
 *   eta:   continuity point parameter (mpfa_eta)
 * Outputs: CSR `data` arrays on the base patterns; NULL = not wanted.
 *   flux, bound_pressure_cell: nnz(FACE_CELL);  vector_source, bound_pressure_vector_source:
 *   nd*nnz(FACE_CELL) (entry p expands to p*nd+j);  bound_flux, bound_pressure_face:
 *   nnz(FACE_BFACE). */
int pb_mpfa_upload(pb_plan *p, const double *perm, const uint8_t *bc, const double *robin_weight,
                   double eta);
/* device-resident assembly of the uploaded problem; want_* select outputs. ms = device time. */
int pb_mpfa_assemble(pb_plan *p, int want_flux_terms, int want_trace_terms,
                     int want_vector_source, float *ms);
int pb_mpfa_download(pb_plan *p, double *flux, double *bound_flux, double *bound_pressure_cell,
                     double *bound_pressure_face, double *vector_source,
                     double *bound_pressure_vector_source);

/* ---- device-resident results ----------------------------------------------------------------------------
 * The value array of one output matrix can be MOVED out of the plan as a pb_values handle: the matrix then
 * stays in HBM until the caller asks for it (the Python layer stores scipy-compatible matrices whose data /
 * indices are downloaded on first touch), and the plan allocates a fresh array at its next assemble.  Keys: */
#define PB_OUT_FLUX 0
#define PB_OUT_BOUND_FLUX 1
#define PB_OUT_BOUND_PRESSURE_CELL 2
#define PB_OUT_BOUND_PRESSURE_FACE 3
#define PB_OUT_VECTOR_SOURCE 4
#define PB_OUT_BOUND_PRESSURE_VECTOR_SOURCE 5
#define PB_OUT_STRESS 6
#define PB_OUT_BOUND_STRESS 7
#define PB_OUT_BOUND_DISPLACEMENT_CELL 8
#define PB_OUT_BOUND_DISPLACEMENT_FACE 9
/* Biot, coupling tensor q: PB_OUT_BIOT + 5*q + {0 displacement_divergence, 1 boundary_displacement_divergence,
 * 2 scalar_gradient, 3 mpsa_consistency, 4 bound_displacement_pressure} */
#define PB_OUT_BIOT 10
typedef struct pb_values pb_values; /* opaque: device array of doubles */
int pb_plan_take_output(pb_plan *p, int key, pb_values **out);
int64_t pb_values_size(const pb_values *v);
int pb_values_download(pb_values *v, double *host); /* D2H of all values (page-locked host buffer: full PCIe rate) */
int pb_values_checksum(pb_values *v, double *sum, double *sum_of_squares); /* device reduction, 16-byte read */
void pb_values_destroy(pb_values *v);

/* One output matrix as a device CSR handle (block-expanded pattern + a copy of the values): operand of the
 * device-side AD chain below.  which / br / bc as in pb_plan_pattern_expanded. */
int pb_plan_output_csr(pb_plan *p, const pb_values *v, int which, int br, int bc, struct pb_csr **out);

/* Device-side system of the flow problem, replacing the host scipy products of
 * FVElliptic.assemble_matrix_rhs (numerics/fv/fv_elliptic.py:67-112):
 *   A = div @ flux  on the CELL_CELL pattern, kept in HBM as a device CSR handle, no D2H of the matrices;
 *   b = -div @ (bound_flux @ bc_values) [- div @ (vector_source @ v)]   (host vectors in/out).
 * The discretization matrices are given by their value handles (NULL = the plan's last assembled arrays). */
int pb_mpfa_system(pb_plan *p, const pb_values *flux, struct pb_csr **out);
int pb_mpfa_rhs(pb_plan *p, const pb_values *bound_flux, const pb_values *vector_source_discr,
                const double *bc_values, const double *vector_source, double *rhs);
/* Same for mechanics (Mpsa.assemble_matrix_rhs, numerics/fv/mpsa.py:486-529): A = div_nd @ stress
 * (nd x nd blocks on the CELL_CELL pattern, row c*nd+i, column k*nd+j) as a device CSR and
 * b = -div_nd @ (bound_stress @ bc_values) + source  (bc_values: nf*nd face-major, source: nc*nd). */
int pb_mpsa_system(pb_plan *p, const pb_values *stress, struct pb_csr **out);
int pb_mpsa_rhs(pb_plan *p, const pb_values *bound_stress, const double *bc_values, const double *source,
                double *rhs);

/* ---- MPSA / Biot ------------------------------------------------------------------------ */
/* Replaces Mpsa._stress_discretization (numerics/fv/mpsa.py:531-781),
 * _create_inverse_gradient_matrix (:784-930), _tensor_vector_prod (:1520-1675),
 * _eliminate_ncasym (:1932-2000), _create_bound_rhs (:984-1185), _reconstruct_displacement
 * (:1187-1275) and, with n_alpha > 0, Biot._local_discretization (numerics/fv/biot.py:714-878).
 *   stiffness: FourthOrderTensor.values (9,9,nc) row-major (params/tensor.py:348)
 *   bc:        (nd, nf) codes PB_BC_* row-major (BoundaryConditionVectorial.is_dir/is_neu/is_rob)
 *   robin_weight: (nd,nd,nf) row-major or NULL
 *   alpha:     n_alpha coupling tensors, each (3,3,nc) row-major (scalar_vector_mappings)
 * Outputs: data arrays; block expansion of the base patterns, row f*nd+i, column c*nd+j:
 *   stress, bound_displacement_cell: nd*nd*nnz(FACE_CELL); bound_stress,
 *   bound_displacement_face: nd*nd*nnz(FACE_BFACE); per coupling tensor:
 *   displacement_divergence nd*nnz(CELL_CELL), boundary_displacement_divergence
 *   nd*nnz(CELL_BFACE), scalar_gradient / bound_displacement_pressure nd*nnz(FACE_CELL),
 *   mpsa_consistency nnz(CELL_CELL). */
int pb_mpsa_upload(pb_plan *p, const double *stiffness, const uint8_t *bc,
                   const double *robin_weight, double eta, int n_alpha, const double *alpha);
/* Boundary conditions in a rotated basis (BoundaryConditionVectorial.basis, params/bc.py; applied to the
 * boundary equations by ExcludeBoundaries, numerics/fv/_fvutils.py:765-945): basis (nd,nd,nf) row-major,
 * NULL = identity.  Call after pb_mpsa_upload (which resets it to the identity). */
int pb_mpsa_set_basis(pb_plan *p, const double *basis);
int pb_mpsa_assemble(pb_plan *p, float *ms);
int pb_mpsa_download(pb_plan *p, double *stress, double *bound_stress,
                     double *bound_displacement_cell, double *bound_displacement_face);
int pb_biot_download(pb_plan *p, int which_alpha, double *displacement_divergence,
                     double *boundary_displacement_divergence, double *scalar_gradient,
                     double *mpsa_consistency, double *bound_displacement_pressure);

/* ---- CSR SpMV ---------------------------------------------------------------------------- */
/* Replaces the scipy `M @ val` of AdArray.__rmatmul__ (numerics/ad/forward_mode.py:565-595)
 * and the residual chain of EquationSystem.assemble(evaluate_jacobian=False)
 * (numerics/ad/equation_system.py:1579-1713).  y = A x (+ beta*y).  */
typedef struct pb_csr pb_csr; /* opaque: device-resident CSR matrix */

/* ---- two-point flux approximation and first-order upwinding (one thread per face) ----------------
 * A pb_facegrid is the face-indexed device view of a grid of ANY dimension (1-D lines and 2-D planes
 * embedded in 3-D included): the face -> cell table built from cell_faces (nf x nc CSC, +-1 data) and
 * face_normals / face_centers (3 x nf), cell_centers (3 x nc), row-major.  No interaction-region plan.
 * Replaces Tpfa.discretize (numerics/fv/tpfa.py:40-280), incl. the 1-D delegation of MPFA / MPSA
 * (mpfa.py:690-712, mpsa.py:666-697), and Upwind.discretize (numerics/fv/upwind.py:150-300).
 * bc_bits (nf): bits 0-1 = PB_BC_* effective code, bit 2 = raw is_dir, bit 3 = raw is_neu.
 * pb_tpfa: fc_indptr = row pointer of cell_faces in CSR-by-face form with ascending columns; value
 * arrays in that pattern (flux, bound_pressure_cell: nnz; vector sources: nnz*vdim, entry-major) and
 * the two diagonals (nf).  pb_upwind: upstream cell per face (-1 = face removed from the matrix) and the
 * diagonals of the Neumann / Dirichlet-inflow boundary matrices.  Host pointers; outputs may be NULL
 * for pb_tpfa. */
typedef struct pb_facegrid pb_facegrid; /* opaque */
int pb_facegrid_create(int64_t nc, int64_t nf, const int32_t *cf_indptr, const int32_t *cf_indices,
                       const int8_t *cf_data, const double *face_normals, const double *face_centers,
                       const double *cell_centers, pb_facegrid **out);
void pb_facegrid_destroy(pb_facegrid *g);
int pb_tpfa(pb_facegrid *g, const double *permeability, const uint8_t *bc_bits, const int32_t *fc_indptr,
            int vdim, double *flux, double *bound_pressure_cell, double *vector_source,
            double *bound_pressure_vector_source, double *bound_flux_diag,
            double *bound_pressure_face_diag);
/* Differentiable TPFA (csrc/tpfa_diff.cuh; reference numerics/fv/tpfa.py:281-760 DifferentiableTpfa and the AD
 * expression of models/constitutive_laws.py:1544-1583): k = 9 * nc doubles, the 3 x 3 tensor of cell c at k[9c..9c+8]
 * row-major; fc_indptr as for pb_tpfa (half-faces numbered by face, then by cell).  Outputs: half-face
 * transmissibilities t_hf (nhf), face transmissibilities T (nf), dT/dk (nhf * 9: the 9 derivatives with respect to the
 * tensor of the half-face's cell).  Host pointers. */
int pb_tpfa_diff(pb_facegrid *g, const double *k, const int32_t *fc_indptr, double *t_hf, double *T, double *dT_dk);
int pb_upwind(pb_facegrid *g, const double *darcy_flux, const uint8_t *bc_bits, int32_t *upstream_cell,
              double *neumann_diag, double *dirichlet_diag);

/* ---- mixed (dual) discretizations of Darcy flow: MVEM and RT0 (csrc/dual_cell.cuh; reference numerics/vem/mvem.py,
 * numerics/fem/rt0.py) -------------------------------------------------------------------------------------------------
 * A pb_dual holds the topology of a grid of dimension nd (1, 2 or 3): cell_faces (nf x nc CSC, +-1 data, the faces of
 * every cell in ascending order) and face_nodes (nn x nf CSC).  pb_dual_mass_pattern returns the FACE x FACE pattern of
 * the mass matrix (row f: every face sharing a cell with f, ascending), built on the device at the first call and kept
 * on the handle; indptr (nf + 1) / indices (*nnz) may be NULL to query the size.  pb_dual_discretize runs one thread
 * per entry of cell_faces.  Geometry in the grid's own frame, each (3 x n) row-major: nodes, face_normals,
 * face_centers, cell_centers; cell_volumes (nc); perm (3 x 3 x nc) row-major, expressed in the frame; rot (3 x 3)
 * row-major, the frame's axes as rows.  Outputs (host): mass values (*nnz) in the pattern; proj values
 * (3 cf_indptr[nc]): row 3c + a of the (3 nc x nf) flux reconstruction holds the faces of c in cell_faces order, at
 * 3 cf_indptr[c] + a n_c + i.  *bad_cell: the smallest cell failing the MVEM consistency test allclose(G, F D) of
 * mvem.py, or -1.  PB_DUAL_RT0 needs nd + 1 faces in every cell.  mass / proj may be NULL: the values stay on the
 * handle either way (until the next call), for pb_dual_download and pb_dual_system.
 * pb_dual_system assembles the saddle-point system of dual_elliptic.py assemble_matrix_rhs from those values on the
 * device: the (nf + nc) square matrix [[mass, div^T], [div, 0]], div = -cell_faces^T, faces first (row f: the mass row,
 * then the columns nf + c of the face's cells; row nf + c: the cell's faces), with codes (nf, PB_BC_*; internal and
 * interior faces PB_BC_INTERIOR): Neumann rows cleared with *norm = |mass|_inf (device reduction) on the diagonal,
 * 1 / (robin_weight area) added on Robin diagonals; rhs (nf + nc, host) = proj^T vector_source (vector_source: 3 nc or
 * NULL) + the Dirichlet / Robin / Neumann terms of assemble_rhs with the sign of each face's first cell. */
#define PB_DUAL_MVEM 0
#define PB_DUAL_RT0 1
typedef struct pb_dual pb_dual; /* opaque */
int pb_dual_create(int nd, int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_indptr, const int32_t *cf_indices,
                   const int8_t *cf_data, const int32_t *fn_indptr, const int32_t *fn_indices, pb_dual **out);
void pb_dual_destroy(pb_dual *d);
int pb_dual_mass_pattern(pb_dual *d, int64_t *nnz, int32_t *indptr, int32_t *indices);
int pb_dual_discretize(pb_dual *d, int method, const double *nodes, const double *face_normals,
                       const double *face_centers, const double *cell_centers, const double *cell_volumes,
                       const double *perm, const double *rot, double *mass, double *proj, int64_t *bad_cell,
                       float *kernel_ms);
int pb_dual_download(pb_dual *d, double *mass, double *proj);
int pb_dual_system(pb_dual *d, const uint8_t *codes, const double *robin_weight, const double *face_areas,
                   const double *bc_values, const double *vector_source, pb_csr **out, double *rhs, double *norm);

/* Hybridization (csrc/dual_hybrid.cuh): every cell's local saddle system is condensed exactly onto one pressure
 * lambda per face (reference numerics/vem/hybrid.py), one warp per cell; cells of at most 32 faces (PB_ENOTIMPL).
 * pb_dual_hybrid_system returns the nf x nf face matrix in the mass pattern (*out) and its right-hand side (rhs, nf,
 * host); pb_dual_hybrid_recover takes lambda (nf, host) and writes [u; p] (nf + nc, host), each u_f by the face's
 * first cell.  *kernel_ms: the per-cell kernel.  Two modes:
 *   PB_DUAL_HYBRID_VEM: HybridDualVEM.matrix_rhs / compute_up.  Geometry as pb_dual_discretize, with perm as given
 *     (not rotated, as hybrid.py reads it) and aperture (nc) scaling cell volumes and normals; values = [bc_values (nf);
 *     source (nc)]; codes PB_BC_DIR / PB_BC_NEU.  Dirichlet rows are cleared with |H|_inf (before the boundary
 *     conditions) on the diagonal and norm bc_values in rhs, Neumann faces add s bc_values area (s: the sign of the
 *     face's first cell).  *bad_cell: as pb_dual_discretize.
 *   PB_DUAL_HYBRID_SADDLE: the face system of the saddle point of pb_dual_system, from the values and geometry of the
 *     last pb_dual_discretize (geometry pointers and aperture NULL); values = any right-hand side b (nf + nc) of that
 *     system; codes and robin_weight / face_areas as pb_dual_system.  Faces with a given pressure (Dirichlet, and
 *     boundary faces without a condition) get identity rows and zeroed columns, Robin faces add -robin_weight area on
 *     the diagonal, Neumann faces the flux s b_f / |mass|_inf; the face right-hand side b_f enters the local system
 *     of the face's first cell.  [u; p] then solves the saddle-point system with right-hand side b.
 * PB_ESINGULAR: a singular local matrix (named by cell). */
#define PB_DUAL_HYBRID_VEM 0
#define PB_DUAL_HYBRID_SADDLE 1
int pb_dual_hybrid_system(pb_dual *d, int mode, const double *nodes, const double *face_normals,
                          const double *face_centers, const double *cell_centers, const double *cell_volumes,
                          const double *perm, const double *rot, const double *aperture, const uint8_t *codes,
                          const double *robin_weight, const double *face_areas, const double *values, pb_csr **out,
                          double *rhs, int64_t *bad_cell, float *kernel_ms);
int pb_dual_hybrid_recover(pb_dual *d, int mode, const double *nodes, const double *face_normals,
                           const double *face_centers, const double *cell_centers, const double *cell_volumes,
                           const double *perm, const double *rot, const double *aperture, const uint8_t *codes,
                           const double *values, const double *lambda, double *up, float *kernel_ms);

/* ---- two-point stress approximation (csrc/tpsa_face.cuh; reference numerics/fv/tpsa.py:376-1430) ------------------
 * One thread per face writes every value of the 14 TPSA matrices in that face's rows.  nr = nd in 3-D (the rotation
 * is a 3-vector) and nr = 1 in 2-D (a scalar).  Shapes (rows x columns) and the block of one (face, cell) entry or of
 * one face:
 *   PB_TPSA_STRESS                          nd nf x nd nc   kron(., I_nd): nd diagonal values per (face, cell)
 *   PB_TPSA_STRESS_ROTATION                 nd nf x nr nc   nd x nr
 *   PB_TPSA_STRESS_TOTAL_PRESSURE           nd nf x nc      nd x 1
 *   PB_TPSA_ROTATION_DISPLACEMENT           nr nf x nd nc   nr x nd
 *   PB_TPSA_ROTATION_ROTATION               nr nf x nr nc   nr x nr
 *   PB_TPSA_SOLID_MASS_DISPLACEMENT         nf x nd nc      1 x nd
 *   PB_TPSA_SOLID_MASS_TOTAL_PRESSURE       nf x nc         1 x 1
 *   PB_TPSA_BOUND_DISPLACEMENT_CELL         nd nf x nd nc   kron(., I_nd): nd diagonal values per (face, cell)
 *   PB_TPSA_BOUND_DISPLACEMENT_ROTATION_CELL       nd nf x nr nc  nd x nr
 *   PB_TPSA_BOUND_DISPLACEMENT_SOLID_PRESSURE_CELL nd nf x nc     nd x 1
 *   PB_TPSA_BOUND_STRESS                    nd nf x nd nf   kron(., I_nd): nd diagonal values per face
 *   PB_TPSA_BOUND_ROTATION_DISPLACEMENT     nr nf x nd nf   nr x nd per face
 *   PB_TPSA_BOUND_MASS_DISPLACEMENT         nf x nd nf      1 x nd per face
 *   PB_TPSA_BOUND_DISPLACEMENT_FACE         nd nf x nd nf   kron(., I_nd): nd diagonal values per face
 * Cell terms follow the pattern of cell_faces in CSR-by-face form with ascending columns (fc_indptr, as for
 * pb_tpfa), block-expanded: their value arrays are the CSR data of the expanded matrices (row f*br + i holds the
 * blocks of the face's cells one after the other; kron(., I_nd) terms are nd x 1 blocks in column c*nd + i).  Face
 * terms are the br x bc blocks row-major, face after face.
 *   mu:         FourthOrderTensor.mu (nc), finite and > 0
 *   codes:      nd * nf PB_BC_* codes, at f*nd + i (is_dir / is_neu / is_rob raveled in "F" order); PB_BC_INTERIOR
 *               where no flag is set (interior and internal faces)
 *   robin_diag: nd * nf diagonal Robin weights at f*nd + i, or NULL when no component is Robin
 *   face_flags: nf bytes, non-zero for the faces of sd.get_all_boundary_faces(); such a face has exactly one cell
 *   out:        PB_TPSA_NTERMS host pointers, each may be NULL
 *   kernel_ms:  device time of the kernel (may be NULL)
 * The face areas must have been set with pb_facegrid_set_face_areas. */
enum {
    PB_TPSA_STRESS = 0,
    PB_TPSA_STRESS_ROTATION = 1,
    PB_TPSA_STRESS_TOTAL_PRESSURE = 2,
    PB_TPSA_ROTATION_DISPLACEMENT = 3,
    PB_TPSA_ROTATION_ROTATION = 4,
    PB_TPSA_SOLID_MASS_DISPLACEMENT = 5,
    PB_TPSA_SOLID_MASS_TOTAL_PRESSURE = 6,
    PB_TPSA_BOUND_DISPLACEMENT_CELL = 7,
    PB_TPSA_BOUND_DISPLACEMENT_ROTATION_CELL = 8,
    PB_TPSA_BOUND_DISPLACEMENT_SOLID_PRESSURE_CELL = 9,
    PB_TPSA_BOUND_STRESS = 10,
    PB_TPSA_BOUND_ROTATION_DISPLACEMENT = 11,
    PB_TPSA_BOUND_MASS_DISPLACEMENT = 12,
    PB_TPSA_BOUND_DISPLACEMENT_FACE = 13,
    PB_TPSA_NTERMS = 14
};
/* face areas (nf, host pointer) of a pb_facegrid, read by pb_tpsa */
int pb_facegrid_set_face_areas(pb_facegrid *g, const double *face_areas);
int pb_tpsa(pb_facegrid *g, int nd, const double *mu, const uint8_t *codes, const double *robin_diag,
            const uint8_t *face_flags, const int32_t *fc_indptr, double **out, float *kernel_ms);

/* The linear system of the TPSA three-field elasticity model (csrc/tpsa_system.cuh; reference
 * models/momentum_balance.py:82-106, 250-280, 344-368 and models/constitutive_laws.py:3064-3296) on one grid without
 * fractures, assembled on the device:
 *   momentum     -div_nd (S_u u + S_r r + S_p p + B_s g)               - f   = 0
 *   angular      -vol/mu r + div_nr (R_u u + R_r r + B_r g)            - s_r = 0
 *   solid mass   -vol/lambda p + div (M_u u + M_p p + B_m g)           - s_p = 0
 * with the PB_TPSA_* terms above (S_u = STRESS, S_r = STRESS_ROTATION, S_p = STRESS_TOTAL_PRESSURE, R_u =
 * ROTATION_DISPLACEMENT, R_r = ROTATION_ROTATION, M_u = SOLID_MASS_DISPLACEMENT, M_p = SOLID_MASS_TOTAL_PRESSURE, B_s =
 * BOUND_STRESS, B_r = BOUND_ROTATION_DISPLACEMENT, B_m = BOUND_MASS_DISPLACEMENT) and div = cell_faces^T.  Unknowns and
 * equations are numbered cell by cell, [u_c (nd), r_c (nr), p_c]: row / column c*(nd+nr+1) + l, so the diagonal
 * (nd+nr+1)^2 blocks are the cell blocks.  Only the structurally non-zero entries are stored (u-u diagonal, r-p and p-r
 * zero: 37 of 49 entries per block in 3-D, 12 of 16 in 2-D); rows are sorted.
 * pb_tpsa_system: A as a new device CSR.  mu, codes, robin_diag, face_flags as for pb_tpsa; lambda (nc): the first
 * Lame parameter, finite and > 0; cell_volumes (nc).  Host pointers.  The face areas must have been set.  The row
 * pattern is built on the device at the first call for a dimension and kept on the handle; the face values of the
 * last call stay on the handle for pb_tpsa_rhs.  No atomics: two calls give bit-identical values.  stage_ms (may be
 * NULL): device times of the face kernel and of the row gather, 2 floats.
 * pb_tpsa_rhs: b = -R(0) of the system last assembled on g, written to the DEVICE array rhs_dev (nc*(nd+nr+1)).
 * bc_values: nd*nf face-major (the model's combined mechanical boundary operator); body_force (nd*nc), angular_source
 * (nr*nc), mass_source (nc): cell-major host arrays, each may be NULL (zero). */
int pb_tpsa_system(pb_facegrid *g, int nd, const double *mu, const double *lambda, const double *cell_volumes,
                   const uint8_t *codes, const double *robin_diag, const uint8_t *face_flags, struct pb_csr **out,
                   float *stage_ms);
int pb_tpsa_rhs(pb_facegrid *g, const double *bc_values, const double *body_force, const double *angular_source,
                const double *mass_source, double *rhs_dev);

/* The Jacobian of the TPSA poromechanics model (pp.Poromechanics + TpsaPoromechanicsMixin; reference
 * models/poromechanics.py:92-136, 177-213, models/constitutive_laws.py:3299-3374) on one grid without fractures:
 * four fields per cell, [u_c (nd), r_c (nr), p_t_c, p_c], B = nd + nr + 2 (5 in 2-D, 8 in 3-D), row / column c*B + l.
 * The mechanics rows are those of pb_tpsa_system, the solid-mass row extended by -vol alpha/lambda p (its p entry is
 * stored for every face neighbour, 0 off the cell's own block).  The fluid-mass row of c holds the p column of every
 * cell of row c of flux_pattern (div @ flux of the MPFA discretization, nc x nc, sorted rows) and the whole own block.
 * pb_tpsa_poro_system: the matrix with its mechanics rows, fluid rows 0, as a new device CSR.  Arguments as for
 * pb_tpsa_system; alpha (nc, host): the Biot coefficient, finite.  The row pattern is built on the device at the first
 * call for a dimension and flux pattern and kept on the handle.  No atomics: two calls give bit-identical values.
 * pb_tpsa_poro_rhs: -R(0) of the mechanics rows (the right-hand side of pb_tpsa_rhs), 0 in the fluid rows, to the DEVICE
 * array rhs_dev (nc*B).
 * pb_tpsa_poro_fluid_rows: the fluid rows at one Newton step, on `stream`, nothing copied to the host: row c of jf
 * (nc x 2 nc device CSR, columns [p_t | p], the field-ordered Jacobian of the fluid mass balance) into the fixed
 * pattern of a (the matrix of pb_tpsa_poro_system on g), and neg_res_dev[c] (-R of the fluid mass balance, device) into
 * rhs_dev[c*B + B-1].  Entries of jf outside the pattern are counted into *missing_dev (device int, may be NULL). */
int pb_tpsa_poro_system(pb_facegrid *g, int nd, const double *mu, const double *lambda, const double *alpha,
                        const double *cell_volumes, const uint8_t *codes, const double *robin_diag,
                        const uint8_t *face_flags, const struct pb_csr *flux_pattern, struct pb_csr **out,
                        float *stage_ms);
int pb_tpsa_poro_rhs(pb_facegrid *g, const double *bc_values, const double *body_force, const double *angular_source,
                     const double *mass_source, double *rhs_dev);
int pb_tpsa_poro_fluid_rows(pb_facegrid *g, struct pb_csr *a, const struct pb_csr *jf, const double *neg_res_dev,
                            double *rhs_dev, int *missing_dev, uint64_t stream);

/* The Jacobian of the TPSA thermo-poromechanics model (pp.Thermoporomechanics + TpsaPoromechanicsMixin) on one grid
 * without fractures: five fields per cell, [u_c (nd), r_c (nr), p_t_c, p_c, T_c], B = nd + nr + 3 (6 in 2-D, 9 in 3-D).
 * The mechanics rows are those of pb_tpsa_poro_system, with no T column (the reference's TPSA stress has no thermal
 * term).  The mass row and then the energy row of c each hold the whole own block and the p and T columns of every
 * other cell of row c of flux_pattern (the union of the Darcy and Fourier div @ flux patterns, nc x nc, sorted rows).
 * pb_tpsa_thm_system / pb_tpsa_thm_rhs: as pb_tpsa_poro_system / pb_tpsa_poro_rhs, 0 in the mass and energy rows.
 * pb_tpsa_thm_balance_rows: the mass and energy rows at one Newton step, on `stream`: row c (mass) and nc + c (energy)
 * of jf (2 nc x 3 nc device CSR, columns [p_t | p | T]) into the fixed pattern of a, neg_res_dev[c] / [nc + c] into
 * rhs_dev[c*B + B-2] / [c*B + B-1]; entries outside the pattern are counted into *missing_dev (may be NULL). */
int pb_tpsa_thm_system(pb_facegrid *g, int nd, const double *mu, const double *lambda, const double *alpha,
                       const double *cell_volumes, const uint8_t *codes, const double *robin_diag,
                       const uint8_t *face_flags, const struct pb_csr *flux_pattern, struct pb_csr **out,
                       float *stage_ms);
int pb_tpsa_thm_rhs(pb_facegrid *g, const double *bc_values, const double *body_force, const double *angular_source,
                    const double *mass_source, double *rhs_dev);
int pb_tpsa_thm_balance_rows(pb_facegrid *g, struct pb_csr *a, const struct pb_csr *jf, const double *neg_res_dev,
                             double *rhs_dev, int *missing_dev, uint64_t stream);

/* The Jacobian of the TPSA elasticity model with fractures in frictional contact (pp.MomentumBalance +
 * TpsaMomentumBalanceMixin on a fractured medium; reference models/momentum_balance.py:127-183,
 * models/constitutive_laws.py:3064-3248, models/contact_mechanics.py:80-245) on a 2-D or 3-D matrix whose fracture faces
 * are internal Dirichlet faces (one cell each) matched one to one with the mortar cells of the interfaces.  Fracture cells
 * (nk) and mortar cells (nm = 2 nk) are numbered over all fractures / interfaces one after the other.
 *   unknowns   [u_c, r_c, p_c per cell (B = nd+nr+1) | t: nd per fracture cell | u_j: nd per mortar cell]
 *   equations  [the three TPSA balances per cell | interface force balance: nd per mortar cell | normal law: one per
 *               fracture cell | tangential law: nd-1 per fracture cell]
 * The balance rows are those of pb_tpsa_system with the interface displacement on the fracture faces, g + Pi^avg u_j:
 * momentum row i of c gains -s_f B_s[f,i] w_m2p in column u_j(m,i), the angular and solid-mass rows +s_f B_r[f] w_m2p
 * and +s_f B_m[f] w_m2p in the nd columns of u_j(m) (s_f: the sign of c on f).  Force row (m, i) is
 * w_p2m s_f sigma[f,i] + vol_m T_c sign_m sum_j R_k[j,i] t_k,j with the three-field stress
 * sigma = S_u u + S_r r + S_p p + B_s (g + w_m2p u_j).  Each contact row holds the 3 nd columns [t_k | u_j(m1) | u_j(m2)],
 * 0 until pb_tpsa_contact_rows writes them.  Rows are sorted.
 * pb_tpsa_contact_system: the matrix as a new device CSR.  Arguments as for pb_tpsa_system, plus per mortar cell (host
 * arrays of num_mortar): its matrix face, fracture cell, mortar_to_primary_avg and primary_to_mortar_int weights, side
 * sign and volume (times its secondary_to_mortar_int weight); frames: the nd x nd local coordinates of every fracture cell,
 * row-major (the nd-1 tangents, then the normal); characteristic_traction: T_c.  A face with more than one mortar cell,
 * a fracture face without exactly one cell, a fracture cell without exactly two mortar cells or an index out of range
 * is PB_EINVAL.  The row pattern is built on the device at the first call for a dimension and interface topology and
 * kept on the handle; the patterns of pb_tpsa_system / pb_tpsa_poro_system / pb_tpsa_thm_system are not touched.  The
 * face values are shared: like those entry points, a call replaces the face values that pb_tpsa_rhs, pb_tpsa_poro_rhs and
 * pb_tpsa_thm_rhs read (the right-hand sides follow the last system assembled on g).  No
 * atomics: two calls give bit-identical values.  stage_ms (may be NULL): device times of the face kernel and of the
 * row writes, 2 floats.
 * pb_tpsa_contact_rhs: b = -R(0) of the balance and force rows (the right-hand side of pb_tpsa_rhs, and
 * -w_p2m s_f B_s g in the force rows), 0 in the contact rows, to the DEVICE array rhs_dev.  Reads the face values of
 * the last system assembled on g.
 * pb_tpsa_contact_rows: the contact rows at one Newton step, on `stream`, nothing copied to the host: row r of jc
 * (nd nk x nd (nk + nm) device CSR, the Jacobian of the [normal | tangential] laws in the variables [t | u_j]) into the
 * fixed pattern of a at column offset B nc, and neg_res_dev[r] into the entry of rhs_dev of that row.  Entries of jc
 * outside the pattern are counted into *missing_dev (device int, may be NULL). */
int pb_tpsa_contact_system(pb_facegrid *g, int nd, const double *mu, const double *lambda, const double *cell_volumes,
                           const uint8_t *codes, const double *robin_diag, const uint8_t *face_flags,
                           int64_t num_mortar, int64_t num_fracture_cells, const int32_t *mortar_face,
                           const int32_t *mortar_cell, const double *m2p_weight, const double *p2m_weight,
                           const double *mortar_sign, const double *mortar_volume, const double *frames,
                           double characteristic_traction, struct pb_csr **out, float *stage_ms);
int pb_tpsa_contact_rhs(pb_facegrid *g, const double *bc_values, const double *body_force, const double *angular_source,
                        const double *mass_source, double *rhs_dev);
int pb_tpsa_contact_rows(pb_facegrid *g, struct pb_csr *a, const struct pb_csr *jc, const double *neg_res_dev,
                         double *rhs_dev, int *missing_dev, uint64_t stream);

/* Interface upwinding (UpwindCoupling.discretize, numerics/fv/upwind.py:427-528): per mortar cell the sign of the
 * interface flux and the masks "upstream is the higher-dimensional side" / "... the lower-dimensional side".
 * Host pointers, n doubles each. */
int pb_upwind_coupling(int64_t n, const double *interface_flux, double *sign, double *from_primary,
                       double *from_secondary);

/* ---- Grid.compute_geometry for 3-D grids (csrc/geometry.cu; reference grids/grid.py:362-381, 572-778) ---------
 * Face normals (area weighted) / centres / areas and cell centres / volumes of a grid of general polyhedral cells
 * from its topology and nodes: each face is fanned into triangles around the mean of its nodes, each cell into
 * tetrahedra around the mean of its faces' centres.  Host arrays in the reference's layouts: CSC of cell_faces
 * (nf x nc, row indices ascending inside a column, data +-1), CSC of face_nodes (nn x nf, the nodes of a face in loop
 * order), nodes (3, nn) row-major; outputs (3, nf), (3, nf), (nf), (3, nc), (nc).  kernel_ms (may be NULL) = device
 * time of the two kernels.  PB_EINVAL ("Some tetrahedra have negative volume", grid.py:754; cell in
 * pb_last_error_node()) for inverted cells. */
int pb_compute_geometry_3d(int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_indptr, const int32_t *cf_indices,
                           const int8_t *cf_data, const int32_t *fn_indptr, const int32_t *fn_indices,
                           const double *nodes, double *face_normals, double *face_centers, double *face_areas,
                           double *cell_centers, double *cell_volumes, float *kernel_ms);

/* ---- sharding of ONE grid across ranks (csrc/shard.cu; host code) ---------------------------------------------
 * This rank's share of a grid from the GLOBAL topology: replaces the reference's memory-splitting chain
 * _fvutils.subproblems (numerics/fv/_fvutils.py:414-539) -> partition.extract_subgrid (grids/partition.py:540-640)
 * for this path.  cf_* / fn_*: CSC arrays of cell_faces (nf x nc, data +-1) and face_nodes (nn x nf); part: rank of
 * each cell.  Shard cells = every cell with a face holding a node of an own cell (one halo layer), OWN CELLS FIRST
 * (ascending), then the halo; faces / nodes ascending.  pb_shard_sizes: {cells, faces, nodes, own cells, nnz of the
 * local cell_faces, nnz of the local face_nodes}.  pb_shard_fill: local->global maps, per local face the flags
 * "row kept by this rank" / "cut face of the overlap" / "one cell inside the shard", per local node "interaction
 * region assembled by this rank", and the local CSC arrays (any output may be NULL). */
typedef struct pb_shard pb_shard; /* opaque */
int pb_shard_create(int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_indptr, const int32_t *cf_indices,
                    const double *cf_data, const int32_t *fn_indptr, const int32_t *fn_indices,
                    const int64_t *part, int64_t rank, pb_shard **out);
int pb_shard_sizes(const pb_shard *s, int64_t *sizes6);
int pb_shard_fill(const pb_shard *s, int64_t *cells, int64_t *faces, int64_t *nodes, uint8_t *own_face,
                  uint8_t *cut_face, uint8_t *single_face, uint8_t *own_node, int32_t *cf_indptr,
                  int32_t *cf_indices, double *cf_data, int32_t *fn_indptr, int32_t *fn_indices);
void pb_shard_destroy(pb_shard *s);
/* dst[r, j] = src[r, idx[j]]: the (3, n) geometry arrays of a sub-grid (row-major host arrays) */
int pb_gather_columns(const double *src, int64_t nrows, int64_t ncols, const int64_t *idx, int64_t n, double *dst);

/* device-resident CSR matrix */
int pb_csr_create(int64_t nrows, int64_t ncols, int64_t nnz, const int32_t *indptr,
                  const int32_t *indices, const double *data, pb_csr **out);
void pb_csr_destroy(pb_csr *a);
/* Keep the first nrows rows (a row-partitioned system: the rows of a rank's own cells come first). */
int pb_csr_truncate_rows(pb_csr *a, int64_t nrows);
/* lanes per row the SpMV of this matrix runs with (autotuned at creation) */
int pb_csr_lanes_per_row(const pb_csr *a);
/* diagonal (min(nrows, ncols) doubles, host) -- the Jacobi preconditioner of the Krylov solve */
int pb_csr_diagonal(pb_csr *a, double *diag);
/* ---- device-side sparse algebra of the AD Jacobian chain (csrc/sparse_ops.cu) ---------------------------------
 * M @ jac (AdArray.__rmatmul__, numerics/ad/forward_mode.py:565-595), diag(v) @ jac (:613-616), jac + jac,
 * the block concatenation of MergedOperator.parse (numerics/ad/ad_utils.py:597-664) and the vstack of
 * EquationSystem.assemble (numerics/ad/equation_system.py:1695-1713), on matrices that stay in HBM.
 * All results are new handles with sorted rows.  d_dev: DEVICE vector. */
int pb_csr_spgemm(const pb_csr *a, const pb_csr *b, pb_csr **out);                      /* C = A @ B */
int pb_csr_axpby(double alpha, const pb_csr *a, double beta, const pb_csr *b, pb_csr **out); /* C = alpha A + beta B */
int pb_csr_scale_dev(const pb_csr *a, const double *d_dev, int by_cols, pb_csr **out);  /* diag(d) A  |  A diag(d) */
/* nbr x nbc grid of blocks, row-major, NULL = zero block; row_sizes (nbr) / col_sizes (nbc) */
int pb_csr_bmat(int nbr, int nbc, const pb_csr *const *blocks, const int64_t *row_sizes, const int64_t *col_sizes,
                pb_csr **out);
/* sum and sum of squares of the stored values (device reduction) */
int pb_csr_checksum(pb_csr *a, double *sum, double *sum_of_squares);
/* copy a device-resident matrix back (indptr nrows+1, indices nnz, data nnz); sizes via pb_csr_shape */
int pb_csr_shape(const pb_csr *a, int64_t *nrows, int64_t *ncols, int64_t *nnz);
int pb_csr_download(pb_csr *a, int32_t *indptr, int32_t *indices, double *data);
/* host vectors in/out (H2D + kernel + D2H) */
int pb_csr_spmv(pb_csr *a, const double *x, double *y);
/* device pointers (e.g. torch tensors' data_ptr()); stream = cudaStream_t as integer (0 = default) */
int pb_csr_spmv_dev(pb_csr *a, const double *x_dev, double *y_dev, uint64_t stream);
/* y = A x on device pointers with the Krylov dot products in the epilogue: *d1 += (w1, y), *d2 += (w2, y)
 * (w2 NULL: (y, y)); d1 / d2 are device addresses or NULL. */
int pb_csr_spmv_dots_dev(pb_csr *a, const double *x_dev, double *y_dev, const double *w1_dev, double *d1_dev,
                         const double *w2_dev, double *d2_dev, uint64_t stream);

/* ---- fused vector kernels of the Jacobi-BiCGStab (csrc/krylov.cu; SURVEY 8f rank 1, replaces the direct solve of
 * models/solution_strategy.py:830-884).  All pointers are DEVICE pointers; `scal` is the 14-double scalar buffer
 * described in krylov.cu (every scalar of the recurrence stays on the device; the caller all-reduces slices of it
 * between the kernels under torch.distributed and polls it every few iterations); cur = iteration parity. */
int pb_kry_init(int64_t n, const double *b, double *x, double *r, double *rhat, double *p, double *v, double *scal,
                double tol, uint64_t stream);
int pb_kry_seed(double *scal, uint64_t stream);
/* minv / bs: the preconditioner M^-1 -- bs = 1: inverse diagonal (n doubles, Jacobi); bs = 2, 3, 4, 5, 7, 8: inverted
 * bs x bs diagonal blocks, row-major (n/bs blocks; block Jacobi over the unknowns of a cell: the displacement components
 * of the MPSA system (2, 3), [u, r, p] of the TPSA system (4 in 2-D, 7 in 3-D) or [u, r, p_t, p] of the TPSA
 * poromechanics system (5, 8)); NULL: none */
int pb_kry_p(int64_t n, const double *r, double *p, const double *v, const double *minv, double *ph, double *scal,
             int cur, int bs, uint64_t stream);
int pb_kry_s(int64_t n, const double *r, const double *v, const double *minv, double *s, double *sh, double *scal,
             int cur, int bs, uint64_t stream);
/* inverses of the first nblocks bs x bs diagonal blocks of a device CSR, to a DEVICE array (nblocks*bs*bs doubles);
 * bs in {1, 2, 3, 4, 5, 7, 8}.  A singular block is replaced by the inverse of its diagonal (1 where that entry is 0). */
int pb_csr_block_diag_inv_dev(const pb_csr *a, int bs, int64_t nblocks, double *out_dev, uint64_t stream);
int pb_kry_xr(int64_t n, double *x, const double *ph, const double *sh, const double *s, const double *t, double *r,
              const double *rhat, double *scal, int cur, int carry /* 1 on exactly one rank */, uint64_t stream);

/* ---- restarted GMRES(m) with a grouped block-Jacobi preconditioner (csrc/gmres.cu): the device solve of the Newton
 * updates of the fractured contact models.  All pointers except `a` are DEVICE pointers.
 * Groups: gptr (ngroups + 1, int64) into grows / gcols (int32): group g is rows grows[gptr[g] .. gptr[g+1]) and columns
 * gcols[same range], of equal size <= 32; the groups partition all rows and all columns (checked by the caller).
 * inv_off (int64, ngroups): offset of the row-major inverse of group g in `inv` (prefix sum of the squared sizes);
 * grp_of (int32, n): the group of every position of the grouped order. */
/* inverses of the blocks J[R_g, C_g] by Gauss-Jordan with partial pivoting; synchronises `stream`.  A zero or non-finite
 * pivot returns PB_ESINGULAR naming the lowest failing group; status_dev: one int32 of device scratch. */
int pb_group_inv_dev(const pb_csr *a, int64_t ngroups, const int64_t *gptr, const int32_t *grows, const int32_t *gcols,
                     const int64_t *inv_off, int smax, double *inv_out, int32_t *status_dev, uint64_t stream);
/* z[C_g] = inv_g y[R_g] for every group (accumulate != 0: z[C_g] +=) */
int pb_group_apply_dev(int64_t n, const int32_t *grp_of, const int64_t *gptr, const int32_t *grows, const int32_t *gcols,
                       const int64_t *inv_off, const double *inv, const double *y, double *z, int accumulate,
                       uint64_t stream);
/* doubles of the GMRES scalar buffer for restart length m (1 <= m <= 128), -1 otherwise */
int64_t pb_gmres_scal_size(int m);
/* V: (m + 1) n basis, z: n, partial: nblk (m + 2) per-block partial sums, scal: pb_gmres_scal_size(m).  init: x = 0,
 * V_0 = b, |b| and the tolerance tol |b|.  step j (0 <= j < m): one Arnoldi step with CGS2 and the Givens update, a
 * no-op once the cycle's DONE flag is set.  cycle_end: x += M^-1 V y, V_0 = b - A x and its norm (the next cycle's
 * start).  inv == NULL: no preconditioner (the group arrays are not read). */
int pb_gmres_init(int64_t n, int m, const double *b, double *x, double *V, double *partial, int nblk, double *scal,
                  double tol, uint64_t stream);
int pb_gmres_step(pb_csr *a, int64_t n, int m, int j, double *V, double *z, double *partial, int nblk, double *scal,
                  const int32_t *grp_of, const int64_t *gptr, const int32_t *grows, const int32_t *gcols,
                  const int64_t *inv_off, const double *inv, uint64_t stream);
int pb_gmres_cycle_end(pb_csr *a, int64_t n, int m, const double *b, double *x, double *V, double *z, double *partial,
                       int nblk, double *scal, const int32_t *grp_of, const int64_t *gptr, const int32_t *grows,
                       const int32_t *gcols, const int64_t *inv_off, const double *inv, uint64_t stream);

/* time `reps` device SpMVs with CUDA events on the launching stream; returns mean ms */
int pb_csr_spmv_bench(pb_csr *a, int reps, float *mean_ms);

#ifdef __cplusplus
}
#endif
#endif /* POREB200_H */
