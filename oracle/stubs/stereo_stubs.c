// TEST INFRASTRUCTURE ONLY. The LAPACK symbol the reference's stereo.c pulls in (LAPACK is not in this image):
// dgeev_ (stereo.c:177-272), the eigenvalues of the 4x4 companion matrix of the pinhole quartic. It calls a hook that
// oracle/stereo_ref.py fills with numpy.linalg.eigvals, which is LAPACK's own dgeev. With no hook set it fails loudly.
#include <stdio.h>

// The eigenvalues (wr, wi) of the n x n column-major matrix a (leading dimension lda); returns LAPACK's info
typedef int (*oracle_dgeev_hook_t)(int n, const double* a, int lda, double* wr, double* wi);
oracle_dgeev_hook_t oracle_dgeev_hook = 0;

// dgeev_ with jobvl = jobvr = 'N' (no eigenvectors), the only use stereo.c makes of it
int dgeev_(char* jobvl, char* jobvr, int* n, double* a, int* lda, double* wr, double* wi, double* vl, int* ldvl,
           double* vr, int* ldvr, double* work, int* lwork, int* info)
{
    (void)jobvl; (void)jobvr; (void)vl; (void)ldvl; (void)vr; (void)ldvr;
    if(oracle_dgeev_hook == 0)
    {
        fprintf(stderr, "oracle/_ref: dgeev_() called with no eigenvalue hook set (oracle/stereo_ref.py sets it)\n");
        *info = -1000;
        return 0;
    }
    if(*lwork == -1) { work[0] = 1.; *info = 0; return 0; }   // the storage query: this stand-in needs no work space
    *info = oracle_dgeev_hook(*n, a, *lda, wr, wi);
    return 0;
}
